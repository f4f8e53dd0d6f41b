/* libxsmm_b200 -- type/enum surface of the LIBXSMM 2.x C API, re-stated for the H100 (sm_90a) backend.
 *
 * This header is written from scratch; it mirrors names, enumerator VALUES and struct layouts of
 * the reference's include/libxsmm_typedefs.h so that callers compiled against either header are
 * ABI compatible. Enumerations are produced from X-macro tables (one row per enumerator) which
 * are also consumed by the host runtime (name lookup, validation).
 *   datatype enum ............ reference include/libxsmm_typedefs.h:218-246
 *   meltw flag/type enums .... reference include/libxsmm_typedefs.h:248-444
 *   gemm flags ............... reference include/libxsmm_typedefs.h:468-529
 *   argument structs ......... reference include/libxsmm_typedefs.h:570-725
 *   shapes / configs ......... reference include/libxsmm_typedefs.h:727-778
 *   function pointer types ... reference include/libxsmm_typedefs.h:690-701, 780-792
 */
#ifndef LIBXSMM_TYPEDEFS_H
#define LIBXSMM_TYPEDEFS_H

#include <stddef.h>
#include <stdint.h>

#if defined(__cplusplus)
# define LIBXSMM_EXTERN_C extern "C"
# define LIBXSMM_ARGDEF(ARG, DEFAULT) ARG = DEFAULT
#else
# define LIBXSMM_EXTERN_C
# define LIBXSMM_ARGDEF(ARG, DEFAULT) ARG
#endif
#if !defined(LIBXSMM_API)
# define LIBXSMM_API LIBXSMM_EXTERN_C __attribute__((visibility("default")))
#endif
#define LIBXSMM_APIVAR_PUBLIC(DECL) LIBXSMM_EXTERN_C __attribute__((visibility("default"))) extern DECL

/* LP64 build only (reference: LIBXSMM_CONFIG_ILP64 0) */
#define LIBXSMM_ILP64 0
#define LIBXSMM_BLASINT_NBITS 32
#define LIBXSMM_BLASINT int
typedef LIBXSMM_BLASINT libxsmm_blasint;
typedef unsigned long long libxsmm_timer_tickint;
typedef unsigned int libxsmm_bitfield;
typedef unsigned short libxsmm_bfloat16;
typedef unsigned short libxsmm_float16;
typedef unsigned char libxsmm_bfloat8;
typedef unsigned char libxsmm_hfloat8;

#define LIBXSMM_PREFETCH_NONE 0
#define LIBXSMM_PREFETCH_AUTO 0
#define LIBXSMM_ALPHA 1
#define LIBXSMM_BETA 1
#define LIBXSMM_DESCRIPTOR_MAXSIZE 96
#define LIBXSMM_DESCRIPTOR_SIGSIZE 32

#include "libxsmm_macros.h"   /* LIBXSMM_UPDIV, LIBXSMM_UP, LIBXSMM_MIN, LIBXSMM_MAX, LIBXSMM_ALIGNMENT, ... */

/* ---- element types: X(name, bytes) in enumerator order (values 0..26) ------------------------ */
#define LIBXSMM_B200_DATATYPES(X) \
  X(F64, 8) X(F32, 4) X(BF16, 2) X(F16, 2) X(BF8, 1) X(HF8, 1) X(I64, 8) X(U64, 8) X(I32, 4) \
  X(U32, 4) X(I16, 2) X(U16, 2) X(I8, 1) X(U8, 1) X(MXBF8, 1) X(MXHF8, 1) X(MXBF6, 1) \
  X(MXHF6, 1) X(I4X2, 1) X(U4X2, 1) X(MXFP4X2, 1) X(NVFP4X2, 1) X(I2X4, 1) X(I1X8, 1) \
  X(BF32, 4) X(IMPLICIT, 0) X(UNSUPPORTED, 0)
typedef enum libxsmm_datatype {
#define LIBXSMM_B200_X(NAME, BYTES) LIBXSMM_DATATYPE_##NAME,
  LIBXSMM_B200_DATATYPES(LIBXSMM_B200_X)
#undef LIBXSMM_B200_X
  LIBXSMM_DATATYPE_B200_COUNT
} libxsmm_datatype;

LIBXSMM_API unsigned char libxsmm_typesize(libxsmm_datatype datatype);
#define LIBXSMM_TYPESIZE(ENUM) ((int)libxsmm_typesize((libxsmm_datatype)(ENUM)))

typedef enum libxsmm_meltw_operation {
  LIBXSMM_MELTW_OPERATION_NONE = 0, LIBXSMM_MELTW_OPERATION_UNARY = 1,
  LIBXSMM_MELTW_OPERATION_BINARY = 2, LIBXSMM_MELTW_OPERATION_TERNARY = 3
} libxsmm_meltw_operation;

/* ---- unary flags ------------------------------------------------------------------------------ */
#define LIBXSMM_B200_UNARY_FLAGS(X) \
  X(NONE, 0) X(BITMASK_2BYTEMULT, 1) X(BCAST_ROW, 2) X(BCAST_COL, 4) X(BCAST_SCALAR, 8) \
  X(REDUCE_COLS, 16) X(REDUCE_ROWS, 32) X(REDUCE_INIT_ACC, 64) X(IDX_SIZE_4BYTES, 128) \
  X(IDX_SIZE_8BYTES, 256) X(REDUCE_INF_ACC, 512) X(REDUCE_NO_PREFETCH, 1024) \
  X(REDUCE_RECORD_ARGOP, 2048) X(STOCHASTIC_ROUND, 4096) X(GS_ROWS, 16) X(GS_COLS, 32) \
  X(GS_OFFS, 8192) X(NTS_HINT, 16384) X(NO_SCF_QUANT, 1024) X(SIGN_SAT_QUANT, 16)
typedef enum libxsmm_meltw_unary_flags {
#define LIBXSMM_B200_X(NAME, VALUE) LIBXSMM_MELTW_FLAG_UNARY_##NAME = VALUE,
  LIBXSMM_B200_UNARY_FLAGS(LIBXSMM_B200_X)
#undef LIBXSMM_B200_X
  LIBXSMM_MELTW_FLAG_UNARY_B200_END = 32768
} libxsmm_meltw_unary_flags;

/* ---- unary operation kinds -------------------------------------------------------------------- */
#define LIBXSMM_B200_UNARY_TYPES(X) \
  X(NONE, 0) X(IDENTITY, 1) X(XOR, 2) X(X2, 3) X(SQRT, 4) X(RELU, 5) X(RELU_INV, 6) X(TANH, 7) \
  X(TANH_INV, 8) X(SIGMOID, 9) X(SIGMOID_INV, 10) X(GELU, 11) X(GELU_INV, 12) X(NEGATE, 13) \
  X(INC, 14) X(RECIPROCAL, 15) X(RECIPROCAL_SQRT, 16) X(EXP, 17) X(REDUCE_X_OP_ADD, 18) \
  X(REDUCE_X2_OP_ADD, 19) X(REDUCE_X_X2_OP_ADD, 20) X(REDUCE_X_OP_MAX, 21) X(REDUCE_X_OP_MUL, 22) \
  X(REDUCE_X_OP_ADD_NCNC_FORMAT, 23) X(REDUCE_TO_SCALAR_OP_ADD, 24) X(DROPOUT, 25) \
  X(DROPOUT_INV, 26) X(REPLICATE_COL_VAR, 27) X(TRANSFORM_NORM_TO_VNNI2, 28) \
  X(TRANSFORM_NORM_TO_NORMT, 29) X(TRANSFORM_VNNI2_TO_VNNI2T, 30) X(TRANSFORM_NORM_TO_VNNI2T, 31) \
  X(TRANSFORM_NORM_TO_VNNI2_PAD, 32) X(UNZIP, 33) X(LEAKY_RELU, 34) X(LEAKY_RELU_INV, 35) \
  X(ELU, 36) X(ELU_INV, 37) X(STOCHASTIC_ROUND, 38) X(TRANSFORM_PADM_MOD2, 39) \
  X(TRANSFORM_PADN_MOD2, 40) X(TRANSFORM_PADNM_MOD2, 41) X(QUANT, 42) X(DEQUANT, 43) \
  X(REDUCE_COLS_IDX_OP_ADD, 44) X(DECOMPRESS_SPARSE_FACTOR_1, 45) X(DECOMPRESS_SPARSE_FACTOR_2, 46) \
  X(DECOMPRESS_SPARSE_FACTOR_4, 47) X(DECOMPRESS_SPARSE_FACTOR_8, 48) \
  X(DECOMPRESS_SPARSE_FACTOR_16, 49) X(DECOMPRESS_SPARSE_FACTOR_32, 50) X(GATHER, 51) \
  X(SCATTER, 52) X(REDUCE_COLS_IDX_OP_MAX, 53) X(TRANSFORM_NORM_TO_VNNI4, 54) \
  X(TRANSFORM_VNNI4_TO_VNNI4T, 55) X(TRANSFORM_NORM_TO_VNNI4T, 56) \
  X(TRANSFORM_NORM_TO_VNNI4_PAD, 57) X(TRANSFORM_PADM_MOD4, 58) X(TRANSFORM_PADN_MOD4, 59) \
  X(TRANSFORM_PADNM_MOD4, 60) X(TRANSFORM_VNNI4_TO_NORM, 61) X(TRANSFORM_VNNI4_TO_VNNI2, 62) \
  X(DUMP, 63) X(DECOMP_FP32_TO_BF16X2, 64) X(DECOMP_FP32_TO_BF16X3, 65) \
  X(TRANSFORM_VNNI4T_TO_NORM, 66) X(TRANSFORM_VNNI2T_TO_NORM, 67) X(REDUCE_COLS_IDX_OP_MIN, 68) \
  X(REDUCE_X_OP_MIN, 69) X(REDUCE_X_OP_ABSMAX, 70) X(TRANSFORM_NORM_TO_VNNI8, 71) \
  X(TRANSFORM_VNNI8_TO_VNNI8T, 72) X(TRANSFORM_NORM_TO_VNNI8T, 73) \
  X(TRANSFORM_NORM_TO_VNNI8_PAD, 74) X(TRANSFORM_VNNI8T_TO_NORM, 75) X(TRANSFORM_VNNI8_TO_NORM, 76)
typedef enum libxsmm_meltw_unary_type {
#define LIBXSMM_B200_X(NAME, VALUE) LIBXSMM_MELTW_TYPE_UNARY_##NAME = VALUE,
  LIBXSMM_B200_UNARY_TYPES(LIBXSMM_B200_X)
#undef LIBXSMM_B200_X
  LIBXSMM_MELTW_TYPE_UNARY_B200_END = 77
} libxsmm_meltw_unary_type;

/* ---- binary ----------------------------------------------------------------------------------- */
#define LIBXSMM_B200_BINARY_FLAGS(X) \
  X(NONE, 0) X(BCAST_ROW_IN_0, 1) X(BCAST_ROW_IN_1, 2) X(BCAST_COL_IN_0, 4) X(BCAST_COL_IN_1, 8) \
  X(BCAST_SCALAR_IN_0, 16) X(BCAST_SCALAR_IN_1, 32) X(STOCHASTIC_ROUND, 64) \
  X(BITMASK_2BYTEMULT, 128) X(NTS_HINT, 256)
typedef enum libxsmm_meltw_binary_flags {
#define LIBXSMM_B200_X(NAME, VALUE) LIBXSMM_MELTW_FLAG_BINARY_##NAME = VALUE,
  LIBXSMM_B200_BINARY_FLAGS(LIBXSMM_B200_X)
#undef LIBXSMM_B200_X
  LIBXSMM_MELTW_FLAG_BINARY_B200_END = 512
} libxsmm_meltw_binary_flags;

#define LIBXSMM_B200_BINARY_TYPES(X) \
  X(NONE, 0) X(ADD, 1) X(MUL, 2) X(SUB, 3) X(DIV, 4) X(MULADD, 5) X(MATMUL, 6) \
  X(MUL_AND_REDUCE_TO_SCALAR_OP_ADD, 7) X(PACK, 8) X(MAX, 9) X(MIN, 10) X(BRGEMM, 11) \
  X(BRGEMM_B_TRANS, 12) X(BRGEMM_A_TRANS, 13) X(BRGEMM_A_TRANS_B_TRANS, 14) X(BRGEMM_A_VNNI, 15) \
  X(BRGEMM_A_VNNI_B_TRANS, 16) X(BRGEMM_A_VNNI_TRANS, 17) X(BRGEMM_A_VNNI_TRANS_B_TRANS, 18) \
  X(MATMUL_B_TRANS, 19) X(MATMUL_A_TRANS, 20) X(MATMUL_A_TRANS_B_TRANS, 21) X(MATMUL_A_VNNI, 22) \
  X(MATMUL_A_VNNI_B_TRANS, 23) X(MATMUL_A_VNNI_TRANS, 24) X(MATMUL_A_VNNI_TRANS_B_TRANS, 25) \
  X(ZIP, 26) X(CMP_OP_GT, 27) X(CMP_OP_GE, 28) X(CMP_OP_LT, 29) X(CMP_OP_LE, 30) \
  X(CMP_OP_EQ, 31) X(CMP_OP_NE, 32)
typedef enum libxsmm_meltw_binary_type {
#define LIBXSMM_B200_X(NAME, VALUE) LIBXSMM_MELTW_TYPE_BINARY_##NAME = VALUE,
  LIBXSMM_B200_BINARY_TYPES(LIBXSMM_B200_X)
#undef LIBXSMM_B200_X
  LIBXSMM_MELTW_TYPE_BINARY_B200_END = 33
} libxsmm_meltw_binary_type;

/* ---- ternary ---------------------------------------------------------------------------------- */
#define LIBXSMM_B200_TERNARY_FLAGS(X) \
  X(NONE, 0) X(BCAST_ROW_IN_0, 1) X(BCAST_ROW_IN_1, 2) X(BCAST_ROW_IN_2, 4) X(BCAST_COL_IN_0, 8) \
  X(BCAST_COL_IN_1, 16) X(BCAST_COL_IN_2, 32) X(BCAST_SCALAR_IN_0, 64) X(BCAST_SCALAR_IN_1, 128) \
  X(BCAST_SCALAR_IN_2, 256) X(REUSE_IN_2_AS_OUT, 512) X(BITMASK_2BYTEMULT, 1024) \
  X(STOCHASTIC_ROUND, 2048)
typedef enum libxsmm_meltw_ternary_flags {
#define LIBXSMM_B200_X(NAME, VALUE) LIBXSMM_MELTW_FLAG_TERNARY_##NAME = VALUE,
  LIBXSMM_B200_TERNARY_FLAGS(LIBXSMM_B200_X)
#undef LIBXSMM_B200_X
  LIBXSMM_MELTW_FLAG_TERNARY_B200_END = 4096
} libxsmm_meltw_ternary_flags;

#define LIBXSMM_B200_TERNARY_TYPES(X) \
  X(NONE, 0) X(MULADD, 1) X(MATMUL, 2) X(SELECT, 3) X(NMULADD, 4) X(BRGEMM, 5) \
  X(BRGEMM_B_TRANS, 6) X(BRGEMM_A_TRANS, 7) X(BRGEMM_A_TRANS_B_TRANS, 8) X(BRGEMM_A_VNNI, 9) \
  X(BRGEMM_A_VNNI_B_TRANS, 10) X(BRGEMM_A_VNNI_TRANS, 11) X(BRGEMM_A_VNNI_TRANS_B_TRANS, 12) \
  X(MATMUL_B_TRANS, 13) X(MATMUL_A_TRANS, 14) X(MATMUL_A_TRANS_B_TRANS, 15) X(MATMUL_A_VNNI, 16) \
  X(MATMUL_A_VNNI_B_TRANS, 17) X(MATMUL_A_VNNI_TRANS, 18) X(MATMUL_A_VNNI_TRANS_B_TRANS, 19)
typedef enum libxsmm_meltw_ternary_type {
#define LIBXSMM_B200_X(NAME, VALUE) LIBXSMM_MELTW_TYPE_TERNARY_##NAME = VALUE,
  LIBXSMM_B200_TERNARY_TYPES(LIBXSMM_B200_X)
#undef LIBXSMM_B200_X
  LIBXSMM_MELTW_TYPE_TERNARY_B200_END = 20
} libxsmm_meltw_ternary_type;

/* ---- GEMM flags ------------------------------------------------------------------------------- */
typedef enum libxsmm_basic_gemm_flags {
  LIBXSMM_BASIC_GEMM_FLAG_NONE = 0, LIBXSMM_BASIC_GEMM_FLAG_TRANS_A = 1,
  LIBXSMM_BASIC_GEMM_FLAG_TRANS_B = 2, LIBXSMM_BASIC_GEMM_FLAG_TRANS_AB = 3,
  LIBXSMM_BASIC_GEMM_FLAG_BETA_0 = 4, LIBXSMM_BASIC_GEMM_FLAG_ALIGN_A = 8,
  LIBXSMM_BASIC_GEMM_FLAG_ALIGN_C = 16, LIBXSMM_BASIC_GEMM_FLAG_ALIGN_C_NTS_HINT = 1024 | 16,
  LIBXSMM_BASIC_GEMM_FLAG_INVALID = 524288
} libxsmm_basic_gemm_flags;

#define LIBXSMM_B200_GEMM_FLAGS(X) \
  X(NONE, 0) X(TRANS_A, 1) X(TRANS_B, 2) X(TRANS_AB, 3) X(BETA_0, 4) X(ALIGN_A, 8) \
  X(ALIGN_C, 16) X(ALIGN_C_NTS_HINT, 32 | 16) X(NO_RESET_TILECONFIG, 64) \
  X(NO_SETUP_TILECONFIG, 128) X(VNNI_A, 256) X(VNNI_B, 512) X(VNNI_C, 1024) \
  X(USE_XGEMM_ABI, 2048) X(USE_XGEMM_EXT_ABI, 4096) X(DESC_ISBIG, 8192) \
  X(BATCH_REDUCE_ADDRESS, 8192) X(BATCH_REDUCE_OFFSET, 16384) X(BATCH_REDUCE_STRIDE, 32768) \
  X(USE_COL_VEC_SCF, 65536) X(USE_COL_VEC_ZPT, 131072) X(INTLV_A_FORMAT, 262144) \
  X(DECOMPRESS_A_VIA_BITMASK, 524288) X(USE_MxK_ZPT, 1048576) X(USE_MxK_SCF, 2097152) \
  X(ALIGN_C_NTS_HINT_BETA_0, 4 | 48) X(ALIGN_C_NTS_HINT_BATCH_REDUCE_ADDRESS, 8192 | 48) \
  X(ALIGN_C_NTS_HINT_BETA_0_BATCH_REDUCE_ADDRESS, 4 | 48 | 8192) \
  X(ALIGN_C_NTS_HINT_BATCH_REDUCE_OFFSET, 16384 | 48) \
  X(ALIGN_C_NTS_HINT_BETA_0_BATCH_REDUCE_OFFSET, 4 | 48 | 16384) \
  X(ALIGN_C_NTS_HINT_BATCH_REDUCE_STRIDE, 32768 | 48) \
  X(ALIGN_C_NTS_HINT_BETA_0_BATCH_REDUCE_STRIDE, 4 | 48 | 32768) X(INVALID, 4194304)
typedef enum libxsmm_gemm_flags {
#define LIBXSMM_B200_X(NAME, VALUE) LIBXSMM_GEMM_FLAG_##NAME = (VALUE),
  LIBXSMM_B200_GEMM_FLAGS(LIBXSMM_B200_X)
#undef LIBXSMM_B200_X
  LIBXSMM_GEMM_FLAG_B200_END = 8388608
} libxsmm_gemm_flags;

/* BLAS transpose characters to flags: only 'N' / 'n' means "as is", so 'T' and the conjugate request 'C' both transpose
 * (reference include/libxsmm_macros.h:278-281; tests/gemmflags.c is the truth table) */
#define LIBXSMM_B200_TRANSPOSED(CH) (!('N' == (CH) || 'n' == (CH)))
#define LIBXSMM_GEMM_FLAGS(TRANSA, TRANSB) (libxsmm_bitfield)( \
  (LIBXSMM_B200_TRANSPOSED(TRANSA) ? LIBXSMM_GEMM_FLAG_TRANS_A : 0) | (LIBXSMM_B200_TRANSPOSED(TRANSB) ? LIBXSMM_GEMM_FLAG_TRANS_B : 0))
/* the same from POINTERS to the characters, where a NULL pointer keeps the transpose bit of DEFAULT; all other bits of DEFAULT
 * pass through (reference :283-287) */
#define LIBXSMM_B200_PTRANS(PCH, BIT, DEFAULT) \
  ((NULL != (const void*)(PCH)) ? (LIBXSMM_B200_TRANSPOSED(*(const char*)(PCH)) ? (BIT) : 0) : ((BIT) & (DEFAULT)))
#define LIBXSMM_GEMM_PFLAGS(TRANSA, TRANSB, DEFAULT) (libxsmm_bitfield)( \
  LIBXSMM_B200_PTRANS(TRANSA, LIBXSMM_GEMM_FLAG_TRANS_A, DEFAULT) | LIBXSMM_B200_PTRANS(TRANSB, LIBXSMM_GEMM_FLAG_TRANS_B, DEFAULT) | \
  ((DEFAULT) & ~(LIBXSMM_GEMM_FLAG_TRANS_A | LIBXSMM_GEMM_FLAG_TRANS_B)))

typedef enum libxsmm_gemm_prefetch_type {
  LIBXSMM_GEMM_PREFETCH_NONE = 0, LIBXSMM_GEMM_PREFETCH_AL2 = 1, LIBXSMM_GEMM_PREFETCH_BL2 = 2
} libxsmm_gemm_prefetch_type;

typedef enum libxsmm_gemm_batch_reduce_type {
  LIBXSMM_GEMM_BATCH_REDUCE_NONE = 0, LIBXSMM_GEMM_BATCH_REDUCE_ADDRESS = 1,
  LIBXSMM_GEMM_BATCH_REDUCE_OFFSET = 2, LIBXSMM_GEMM_BATCH_REDUCE_STRIDE = 4
} libxsmm_gemm_batch_reduce_type;

typedef enum libxsmm_kernel_kind {
  LIBXSMM_KERNEL_KIND_MATMUL = 0, LIBXSMM_KERNEL_KIND_MELTW = 1, LIBXSMM_KERNEL_KIND_MEQN = 2,
  LIBXSMM_KERNEL_KIND_USER = 3, LIBXSMM_KERNEL_UNREGISTERED = 4
} libxsmm_kernel_kind;

/* ---- argument structs (six/four pointer slots; see SURVEY.md appendix A/C for slot meaning) ---- */
typedef struct libxsmm_matrix_arg {
  void *primary, *secondary, *tertiary, *quaternary, *quinary, *senary;
} libxsmm_matrix_arg;
typedef struct libxsmm_matrix_op_arg {
  void *primary, *secondary, *tertiary, *quaternary;
} libxsmm_matrix_op_arg;

/* ---- matrix equations (include/libxsmm_typedefs.h:586-694 of the reference): argument description and call structs ---- */
typedef enum libxsmm_matrix_arg_type { LIBXSMM_MATRIX_ARG_TYPE_SINGULAR = 0, LIBXSMM_MATRIX_ARG_TYPE_SET = 1 } libxsmm_matrix_arg_type;
typedef enum libxsmm_matrix_arg_set_type {
  LIBXSMM_MATRIX_ARG_SET_TYPE_NONE = 0, LIBXSMM_MATRIX_ARG_SET_TYPE_ABS_ADDRESS = 1, LIBXSMM_MATRIX_ARG_SET_TYPE_OFFSET_BASE = 2,
  LIBXSMM_MATRIX_ARG_SET_TYPE_STRIDE_BASE = 3
} libxsmm_matrix_arg_set_type;
typedef struct libxsmm_meqn_arg_shape { libxsmm_blasint m, n, ld; libxsmm_datatype type; } libxsmm_meqn_arg_shape;
typedef struct libxsmm_matrix_arg_attributes {
  libxsmm_matrix_arg_type type; libxsmm_matrix_arg_set_type set_type; libxsmm_blasint set_cardinality_hint, set_stride_hint;
} libxsmm_matrix_arg_attributes;
typedef struct libxsmm_meqn_op_metadata { libxsmm_blasint eqn_idx, op_arg_pos; } libxsmm_meqn_op_metadata;
typedef struct libxsmm_meqn_arg_metadata { libxsmm_blasint eqn_idx, in_arg_pos; } libxsmm_meqn_arg_metadata;
typedef struct libxsmm_meqn_param {
  const libxsmm_matrix_op_arg* ops_args;    /* per-operation parameters, indexed by op_arg_pos */
  const libxsmm_matrix_arg* inputs;         /* input matrices, indexed by in_arg_pos */
  libxsmm_matrix_arg output;
} libxsmm_meqn_param;
typedef void (*libxsmm_meqn_function)(const libxsmm_meqn_param* in_struct);


typedef struct libxsmm_meltw_unary_shape {
  libxsmm_blasint m, n, ldi, ldo;
  libxsmm_datatype in0_type, out_type, comp_type;
} libxsmm_meltw_unary_shape;
typedef struct libxsmm_meltw_binary_shape {
  libxsmm_blasint m, n, ldi, ldi2, ldo;
  libxsmm_datatype in0_type, in1_type, out_type, comp_type;
} libxsmm_meltw_binary_shape;
typedef struct libxsmm_meltw_ternary_shape {
  libxsmm_blasint m, n, ldi, ldi2, ldi3, ldo;
  libxsmm_datatype in0_type, in1_type, in2_type, out_type, comp_type;
} libxsmm_meltw_ternary_shape;

typedef struct libxsmm_meltw_unary_param {
  libxsmm_matrix_op_arg op; libxsmm_matrix_arg in; libxsmm_matrix_arg out;
} libxsmm_meltw_unary_param;
typedef struct libxsmm_meltw_binary_param {
  libxsmm_matrix_op_arg op; libxsmm_matrix_arg in0; libxsmm_matrix_arg in1; libxsmm_matrix_arg out;
} libxsmm_meltw_binary_param;
typedef struct libxsmm_meltw_ternary_param {
  libxsmm_matrix_op_arg op; libxsmm_matrix_arg in0; libxsmm_matrix_arg in1; libxsmm_matrix_arg in2;
  libxsmm_matrix_arg out;
} libxsmm_meltw_ternary_param;

typedef void (*libxsmm_meltwfunction_unary)(const libxsmm_meltw_unary_param* in_struct);
typedef void (*libxsmm_meltwfunction_binary)(const libxsmm_meltw_binary_param* in_struct);
typedef void (*libxsmm_meltwfunction_ternary)(const libxsmm_meltw_ternary_param* in_struct);
typedef union libxsmm_xmeltwfunction {
  void (*xmeltw)(const void* in_struct);
  libxsmm_meltwfunction_unary meltw_unary;
  libxsmm_meltwfunction_binary meltw_binary;
  libxsmm_meltwfunction_ternary meltw_ternary;
} libxsmm_xmeltwfunction;

typedef void (*libxsmm_dmmfunction)(const double* a, const double* b, double* c);
typedef void (*libxsmm_smmfunction)(const float* a, const float* b, float* c);

typedef struct libxsmm_gemm_param {
  libxsmm_matrix_op_arg op; libxsmm_matrix_arg a; libxsmm_matrix_arg b; libxsmm_matrix_arg c;
} libxsmm_gemm_param;
typedef struct libxsmm_gemm_ext_param {
  libxsmm_matrix_op_arg op; libxsmm_matrix_arg a; libxsmm_matrix_arg b; libxsmm_matrix_arg c;
  libxsmm_matrix_arg d; libxsmm_matrix_arg ap; libxsmm_matrix_arg bp; libxsmm_matrix_arg cp;
} libxsmm_gemm_ext_param;

typedef struct libxsmm_gemm_shape {
  libxsmm_blasint m, n, k, lda, ldb, ldc;
  libxsmm_datatype a_in_type, b_in_type, out_type, comp_type;
} libxsmm_gemm_shape;
typedef struct libxsmm_gemm_batch_reduce_config {
  libxsmm_gemm_batch_reduce_type br_type;
  libxsmm_blasint br_stride_a_hint, br_stride_b_hint;   /* bytes */
  unsigned char br_unroll_hint;
} libxsmm_gemm_batch_reduce_config;
typedef struct libxsmm_spgemm_config {
  libxsmm_blasint packed_width, bk, bn;
} libxsmm_spgemm_config;
typedef struct libxsmm_gemm_ext_unary_argops {
  libxsmm_blasint ldap; libxsmm_meltw_unary_type ap_unary_type; libxsmm_bitfield ap_unary_flags;
  libxsmm_blasint store_ap;
  libxsmm_blasint ldbp; libxsmm_meltw_unary_type bp_unary_type; libxsmm_bitfield bp_unary_flags;
  libxsmm_blasint store_bp;
  libxsmm_blasint ldcp; libxsmm_meltw_unary_type cp_unary_type; libxsmm_bitfield cp_unary_flags;
  libxsmm_blasint store_cp;
} libxsmm_gemm_ext_unary_argops;
typedef struct libxsmm_gemm_ext_binary_postops {
  libxsmm_blasint ldd; libxsmm_datatype d_in_type; libxsmm_meltw_binary_type d_binary_type;
  libxsmm_bitfield d_binary_flags;
} libxsmm_gemm_ext_binary_postops;
typedef struct libxsmm_tilecfg_state { unsigned char tileconfig[64]; } libxsmm_tilecfg_state;

typedef void (*libxsmm_gemmfunction)(const libxsmm_gemm_param* in_struct);
typedef void (*libxsmm_gemmfunction_ext)(const libxsmm_gemm_ext_param* in_struct);
typedef void (*libxsmm_tilecfgfunction)(const libxsmm_tilecfg_state* in_struct);
typedef union libxsmm_xmmfunction {
  const void* ptr_const; void* ptr;
  void (*xmm)(const void* a, const void* b, void* c);
  void (*xgemm)(const void* in_struct);
  libxsmm_dmmfunction dmm; libxsmm_smmfunction smm;
  libxsmm_gemmfunction gemm; libxsmm_gemmfunction_ext gemm_ext;
  libxsmm_tilecfgfunction tilecfg;
} libxsmm_xmmfunction;

/* ---- query structs ---------------------------------------------------------------------------- */
typedef struct libxsmm_mmkernel_info {
  libxsmm_datatype iprecision, oprecision;
  libxsmm_gemm_prefetch_type prefetch;
  unsigned int lda, ldb, ldc, m, n, k;
  int flags;
} libxsmm_mmkernel_info;
typedef struct libxsmm_meltwkernel_info {
  unsigned int ldi, ldo, m, n, datatype, flags, operation;
} libxsmm_meltwkernel_info;
typedef struct libxsmm_kernel_info {
  libxsmm_kernel_kind kind; unsigned int nflops; size_t code_size; unsigned int is_reference_kernel;
} libxsmm_kernel_info;
typedef struct libxsmm_registry_info { size_t capacity, size, nbytes, nstatic, ncache; } libxsmm_registry_info;

/* opaque descriptors (layout private to the runtime, see csrc/xb_internal.h) */
typedef struct libxsmm_descriptor_blob { char data[LIBXSMM_DESCRIPTOR_MAXSIZE]; } libxsmm_descriptor_blob;
typedef struct libxsmm_gemm_descriptor libxsmm_gemm_descriptor;
typedef struct libxsmm_meltw_descriptor libxsmm_meltw_descriptor;

#endif /* LIBXSMM_TYPEDEFS_H */
