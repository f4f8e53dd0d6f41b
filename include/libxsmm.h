/* libxsmm_b200 -- drop-in C API of LIBXSMM's tensor-processing-primitive hot path.
 *
 * Every entry point below keeps the name, argument meaning and error behaviour (NULL on
 * unsupported/failed, library is mute unless libxsmm_verbosity != 0) of the reference API, but the
 * handle that dispatch returns launches a hand-written sm_90a CUDA kernel instead of JIT'ed x86.
 * Each declaration cites the reference interface it replaces (file:line in /root/reference).
 * Additive, GPU-only entry points (batch launch, streams, device memory) live in libxsmm_b200.h.
 */
#ifndef LIBXSMM_H
#define LIBXSMM_H

#include "libxsmm_typedefs.h"
#include "libxsmm_fsspmdm.h"
#include "libxsmm_b200.h"

#define LIBXSMM_VERSION_MAJOR 2
#define LIBXSMM_VERSION_MINOR 0
#define LIBXSMM_VERSION_UPDATE 0
#define LIBXSMM_B200 1

#if defined(__cplusplus)
extern "C" {
#endif

/* public state words (reference include/libxsmm_generator.h:214-222); LIBXSMM_INIT reads ninit */
LIBXSMM_APIVAR_PUBLIC(unsigned int libxsmm_ninit);
LIBXSMM_APIVAR_PUBLIC(int libxsmm_target_archid);
LIBXSMM_APIVAR_PUBLIC(int libxsmm_verbosity);
#define LIBXSMM_INIT if (2 > libxsmm_ninit) libxsmm_init();

/* ---- lifetime / environment (reference include/libxsmm.h:62-100) ------------------------------- */
LIBXSMM_API void libxsmm_init(void);
LIBXSMM_API void libxsmm_finalize(void);
LIBXSMM_API int libxsmm_get_target_archid(void);
LIBXSMM_API void libxsmm_set_target_archid(int id);
LIBXSMM_API const char* libxsmm_get_target_arch(void);          /* returns "sm_90a" */
LIBXSMM_API void libxsmm_set_target_arch(const char* arch);     /* accepted and ignored */
LIBXSMM_API const char* libxsmm_get_typename(libxsmm_datatype datatype);
LIBXSMM_API int libxsmm_get_verbosity(void);
LIBXSMM_API void libxsmm_set_verbosity(int level);

/* ---- introspection (reference include/libxsmm.h:102-117) --------------------------------------- */
LIBXSMM_API int libxsmm_get_mmkernel_info(libxsmm_xmmfunction kernel, libxsmm_mmkernel_info* info);
LIBXSMM_API int libxsmm_get_meltwkernel_info(libxsmm_xmeltwfunction kernel, libxsmm_meltwkernel_info* info);
LIBXSMM_API int libxsmm_get_kernel_info(const void* kernel, libxsmm_kernel_info* info);
LIBXSMM_API int libxsmm_get_registry_info(libxsmm_registry_info* info);
/* enumerate the registry by kind (reference include/libxsmm.h:105-108): LIBXSMM_KERNEL_KIND_USER yields the VALUE of every entry made with
 * libxsmm_xregister (and its key through `key`, may be NULL); the kernel kinds yield the callable of every registered handle. _next accepts
 * an entry that was released after it was returned (tests/registry.c:133-137). NULL ends the enumeration. */
LIBXSMM_API void* libxsmm_get_registry_begin(libxsmm_kernel_kind kind, const void** key);
LIBXSMM_API void* libxsmm_get_registry_next(const void* regentry, const void** key);

/* ---- shape/config constructors (reference include/libxsmm_generator.h:20-43) ------------------- */
LIBXSMM_API libxsmm_gemm_shape libxsmm_create_gemm_shape(libxsmm_blasint m, libxsmm_blasint n, libxsmm_blasint k,
  libxsmm_blasint lda, libxsmm_blasint ldb, libxsmm_blasint ldc,
  libxsmm_datatype a_in_type, libxsmm_datatype b_in_type, libxsmm_datatype out_type, libxsmm_datatype comp_type);
LIBXSMM_API libxsmm_gemm_batch_reduce_config libxsmm_create_gemm_batch_reduce_config(
  libxsmm_gemm_batch_reduce_type br_type, libxsmm_blasint br_stride_a_hint, libxsmm_blasint br_stride_b_hint,
  unsigned char br_unroll_hint);
LIBXSMM_API libxsmm_gemm_ext_unary_argops libxsmm_create_gemm_ext_unary_argops(
  libxsmm_blasint ldap, libxsmm_meltw_unary_type ap_unary_type, libxsmm_bitfield ap_unary_flags, libxsmm_blasint store_ap,
  libxsmm_blasint ldbp, libxsmm_meltw_unary_type bp_unary_type, libxsmm_bitfield bp_unary_flags, libxsmm_blasint store_bp,
  libxsmm_blasint ldcp, libxsmm_meltw_unary_type cp_unary_type, libxsmm_bitfield cp_unary_flags, libxsmm_blasint store_cp);
LIBXSMM_API libxsmm_gemm_ext_binary_postops libxsmm_create_gemm_ext_binary_postops(
  libxsmm_blasint ldd, libxsmm_datatype d_in_type, libxsmm_meltw_binary_type d_binary_type, libxsmm_bitfield d_binary_flags);
LIBXSMM_API libxsmm_meltw_unary_shape libxsmm_create_meltw_unary_shape(libxsmm_blasint m, libxsmm_blasint n,
  libxsmm_blasint ldi, libxsmm_blasint ldo, libxsmm_datatype in0_type, libxsmm_datatype out_type, libxsmm_datatype comp_type);
LIBXSMM_API libxsmm_meltw_binary_shape libxsmm_create_meltw_binary_shape(libxsmm_blasint m, libxsmm_blasint n,
  libxsmm_blasint ldi, libxsmm_blasint ldi2, libxsmm_blasint ldo,
  libxsmm_datatype in0_type, libxsmm_datatype in1_type, libxsmm_datatype out_type, libxsmm_datatype comp_type);
LIBXSMM_API libxsmm_meltw_ternary_shape libxsmm_create_meltw_ternary_shape(libxsmm_blasint m, libxsmm_blasint n,
  libxsmm_blasint ldi, libxsmm_blasint ldi2, libxsmm_blasint ldi3, libxsmm_blasint ldo,
  libxsmm_datatype in0_type, libxsmm_datatype in1_type, libxsmm_datatype in2_type, libxsmm_datatype out_type,
  libxsmm_datatype comp_type);

/* ---- dense GEMM / BRGEMM dispatch (reference include/libxsmm.h:128-140, src/libxsmm_main.c:3390-3446) -- */
LIBXSMM_API libxsmm_gemmfunction libxsmm_dispatch_gemm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags);
LIBXSMM_API libxsmm_gemmfunction libxsmm_dispatch_brgemm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags,
  const libxsmm_gemm_batch_reduce_config brgemm_config);
LIBXSMM_API libxsmm_gemmfunction_ext libxsmm_dispatch_brgemm_ext(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags,
  const libxsmm_gemm_batch_reduce_config brgemm_config,
  const libxsmm_gemm_ext_unary_argops unary_argops, const libxsmm_gemm_ext_binary_postops binary_postops);
/* AMX tile (re)configuration has no GPU meaning: returns a callable no-op (include/libxsmm.h:139) */
LIBXSMM_API libxsmm_tilecfgfunction libxsmm_dispatch_tilecfg_gemm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags);

/* ---- matrix-eltwise dispatch (reference include/libxsmm.h:142-146, src/libxsmm_main.c:3449-3511) -- */
LIBXSMM_API libxsmm_meltwfunction_unary libxsmm_dispatch_meltw_unary(const libxsmm_meltw_unary_type unary_type,
  const libxsmm_meltw_unary_shape unary_shape, const libxsmm_bitfield unary_flags);
LIBXSMM_API libxsmm_meltwfunction_binary libxsmm_dispatch_meltw_binary(const libxsmm_meltw_binary_type binary_type,
  const libxsmm_meltw_binary_shape binary_shape, const libxsmm_bitfield binary_flags);
LIBXSMM_API libxsmm_meltwfunction_ternary libxsmm_dispatch_meltw_ternary(const libxsmm_meltw_ternary_type ternary_type,
  const libxsmm_meltw_ternary_shape ternary_shape, const libxsmm_bitfield ternary_flags);
/* descriptor route (reference include/libxsmm.h:143, include/libxsmm_generator.h:48-57): the blob is filled by one of the two
 * init helpers; dispatch returns the same handle the typed dispatcher above returns for the same operation */
LIBXSMM_API libxsmm_meltw_descriptor* libxsmm_meltw_descriptor_init(libxsmm_descriptor_blob* blob,
  libxsmm_datatype in_type, libxsmm_datatype out_type, libxsmm_blasint m, libxsmm_blasint n, libxsmm_blasint ldi, libxsmm_blasint ldo,
  unsigned short flags, unsigned short param, unsigned char operation);
LIBXSMM_API libxsmm_meltw_descriptor* libxsmm_meltw_descriptor_init2(libxsmm_descriptor_blob* blob,
  libxsmm_datatype in0_type, libxsmm_datatype in1_type, libxsmm_datatype in2_type, libxsmm_datatype comp_type, libxsmm_datatype out_type,
  libxsmm_blasint m, libxsmm_blasint n, libxsmm_blasint ldi, libxsmm_blasint ldo, libxsmm_blasint ldi2, libxsmm_blasint ldi3,
  unsigned short flags, unsigned short param, unsigned char operation);
LIBXSMM_API libxsmm_xmeltwfunction libxsmm_dispatch_meltw(const libxsmm_meltw_descriptor* descriptor);

/* ---- packed sparse GEMM (reference include/libxsmm.h:170-192, src/libxsmm_main.c:3553-3731) ------
 * which operand is sparse follows the reference's convention: the one whose leading dimension in the
 * shape is 0 (lda==0: A sparse, ldb==0: B sparse, ldc==0: C sparse). Handles are caller-owned and
 * freed with libxsmm_release_kernel. */
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_spgemm_csr(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width,
  const unsigned int* row_ptr, const unsigned int* column_idx, const void* values);
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_spgemm_csc(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width,
  const unsigned int* column_ptr, const unsigned int* row_idx, const void* values);
/* ---- matrix equations: a tree of element-wise / reduction nodes built in pre-order, evaluated by one call (reference
 * include/libxsmm.h:149-162). GEMM nodes are not available in this backend (dispatch returns NULL for such trees). ---- */
LIBXSMM_API libxsmm_blasint libxsmm_meqn_create(void);
LIBXSMM_API libxsmm_meqn_arg_shape libxsmm_create_meqn_arg_shape(const libxsmm_blasint m, const libxsmm_blasint n, const libxsmm_blasint ld, const libxsmm_datatype type);
LIBXSMM_API libxsmm_matrix_arg_attributes libxsmm_create_matrix_arg_attributes(const libxsmm_matrix_arg_type type, const libxsmm_matrix_arg_set_type set_type,
  const libxsmm_blasint set_cardinality_hint, const libxsmm_blasint set_stride_hint);
LIBXSMM_API libxsmm_meqn_arg_metadata libxsmm_create_meqn_arg_metadata(const libxsmm_blasint eqn_idx, const libxsmm_blasint in_arg_pos);
LIBXSMM_API libxsmm_meqn_op_metadata libxsmm_create_meqn_op_metadata(const libxsmm_blasint eqn_idx, const libxsmm_blasint op_arg_pos);
LIBXSMM_API int libxsmm_meqn_push_back_arg(const libxsmm_meqn_arg_metadata arg_metadata, const libxsmm_meqn_arg_shape arg_shape, libxsmm_matrix_arg_attributes arg_attr);
LIBXSMM_API int libxsmm_meqn_push_back_unary_op(const libxsmm_meqn_op_metadata op_metadata, const libxsmm_meltw_unary_type type, const libxsmm_datatype dtype, const libxsmm_bitfield flags);
LIBXSMM_API int libxsmm_meqn_push_back_binary_op(const libxsmm_meqn_op_metadata op_metadata, const libxsmm_meltw_binary_type type, const libxsmm_datatype dtype, const libxsmm_bitfield flags);
LIBXSMM_API int libxsmm_meqn_push_back_ternary_op(const libxsmm_meqn_op_metadata op_metadata, const libxsmm_meltw_ternary_type type, const libxsmm_datatype dtype, const libxsmm_bitfield flags);
LIBXSMM_API void libxsmm_meqn_tree_print(const libxsmm_blasint idx);
LIBXSMM_API void libxsmm_meqn_rpn_print(const libxsmm_blasint idx);
LIBXSMM_API libxsmm_meqn_function libxsmm_dispatch_meqn(const libxsmm_blasint idx, const libxsmm_meqn_arg_shape out_shape);

/* ---- user key/value registry (reference include/libxsmm.h:106-125): binary keys up to LIBXSMM_DESCRIPTOR_MAXSIZE bytes ---- */
LIBXSMM_API void* libxsmm_xregister(const void* key, size_t key_size, size_t value_size, const void* value_init);
LIBXSMM_API void* libxsmm_xdispatch(const void* key, size_t key_size);
LIBXSMM_API void libxsmm_xrelease(const void* key, size_t key_size);

/* packed DENSE GEMM (EDGE/SeisSol): every matrix element is a vector of `packed_width` independent problems (innermost);
 * F32 / F64; caller-owned handles (libxsmm_release_kernel). Layouts [row][col][packed] with the leading dimensions counted in vectors:
 *   libxsmm_create_packed_gemm        C[n][m][p] (+)= A[k][m][p] * B[n][k][p]
 *   libxsmm_create_packed_gemm_ac_rm  C[m][n][p] (+)= A[m][k][p] * B[k][n]        (B is a plain row-major matrix)
 *   libxsmm_create_packed_gemm_bc_rm  C[m][n][p] (+)= A[m][k]    * B[k][n][p]     (A is a plain row-major matrix) */
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_gemm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width);
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_gemm_ac_rm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width);
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_gemm_bc_rm(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width);
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_spgemm_bcsc(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_spgemm_config spgemm_config);
LIBXSMM_API libxsmm_tilecfgfunction libxsmm_create_tilecfg_packed_spgemm_bcsc(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_spgemm_config spgemm_config);
/* sparse A kept on chip, dense row-major B/C (reference include/libxsmm.h:216-223, used by fsspmdm) */
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_spgemm_csr_areg(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint max_N,
  const unsigned int* row_ptr, const unsigned int* column_idx, const double* values);
LIBXSMM_API void libxsmm_release_kernel(const void* kernel);      /* reference include/libxsmm.h:229 */

/* ---- memory (reference include/libxsmm_malloc.h:17-31): backed by CUDA managed memory so that
 * buffers obtained here are valid on host and device ------------------------------------------- */
LIBXSMM_API void* libxsmm_malloc(size_t size);
LIBXSMM_API void* libxsmm_aligned_malloc(size_t size, size_t alignment);
LIBXSMM_API void libxsmm_free(const void* memory);

/* ---- conversions the kernels are bit-compatible with (reference src/libxsmm_math.c:587-830) ---- */
LIBXSMM_API float libxsmm_convert_bf16_to_f32(libxsmm_bfloat16 in);
LIBXSMM_API float libxsmm_convert_f16_to_f32(libxsmm_float16 in);
LIBXSMM_API libxsmm_bfloat16 libxsmm_convert_f32_to_bf16_rne(float in);
LIBXSMM_API libxsmm_float16 libxsmm_convert_f32_to_f16(float in);

#if defined(__cplusplus)
}
#endif
#endif /* LIBXSMM_H */
