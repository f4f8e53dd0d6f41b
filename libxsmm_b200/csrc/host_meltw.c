/* libxsmm_b200 -- host side of the matrix-eltwise (TPP) handles: shape constructors, dispatch into the
 * registry and the invocation glue that turns a reference argument struct into a kernel launch.
 *
 * Reference roles: src/libxsmm_main.c:3449-3511 (libxsmm_dispatch_meltw_{unary,binary,ternary}),
 * src/libxsmm_generator.c:90-116 (descriptor), argument slots per SURVEY.md appendix C /
 * src/generator_mateltwise_reference_impl.c. Unsupported (op, datatype) pairs answer NULL.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "xb_internal.h"
#include "xb_device.cuh"

extern int xb_host_registry_get(int kind, const void* key, size_t key_size, unsigned int nflops);

LIBXSMM_API libxsmm_meltw_unary_shape libxsmm_create_meltw_unary_shape(libxsmm_blasint m, libxsmm_blasint n,
  libxsmm_blasint ldi, libxsmm_blasint ldo, libxsmm_datatype in0_type, libxsmm_datatype out_type, libxsmm_datatype comp_type)
{
  libxsmm_meltw_unary_shape s;
  memset(&s, 0, sizeof(s));
  s.m = m; s.n = n; s.ldi = ldi; s.ldo = ldo; s.in0_type = in0_type; s.out_type = out_type; s.comp_type = comp_type;
  return s;
}

LIBXSMM_API libxsmm_meltw_binary_shape libxsmm_create_meltw_binary_shape(libxsmm_blasint m, libxsmm_blasint n,
  libxsmm_blasint ldi, libxsmm_blasint ldi2, libxsmm_blasint ldo,
  libxsmm_datatype in0_type, libxsmm_datatype in1_type, libxsmm_datatype out_type, libxsmm_datatype comp_type)
{
  libxsmm_meltw_binary_shape s;
  memset(&s, 0, sizeof(s));
  s.m = m; s.n = n; s.ldi = ldi; s.ldi2 = ldi2; s.ldo = ldo;
  s.in0_type = in0_type; s.in1_type = in1_type; s.out_type = out_type; s.comp_type = comp_type;
  return s;
}

LIBXSMM_API libxsmm_meltw_ternary_shape libxsmm_create_meltw_ternary_shape(libxsmm_blasint m, libxsmm_blasint n,
  libxsmm_blasint ldi, libxsmm_blasint ldi2, libxsmm_blasint ldi3, libxsmm_blasint ldo,
  libxsmm_datatype in0_type, libxsmm_datatype in1_type, libxsmm_datatype in2_type, libxsmm_datatype out_type,
  libxsmm_datatype comp_type)
{
  libxsmm_meltw_ternary_shape s;
  memset(&s, 0, sizeof(s));
  s.m = m; s.n = n; s.ldi = ldi; s.ldi2 = ldi2; s.ldi3 = ldi3; s.ldo = ldo;
  s.in0_type = in0_type; s.in1_type = in1_type; s.in2_type = in2_type; s.out_type = out_type; s.comp_type = comp_type;
  return s;
}

/* ---- the rules: which family serves a descriptor, and which side operands its calls carry --------------------------------- */
static int is_f(int t) {
  return t == LIBXSMM_DATATYPE_F32 || t == LIBXSMM_DATATYPE_BF16 || t == LIBXSMM_DATATYPE_F16 || t == LIBXSMM_DATATYPE_BF8 || t == LIBXSMM_DATATYPE_HF8;
}
static int is_i(int t) { return t == LIBXSMM_DATATYPE_I8 || t == LIBXSMM_DATATYPE_I16 || t == LIBXSMM_DATATYPE_I32; }

int xb_meltw_family(const xb_meltw_desc* d) {
  const int f_in_out = is_f(d->t_in0) && is_f(d->t_out), ts = xb_dev_typesize(d->t_in0);
  const int in64 = d->t_in0 == LIBXSMM_DATATYPE_F64 && d->t_out == LIBXSMM_DATATYPE_F64;
  if (d->op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    switch (d->op) {
      case LIBXSMM_MELTW_TYPE_UNARY_IDENTITY: case LIBXSMM_MELTW_TYPE_UNARY_XOR: case LIBXSMM_MELTW_TYPE_UNARY_X2: case LIBXSMM_MELTW_TYPE_UNARY_DUMP:
      case LIBXSMM_MELTW_TYPE_UNARY_SQRT: case LIBXSMM_MELTW_TYPE_UNARY_NEGATE: case LIBXSMM_MELTW_TYPE_UNARY_INC:
      case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL: case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL_SQRT:
        if (in64 && d->t_comp == LIBXSMM_DATATYPE_F64) return (d->op == LIBXSMM_MELTW_TYPE_UNARY_DUMP) ? XB_FAM_NONE : XB_FAM_MAP;
        return f_in_out ? XB_FAM_MAP : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TANH: case LIBXSMM_MELTW_TYPE_UNARY_TANH_INV: case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID:
      case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID_INV: case LIBXSMM_MELTW_TYPE_UNARY_GELU: case LIBXSMM_MELTW_TYPE_UNARY_GELU_INV:
      case LIBXSMM_MELTW_TYPE_UNARY_EXP: case LIBXSMM_MELTW_TYPE_UNARY_REPLICATE_COL_VAR:
      case LIBXSMM_MELTW_TYPE_UNARY_RELU: case LIBXSMM_MELTW_TYPE_UNARY_RELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU:
      case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_ELU: case LIBXSMM_MELTW_TYPE_UNARY_ELU_INV:
        return f_in_out ? XB_FAM_MAP : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MAX:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MIN: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MAX:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MIN:
        return (in64 || f_in_out) ? XB_FAM_REDUCE : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD: return (in64 || f_in_out) ? XB_FAM_SCALAR : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT: return XB_FAM_TRANSFORM;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2_TO_VNNI2T:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2T_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4T:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4T_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8T:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8T_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD2:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD2:
        return (ts == 2) ? XB_FAM_TRANSFORM : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI4T:
        return (ts <= 2) ? XB_FAM_TRANSFORM : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD4:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI2:
        return (ts == 1) ? XB_FAM_TRANSFORM : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8_TO_VNNI8T:
        return (ts >= 1 && ts <= 2) ? XB_FAM_TRANSFORM : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_GATHER: case LIBXSMM_MELTW_TYPE_UNARY_SCATTER: return (ts >= 1 && ts <= 4) ? XB_FAM_GS : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_QUANT:
        if (d->t_in0 == LIBXSMM_DATATYPE_BF16 && (d->t_out == LIBXSMM_DATATYPE_MXFP4X2 || d->t_out == LIBXSMM_DATATYPE_NVFP4X2 || d->t_out == LIBXSMM_DATATYPE_MXBF8)) return XB_FAM_MXQUANT;
        return (d->t_in0 == LIBXSMM_DATATYPE_F32 && is_i(d->t_out)) ? XB_FAM_QUANT : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_DEQUANT: return (d->t_out == LIBXSMM_DATATYPE_F32 && is_i(d->t_in0)) ? XB_FAM_QUANT : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_DROPOUT: case LIBXSMM_MELTW_TYPE_UNARY_DROPOUT_INV: return f_in_out ? XB_FAM_DROPOUT : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_UNZIP: case LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X2: case LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X3:
        return (d->t_in0 == LIBXSMM_DATATYPE_F32) ? XB_FAM_SPLIT : XB_FAM_NONE;
      default: return XB_FAM_NONE;
    }
  }
  if (d->op_class == LIBXSMM_MELTW_OPERATION_BINARY) {
    const int all64 = in64 && d->t_in1 == LIBXSMM_DATATYPE_F64 && d->t_comp == LIBXSMM_DATATYPE_F64, f3 = f_in_out && is_f(d->t_in1);
    switch (d->op) {
      case LIBXSMM_MELTW_TYPE_BINARY_ADD: case LIBXSMM_MELTW_TYPE_BINARY_MUL: case LIBXSMM_MELTW_TYPE_BINARY_SUB:
      case LIBXSMM_MELTW_TYPE_BINARY_DIV: case LIBXSMM_MELTW_TYPE_BINARY_MULADD: case LIBXSMM_MELTW_TYPE_BINARY_MAX:
      case LIBXSMM_MELTW_TYPE_BINARY_MIN:
        return (all64 || f3) ? XB_FAM_MAP : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GE: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LT:
      case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LE: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_EQ: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_NE:
        return (is_f(d->t_in0) && is_f(d->t_in1)) ? XB_FAM_MAP : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_BINARY_ZIP:
        return (d->t_in0 == LIBXSMM_DATATYPE_U16 || d->t_in0 == LIBXSMM_DATATYPE_BF16 || d->t_in0 == LIBXSMM_DATATYPE_I16) ? XB_FAM_MAP : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD: return (all64 || f3) ? XB_FAM_SCALAR : XB_FAM_NONE;
      default: return XB_FAM_NONE;
    }
  }
  if (d->op_class == LIBXSMM_MELTW_OPERATION_TERNARY) {
    const int f3 = f_in_out && is_f(d->t_in1);
    switch (d->op) {
      case LIBXSMM_MELTW_TYPE_TERNARY_SELECT:
        return ((in64 && d->t_in1 == LIBXSMM_DATATYPE_F64 && d->t_in2 == LIBXSMM_DATATYPE_F64 && d->t_comp == LIBXSMM_DATATYPE_F64) || f3) ? XB_FAM_MAP : XB_FAM_NONE;
      case LIBXSMM_MELTW_TYPE_TERNARY_MULADD: case LIBXSMM_MELTW_TYPE_TERNARY_NMULADD: return (f3 && is_f(d->t_in2)) ? XB_FAM_MAP : XB_FAM_NONE;
      default: return XB_FAM_NONE;
    }
  }
  return XB_FAM_NONE;
}

/* Which side operands a call of a served descriptor carries (reference src/generator_mateltwise_reference_impl.c: the relu family
 * :2138-2194, dropout :2091 and :43-73, quantisers :2195-2360, reductions :1065-1443, gather / scatter :1444-1794). Stochastic rounding
 * draws from op.secondary when it rounds to BF8 (:310-316): in the element-wise unary ops of the generic loop (:2470-2498) over a
 * non-F64 input, and in every binary map and ternary op. */
int xb_meltw_sides(const xb_meltw_desc* d) {
  const int fam = xb_meltw_family(d);
  const unsigned int f = d->flags;
  const int to_bf8 = d->t_out == LIBXSMM_DATATYPE_BF8;
  const int sr = ((f & LIBXSMM_MELTW_FLAG_UNARY_STOCHASTIC_ROUND) && to_bf8 && d->t_in0 != LIBXSMM_DATATYPE_F64) ? XB_MSIDE_STATE : 0;
  if (d->op_class == LIBXSMM_MELTW_OPERATION_BINARY) {
    return ((f & LIBXSMM_MELTW_FLAG_BINARY_STOCHASTIC_ROUND) && to_bf8 && d->op < LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT
            && d->op != LIBXSMM_MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD && d->op != LIBXSMM_MELTW_TYPE_BINARY_ZIP) ? XB_MSIDE_STATE : 0;
  }
  if (d->op_class == LIBXSMM_MELTW_OPERATION_TERNARY) return ((f & LIBXSMM_MELTW_FLAG_TERNARY_STOCHASTIC_ROUND) && to_bf8) ? XB_MSIDE_STATE : 0;
  switch (d->op) {
    case LIBXSMM_MELTW_TYPE_UNARY_RELU: return (f & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) ? XB_MSIDE_MASK_OUT : 0;
    case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU: case LIBXSMM_MELTW_TYPE_UNARY_ELU:
      return XB_MSIDE_ALPHA | ((f & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) ? XB_MSIDE_MASK_OUT : 0);
    case LIBXSMM_MELTW_TYPE_UNARY_RELU_INV: return XB_MSIDE_IN_AUX;
    case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_ELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_DROPOUT_INV:
      return XB_MSIDE_ALPHA | XB_MSIDE_IN_AUX;
    case LIBXSMM_MELTW_TYPE_UNARY_DROPOUT:
      return XB_MSIDE_ALPHA | XB_MSIDE_STATE | ((f & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) ? XB_MSIDE_MASK_OUT : 0);
    case LIBXSMM_MELTW_TYPE_UNARY_QUANT: case LIBXSMM_MELTW_TYPE_UNARY_DEQUANT:   /* the scale: NO_SCF_QUANT or a NULL pointer stand for 1 */
      return (fam == XB_FAM_MXQUANT) ? XB_MSIDE_OUT_AUX : XB_MSIDE_IN_AUX;
    case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MAX: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MIN: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX:
      return ((f & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP) && !(f & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_ROWS)) ? XB_MSIDE_ARGOP : 0;
    case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MAX: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MIN:
      if (f & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP) return XB_MSIDE_IN_AUX | XB_MSIDE_COUNT | XB_MSIDE_RUNTIME | XB_MSIDE_ARGOP;
      /* fall through */
    case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_ADD: return XB_MSIDE_IN_AUX | XB_MSIDE_COUNT | XB_MSIDE_RUNTIME;
    case LIBXSMM_MELTW_TYPE_UNARY_GATHER: return XB_MSIDE_IN_AUX | XB_MSIDE_RUNTIME;
    case LIBXSMM_MELTW_TYPE_UNARY_SCATTER: case LIBXSMM_MELTW_TYPE_UNARY_UNZIP: case LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X2:
    case LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X3: return XB_MSIDE_OUT_AUX | XB_MSIDE_RUNTIME;
    case LIBXSMM_MELTW_TYPE_UNARY_REPLICATE_COL_VAR: return XB_MSIDE_COUNT | sr;
    case LIBXSMM_MELTW_TYPE_UNARY_DUMP: return XB_MSIDE_COPY_OUT | sr;
    default: return (fam == XB_FAM_MAP) ? sr : 0;       /* the other maps of the generic loop; transforms and reductions carry nothing */
  }
}

static const void* xb_dispatch_meltw(xb_meltw_desc* d) {
  int slot;
  LIBXSMM_INIT
  if (d->m <= 0 || d->n <= 0 || xb_meltw_family(d) == XB_FAM_NONE) return NULL;
  slot = xb_host_registry_get(XB_KIND_MELTW, d, sizeof(*d), 0);
  return (slot < 0) ? NULL : xb_thunk(slot);
}

LIBXSMM_API libxsmm_meltwfunction_unary libxsmm_dispatch_meltw_unary(const libxsmm_meltw_unary_type unary_type,
  const libxsmm_meltw_unary_shape s, const libxsmm_bitfield unary_flags)
{
  xb_meltw_desc d;
  memset(&d, 0, sizeof(d));
  d.op_class = LIBXSMM_MELTW_OPERATION_UNARY; d.op = (int)unary_type; d.flags = unary_flags;
  d.m = s.m; d.n = s.n; d.ldi = s.ldi; d.ldo = s.ldo;
  d.t_in0 = (int)s.in0_type; d.t_in1 = d.t_in2 = LIBXSMM_DATATYPE_UNSUPPORTED; d.t_out = (int)s.out_type; d.t_comp = (int)s.comp_type;
  return (libxsmm_meltwfunction_unary)xb_dispatch_meltw(&d);
}

LIBXSMM_API libxsmm_meltwfunction_binary libxsmm_dispatch_meltw_binary(const libxsmm_meltw_binary_type binary_type,
  const libxsmm_meltw_binary_shape s, const libxsmm_bitfield binary_flags)
{
  xb_meltw_desc d;
  memset(&d, 0, sizeof(d));
  d.op_class = LIBXSMM_MELTW_OPERATION_BINARY; d.op = (int)binary_type; d.flags = binary_flags;
  d.m = s.m; d.n = s.n; d.ldi = s.ldi; d.ldi2 = s.ldi2; d.ldo = s.ldo;
  d.t_in0 = (int)s.in0_type; d.t_in1 = (int)s.in1_type; d.t_in2 = LIBXSMM_DATATYPE_UNSUPPORTED; d.t_out = (int)s.out_type; d.t_comp = (int)s.comp_type;
  return (libxsmm_meltwfunction_binary)xb_dispatch_meltw(&d);
}

LIBXSMM_API libxsmm_meltwfunction_ternary libxsmm_dispatch_meltw_ternary(const libxsmm_meltw_ternary_type ternary_type,
  const libxsmm_meltw_ternary_shape s, const libxsmm_bitfield ternary_flags)
{
  xb_meltw_desc d;
  memset(&d, 0, sizeof(d));
  d.op_class = LIBXSMM_MELTW_OPERATION_TERNARY; d.op = (int)ternary_type; d.flags = ternary_flags;
  d.m = s.m; d.n = s.n; d.ldi = s.ldi; d.ldi2 = s.ldi2; d.ldi3 = s.ldi3; d.ldo = s.ldo;
  d.t_in0 = (int)s.in0_type; d.t_in1 = (int)s.in1_type; d.t_in2 = (int)s.in2_type; d.t_out = (int)s.out_type; d.t_comp = (int)s.comp_type;
  return (libxsmm_meltwfunction_ternary)xb_dispatch_meltw(&d);
}

/* ---- descriptor-based dispatch (reference include/libxsmm.h:143, include/libxsmm_generator.h:48-57) ---------------
 * libxsmm_dispatch_meltw takes the library's packed descriptor (reference src/libxsmm_main.h:292-302): six 32-bit
 * extents, the five datatypes in 6-bit fields (IN0 [5:0], IN1 [11:6], IN2 [17:12], OUT [23:18], COMP [29:24]), the
 * flags and the operation class (bits 2:0) / operation type (bits 15:3). Callers fill it through the two init helpers. */
struct libxsmm_meltw_descriptor {
  unsigned int m, n, ldi, ldo, ldi2, ldi3;
  unsigned int datatypes;
  unsigned short flags;
  unsigned short param_operation;
} __attribute__((packed));

static unsigned int xb_meltw_pack_types(int in0, int in1, int in2, int out, int comp) {
  return ((unsigned int)in0 & 0x3fu) | (((unsigned int)in1 & 0x3fu) << 6) | (((unsigned int)in2 & 0x3fu) << 12)
       | (((unsigned int)out & 0x3fu) << 18) | (((unsigned int)comp & 0x3fu) << 24);
}

LIBXSMM_API libxsmm_meltw_descriptor* libxsmm_meltw_descriptor_init2(libxsmm_descriptor_blob* blob,
  libxsmm_datatype in0_type, libxsmm_datatype in1_type, libxsmm_datatype in2_type, libxsmm_datatype comp_type, libxsmm_datatype out_type,
  libxsmm_blasint m, libxsmm_blasint n, libxsmm_blasint ldi, libxsmm_blasint ldo, libxsmm_blasint ldi2, libxsmm_blasint ldi3,
  unsigned short flags, unsigned short param, unsigned char operation)
{
  libxsmm_meltw_descriptor* d = (libxsmm_meltw_descriptor*)blob;
  if (blob == NULL) return NULL;
  memset(blob, 0, sizeof(*blob));
  d->m = (unsigned int)m; d->n = (unsigned int)n; d->ldi = (unsigned int)ldi; d->ldo = (unsigned int)ldo; d->ldi2 = (unsigned int)ldi2; d->ldi3 = (unsigned int)ldi3;
  d->datatypes = xb_meltw_pack_types((int)in0_type, (int)in1_type, (int)in2_type, (int)out_type, (int)comp_type);
  d->flags = flags;
  d->param_operation = (unsigned short)((operation & 0x7u) | ((unsigned int)param << 3));
  return d;
}

LIBXSMM_API libxsmm_meltw_descriptor* libxsmm_meltw_descriptor_init(libxsmm_descriptor_blob* blob,
  libxsmm_datatype in_type, libxsmm_datatype out_type, libxsmm_blasint m, libxsmm_blasint n, libxsmm_blasint ldi, libxsmm_blasint ldo,
  unsigned short flags, unsigned short param, unsigned char operation)
{
  return libxsmm_meltw_descriptor_init2(blob, in_type, LIBXSMM_DATATYPE_IMPLICIT, LIBXSMM_DATATYPE_IMPLICIT, LIBXSMM_DATATYPE_IMPLICIT, out_type,
                                        m, n, ldi, ldo, 0, 0, flags, param, operation);
}

LIBXSMM_API libxsmm_xmeltwfunction libxsmm_dispatch_meltw(const libxsmm_meltw_descriptor* descriptor) {
  libxsmm_xmeltwfunction result;
  xb_meltw_desc d;
  result.xmeltw = NULL;
  if (descriptor == NULL) return result;
  memset(&d, 0, sizeof(d));
  d.op_class = (int)(descriptor->param_operation & 0x7u); d.op = (int)(descriptor->param_operation >> 3); d.flags = descriptor->flags;
  d.m = (int)descriptor->m; d.n = (int)descriptor->n; d.ldi = (int)descriptor->ldi; d.ldo = (int)descriptor->ldo;
  d.t_in0 = (int)(descriptor->datatypes & 0x3fu); d.t_out = (int)((descriptor->datatypes >> 18) & 0x3fu); d.t_comp = (int)((descriptor->datatypes >> 24) & 0x3fu);
  /* the registry key is the one the typed dispatchers build, so both routes return the identical handle */
  d.t_in1 = d.t_in2 = LIBXSMM_DATATYPE_UNSUPPORTED;
  if (d.op_class == LIBXSMM_MELTW_OPERATION_BINARY || d.op_class == LIBXSMM_MELTW_OPERATION_TERNARY) {
    d.ldi2 = (int)descriptor->ldi2; d.t_in1 = (int)((descriptor->datatypes >> 6) & 0x3fu);
  }
  if (d.op_class == LIBXSMM_MELTW_OPERATION_TERNARY) { d.ldi3 = (int)descriptor->ldi3; d.t_in2 = (int)((descriptor->datatypes >> 12) & 0x3fu); }
  if (d.op_class != LIBXSMM_MELTW_OPERATION_UNARY && d.op_class != LIBXSMM_MELTW_OPERATION_BINARY && d.op_class != LIBXSMM_MELTW_OPERATION_TERNARY) return result;
  result.xmeltw = (void (*)(const void*))(uintptr_t)xb_dispatch_meltw(&d);
  return result;
}

/* ---- invocation -------------------------------------------------------------------------------------------- */
typedef struct xb_stage { void* host; void* dev; size_t bytes; } xb_stage;
/* batch: nothing is staged; operands pass through, a pageable one sets `pageable`, and every output is recorded in out[] with the
 * bytes one call writes through it (the batch form checks its stride against them) */
typedef struct xb_stager { xb_stage out[4]; int nout; int staged; int failed; int batch; int pageable; } xb_stager;

static const void* stage_in(xb_stager* st, const void* p, size_t bytes) {
  if (st->batch) { if (p != NULL && xb_rt_ptr_kind(p) == 0) st->pageable = 1; return p; }
  if (p == NULL || xb_rt_ptr_kind(p) != 0) return p;
  else {
    void* d = xb_rt_scratch(bytes ? bytes : 1);
    if (d == NULL) { st->failed = 1; return NULL; }
    xb_rt_upload(d, p, bytes);
    st->staged = 1;
    return d;
  }
}
/* output staged in AND out (partial writes must preserve what the kernel does not touch) */
static void* stage_inout(xb_stager* st, void* p, size_t bytes) {
  if (st->batch) {
    if (p == NULL) return p;
    if (xb_rt_ptr_kind(p) == 0) st->pageable = 1;
    if (st->nout >= 4) { st->failed = 1; return p; }
    st->out[st->nout].host = st->out[st->nout].dev = p; st->out[st->nout].bytes = bytes; ++st->nout;
    return p;
  }
  if (p == NULL || xb_rt_ptr_kind(p) != 0) return p;
  else {
    void* d = xb_rt_scratch(bytes ? bytes : 1);
    if (d == NULL || st->nout >= 4) { st->failed = 1; return NULL; }
    xb_rt_upload(d, p, bytes);
    st->out[st->nout].host = p; st->out[st->nout].dev = d; st->out[st->nout].bytes = bytes; ++st->nout;
    st->staged = 1;
    return d;
  }
}

static size_t in_extent(const xb_meltw_desc* d, unsigned int row, unsigned int col, unsigned int sca, long long ld, long long n) {
  if (row) return (size_t)((n - 1) * ld + 1);
  if (col) return (size_t)d->m;
  if (sca) return 1;
  return (size_t)((n - 1) * ld + d->m);
}

/* STOCHASTIC_ROUND to BF8 (libxsmm_elementwise_store_value, :310-316): the 4 x 16-word generator state in op.secondary is read and
 * advanced; one random byte per element goes through device scratch */
static void stage_stochastic(xb_stager* st, xb_meltw_args* a, const void* state, long long elements) {
  if (state == NULL || elements <= 0) { st->failed = 1; return; }
  a->rng = stage_inout(st, (void*)(uintptr_t)state, 64 * sizeof(unsigned int));
  a->rnd8 = (unsigned char*)xb_rt_scratch((size_t)elements);
  if (a->rng == NULL || a->rnd8 == NULL) st->failed = 1;
}

/* the kernel arguments of one call: operands staged through `st` (or, for a batch, checked and recorded there). Returns 1 if the
 * call cannot run; the error is noted and the scratch arena reset. */
static int meltw_args(const xb_meltw_desc* d, const void* param, xb_meltw_args* out_args, xb_stager* pst) {
  xb_meltw_args a; xb_stager st = *pst;
  const size_t ts_in = libxsmm_typesize((libxsmm_datatype)d->t_in0), ts_out = libxsmm_typesize((libxsmm_datatype)d->t_out);
  const size_t mask_ld_i = (size_t)LIBXSMM_UP(d->ldi, 16);
  memset(&a, 0, sizeof(a));
  if (d->op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    const libxsmm_meltw_unary_param* p = (const libxsmm_meltw_unary_param*)param;
    const int op = d->op, sides = xb_meltw_sides(d);
    const size_t idx = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_IDX_SIZE_4BYTES) ? 4 : 8;
    long long n = d->n;
    size_t ext_in, ext_out = ((size_t)(d->n - 1) * d->ldo + d->m) * ts_out, mx_scales = 0;
    if ((sides & (XB_MSIDE_COUNT | XB_MSIDE_RUNTIME)) == XB_MSIDE_COUNT) {       /* op.primary: the run-time column count */
      n = (long long)*(const unsigned long long*)p->op.primary; a.n_rt = (unsigned long long)n; ext_out = ((size_t)(n - 1) * d->ldo + d->m) * ts_out;
    }
    ext_in = in_extent(d, d->flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_ROW, (d->flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_COL) | (op == LIBXSMM_MELTW_TYPE_UNARY_REPLICATE_COL_VAR),
                       d->flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_SCALAR, d->ldi, n) * ts_in;
    a.alpha = (sides & XB_MSIDE_ALPHA) ? xb_meltw_scalar(p->op.primary) : 1.0f;
    if (xb_meltw_family(d) == XB_FAM_QUANT && (d->flags & LIBXSMM_MELTW_FLAG_UNARY_NO_SCF_QUANT) == 0 && p->in.secondary != NULL) a.alpha = *(const float*)p->in.secondary;
    if (xb_meltw_family(d) == XB_FAM_MXQUANT) {   /* block formats: 4-bit data at ldo/2 bytes per column, one scale byte per block in out.secondary (reference :2247-2326) */
      const int blk = (d->t_out == LIBXSMM_DATATYPE_NVFP4X2) ? 16 : 32;
      const size_t per = (d->t_out == LIBXSMM_DATATYPE_MXBF8) ? 1 : 2;
      ext_out = ((size_t)(d->n - 1) * (d->ldo / per) + (size_t)(d->m / blk) * blk / per);
      mx_scales = ((size_t)(d->n - 1) * (d->ldo / blk) + (size_t)(d->m / blk));
    }
    /* shapes of the data-movement and reduction families */
    if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT) ext_out = ((size_t)(d->m - 1) * d->ldo + d->n) * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD) ext_out = (size_t)d->ldo * LIBXSMM_UP(d->n, 2) * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4_PAD) ext_out = (size_t)d->ldo * LIBXSMM_UP(d->n, 4) * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2T || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4T) ext_out = (size_t)d->ldo * d->m * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2_TO_VNNI2T || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI4T) { ext_in = (size_t)d->ldi * d->n * ts_in; ext_out = (size_t)d->ldo * d->m * ts_out; }
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2T_TO_NORM || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4T_TO_NORM) { ext_in = (size_t)d->ldi * d->n * ts_in; ext_out = ((size_t)(d->m - 1) * d->ldo + d->n) * ts_out; }
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_NORM) ext_in = (size_t)d->ldi * LIBXSMM_UP(d->n, 4) * ts_in;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8_PAD) ext_out = (size_t)d->ldo * LIBXSMM_UP(d->n, 8) * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8T) ext_out = (size_t)d->ldo * d->m * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8_TO_VNNI8T) { ext_in = (size_t)d->ldi * d->n * ts_in; ext_out = (size_t)d->ldo * d->m * ts_out; }
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8T_TO_NORM) { ext_in = (size_t)d->ldi * d->n * ts_in; ext_out = ((size_t)(d->m - 1) * d->ldo + d->n) * ts_out; }
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI2) { ext_in = (size_t)d->ldi * LIBXSMM_UP(d->n, 4) * ts_in; ext_out = (size_t)d->ldo * LIBXSMM_UP(d->n, 2) * ts_out; }
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD2 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD2) ext_out = (size_t)d->ldo * LIBXSMM_UP(d->n, 2) * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD4 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD4) ext_out = (size_t)d->ldo * LIBXSMM_UP(d->n, 4) * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD2 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4) ext_out = (size_t)d->ldo * d->n * ts_out;
    else if (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD) ext_out = ts_out;
    else if (op >= LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ADD && op <= LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MAX) {
      const size_t rs = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_ROWS) ? (size_t)d->n : (size_t)d->ldo;
      ext_out = rs * ts_out * ((op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD) ? 2 : 1);
    } else if (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MIN || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX) {
      ext_out = ((d->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_ROWS) ? (size_t)d->n : (size_t)d->m) * ts_out;
    }
    if ((sides & XB_MSIDE_RUNTIME) && xb_meltw_family(d) != XB_FAM_SPLIT) {
      /* extents depend on run-time indices: operands must be device-accessible (device, managed or pinned) */
      if (xb_rt_ptr_kind(p->in.primary) == 0 || xb_rt_ptr_kind(p->out.primary) == 0) { xb_rt_note_error(1, "meltw: indexed op needs device-accessible memory"); return 1; }
      a.in0 = p->in.primary; a.out = p->out.primary; a.in_aux = p->in.secondary; a.out_aux = p->out.secondary;
      if (sides & XB_MSIDE_COUNT) {                  /* in.tertiary: the number of column indices in in.secondary */
        a.n_rt = *(const unsigned long long*)p->in.tertiary;
        a.in_aux = stage_in(&st, p->in.secondary, (size_t)a.n_rt * idx);
      } else {
        const size_t isz = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_IDX_SIZE_8BYTES) ? 8 : 4;
        const size_t cnt = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_GS_COLS) ? (size_t)d->n : ((d->flags & LIBXSMM_MELTW_FLAG_UNARY_GS_ROWS) ? (size_t)d->m : (size_t)d->m * d->n);
        if (sides & XB_MSIDE_IN_AUX) a.in_aux = stage_in(&st, p->in.secondary, cnt * isz);
        else a.out_aux = (void*)(uintptr_t)stage_in(&st, p->out.secondary, cnt * isz);
      }
    } else {
      a.in0 = stage_in(&st, p->in.primary, ext_in);
      if (sides & XB_MSIDE_RUNTIME) {
        /* several bf16 planes behind ONE output pointer at caller-given byte distances (out.secondary): the output must be
         * device-accessible, there is no single extent to stage */
        const unsigned long long* offs = (const unsigned long long*)p->out.secondary;
        const int noff = (op == LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X3) ? 2 : 1;
        if (offs == NULL || xb_rt_ptr_kind(p->out.primary) == 0) { xb_rt_note_error(1, "meltw: unzip/decomp need a device-accessible output and plane offsets"); xb_rt_scratch_reset(); return 1; }
        if (xb_rt_ptr_kind(offs) == 1) xb_rt_memcpy(a.off, offs, noff * sizeof(unsigned long long)); else memcpy(a.off, offs, noff * sizeof(unsigned long long));
        a.out = p->out.primary;
      } else a.out = stage_inout(&st, p->out.primary, ext_out);
      if ((sides & XB_MSIDE_OUT_AUX) && mx_scales != 0) { a.out_aux = stage_inout(&st, p->out.secondary, mx_scales); if (a.out_aux == NULL) st.failed = 1; }
      if (sides & XB_MSIDE_COPY_OUT) { a.out_aux = stage_inout(&st, p->out.secondary, ext_out); if (a.out_aux == NULL) st.failed = 1; }
      if ((sides & XB_MSIDE_STATE) && xb_meltw_family(d) != XB_FAM_DROPOUT) stage_stochastic(&st, &a, p->op.secondary, (long long)d->m * n);
      else if (sides & XB_MSIDE_STATE) {             /* dropout: op.secondary, generator state, read AND advanced (:2091, :43-73) */
        a.rng = stage_inout(&st, p->op.secondary, 64 * sizeof(unsigned int));
        a.rnd = (float*)xb_rt_scratch((size_t)LIBXSMM_UPDIV(d->m, 16) * d->n * 16 * sizeof(float));
        if (a.rng == NULL || a.rnd == NULL) st.failed = 1;
      }
      if (sides & XB_MSIDE_MASK_OUT) a.out_aux = stage_inout(&st, p->out.secondary, xb_meltw_mask_bytes(d->ldo, d->n));
      if ((sides & XB_MSIDE_IN_AUX) && xb_meltw_family(d) != XB_FAM_QUANT) {   /* the forward output of ELU_INV, else a bit mask */
        const size_t mld = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) ? mask_ld_i : (size_t)d->ldi;
        a.in_aux = stage_in(&st, p->in.secondary, (op == LIBXSMM_MELTW_TYPE_UNARY_ELU_INV) ? ((size_t)(d->n - 1) * d->ldi + d->m) * ts_in : (mld / 8) * (size_t)d->n + 1);
      }
    }
    /* arg-max/min column indices land in out.secondary (reference :1243-1275), staged in and out so that a pageable index buffer is
     * never handed to the kernel */
    if (sides & XB_MSIDE_ARGOP) { a.out_aux = stage_inout(&st, p->out.secondary, (size_t)d->m * idx); if (a.out_aux == NULL) st.failed = 1; }
  } else if (d->op_class == LIBXSMM_MELTW_OPERATION_BINARY) {
    const libxsmm_meltw_binary_param* p = (const libxsmm_meltw_binary_param*)param;
    const size_t ts1 = libxsmm_typesize((libxsmm_datatype)d->t_in1);
    size_t ext_out = ((size_t)(d->n - 1) * d->ldo + d->m) * ts_out;
    if (d->op >= LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT) ext_out = xb_meltw_mask_bytes(d->ldo, d->n);
    if (d->op == LIBXSMM_MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD) ext_out = ts_out;
    if (d->op == LIBXSMM_MELTW_TYPE_BINARY_ZIP) ext_out = ((size_t)(d->n - 1) * d->ldo + d->m) * 4;
    a.in0 = stage_in(&st, p->in0.primary, in_extent(d, d->flags & LIBXSMM_MELTW_FLAG_BINARY_BCAST_ROW_IN_0, d->flags & LIBXSMM_MELTW_FLAG_BINARY_BCAST_COL_IN_0,
                                                     d->flags & LIBXSMM_MELTW_FLAG_BINARY_BCAST_SCALAR_IN_0, d->ldi, d->n) * ts_in);
    a.in1 = stage_in(&st, p->in1.primary, in_extent(d, d->flags & LIBXSMM_MELTW_FLAG_BINARY_BCAST_ROW_IN_1, d->flags & LIBXSMM_MELTW_FLAG_BINARY_BCAST_COL_IN_1,
                                                     d->flags & LIBXSMM_MELTW_FLAG_BINARY_BCAST_SCALAR_IN_1, d->ldi2, d->n) * ts1);
    a.out = stage_inout(&st, p->out.primary, ext_out);
    if (xb_meltw_sides(d) & XB_MSIDE_STATE) stage_stochastic(&st, &a, p->op.secondary, (long long)d->m * d->n);
  } else {
    const libxsmm_meltw_ternary_param* p = (const libxsmm_meltw_ternary_param*)param;
    const size_t ts1 = libxsmm_typesize((libxsmm_datatype)d->t_in1), ts2 = libxsmm_typesize((libxsmm_datatype)d->t_in2);
    a.in0 = stage_in(&st, p->in0.primary, in_extent(d, d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_0, d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_0,
                                                     d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_0, d->ldi, d->n) * ts_in);
    a.in1 = stage_in(&st, p->in1.primary, in_extent(d, d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_1, d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_1,
                                                     d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_1, d->ldi2, d->n) * ts1);
    if (d->op == LIBXSMM_MELTW_TYPE_TERNARY_SELECT) a.in2 = stage_in(&st, p->in2.primary, xb_meltw_mask_bytes(d->ldi3, d->n));
    else a.in2 = stage_in(&st, p->in2.primary, in_extent(d, d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_2, d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_2,
                                                          d->flags & LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_2, d->ldi3, d->n) * ts2);
    a.out = stage_inout(&st, p->out.primary, ((size_t)(d->n - 1) * d->ldo + d->m) * ts_out);
    if (xb_meltw_sides(d) & XB_MSIDE_STATE) stage_stochastic(&st, &a, p->op.secondary, (long long)d->m * d->n);
  }
  *pst = st; *out_args = a;
  if (st.failed) { xb_rt_note_error(2, "meltw: staging failed"); xb_rt_scratch_reset(); return 1; }
  return 0;
}

void xb_invoke_meltw(const xb_slot* s, const void* param) {
  const xb_meltw_desc* d = &s->u.meltw;
  xb_meltw_args a; xb_stager st;
  int rc, i;
  memset(&st, 0, sizeof(st));
  if (meltw_args(d, param, &a, &st) != 0) return;
  rc = xb_meltw_launch(d, &a);
  if (rc != 0) { xb_rt_scratch_reset(); return; }
  for (i = 0; i < st.nout; ++i) xb_rt_memcpy_async(st.out[i].host, st.out[i].dev, st.out[i].bytes);
  if (st.staged || xb_rt_blocking()) { xb_rt_sync(); xb_rt_scratch_reset(); }
}

/* ---- strided batch: `count` calls of one handle in one launch ------------------------------------------------------------
 * Calls whose kernel carries per-call state or run-time extents are refused: the dropout generator chains call to call, stochastic
 * rounding draws from a state in op.secondary, the others read their extents, indices or plane offsets at run time. */
int xb_meltw_batchable(const xb_meltw_desc* d) {
  const unsigned int sr = (d->op_class == LIBXSMM_MELTW_OPERATION_UNARY) ? LIBXSMM_MELTW_FLAG_UNARY_STOCHASTIC_ROUND
                        : (d->op_class == LIBXSMM_MELTW_OPERATION_BINARY ? LIBXSMM_MELTW_FLAG_BINARY_STOCHASTIC_ROUND : LIBXSMM_MELTW_FLAG_TERNARY_STOCHASTIC_ROUND);
  /* kept as it was (a follow-up): the STOCHASTIC_ROUND flag refuses the batch even where the op does not round stochastically */
  return (xb_meltw_sides(d) & (XB_MSIDE_STATE | XB_MSIDE_COUNT | XB_MSIDE_RUNTIME)) == 0 && (d->flags & sr) == 0;
}

float xb_meltw_scalar(const void* p) {
  float v;
  if (xb_rt_ptr_kind(p) == 1) xb_rt_memcpy(&v, p, sizeof(v)); else v = *(const float*)p;
  return v;
}

LIBXSMM_API int libxsmm_b200_meltw_batch_strided(const void* kernel, const void* param, const libxsmm_b200_meltw_strides* strides, long long count) {
  const xb_slot* s = xb_slot_of(kernel);
  const xb_meltw_desc* d;
  xb_meltw_args a; xb_stager st;
  void* outs[2] = { NULL, NULL }; long long out_strides[2] = { 0, 0 };
  int rc, i, k;
  if (s == NULL || s->kind != XB_KIND_MELTW || param == NULL || strides == NULL || count < 0) return -1;
  d = &s->u.meltw;
  if (!xb_meltw_batchable(d)) return LIBXSMM_B200_ERROR_NOT_BATCHABLE;
  if (strides->in0 < 0 || strides->in1 < 0 || strides->in2 < 0 || strides->in_aux < 0 || strides->out < 0 || strides->out_aux < 0) return -1;
  if (count == 0) return 0;
  memset(&st, 0, sizeof(st)); st.batch = 1;
  if (meltw_args(d, param, &a, &st) != 0) return -1;
  if (st.pageable) return -4;                           /* no staging path: device, managed or pinned operands only */
  /* every output a call writes must not reach into the next call's */
  if (d->op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    const libxsmm_meltw_unary_param* p = (const libxsmm_meltw_unary_param*)param;
    outs[0] = p->out.primary; outs[1] = p->out.secondary; out_strides[0] = strides->out; out_strides[1] = strides->out_aux;
    a.s_in0 = strides->in0; a.s_in_aux = strides->in_aux; a.s_out = strides->out; a.s_out_aux = strides->out_aux;
  } else {
    outs[0] = (d->op_class == LIBXSMM_MELTW_OPERATION_BINARY) ? ((const libxsmm_meltw_binary_param*)param)->out.primary
                                                               : ((const libxsmm_meltw_ternary_param*)param)->out.primary;
    out_strides[0] = strides->out;
    a.s_in0 = strides->in0; a.s_in1 = strides->in1; a.s_in2 = strides->in2; a.s_out = strides->out;
  }
  if (count > 1) for (i = 0; i < st.nout; ++i) for (k = 0; k < 2; ++k) {
    if (outs[k] != NULL && st.out[i].host == outs[k] && out_strides[k] < (long long)st.out[i].bytes) return -1;
  }
  a.count = count;
  rc = xb_meltw_launch(d, &a);
  if (rc == 0 && xb_rt_blocking()) rc = xb_rt_sync();
  return rc;
}
