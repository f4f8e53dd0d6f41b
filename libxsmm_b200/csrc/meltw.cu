// libxsmm_b200 -- matrix-eltwise (TPP) kernels for sm_90a: unary / binary / ternary maps with
// row/column/scalar broadcast and bitmasks, reductions, layout transforms, gather/scatter and
// (de)quantisation. All matrices are column-major, element (i,j) at i + j*ld.
//
// Semantics follow the reference's portable kernels in src/generator_mateltwise_reference_impl.c:
//   operand indexing with broadcast ........ :241-272      generic unary ops ........... :76-139, :2470-2498
//   RELU/LEAKY_RELU/ELU (+bitmask), inverse  :2138-2194    reductions .................. :1065-1443
//   gather / scatter ........................ :1444-1794    transforms .................. :377-1062
//   quant / dequant ......................... :2195-2360    binary / ternary ............ :2505-2660
// Values are loaded to f32 (bf16 loads flush denormals like libxsmm_convert_bf16_to_f32), computed in
// f32 (f64 only if every type is F64) and stored with round-to-nearest-even. Data-movement kernels
// (transforms, gather/scatter) are bit-exact. Mapping: one warp per (column, 32-row chunk), so loads
// and stores are coalesced along i and a bitmask byte is assembled with one __ballot_sync.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <float.h>
#include <type_traits>
#include "xb_internal.h"
#include "xb_device.cuh"

namespace {

enum { FAM_NONE = 0, FAM_MAP, FAM_REDUCE, FAM_SCALAR, FAM_TRANSFORM, FAM_GS, FAM_QUANT, FAM_DROPOUT, FAM_SPLIT, FAM_MXQUANT };

__host__ __device__ inline bool is_f(int t) {
  return t == LIBXSMM_DATATYPE_F32 || t == LIBXSMM_DATATYPE_BF16 || t == LIBXSMM_DATATYPE_F16 || t == LIBXSMM_DATATYPE_BF8 || t == LIBXSMM_DATATYPE_HF8;
}

__host__ __device__ inline int family_of(const xb_meltw_desc& d) {
  if (d.op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    switch (d.op) {
      case LIBXSMM_MELTW_TYPE_UNARY_IDENTITY: case LIBXSMM_MELTW_TYPE_UNARY_XOR: case LIBXSMM_MELTW_TYPE_UNARY_X2: case LIBXSMM_MELTW_TYPE_UNARY_DUMP:
      case LIBXSMM_MELTW_TYPE_UNARY_SQRT: case LIBXSMM_MELTW_TYPE_UNARY_NEGATE: case LIBXSMM_MELTW_TYPE_UNARY_INC:
      case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL: case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL_SQRT:
        if (d.t_in0 == LIBXSMM_DATATYPE_F64 && d.t_out == LIBXSMM_DATATYPE_F64 && d.t_comp == LIBXSMM_DATATYPE_F64) return (d.op == LIBXSMM_MELTW_TYPE_UNARY_DUMP) ? FAM_NONE : FAM_MAP;
        return (is_f(d.t_in0) && is_f(d.t_out)) ? FAM_MAP : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TANH: case LIBXSMM_MELTW_TYPE_UNARY_TANH_INV: case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID:
      case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID_INV: case LIBXSMM_MELTW_TYPE_UNARY_GELU: case LIBXSMM_MELTW_TYPE_UNARY_GELU_INV:
      case LIBXSMM_MELTW_TYPE_UNARY_EXP: case LIBXSMM_MELTW_TYPE_UNARY_REPLICATE_COL_VAR:
      case LIBXSMM_MELTW_TYPE_UNARY_RELU: case LIBXSMM_MELTW_TYPE_UNARY_RELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU:
      case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_ELU: case LIBXSMM_MELTW_TYPE_UNARY_ELU_INV:
        return (is_f(d.t_in0) && is_f(d.t_out)) ? FAM_MAP : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MAX:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MIN: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MAX:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MIN:
        if (d.t_in0 == LIBXSMM_DATATYPE_F64 && d.t_out == LIBXSMM_DATATYPE_F64) return FAM_REDUCE;
        return (is_f(d.t_in0) && is_f(d.t_out)) ? FAM_REDUCE : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD:
        if (d.t_in0 == LIBXSMM_DATATYPE_F64 && d.t_out == LIBXSMM_DATATYPE_F64) return FAM_SCALAR;
        return (is_f(d.t_in0) && is_f(d.t_out)) ? FAM_SCALAR : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT: return FAM_TRANSFORM;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2_TO_VNNI2T:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2T_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4T:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4T_TO_NORM:
        return (xb_dev_typesize(d.t_in0) == 2) ? FAM_TRANSFORM : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI4T:
        return (xb_dev_typesize(d.t_in0) <= 2) ? FAM_TRANSFORM : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_NORM:
        return (xb_dev_typesize(d.t_in0) == 1) ? FAM_TRANSFORM : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_GATHER: case LIBXSMM_MELTW_TYPE_UNARY_SCATTER:
        return (xb_dev_typesize(d.t_in0) <= 4 && xb_dev_typesize(d.t_in0) >= 1) ? FAM_GS : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_QUANT:
        if (d.t_in0 == LIBXSMM_DATATYPE_BF16 && (d.t_out == LIBXSMM_DATATYPE_MXFP4X2 || d.t_out == LIBXSMM_DATATYPE_NVFP4X2 || d.t_out == LIBXSMM_DATATYPE_MXBF8)) return FAM_MXQUANT;
        return (d.t_in0 == LIBXSMM_DATATYPE_F32 && (d.t_out == LIBXSMM_DATATYPE_I8 || d.t_out == LIBXSMM_DATATYPE_I16 || d.t_out == LIBXSMM_DATATYPE_I32)) ? FAM_QUANT : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_DEQUANT:
        return (d.t_out == LIBXSMM_DATATYPE_F32 && (d.t_in0 == LIBXSMM_DATATYPE_I8 || d.t_in0 == LIBXSMM_DATATYPE_I16 || d.t_in0 == LIBXSMM_DATATYPE_I32)) ? FAM_QUANT : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8_TO_VNNI8T:
        return (xb_dev_typesize(d.t_in0) <= 2 && xb_dev_typesize(d.t_in0) >= 1) ? FAM_TRANSFORM : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8T_TO_NORM:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD2:
        return (xb_dev_typesize(d.t_in0) == 2) ? FAM_TRANSFORM : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD4:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI2:
        return (xb_dev_typesize(d.t_in0) == 1) ? FAM_TRANSFORM : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_DROPOUT: case LIBXSMM_MELTW_TYPE_UNARY_DROPOUT_INV:
        return (is_f(d.t_in0) && is_f(d.t_out)) ? FAM_DROPOUT : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_UNARY_UNZIP: case LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X2: case LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X3:
        return (d.t_in0 == LIBXSMM_DATATYPE_F32) ? FAM_SPLIT : FAM_NONE;
      default: return FAM_NONE;
    }
  }
  if (d.op_class == LIBXSMM_MELTW_OPERATION_BINARY) {
    const bool all64 = d.t_in0 == LIBXSMM_DATATYPE_F64 && d.t_in1 == LIBXSMM_DATATYPE_F64 && d.t_out == LIBXSMM_DATATYPE_F64 && d.t_comp == LIBXSMM_DATATYPE_F64;
    switch (d.op) {
      case LIBXSMM_MELTW_TYPE_BINARY_ADD: case LIBXSMM_MELTW_TYPE_BINARY_MUL: case LIBXSMM_MELTW_TYPE_BINARY_SUB:
      case LIBXSMM_MELTW_TYPE_BINARY_DIV: case LIBXSMM_MELTW_TYPE_BINARY_MULADD: case LIBXSMM_MELTW_TYPE_BINARY_MAX:
      case LIBXSMM_MELTW_TYPE_BINARY_MIN:
        return (all64 || (is_f(d.t_in0) && is_f(d.t_in1) && is_f(d.t_out))) ? FAM_MAP : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GE: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LT:
      case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LE: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_EQ: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_NE:
        return (is_f(d.t_in0) && is_f(d.t_in1)) ? FAM_MAP : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_BINARY_ZIP:
        return (d.t_in0 == LIBXSMM_DATATYPE_U16 || d.t_in0 == LIBXSMM_DATATYPE_BF16 || d.t_in0 == LIBXSMM_DATATYPE_I16) ? FAM_MAP : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD:
        return (all64 || (is_f(d.t_in0) && is_f(d.t_in1) && is_f(d.t_out))) ? FAM_SCALAR : FAM_NONE;
      default: return FAM_NONE;
    }
  }
  if (d.op_class == LIBXSMM_MELTW_OPERATION_TERNARY) {
    const bool all64 = d.t_in0 == LIBXSMM_DATATYPE_F64 && d.t_in1 == LIBXSMM_DATATYPE_F64 && d.t_in2 == LIBXSMM_DATATYPE_F64
                    && d.t_out == LIBXSMM_DATATYPE_F64 && d.t_comp == LIBXSMM_DATATYPE_F64;
    switch (d.op) {
      case LIBXSMM_MELTW_TYPE_TERNARY_SELECT: return (all64 || (is_f(d.t_in0) && is_f(d.t_in1) && is_f(d.t_out))) ? FAM_MAP : FAM_NONE;
      case LIBXSMM_MELTW_TYPE_TERNARY_MULADD: case LIBXSMM_MELTW_TYPE_TERNARY_NMULADD:
        return (is_f(d.t_in0) && is_f(d.t_in1) && is_f(d.t_in2) && is_f(d.t_out)) ? FAM_MAP : FAM_NONE;
      default: return FAM_NONE;
    }
  }
  return FAM_NONE;
}

// what a kernel sees of a call: xb_meltw_args without the tile axis, which only the batch instantiations take (as mtiles). The
// kernels' argument struct keeps its former size, so the single-call kernels compile as they did before the axis existed.
struct margs {
  const void* in0; const void* in1; const void* in2; void* out;
  const void* in_aux; void* out_aux;
  float alpha; unsigned long long n_rt; unsigned long long off[2];
  void* rng; float* rnd; unsigned char* rnd8;
};
struct mtiles { long long count, s_in0, s_in1, s_in2, s_in_aux, s_out, s_out_aux; };

// ---- typed load/store -----------------------------------------------------------------------------------
__device__ __forceinline__ float ld_f32(const void* p, long long idx, int t) {
  if (t == LIBXSMM_DATATYPE_F32) return ((const float*)p)[idx];
  if (t == LIBXSMM_DATATYPE_BF16) { unsigned short h = ((const unsigned short*)p)[idx]; if ((h & 0x7f80) == 0) h &= 0x8000; return xb_bf16_to_f32(h); }
  if (t == LIBXSMM_DATATYPE_BF8) return xb_bf8_to_f32(((const unsigned char*)p)[idx]);
  if (t == LIBXSMM_DATATYPE_HF8) return xb_hf8_to_f32(((const unsigned char*)p)[idx]);
  return xb_f16_to_f32(((const unsigned short*)p)[idx]);
}
__device__ __forceinline__ void st_f32(void* p, long long idx, int t, float v) {
  if (t == LIBXSMM_DATATYPE_F32) ((float*)p)[idx] = v;
  else if (t == LIBXSMM_DATATYPE_BF16) ((unsigned short*)p)[idx] = xb_f32_to_bf16_rne(v);
  else if (t == LIBXSMM_DATATYPE_BF8) ((unsigned char*)p)[idx] = xb_f32_to_bf8(v);
  else if (t == LIBXSMM_DATATYPE_HF8) ((unsigned char*)p)[idx] = xb_f32_to_hf8(v);
  else ((unsigned short*)p)[idx] = xb_f32_to_f16(v);
}
// f32 -> bf8 with a random byte added below the kept bits (libxsmm_stochastic_convert_fp32_bf8, src/libxsmm_lpflt_quant.c:332-368):
// normal numbers only; f16-subnormal magnitudes round to nearest even, Inf/NaN pass through
__device__ __forceinline__ unsigned char bf8_stochastic(float v, unsigned int rnd) {
  unsigned int h = xb_f32_to_f16(v);
  if ((h & 0x7c00u) == 0x7c00u) { if (h & 0x03ffu) h |= 0x0200u; }
  else if ((h & 0x7c00u) == 0u) h = (h + 0x7fu + ((h >> 8) & 1u)) & 0xffffu;
  else h = (h + rnd) & 0xffffu;
  return (unsigned char)(h >> 8);
}
// store of the map kernels: element (i, j) is the (j*m + i)-th the reference visits, which selects its random byte
__device__ __forceinline__ void st_map(const xb_meltw_desc& d, const margs& a, long long oi, int i, int j, float v) {
  if (a.rnd8 != nullptr) ((unsigned char*)a.out)[oi] = bf8_stochastic(v, a.rnd8[(long long)j * d.m + i]);
  else st_f32(a.out, oi, d.t_out, v);
}
// operand index with broadcast flags; which: 0,1,2 = in0,in1,in2
__device__ __forceinline__ long long bidx(const xb_meltw_desc& d, int which, int i, int j, long long ld) {
  unsigned int row = 0, col = 0, sca = 0;
  if (d.op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    if (which == 0) { row = d.flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_ROW; col = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_COL) | (d.op == LIBXSMM_MELTW_TYPE_UNARY_REPLICATE_COL_VAR); sca = d.flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_SCALAR; }
  } else if (d.op_class == LIBXSMM_MELTW_OPERATION_BINARY) {
    row = d.flags & (which == 0 ? LIBXSMM_MELTW_FLAG_BINARY_BCAST_ROW_IN_0 : LIBXSMM_MELTW_FLAG_BINARY_BCAST_ROW_IN_1);
    col = d.flags & (which == 0 ? LIBXSMM_MELTW_FLAG_BINARY_BCAST_COL_IN_0 : LIBXSMM_MELTW_FLAG_BINARY_BCAST_COL_IN_1);
    sca = d.flags & (which == 0 ? LIBXSMM_MELTW_FLAG_BINARY_BCAST_SCALAR_IN_0 : LIBXSMM_MELTW_FLAG_BINARY_BCAST_SCALAR_IN_1);
    if (which > 1) row = col = sca = 0;
  } else {
    const unsigned int r[3] = { LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_0, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_1, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_2 };
    const unsigned int c[3] = { LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_0, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_1, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_2 };
    const unsigned int s[3] = { LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_0, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_1, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_2 };
    row = d.flags & r[which]; col = d.flags & c[which]; sca = d.flags & s[which];
  }
  if (row) return (long long)j * ld;
  if (col) return i;
  if (sca) return 0;
  return i + (long long)j * ld;
}

__device__ __forceinline__ float sigmoidf_ref(float x) { return (tanhf(x / 2.0f) + 1.0f) / 2.0f; }

__device__ __forceinline__ float unary_f32(float x, int op) {
  switch (op) {
    case LIBXSMM_MELTW_TYPE_UNARY_NEGATE: return -1.0f * x;
    case LIBXSMM_MELTW_TYPE_UNARY_X2: return x * x;
    case LIBXSMM_MELTW_TYPE_UNARY_XOR: return 0.0f;
    case LIBXSMM_MELTW_TYPE_UNARY_TANH: return tanhf(x);
    case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID: return sigmoidf_ref(x);
    case LIBXSMM_MELTW_TYPE_UNARY_GELU: return (erff(x / sqrtf(2.0f)) + 1.0f) * 0.5f * x;
    case LIBXSMM_MELTW_TYPE_UNARY_GELU_INV: return 0.5f + 0.5f * erff(x / sqrtf(2.0f)) + x / sqrtf(2.0f * 3.14159265358979323846f) * expf(-0.5f * x * x);
    case LIBXSMM_MELTW_TYPE_UNARY_TANH_INV: { const float t = tanhf(x); return 1.0f - t * t; }
    case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID_INV: { const float s = sigmoidf_ref(x); return s * (1.0f - s); }
    case LIBXSMM_MELTW_TYPE_UNARY_SQRT: return sqrtf(x);
    case LIBXSMM_MELTW_TYPE_UNARY_INC: return x + 1.0f;
    case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL: return 1.0f / x;
    case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL_SQRT: return 1.0f / sqrtf(x);
    case LIBXSMM_MELTW_TYPE_UNARY_EXP: return expf(x);
    default: return x;   // IDENTITY, REPLICATE_COL_VAR
  }
}
__device__ __forceinline__ double unary_f64(double x, int op) {
  switch (op) {
    case LIBXSMM_MELTW_TYPE_UNARY_NEGATE: return -1.0 * x;
    case LIBXSMM_MELTW_TYPE_UNARY_X2: return x * x;
    case LIBXSMM_MELTW_TYPE_UNARY_XOR: return 0.0;
    case LIBXSMM_MELTW_TYPE_UNARY_SQRT: return sqrt(x);
    case LIBXSMM_MELTW_TYPE_UNARY_INC: return x + 1.0;
    case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL: return 1.0 / x;
    case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL_SQRT: return 1.0 / sqrt(x);
    default: return x;
  }
}
template <typename T> __device__ __forceinline__ T binary_op(T a, T b, T out, int op) {
  switch (op) {
    case LIBXSMM_MELTW_TYPE_BINARY_ADD: return a + b;
    case LIBXSMM_MELTW_TYPE_BINARY_SUB: return a - b;
    case LIBXSMM_MELTW_TYPE_BINARY_MUL: return a * b;
    case LIBXSMM_MELTW_TYPE_BINARY_DIV: return a / b;
    case LIBXSMM_MELTW_TYPE_BINARY_MULADD: return out + a * b;
    case LIBXSMM_MELTW_TYPE_BINARY_MAX: return (a > b) ? a : b;
    case LIBXSMM_MELTW_TYPE_BINARY_MIN: return (a > b) ? b : a;
    default: return out;
  }
}
__device__ __forceinline__ bool cmp_op(float a, float b, int op) {
  switch (op) {
    case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT: return a > b;
    case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GE: return a >= b;
    case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LT: return a < b;
    case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LE: return a <= b;
    case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_EQ: return a == b;
    default: return a != b;
  }
}
__device__ __forceinline__ bool mask_bit(const void* mask, int i, int j, long long mask_ld) {
  return (((const unsigned char*)mask)[i / 8 + (long long)j * (mask_ld / 8)] >> (i % 8)) & 1;
}
// a warp holds 32 consecutive rows [i0, i0+32) of column j; lane bit = predicate. Only bits of valid rows change.
__device__ __forceinline__ void mask_store(void* mask, int i0, int j, long long mask_ld, int m, bool bit, int lane) {
  const unsigned int word = __ballot_sync(0xffffffffu, bit);
  if (lane < 4) {
    const int ib = i0 + lane * 8;
    if (ib < m) {
      unsigned char* dst = (unsigned char*)mask + ib / 8 + (long long)j * (mask_ld / 8);
      const unsigned int valid = (m - ib >= 8) ? 0xffu : ((1u << (m - ib)) - 1u);
      const unsigned int nb = (word >> (lane * 8)) & 0xffu;
      *dst = (unsigned char)((valid == 0xffu) ? nb : ((*dst & ~valid) | (nb & valid)));
    }
  }
}

// ---- tile axis (margs.count): a batch of calls in one launch. blockIdx.y strides the calls, blockIdx.x keeps the
// single call's work split; call t reads and writes through its operands advanced by t times their byte strides. Every kernel
// that takes the axis has a template flag B: a single call launches B = false, whose loop over the calls is the one iteration
// t = 0 and folds away at compile time, so its code and registers are those of the kernel without the axis.

template <typename P> __device__ __forceinline__ P adv(P p, long long t, long long s) { return (P)((const char*)p + t * s); }
__device__ __forceinline__ margs tile_args(const margs& a, const mtiles& s, long long t) {
  margs r = a;
  r.in0 = adv(a.in0, t, s.s_in0); r.in1 = adv(a.in1, t, s.s_in1); r.in2 = adv(a.in2, t, s.s_in2);
  r.in_aux = adv(a.in_aux, t, s.s_in_aux); r.out = (void*)adv(a.out, t, s.s_out); r.out_aux = (void*)adv(a.out_aux, t, s.s_out_aux);
  return r;
}
#define XB_FOR_TILES(A0) _Pragma("unroll 1") for (long long t_ = B ? blockIdx.y : 0; t_ < (B ? tl.count : 1); t_ += B ? gridDim.y : 1)
#define XB_FOR_CALLS(T, COUNT) _Pragma("unroll 1") for (long long T = B ? blockIdx.y : 0; T < (B ? (COUNT) : 1); T += B ? gridDim.y : 1)

// ---- map kernel: unary / binary / ternary elementwise (with masks) ---------------------------------------------
template <bool B>
__global__ void __launch_bounds__(256) meltw_map_kernel(const xb_meltw_desc d, const margs a0, const mtiles tl, const int n_eff) {
  const int lane = threadIdx.x & 31;
  const int chunks = (d.m + 31) / 32;
  const long long nwork = (long long)chunks * n_eff;
  const long long wstride = (long long)gridDim.x * (blockDim.x >> 5);
  const bool f64 = (d.t_out == LIBXSMM_DATATYPE_F64);
  XB_FOR_TILES(a0) {
  const margs a = B ? tile_args(a0, tl, t_) : a0;
  for (long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < nwork; w += wstride) {
    const int j = (int)(w / chunks), i0 = (int)(w % chunks) * 32, i = i0 + lane;
    const bool act = i < d.m;
    const long long oi = i + (long long)j * d.ldo;
    if (d.op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
      const int op = d.op;
      if (f64) {
        if (act) { const double r = unary_f64(((const double*)a.in0)[bidx(d, 0, i, j, d.ldi)], op); ((double*)a.out)[oi] = r; if (op == LIBXSMM_MELTW_TYPE_UNARY_DUMP) ((double*)a.out_aux)[oi] = r; }
        continue;
      }
      const float x = act ? ld_f32(a.in0, bidx(d, 0, i, j, d.ldi), d.t_in0) : 0.0f;
      const bool bitm = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) != 0;
      if (op == LIBXSMM_MELTW_TYPE_UNARY_RELU || op == LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU || op == LIBXSMM_MELTW_TYPE_UNARY_ELU) {
        float y;
        if (op == LIBXSMM_MELTW_TYPE_UNARY_RELU) {
          // (x <= 0) ? 0 : x on the BITS with integer compares: written with a float compare (even in PTX) ptxas fuses it into
          // FMNMX.NAN, which canonicalises a NaN's payload; the reference passes the NaN through untouched
          const unsigned int xb = __float_as_uint(x);
          const bool zero_it = ((int)xb <= 0) && ((xb & 0x7fffffffu) <= 0x7f800000u);
          y = __uint_as_float(zero_it ? 0u : xb);
        }
        else if (op == LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU) y = (x <= 0.0f) ? a.alpha * x : x;
        else y = (x <= 0.0f) ? a.alpha * (expf(x) - 1.0f) : x;
        if (act) st_f32(a.out, oi, d.t_out, y);
        if (bitm) mask_store(a.out_aux, i0, j, ((d.ldo + 15) / 16) * 16, d.m, act && !(x <= 0.0f), lane);
      } else if (op == LIBXSMM_MELTW_TYPE_UNARY_RELU_INV || op == LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU_INV) {
        if (act) {
          const long long mld = bitm ? ((d.ldi + 15) / 16) * 16 : d.ldi;
          const bool bit = mask_bit(a.in_aux, i, j, mld);
          st_f32(a.out, oi, d.t_out, bit ? x : ((op == LIBXSMM_MELTW_TYPE_UNARY_RELU_INV) ? 0.0f : a.alpha * x));
        }
      } else if (op == LIBXSMM_MELTW_TYPE_UNARY_ELU_INV) {
        if (act) { const float fwd = ld_f32(a.in_aux, i + (long long)j * d.ldi, d.t_in0); st_f32(a.out, oi, d.t_out, (fwd > 0) ? x : x * (fwd + a.alpha)); }
      } else if (act) {
        st_map(d, a, oi, i, j, unary_f32(x, op));
        if (op == LIBXSMM_MELTW_TYPE_UNARY_DUMP) {                      // second copy of what was stored (:2478-2493)
          if (a.rnd8 != nullptr) ((unsigned char*)a.out_aux)[oi] = ((unsigned char*)a.out)[oi];
          else st_f32(a.out_aux, oi, d.t_out, x);
        }
      }
    } else if (d.op_class == LIBXSMM_MELTW_OPERATION_BINARY) {
      const int op = d.op;
      if (op == LIBXSMM_MELTW_TYPE_BINARY_ZIP) {
        if (act) ((unsigned int*)a.out)[oi] = (unsigned int)((const unsigned short*)a.in0)[bidx(d, 0, i, j, d.ldi)]
                                            | ((unsigned int)((const unsigned short*)a.in1)[bidx(d, 1, i, j, d.ldi2)] << 16);
        continue;
      }
      if (f64 && op < LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT) {
        if (act) { double* o = (double*)a.out + oi; *o = binary_op<double>(((const double*)a.in0)[bidx(d, 0, i, j, d.ldi)], ((const double*)a.in1)[bidx(d, 1, i, j, d.ldi2)], *o, op); }
        continue;
      }
      const float x = act ? ld_f32(a.in0, bidx(d, 0, i, j, d.ldi), d.t_in0) : 0.0f;
      const float y = act ? ld_f32(a.in1, bidx(d, 1, i, j, d.ldi2), d.t_in1) : 0.0f;
      if (op >= LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT) mask_store(a.out, i0, j, ((d.ldo + 15) / 16) * 16, d.m, act && cmp_op(x, y, op), lane);
      else if (act) {
        const float o = (op == LIBXSMM_MELTW_TYPE_BINARY_MULADD) ? ld_f32(a.out, oi, d.t_out) : 0.0f;
        st_map(d, a, oi, i, j, binary_op<float>(x, y, o, op));
      }
    } else if (act) {
      if (d.op == LIBXSMM_MELTW_TYPE_TERNARY_SELECT) {
        const bool bit = mask_bit(a.in2, i, j, ((d.ldi3 + 15) / 16) * 16);
        if (f64) ((double*)a.out)[oi] = bit ? ((const double*)a.in1)[bidx(d, 1, i, j, d.ldi2)] : ((const double*)a.in0)[bidx(d, 0, i, j, d.ldi)];
        else st_map(d, a, oi, i, j, bit ? ld_f32(a.in1, bidx(d, 1, i, j, d.ldi2), d.t_in1) : ld_f32(a.in0, bidx(d, 0, i, j, d.ldi), d.t_in0));
      } else {
        const float x = ld_f32(a.in0, bidx(d, 0, i, j, d.ldi), d.t_in0), y = ld_f32(a.in1, bidx(d, 1, i, j, d.ldi2), d.t_in1);
        const float z = ld_f32(a.in2, bidx(d, 2, i, j, d.ldi3), d.t_in2);
        st_map(d, a, oi, i, j, (d.op == LIBXSMM_MELTW_TYPE_TERNARY_MULADD) ? (z + x * y) : (y - x * z));
      }
    }
  }
  }
}

// ---- reductions: one warp per result element ------------------------------------------------------------------------
// Sums: lanes stride the reduced dimension, shuffle combine. Max / min / absmax give the reference's sequential fold bit for bit
// (:1215-1428 with LIBXSMM_MAX(A,B) = A < B ? B : A, LIBXSMM_MIN(A,B) = A < B ? A : B, LIBXSMM_ABS(A) = 0 <= A ? A : -A):
//   line   op       start       equal values      NaN element
//   rows   MAX      element 0   earlier kept      ignored; a NaN element 0 sticks
//   rows   ABSMAX   element 0   earlier kept      ignored; a NaN element 0 sticks, its sign flipped once per element folded
//   rows   MIN      element 0   later taken       taken, and the next element replaces it (the fold restarts after it)
//   cols   MAX      -FLT_MAX    later taken       taken, the fold restarts after it (without the -FLT_MAX start)
//   cols   ABSMAX   +0          later taken       like cols MAX, on ABS values (ABS(-0) = -0, ABS flips a NaN's sign)
//   cols   MIN      +FLT_MAX    earlier kept      ignored
//   argop  any      as cols     later taken       ignored (x >= tmp / x <= tmp is false); an index never taken is not written
// Each lane folds one contiguous segment of the line with these rules; the segments combine in lane order (a segment holding a
// NaN that restarts the fold discards everything before it), so the result is the sequential one whatever the segment cut.
// Values are compared through integer keys and moved as bits: a float select could be fused into FMNMX, which returns +0 for
// (-0, +0) and canonicalises NaN payloads.
__device__ __forceinline__ unsigned int mm_bits(float x) { return __float_as_uint(x); }
__device__ __forceinline__ unsigned long long mm_bits(double x) { return (unsigned long long)__double_as_longlong(x); }
__device__ __forceinline__ float mm_from(unsigned int u, float) { return __uint_as_float(u); }
__device__ __forceinline__ double mm_from(unsigned long long u, double) { return __longlong_as_double((long long)u); }
template <typename T> struct mm_traits;
template <> struct mm_traits<float> { typedef unsigned int U; static constexpr U SIGN = 0x80000000u, INF = 0x7f800000u; };
template <> struct mm_traits<double> { typedef unsigned long long U; static constexpr U SIGN = 0x8000000000000000ull, INF = 0x7ff0000000000000ull; };
template <typename T> __device__ __forceinline__ bool mm_isnan(T x) {
  typedef typename mm_traits<T>::U U; return (mm_bits(x) & ~mm_traits<T>::SIGN) > mm_traits<T>::INF;
}
// LIBXSMM_ABS: negative non-zero values and NaNs get their sign flipped, +-0 stay
template <typename T> __device__ __forceinline__ T mm_abs(T x) {
  typedef typename mm_traits<T>::U U; const U u = mm_bits(x);
  const bool flip = mm_isnan(x) || ((u & mm_traits<T>::SIGN) != 0 && (u & ~mm_traits<T>::SIGN) != 0);
  return mm_from(flip ? (u ^ mm_traits<T>::SIGN) : u, x);
}
// order key of a non-NaN value with -0 == +0
template <typename T> __device__ __forceinline__ typename mm_traits<T>::U mm_key(T x) {
  typedef typename mm_traits<T>::U U; U u = mm_bits(x);
  if ((u & ~mm_traits<T>::SIGN) == 0) u = 0;
  return (u & mm_traits<T>::SIGN) ? ~u : (u | mm_traits<T>::SIGN);
}
// x replaces the running value v: max or min, the later one on equal values or the earlier one
template <typename T> __device__ __forceinline__ bool mm_better(T x, T v, bool is_min, bool later) {
  const typename mm_traits<T>::U kx = mm_key(x), kv = mm_key(v);
  return is_min ? (later ? kx <= kv : kx < kv) : (later ? kx >= kv : kx > kv);
}
template <typename T> struct mm_state { T v, nanv; long long pos; int have, reset; };
template <typename T> __device__ __forceinline__ mm_state<T> mm_combine(mm_state<T> l, const mm_state<T>& r, bool is_min, bool later) {
  if (r.reset) return r;
  if (r.have && (!l.have || mm_better(r.v, l.v, is_min, later))) { l.v = r.v; l.pos = r.pos; l.have = 1; }
  return l;
}

template <typename T>
__device__ __forceinline__ T reduce_load(const xb_meltw_desc& d, const void* in0, long long idx) {
  return (sizeof(T) == 8) ? (T)((const double*)in0)[idx] : (T)ld_f32(in0, idx, d.t_in0);
}
template <typename T> __device__ __forceinline__ T warp_sum(T v) { for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o); return v; }

template <typename T, bool B>
__global__ void __launch_bounds__(256) meltw_reduce_kernel(const xb_meltw_desc d, const margs a, const mtiles tl) {
  const int lane = threadIdx.x & 31;
  const bool rows = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_ROWS) != 0;
  const bool init_acc = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_INIT_ACC) != 0;
  const bool argop = !rows && (d.flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP) != 0;
  const bool idx4 = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_IDX_SIZE_4BYTES) != 0;
  const bool f64 = sizeof(T) == 8;
  const int op = d.op;
  const bool by_idx = (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_ADD || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MAX || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MIN);
  const int kind = (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MAX || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MAX) ? 1
                 : (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MIN || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MIN) ? 2
                 : (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX) ? 3 : 0;
  const bool want_x = (op != LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD);
  const bool want_x2 = (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD);
  const int nres = rows ? d.n : d.m;
  const int result_size = rows ? d.n : d.ldo;                 // offset of the x^2 plane (reference :1073-1076)
  const long long len = rows ? d.m : (by_idx ? (long long)a.n_rt : d.n);
  // fold rules of the table above
  const bool is_min = (kind == 2);
  const bool later = argop || (rows ? kind == 2 : kind != 2);
  const bool nan_restarts = !argop && (rows ? kind == 2 : kind != 2);
  XB_FOR_CALLS(t_, tl.count) {                              // the operands of call t_ (a single call: t_ = 0, the kernel's own)
  const void* const in0 = adv(a.in0, t_, tl.s_in0); const void* const in_aux = adv(a.in_aux, t_, tl.s_in_aux);
  void* const out = adv(a.out, t_, tl.s_out); void* const out_aux = adv(a.out_aux, t_, tl.s_out_aux);
  for (int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); o < nres; o += gridDim.x * (blockDim.x >> 5)) {
    if (kind == 0) {
      T sx = 0, sx2 = 0;
      for (long long t = lane; t < len; t += 32) {
        long long idx;
        if (rows) idx = t + (long long)o * d.ldi;
        else { const long long j = by_idx ? (idx4 ? (long long)((const unsigned int*)in_aux)[t] : (long long)((const unsigned long long*)in_aux)[t]) : t; idx = o + j * d.ldi; }
        const T v = reduce_load<T>(d, in0, idx);
        sx += v; sx2 += v * v;
      }
      sx = warp_sum(sx); sx2 = warp_sum(sx2);
      if (lane == 0) {
        if (f64) {
          double* ox = (double*)out; double* ox2 = want_x ? ox + result_size : ox;
          if (want_x) ox[o] = (double)sx + ((init_acc) ? ox[o] : 0.0);
          if (want_x2) ox2[o] = (double)sx2 + ((init_acc) ? ox2[o] : 0.0);
        } else {
          char* base2 = (char*)out + (want_x ? (size_t)result_size * xb_dev_typesize(d.t_out) : 0);
          if (want_x) { float r = (float)sx; if (init_acc && !by_idx) r += ld_f32(out, o, d.t_out); st_f32(out, o, d.t_out, r); }
          if (want_x2) { float r = (float)sx2; if (init_acc) r += ld_f32(base2, o, d.t_out); st_f32(base2, o, d.t_out, r); }
        }
      }
      continue;
    }
    const long long seg = (len + 31) / 32, t0 = lane * seg, t1 = (t0 + seg < len) ? t0 + seg : len;
    mm_state<T> st; st.v = st.nanv = (T)0; st.pos = 0; st.have = 0; st.reset = 0;
    for (long long t = t0; t < t1; ++t) {
      const long long j = rows ? t : (by_idx ? (idx4 ? (long long)((const unsigned int*)in_aux)[t] : (long long)((const unsigned long long*)in_aux)[t]) : t);
      T v = reduce_load<T>(d, in0, rows ? (t + (long long)o * d.ldi) : (o + j * d.ldi));
      if (kind == 3) v = mm_abs(v);
      if (mm_isnan(v)) { if (nan_restarts) { st.reset = 1; st.have = 0; st.nanv = v; } }
      else if (!st.have || mm_better(v, st.v, is_min, later)) { st.v = v; st.pos = j; st.have = 1; }
    }
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      mm_state<T> r;
      r.v = __shfl_down_sync(0xffffffffu, st.v, off); r.nanv = __shfl_down_sync(0xffffffffu, st.nanv, off);
      r.pos = __shfl_down_sync(0xffffffffu, st.pos, off);
      r.have = __shfl_down_sync(0xffffffffu, st.have, off); r.reset = __shfl_down_sync(0xffffffffu, st.reset, off);
      if ((lane & (2 * off - 1)) == 0 && lane + off < 32) st = mm_combine(st, r, is_min, later);
    }
    if (lane == 0) {
      T res; bool taken = false;
      if (rows) {
        const T x0 = reduce_load<T>(d, in0, (long long)o * d.ldi);
        if (kind != 2 && mm_isnan(x0)) {                       // a NaN start sticks; ABS flips it once per element folded
          typedef typename mm_traits<T>::U U;
          res = (kind == 3 && (len & 1)) ? mm_from((U)(mm_bits(x0) ^ mm_traits<T>::SIGN), x0) : x0;
        } else res = st.have ? st.v : st.nanv;
      } else if (st.reset) res = st.have ? st.v : st.nanv;    // after a NaN the fold has no start value
      else {
        const T start = (kind == 1) ? (T)-FLT_MAX : ((kind == 2) ? (T)FLT_MAX : (T)0);
        taken = st.have && mm_better(st.v, start, is_min, later);
        res = taken ? st.v : start;
      }
      if (f64) ((double*)out)[o] = (double)res; else st_f32(out, o, d.t_out, (float)res);
      if (argop && taken && out_aux != nullptr) {
        if (idx4) ((unsigned int*)out_aux)[o] = (unsigned int)st.pos; else ((unsigned long long*)out_aux)[o] = (unsigned long long)st.pos;
      }
    }
  }
  }
}

// whole-matrix reductions to one scalar (one CTA per call; the tests' sizes are tiny, the large case is a dot product)
template <typename T, bool B>
__global__ void __launch_bounds__(1024) meltw_scalar_kernel(const xb_meltw_desc d, const margs a0, const mtiles tl) {
  __shared__ T part[32];
  const bool f64 = sizeof(T) == 8;
  const bool dot = (d.op_class == LIBXSMM_MELTW_OPERATION_BINARY);
  XB_FOR_TILES(a0) {
  const margs a = B ? tile_args(a0, tl, t_) : a0;
  T acc = 0;
  for (long long e = threadIdx.x; e < (long long)d.m * d.n; e += blockDim.x) {
    const int i = (int)(e % d.m), j = (int)(e / d.m);
    T x = f64 ? (T)((const double*)a.in0)[bidx(d, 0, i, j, d.ldi)] : (T)ld_f32(a.in0, bidx(d, 0, i, j, d.ldi), d.t_in0);
    if (dot) x *= f64 ? (T)((const double*)a.in1)[bidx(d, 1, i, j, d.ldi2)] : (T)ld_f32(a.in1, bidx(d, 1, i, j, d.ldi2), d.t_in1);
    acc += x;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    acc = (threadIdx.x < (blockDim.x >> 5)) ? part[threadIdx.x] : (T)0;
    acc = warp_sum(acc);
    if (threadIdx.x == 0) { if (f64) ((double*)a.out)[0] = (double)acc; else st_f32(a.out, 0, d.t_out, (float)acc); }
  }
  if (B && t_ + gridDim.y < tl.count) __syncthreads();       // part[] is reused by the next call of the batch
  }
}

// ---- transforms: one thread per OUTPUT element, pure data movement -------------------------------------------------
template <typename E, bool B>
__global__ void __launch_bounds__(256) meltw_transform_kernel(const xb_meltw_desc d, const margs a0, const mtiles tl) {
  const long long M = d.m, N = d.n, ldi = d.ldi, ldo = d.ldo;
  const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x, nth = (long long)gridDim.x * blockDim.x;
  const E* in0 = (const E*)a0.in0; E* out0 = (E*)a0.out;
  // the element's indices are worked out once and the move repeats for every call of the batch (a single call: once, t_ = 0)
#define XB_PUT(OI, COND, II) { const long long oi_ = (OI), ii_ = (II); const bool c_ = (COND); \
    XB_FOR_CALLS(t_, tl.count) adv(out0, t_, tl.s_out)[oi_] = c_ ? adv(in0, t_, tl.s_in0)[ii_] : (E)0; }
  switch (d.op) {
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT:          // out[j*ldo+i] = in[i*ldi+j], i<N, j<M (:390-417)
      for (long long e = tid; e < M * N; e += nth) { const long long i = e % N, j = e / N; XB_PUT(j * ldo + i, true, i * ldi + j); }
      break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD:
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4_PAD: {
      // whole ldo x Nn output is defined: zero everywhere except out[(j*ldo*v)+(i*v)+j2] = in[((j*v)+j2)*ldi+i] (:541-553, :690-708, :737-759)
      const long long v = (d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2 || d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD) ? 2 : 4;
      const long long Nn = ((N + v - 1) / v) * v;
      for (long long e = tid; e < ldo * Nn; e += nth) {
        const long long j = e / (ldo * v), rem = e % (ldo * v), i = rem / v, j2 = rem % v, col = j * v + j2;
        XB_PUT(e, i < M && col < N, col * ldi + i);   // rows >= N of the last group are zero padding
      }
    } break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4T: {
      const long long v = (d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2T) ? 2 : 4;   // out[(i*ldo*v)+(j*v)+i2] = in[(j*ldi)+(i*v+i2)]
      for (long long e = tid; e < (M / v) * N * v; e += nth) { const long long i2 = e % v, j = (e / v) % N, i = e / (v * N); XB_PUT(i * ldo * v + j * v + i2, true, j * ldi + i * v + i2); }
    } break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2_TO_VNNI2T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI4T: {
      const long long v = (d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2_TO_VNNI2T) ? 2 : 4;  // out[j*ldo*v+j2+(i*v+i2)*v] = in[i*ldi*v+i2+(j*v+j2)*v]
      for (long long e = tid; e < (M / v) * (N / v) * v * v; e += nth) {
        const long long i2 = e % v, j2 = (e / v) % v, i = (e / (v * v)) % (N / v), j = e / (v * v * (N / v));
        XB_PUT(j * ldo * v + j2 + (i * v + i2) * v, true, i * ldi * v + i2 + (j * v + j2) * v);
      }
    } break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2T_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4T_TO_NORM: {
      const long long v = (d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2T_TO_NORM) ? 2 : 4;   // roles of m/n swapped (:620-660)
      const long long Mr = d.n, Nr = d.m;                                                          // out[(j*ldo)+(i*v)+i2] = in[(i*ldi*v)+(j*v+i2)]
      for (long long e = tid; e < (Mr / v) * Nr * v; e += nth) { const long long i2 = e % v, j = (e / v) % Nr, i = e / (v * Nr); XB_PUT(j * ldo + i * v + i2, true, i * ldi * v + j * v + i2); }
    } break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_NORM:            // out[(i*ldo)+j] = in[((i/4)*ldi*4)+j*4+(i%4)], i<N, j<M (:787-803)
      for (long long e = tid; e < M * N; e += nth) { const long long j = e % M, i = e / M; XB_PUT(i * ldo + j, true, (i / 4) * ldi * 4 + j * 4 + (i % 4)); }
      break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8_PAD: {
      // :712-786 -- like VNNI2/VNNI4 with groups of 8 columns; columns past N read as zero here (the reference reads past its input)
      const long long v = 8, Nn = ((N + v - 1) / v) * v;
      for (long long e = tid; e < ldo * Nn; e += nth) {
        const long long j = e / (ldo * v), rem = e % (ldo * v), i = rem / v, j2 = rem % v, col = j * v + j2;
        XB_PUT(e, i < M && col < N, col * ldi + i);
      }
    } break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8T:           // out[(i*ldo*8)+(j*8)+i2] = in[(j*ldi)+(i*8+i2)] (:666-686)
      for (long long e = tid; e < (M / 8) * N * 8; e += nth) { const long long i2 = e % 8, j = (e / 8) % N, i = e / (8 * N); XB_PUT(i * ldo * 8 + j * 8 + i2, true, j * ldi + i * 8 + i2); }
      break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8_TO_VNNI8T:          // out[j*ldo*8+j2+(i*8+i2)*8] = in[i*ldi*8+i2+(j*8+j2)*8] (:489-531)
      for (long long e = tid; e < (M / 8) * (N / 8) * 64; e += nth) {
        const long long i2 = e % 8, j2 = (e / 8) % 8, i = (e / 64) % (N / 8), j = e / (64 * (N / 8));
        XB_PUT(j * ldo * 8 + j2 + (i * 8 + i2) * 8, true, i * ldi * 8 + i2 + (j * 8 + j2) * 8);
      }
      break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8T_TO_NORM: {         // roles of m/n swapped (:581-601)
      const long long Mr = d.n, Nr = d.m;                              // out[(j*ldo)+(i*8)+i2] = in[(i*ldi*8)+(j*8+i2)]
      for (long long e = tid; e < (Mr / 8) * Nr * 8; e += nth) { const long long i2 = e % 8, j = (e / 8) % Nr, i = e / (8 * Nr); XB_PUT(j * ldo + i * 8 + i2, true, i * ldi * 8 + j * 8 + i2); }
    } break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI2:            // out[((i/2)*ldo*2)+j*2+(i%2)] = in[((i/4)*ldi*4)+j*4+(i%4)], i<N, j<M (:806-823)
      for (long long e = tid; e < M * N; e += nth) { const long long j = e % M, i = e / M; XB_PUT((i / 2) * ldo * 2 + j * 2 + (i % 2), true, (i / 4) * ldi * 4 + j * 4 + (i % 4)); }
      break;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD2:
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD4: {
      // copy into a zero-filled ldo x Nn image; Nn rounds N up for the PADN/PADNM kinds, PADM keeps N (:825-960)
      const bool mod4 = (d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4 || d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD4 || d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD4);
      const bool padm_only = (d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD2 || d.op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4);
      const long long v = mod4 ? 4 : 2, Nn = padm_only ? N : ((N + v - 1) / v) * v;
      for (long long e = tid; e < ldo * Nn; e += nth) { const long long i = e % ldo, j = e / ldo; XB_PUT(e, i < M && j < N, j * ldi + i); }
    } break;
    default: break;
  }
#undef XB_PUT
}

// ---- bandwidth versions of the three layout/reduction kernels that matter at size (K7 of SURVEY.md 2.3) ------------------------
// transpose: 64 x 64 tiles through shared memory, one tile per CTA; both the read (rows of the input) and the write (rows of
// the output) are coalesced and every thread has its 16 loads in flight before the first store
template <typename E, bool B>
__global__ void __launch_bounds__(256) meltw_transpose_tiled_kernel(const E* __restrict__ in0, E* __restrict__ out0, long long M, long long N, long long ldi, long long ldo,
                                                                    long long count, long long s_in, long long s_out) {
  __shared__ E tile[64][65];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;                 // 32 x 8 threads
  const long long tiles_j = (M + 63) / 64;
  const long long t = blockIdx.x;
  const long long j0 = (t % tiles_j) * 64, i0 = (t / tiles_j) * 64;       // in[i*ldi + j], j contiguous, j < M, i < N
  XB_FOR_CALLS(c, count) {                                                // calls of a batch
  const E* __restrict__ in = adv(in0, c, s_in);
  E* __restrict__ out = adv(out0, c, s_out);
  E v[16];
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const long long i = i0 + ty + 8 * r;
#pragma unroll
    for (int h = 0; h < 2; ++h) v[2 * r + h] = (i < N && j0 + tx + 32 * h < M) ? in[i * ldi + j0 + tx + 32 * h] : (E)0;
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) { tile[ty + 8 * r][tx] = v[2 * r]; tile[ty + 8 * r][tx + 32] = v[2 * r + 1]; }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const long long j = j0 + ty + 8 * r;
#pragma unroll
    for (int h = 0; h < 2; ++h) if (j < M && i0 + tx + 32 * h < N) out[j * ldo + i0 + tx + 32 * h] = tile[tx + 32 * h][ty + 8 * r];
  }
  if (B && c + gridDim.y < count) __syncthreads();                        // the next call refills the tile
  }
}
// NORM -> VNNI-v pack: a thread takes 4 consecutive rows of one group of v columns: v loads of 4 elements, 4 stores of one
// v-element word each (16 contiguous bytes); zero padding of the last group and of rows [m, ldo) like the generic kernel
template <typename E, int V, bool B>
__global__ void __launch_bounds__(256) meltw_vnni_pack_kernel(const E* __restrict__ in0, E* __restrict__ out0, long long M, long long N, long long ldi, long long ldo,
                                                              long long count, long long s_in, long long s_out) {
  const long long groups = (N + V - 1) / V, quads = (ldo + 3) / 4;
  XB_FOR_CALLS(t, count) {
  const E* __restrict__ in = adv(in0, t, s_in);
  E* __restrict__ out = adv(out0, t, s_out);
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < groups * quads; e += (long long)gridDim.x * blockDim.x) {
    const long long g = e / quads, i0 = (e % quads) * 4;
    E v[V][4];
#pragma unroll
    for (int c = 0; c < V; ++c) {
      const long long col = g * V + c;
#pragma unroll
      for (int r = 0; r < 4; ++r) v[c][r] = (col < N && i0 + r < M) ? in[col * ldi + i0 + r] : (E)0;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) if (i0 + r < ldo) {
#pragma unroll
      for (int c = 0; c < V; ++c) out[(g * ldo + i0 + r) * V + c] = v[c][r];
    }
  }
  }
}
// the same pack with 16-byte accesses: a thread takes R = 16/sizeof(E) consecutive rows of one group of v columns (v loads of
// 16 bytes, v stores of 16 contiguous bytes); needs M, ldi, ldo multiples of R and 16-byte aligned bases
template <typename E, int V, bool B>
__global__ void __launch_bounds__(256) meltw_vnni_pack_vec_kernel(const E* __restrict__ in0, E* __restrict__ out0, long long M, long long N, long long ldi, long long ldo,
                                                                  long long count, long long s_in, long long s_out) {
  constexpr int R = 16 / (int)sizeof(E);
  const long long groups = (N + V - 1) / V, chunks = ldo / R;
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= groups * chunks) return;
  const long long g = e / chunks, i0 = (e % chunks) * R;
  XB_FOR_CALLS(t, count) {
  const E* __restrict__ in = adv(in0, t, s_in);
  E* __restrict__ out = adv(out0, t, s_out);
  union { uint4 q; E e[R]; } src[V];
  union { uint4 q[V]; E e[R * V]; } dst;
#pragma unroll
  for (int c = 0; c < V; ++c) {
    const long long col = g * V + c;
    src[c].q = (col < N && i0 < M) ? *reinterpret_cast<const uint4*>(in + col * ldi + i0) : make_uint4(0u, 0u, 0u, 0u);
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
#pragma unroll
    for (int c = 0; c < V; ++c) dst.e[r * V + c] = src[c].e[r];
  }
  uint4* o = reinterpret_cast<uint4*>(out + (g * ldo + i0) * V);
#pragma unroll
  for (int c = 0; c < V; ++c) o[c] = dst.q[c];
  }
}
// column sums of an f32 matrix with 16-byte loads: a warp covers 128 consecutive rows (one float4 per lane), the 8 warps of a
// CTA take the columns of the CTA's slice round-robin, four columns in flight per warp; the CTA's eight partial sums are added
// in warp order through shared memory
__global__ void __launch_bounds__(256) meltw_reduce_cols_partial_vec_kernel(const float* __restrict__ in, long long M, long long N, long long ldi, float* __restrict__ part, int want_x2) {
  __shared__ float4 sh[2][8][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long i = ((long long)blockIdx.x * 32 + lane) * 4;
  const long long per = (N + gridDim.y - 1) / gridDim.y, j0 = blockIdx.y * per, j1 = (j0 + per < N) ? j0 + per : N;
  float4 sx = make_float4(0.f, 0.f, 0.f, 0.f), sq = sx;
  if (i < M) {
    long long j = j0 + w;
    for (; j + 24 < j1; j += 32) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(in + (j + 8 * u) * ldi + i);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        sx.x += v[u].x; sx.y += v[u].y; sx.z += v[u].z; sx.w += v[u].w;
        sq.x += v[u].x * v[u].x; sq.y += v[u].y * v[u].y; sq.z += v[u].z * v[u].z; sq.w += v[u].w * v[u].w;
      }
    }
    for (; j < j1; j += 8) {
      const float4 v = *reinterpret_cast<const float4*>(in + j * ldi + i);
      sx.x += v.x; sx.y += v.y; sx.z += v.z; sx.w += v.w;
      sq.x += v.x * v.x; sq.y += v.y * v.y; sq.z += v.z * v.z; sq.w += v.w * v.w;
    }
  }
  sh[0][w][lane] = sx; sh[1][w][lane] = sq;
  __syncthreads();
  if (w == 0 && i < M) {
    float4 a = sh[0][0][lane], b = sh[1][0][lane];
    for (int k = 1; k < 8; ++k) {
      const float4 x = sh[0][k][lane], y = sh[1][k][lane];
      a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w; b.x += y.x; b.y += y.y; b.z += y.z; b.w += y.w;
    }
    *reinterpret_cast<float4*>(part + (size_t)blockIdx.y * M + i) = a;
    if (want_x2) *reinterpret_cast<float4*>(part + (size_t)(gridDim.y + blockIdx.y) * M + i) = b;
  }
}
// column reduction (one result per ROW i, the input's contiguous index): lanes take consecutive rows, so every load of a
// warp is one 128-byte line; the columns are cut into gridDim.y slices whose partial sums go to `part` and are added up, in
// slice order, by a second small kernel
__global__ void __launch_bounds__(256) meltw_reduce_cols_partial_kernel(const xb_meltw_desc d, const margs a, float* __restrict__ part, int want_x2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int per = (d.n + gridDim.y - 1) / gridDim.y, j0 = blockIdx.y * per, j1 = (j0 + per < d.n) ? j0 + per : d.n;
  if (i >= d.m) return;
  float sx = 0.0f, sx2 = 0.0f;
  for (int j = j0; j < j1; ++j) { const float v = ld_f32(a.in0, i + (long long)j * d.ldi, d.t_in0); sx += v; sx2 += v * v; }
  part[(size_t)blockIdx.y * d.m + i] = sx;
  if (want_x2) part[(size_t)(gridDim.y + blockIdx.y) * d.m + i] = sx2;
}
__global__ void __launch_bounds__(256) meltw_reduce_cols_final_kernel(const xb_meltw_desc d, const margs a, const float* __restrict__ part, int slices) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.m) return;
  const bool init_acc = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_INIT_ACC) != 0;
  const bool want_x = (d.op != LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD);
  const bool want_x2 = (d.op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD || d.op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD);
  float sx = 0.0f, sx2 = 0.0f;
  for (int s2 = 0; s2 < slices; ++s2) { sx += part[(size_t)s2 * d.m + i]; if (want_x2) sx2 += part[(size_t)(slices + s2) * d.m + i]; }
  char* base2 = (char*)a.out + (want_x ? (size_t)d.ldo * xb_dev_typesize(d.t_out) : 0);
  if (want_x) { if (init_acc) sx += ld_f32(a.out, i, d.t_out); st_f32(a.out, i, d.t_out, sx); }
  if (want_x2) { if (init_acc) sx2 += ld_f32(base2, i, d.t_out); st_f32(base2, i, d.t_out, sx2); }
}

// ---- gather / scatter (:1444-1794) ------------------------------------------------------------------------------------
template <typename E>
__global__ void __launch_bounds__(256) meltw_gs_kernel(const xb_meltw_desc d, const margs a) {
  const E* in = (const E*)a.in0; E* out = (E*)a.out;
  const bool gather = (d.op == LIBXSMM_MELTW_TYPE_UNARY_GATHER);
  const void* idxp = gather ? a.in_aux : (const void*)a.out_aux;
  const bool idx8 = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_IDX_SIZE_8BYTES) != 0;
  const bool cols = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_GS_COLS) != 0, rows = !cols && (d.flags & LIBXSMM_MELTW_FLAG_UNARY_GS_ROWS) != 0;
  const long long M = d.m, N = d.n, ldi = d.ldi, ldo = d.ldo;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < M * N; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e % M, j = e / M;
    const long long sel = cols ? j : (rows ? i : (i + j * M));
    const long long x = idx8 ? (long long)((const unsigned long long*)idxp)[sel] : (long long)((const unsigned int*)idxp)[sel];
    if (gather) out[i + j * ldo] = cols ? in[i + x * ldi] : (rows ? in[x + j * ldi] : in[x]);
    else { if (cols) out[i + x * ldo] = in[i + j * ldi]; else if (rows) out[x + j * ldo] = in[i + j * ldi]; else out[x] = in[i + j * ldi]; }
  }
}

// ---- block-scaled quantisers: bf16 -> MXFP4 (32 rows, E8M0 scale), NVFP4 (16 rows, E4M3 scale), MXBF8 (32 rows, E8M0) -------------
// reference :1796-2073 (block converters) and :2247-2326 (layout: data ld = ldo/2 bytes for the 4-bit formats, scales ld = ldo/block).
// One thread owns one block: the block's values stay in registers between the amax pass and the encode pass.
__device__ __forceinline__ unsigned int mx_e2m1(float a) {             // |x| -> code of {0, .5, 1, 1.5, 2, 3, 4, 6}; ties to the even code
  if (a != a) return 7u;
  unsigned int c = (a > 0.25f) + (a >= 0.75f) + (a > 1.25f) + (a >= 1.75f) + (a > 2.5f) + (a >= 3.5f) + (a > 5.0f);
  return c;
}
__device__ __forceinline__ unsigned int mx_e4m3_scale(float v) {       // RNE, clamp to 448, flush below 2^-10 (:1812-1893)
  const unsigned int u = __float_as_uint(v), sign = (u >> 31) << 7, ef = (u >> 23) & 0xffu, mf = u & 0x7fffffu;
  int e = (int)ef - 127;
  if (ef == 0xffu && mf != 0u) return sign | 0x7fu;
  if (ef == 0xffu || fabsf(v) > 448.0f || e > 8) return sign | 0x78u;
  if (ef == 0u || e < -9) return sign;
  if (e >= -6) {
    unsigned int m = mf >> 20;
    if (((mf >> 19) & 1u) && ((mf & 0x7ffffu) || (m & 1u))) ++m;
    if (m == 8u) { m = 0u; ++e; }
    return (e + 7 >= 15) ? (sign | 0x78u) : (sign | ((unsigned int)(e + 7) << 3) | m);
  }
  const int sh = -6 - e;
  const unsigned int full = 8u | (mf >> 20);
  const bool sticky = ((full & ((1u << (sh - 1)) - 1u)) != 0u) || ((mf & 0xfffffu) != 0u);
  unsigned int m = full >> sh;
  if (((full >> (sh - 1)) & 1u) && (sticky || (m & 1u))) ++m;
  return (m >= 8u) ? (sign | 0x08u) : (sign | (m & 7u));
}
__device__ __forceinline__ float mx_bf16_round(float f) { return __uint_as_float((unsigned int)xb_f32_to_bf16_rne(f) << 16); }
template <int BLK, int KIND, bool B>     // KIND 0: MXFP4, 1: NVFP4, 2: MXBF8
__global__ void __launch_bounds__(128) meltw_mxquant_kernel(const unsigned short* __restrict__ in0, unsigned char* __restrict__ out0, unsigned char* __restrict__ scl0,
                                                            int m, int n, long long ldi, long long ldo,
                                                            long long count, long long s_in, long long s_out, long long s_scl) {
  const long long blocks_m = m / BLK, ld_data = (KIND == 2) ? ldo : ldo / 2, ld_scl = ldo / BLK;
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= blocks_m * n) return;
  const long long b = e % blocks_m, j = e / blocks_m;
  XB_FOR_CALLS(t, count) {
  const unsigned short* __restrict__ in = adv(in0, t, s_in);
  unsigned char* __restrict__ out = adv(out0, t, s_out);
  unsigned char* __restrict__ scl = adv(scl0, t, s_scl);
  const unsigned short* src = in + j * ldi + b * BLK;
  float x[BLK];
  float amax = 0.0f;
#pragma unroll
  for (int k = 0; k < BLK; ++k) { x[k] = __uint_as_float((unsigned int)src[k] << 16); const float a = fabsf(x[k]); if (a > amax || a != a) amax = a; }
  unsigned char* o = out + j * ld_data + b * ((KIND == 2) ? BLK : BLK / 2);
  if (KIND == 1) {
    unsigned int sc = 0u; float sv = 0.0f;
    if (amax != 0.0f) { sc = mx_e4m3_scale(mx_bf16_round(__fmul_rn(mx_bf16_round(amax), __uint_as_float(0x3e2a0000u)))); sv = xb_hf8_to_f32((uint8_t)sc); }
    scl[j * ld_scl + b] = (unsigned char)sc;
    const float rcp = (sv == 0.0f) ? 0.0f : mx_bf16_round(__fdiv_rn(1.0f, mx_bf16_round(sv)));
#pragma unroll
    for (int k = 0; k < BLK / 2; ++k) {
      const unsigned int lo = ((__float_as_uint(x[2 * k]) >> 31) << 3) | mx_e2m1(fabsf(mx_bf16_round(__fmul_rn(x[2 * k], rcp))));
      const unsigned int hi = ((__float_as_uint(x[2 * k + 1]) >> 31) << 3) | mx_e2m1(fabsf(mx_bf16_round(__fmul_rn(x[2 * k + 1], rcp))));
      o[k] = (sv == 0.0f) ? (unsigned char)0 : (unsigned char)((hi << 4) | lo);
    }
  } else {
    int se = (int)((__float_as_uint(amax) >> 23) & 0xffu);
    const bool special = (se == 0xff);
    const int emax = (KIND == 0) ? 2 : 15;
    se = special ? 0xff : (se - emax < 0 ? 0 : se - emax);
    scl[j * ld_scl + b] = (unsigned char)se;
    const float scale = __uint_as_float(((unsigned int)se << 23) | ((se == 0 || special) ? 0x400000u : 0u));
    if (KIND == 0) {
#pragma unroll
      for (int k = 0; k < BLK / 2; ++k) {
        const unsigned int lo = ((__float_as_uint(x[2 * k]) >> 31) << 3) | mx_e2m1(fabsf(__fdiv_rn(x[2 * k], scale)));
        const unsigned int hi = ((__float_as_uint(x[2 * k + 1]) >> 31) << 3) | mx_e2m1(fabsf(__fdiv_rn(x[2 * k + 1], scale)));
        o[k] = special ? (unsigned char)0x77 : (unsigned char)((hi << 4) | lo);
      }
    } else {
#pragma unroll
      for (int k = 0; k < BLK; ++k) o[k] = special ? (unsigned char)0x7b : (unsigned char)xb_f32_to_bf8(__fdiv_rn(x[k], scale));
    }
  }
  }
}

// ---- quant / dequant (:2195-2360) ----------------------------------------------------------------------------------------
template <bool B>
__global__ void __launch_bounds__(256) meltw_quant_kernel(const xb_meltw_desc d, const margs a0, const mtiles tl) {
  const bool quant = (d.op == LIBXSMM_MELTW_TYPE_UNARY_QUANT);
  const bool sat = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_SIGN_SAT_QUANT) != 0;
  XB_FOR_TILES(a0) {
  const margs a = B ? tile_args(a0, tl, t_) : a0;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < (long long)d.m * d.n; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e % d.m), j = (int)(e / d.m);
    const long long ii = bidx(d, 0, i, j, d.ldi), oi = i + (long long)j * d.ldo;
    if (quant) {
      const float r = nearbyintf(((const float*)a.in0)[ii] * a.alpha);
      if (d.t_out == LIBXSMM_DATATYPE_I8) ((signed char*)a.out)[oi] = sat ? (signed char)fminf(fmaxf(r, -128.f), 127.f) : (signed char)(0xff & (int)r);
      else if (d.t_out == LIBXSMM_DATATYPE_I16) ((short*)a.out)[oi] = sat ? (short)fminf(fmaxf(r, -32768.f), 32767.f) : (short)(0xffff & (int)r);
      else ((int*)a.out)[oi] = (int)r;
    } else {
      float v;
      if (d.t_in0 == LIBXSMM_DATATYPE_I8) v = (float)((const signed char*)a.in0)[ii];
      else if (d.t_in0 == LIBXSMM_DATATYPE_I16) v = (float)((const short*)a.in0)[ii];
      else v = (float)((const int*)a.in0)[ii];
      ((float*)a.out)[oi] = v * a.alpha;
    }
  }
  }
}

// ---- dropout (:2361-2422). The reference draws 16 uniform numbers per group of 16 rows from a 16-lane xoshiro128+ state
// (libxsmm_lsfr_Xwide, :43-73) walking the matrix column by column; lane w of group g therefore sees the (g+1)-th number of
// sequence w. Phase 1 (one warp, lanes 0..15 = the 16 sequences) produces the numbers in that order and leaves the advanced
// state behind, phase 2 applies them to all elements in parallel. Sequential in the number of groups -- exact by construction.
__global__ void __launch_bounds__(32) meltw_rng_kernel(unsigned int* __restrict__ state, float* __restrict__ rnd, long long groups) {
  const int w = threadIdx.x;
  if (w >= 16) return;
  unsigned int s0 = state[w], s1 = state[16 + w], s2 = state[32 + w], s3 = state[48 + w];
  for (long long g = 0; g < groups; ++g) {
    rnd[g * 16 + w] = __uint_as_float(0x3f800000u | ((s3 + s0) >> 9)) - 1.0f;
    const unsigned int t = s1 << 9;
    s2 ^= s0; s3 ^= s1; s1 ^= s2; s0 ^= s3; s2 ^= t; s3 = (s3 << 11) | (s3 >> 21);
  }
  state[w] = s0; state[16 + w] = s1; state[32 + w] = s2; state[48 + w] = s3;
}
// random bytes for stochastic rounding: element e draws from sequence e % 16 (libxsmm_lsfr_i32, src/libxsmm_lpflt_quant.c:303-330:
// xoshiro128++ per lane, top byte of the draw); sequential per lane like the dropout generator above
__global__ void __launch_bounds__(32) meltw_rng8_kernel(unsigned int* __restrict__ state, unsigned char* __restrict__ rnd8, long long count) {
  const int w = threadIdx.x;
  if (w >= 16) return;
  unsigned int s0 = state[w], s1 = state[16 + w], s2 = state[32 + w], s3 = state[48 + w];
  for (long long e = w; e < count; e += 16) {
    const unsigned int sum = s0 + s3;
    rnd8[e] = (unsigned char)((((sum << 7) | (sum >> 25)) + s0) >> 24);
    const unsigned int t = s1 << 9;
    s2 ^= s0; s3 ^= s1; s1 ^= s2; s0 ^= s3; s2 ^= t; s3 = (s3 << 11) | (s3 >> 21);
  }
  state[w] = s0; state[16 + w] = s1; state[32 + w] = s2; state[48 + w] = s3;
}
template <bool B>
__global__ void __launch_bounds__(256) meltw_dropout_kernel(const xb_meltw_desc d, const margs a0, const mtiles tl) {
  const int lane = threadIdx.x & 31;
  const int chunks = (d.m + 31) / 32, gpc = (d.m + 15) / 16;
  const bool fwd = (d.op == LIBXSMM_MELTW_TYPE_UNARY_DROPOUT);
  const bool bitm = (d.flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) != 0;
  const float pn = 1.0f - a0.alpha, pi = 1.0f / pn;
  const long long nwork = (long long)chunks * d.n, wstride = (long long)gridDim.x * (blockDim.x >> 5);
  XB_FOR_TILES(a0) {                                        // batches: DROPOUT_INV only (the forward generator chains call to call)
  const margs a = B ? tile_args(a0, tl, t_) : a0;
  for (long long w = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < nwork; w += wstride) {
    const int j = (int)(w / chunks), i0 = (int)(w % chunks) * 32, i = i0 + lane;
    const bool act = i < d.m;
    const float x = act ? ld_f32(a.in0, bidx(d, 0, i, j, d.ldi), d.t_in0) : 0.0f;
    if (fwd) {
      const bool keep = act && (a.rnd[((long long)j * gpc + i / 16) * 16 + (i % 16)] < pn);
      if (act) st_f32(a.out, i + (long long)j * d.ldo, d.t_out, keep ? pi * x : 0.0f);
      if (bitm) mask_store(a.out_aux, i0, j, ((d.ldo + 15) / 16) * 16, d.m, keep, lane);
    } else if (act) {
      const long long mld = bitm ? ((d.ldi + 15) / 16) * 16 : d.ldi;
      st_f32(a.out, i + (long long)j * d.ldo, d.t_out, mask_bit(a.in_aux, i, j, mld) ? x * pi : 0.0f);
    }
  }
  }
}

// ---- f32 -> bf16 planes: UNZIP (low/high halves), DECOMP_FP32_TO_BF16X2/X3 (truncated head + rounded remainders) (:2423-2469)
__global__ void __launch_bounds__(256) meltw_split_kernel(const xb_meltw_desc d, const margs a) {
  const float* in = (const float*)a.in0;
  unsigned short* out = (unsigned short*)a.out;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < (long long)d.m * d.n; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e % d.m), j = (int)(e / d.m);
    const float x = in[bidx(d, 0, i, j, d.ldi)];
    const long long o = i + (long long)j * d.ldo;
    const unsigned int bits = __float_as_uint(x);
    if (d.op == LIBXSMM_MELTW_TYPE_UNARY_UNZIP) {
      out[o] = (unsigned short)(bits & 0xffffu);
      ((unsigned short*)((char*)a.out + a.off[0]))[o] = (unsigned short)(bits >> 16);
    } else {
      const float head = __uint_as_float(bits & 0xffff0000u);
      const float r1 = __fsub_rn(x, head);
      out[o] = (unsigned short)(bits >> 16);
      if (d.op == LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X3) {
        const unsigned int b1 = __float_as_uint(r1);
        const float r2 = __fsub_rn(r1, __uint_as_float(b1 & 0xffff0000u));
        out[o + (long long)(a.off[0] / 2)] = (unsigned short)(b1 >> 16);
        out[o + (long long)(a.off[1] / 2)] = xb_f32_to_bf16_rne(r2);
      } else out[o + (long long)(a.off[0] / 2)] = xb_f32_to_bf16_rne(r1);
    }
  }
}

// grid of a launch: `gx` blocks per call (the single call's grid), and as many calls side by side in y as keep the whole grid within
// `cap` blocks; the kernels stride the remaining calls through blockIdx.y. A single call gets gridDim.y = 1.
dim3 batch_grid(long long gx, long long count, long long cap) {
  long long gy = cap / (gx > 0 ? gx : 1);
  if (gy > count) gy = count;
  if (gy > 65535) gy = 65535;
  if (gy < 1) gy = 1;
  return dim3((unsigned int)gx, (unsigned int)gy);
}

int launch_done(const char* where) {
  xb_rt_count_launch_backend(LIBXSMM_B200_BACKEND_STREAM);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { xb_rt_note_error((int)e, where); return (int)e; }
  return 0;
}

}  // namespace

extern "C" int xb_meltw_supported(const xb_meltw_desc* d) { return family_of(*d) != FAM_NONE; }

// which kernel a call runs (the variant numbers of libxsmm_b200_meltw_variant, include/libxsmm_b200.h). The choice depends on the
// shape and, for the vector kernels, on the alignment of the operands the kernel reads and writes:
//   NORM_TO_NORMT with m*n >= 4096 ................................................. 1 tiled transpose (64 x 64 tiles)
//   NORM_TO_VNNI2(_PAD) 16-bit / NORM_TO_VNNI4(_PAD) 8-bit with ldo*n >= 4096 ........ 2 VNNI pack, or 3 with 16-byte accesses when
//                                                                                      m, ldi, ldo are multiples of 16/size and in0, out
//                                                                                      are 16-byte aligned
//   other transforms ................................................................ 0 generic transform
//   column sum / sum of squares, not F64, m >= 256, m*n >= 2^18 ...................... 5 two-phase column reduction, or 6 with the float4
//                                                                                      partial pass (F32, m % 4 = 0, ldi % 4 = 0, in0
//                                                                                      16-byte aligned)
//   other reductions (rows, max / min / absmax, column-index, F64) ................... 4 warp reduction
//   maps, to-scalar, gather / scatter, quantisers, dropout, unzip / decomp ........... 7
// A batch (a->count > 1) takes the same kernel as its single call, except: the 16-byte VNNI pack also needs both byte strides to be
// multiples of 16, and column sums take the warp reduction (4) -- the two-phase reduction's scratch is sized for one call.
extern "C" int xb_meltw_variant(const xb_meltw_desc* d, const xb_meltw_args* a) {
  const int fam = family_of(*d);
  const bool batch = a->count > 1;
  if (fam == FAM_TRANSFORM) {
    const int ts = xb_dev_typesize(d->t_in0);
    if (d->op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT && (long long)d->m * d->n >= 4096) return 1;
    if ((long long)d->ldo * d->n >= 4096 && ((ts == 2 && (d->op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2 || d->op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD))
                                          || (ts == 1 && (d->op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4 || d->op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4_PAD)))) {
      const int V = (ts == 2) ? 2 : 4, R = 16 / ts;
      const long long items = (long long)((d->n + V - 1) / V) * (d->ldo / R);
      const uintptr_t strides = batch ? (uintptr_t)(a->s_in0 | a->s_out) : 0;
      const bool vec = (d->m % R) == 0 && (d->ldi % R) == 0 && (d->ldo % R) == 0 && (((uintptr_t)a->in0 | (uintptr_t)a->out | strides) & 15) == 0
                    && (items + 255) / 256 <= 0x7fffffffll;
      return vec ? 3 : 2;
    }
    return 0;
  }
  if (fam == FAM_REDUCE) {
    const bool sum_op = (d->op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ADD || d->op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD || d->op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD);
    if (!batch && sum_op && (d->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_ROWS) == 0 && d->t_in0 != LIBXSMM_DATATYPE_F64 && (long long)d->m * d->n >= (1 << 18) && d->m >= 256) {
      return (d->t_in0 == LIBXSMM_DATATYPE_F32 && (d->m % 4) == 0 && (d->ldi % 4) == 0 && ((uintptr_t)a->in0 & 15) == 0) ? 6 : 5;
    }
    return 4;
  }
  return 7;
}

// the same answer for a handle and the argument struct of a call. Pageable operands are answered for the scratch buffers they are
// staged through (256-byte aligned); a NULL param stands for aligned device operands. -1: not a matrix-eltwise handle.
LIBXSMM_API int libxsmm_b200_meltw_variant(const void* kernel, const void* param) {
  const xb_slot* s = xb_slot_of(kernel);
  const void* staged = (const void*)(uintptr_t)256;
  xb_meltw_args a;
  if (s == nullptr || s->kind != XB_KIND_MELTW) return -1;
  memset(&a, 0, sizeof(a));
  a.in0 = staged; a.out = (void*)(uintptr_t)staged;
  if (param != nullptr && s->u.meltw.op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    const libxsmm_meltw_unary_param* p = (const libxsmm_meltw_unary_param*)param;
    if (p->in.primary != nullptr && xb_rt_ptr_kind(p->in.primary) != 0) a.in0 = p->in.primary;
    if (p->out.primary != nullptr && xb_rt_ptr_kind(p->out.primary) != 0) a.out = p->out.primary;
  }
  return xb_meltw_variant(&s->u.meltw, &a);
}

extern "C" int xb_meltw_launch(const xb_meltw_desc* d, const xb_meltw_args* a) {
  cudaStream_t st = (cudaStream_t)xb_rt_stream();
  const int fam = family_of(*d);
  if (d->m <= 0 || d->n <= 0) return 0;
  const int variant = xb_meltw_variant(d, a);
  const long long count = (a->count > 1) ? a->count : 1;   // calls in this launch: every grid below is the single call's in x, calls in y
  const margs ka = { a->in0, a->in1, a->in2, a->out, a->in_aux, a->out_aux, a->alpha, a->n_rt, { a->off[0], a->off[1] }, a->rng, a->rnd, a->rnd8 };
  const mtiles tl = { count, a->s_in0, a->s_in1, a->s_in2, a->s_in_aux, a->s_out, a->s_out_aux };
  if (count > 1 && (fam == FAM_GS || fam == FAM_SPLIT || a->rnd8 != nullptr || a->n_rt != 0
                    || (fam == FAM_DROPOUT && d->op == LIBXSMM_MELTW_TYPE_UNARY_DROPOUT))) {
    xb_rt_note_error(1, "meltw: this operation has per-call state or run-time extents and runs one call per launch"); return 1;
  }
  // the kernels' tile-axis flag: a batch launches <.., true>, a single call <.., false>
  const auto run = [&](auto batched) -> int {
  constexpr bool B = decltype(batched)::value;
  switch (fam) {
    case FAM_MAP: {
      const int n_eff = (d->op_class == LIBXSMM_MELTW_OPERATION_UNARY && d->op == LIBXSMM_MELTW_TYPE_UNARY_REPLICATE_COL_VAR) ? (int)a->n_rt : d->n;
      const long long warps = (long long)((d->m + 31) / 32) * n_eff;
      long long grid = (warps + 7) / 8; if (grid > 132 * 8) grid = 132 * 8; if (grid < 1) return 0;
      if (a->rnd8 != nullptr) {
        meltw_rng8_kernel<<<1, 32, 0, st>>>((unsigned int*)a->rng, a->rnd8, (long long)d->m * n_eff);
        if (launch_done("meltw_rng8") != 0) return 1;
      }
      meltw_map_kernel<B><<<batch_grid(grid, count, 132 * 8), 256, 0, st>>>(*d, ka, tl, n_eff);
      return launch_done("meltw_map");
    }
    case FAM_REDUCE: {
      if (variant == 5 || variant == 6) {
        // big column reduction: coalesced two-phase version (partial sums per column slice, then the slices in order)
        int slices = (int)(((long long)132 * 4 * 128 + d->m - 1) / d->m); if (slices > d->n / 16) slices = d->n / 16; if (slices < 1) slices = 1; if (slices > 256) slices = 256;
        const int want_x2 = (d->op != LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ADD);
        float* part = (float*)xb_rt_scratch((size_t)2 * slices * d->m * sizeof(float));
        if (part == nullptr) { xb_rt_note_error(2, "meltw_reduce: no scratch for the partial sums"); return 1; }
        if (variant == 6) {
          const dim3 gv((d->m + 127) / 128, slices);
          meltw_reduce_cols_partial_vec_kernel<<<gv, 256, 0, st>>>((const float*)a->in0, d->m, d->n, d->ldi, part, want_x2);
        } else {
          const dim3 g((d->m + 255) / 256, slices);
          meltw_reduce_cols_partial_kernel<<<g, 256, 0, st>>>(*d, ka, part, want_x2);
        }
        if (launch_done("meltw_reduce_partial") != 0) return 1;
        meltw_reduce_cols_final_kernel<<<(d->m + 255) / 256, 256, 0, st>>>(*d, ka, part, slices);
        return launch_done("meltw_reduce_final");
      }
      const int nres = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_ROWS) ? d->n : d->m;
      int grid = (nres + 7) / 8; if (grid > 132 * 8) grid = 132 * 8;
      const dim3 g = batch_grid(grid, count, 132 * 8);
      if (d->t_in0 == LIBXSMM_DATATYPE_F64) meltw_reduce_kernel<double, B><<<g, 256, 0, st>>>(*d, ka, tl);
      else meltw_reduce_kernel<float, B><<<g, 256, 0, st>>>(*d, ka, tl);
      return launch_done("meltw_reduce");
    }
    case FAM_SCALAR: {
      const dim3 g = batch_grid(1, count, 132 * 2);
      if (d->t_in0 == LIBXSMM_DATATYPE_F64) meltw_scalar_kernel<double, B><<<g, 1024, 0, st>>>(*d, ka, tl);
      else meltw_scalar_kernel<float, B><<<g, 1024, 0, st>>>(*d, ka, tl);
      return launch_done("meltw_scalar");
    }
    case FAM_TRANSFORM: case FAM_GS: {
      const long long work = (long long)(d->ldo > d->m ? d->ldo : d->m) * ((d->n + 3) / 4 * 4);
      long long grid = (work + 255) / 256; if (grid > 132 * 16) grid = 132 * 16; if (grid < 1) grid = 1;
      const int ts = xb_dev_typesize(d->t_in0);
      const long long si = a->s_in0, so = a->s_out;
      if (variant == 1) {
        const long long tiles = (long long)((d->m + 63) / 64) * ((d->n + 63) / 64);
        if (tiles > 0x7fffffffll) return 1;
        const dim3 tg = batch_grid(tiles, count, 132 * 8);
        if (ts == 8) meltw_transpose_tiled_kernel<unsigned long long, B><<<tg, 256, 0, st>>>((const unsigned long long*)a->in0, (unsigned long long*)a->out, d->m, d->n, d->ldi, d->ldo, count, si, so);
        else if (ts == 4) meltw_transpose_tiled_kernel<unsigned int, B><<<tg, 256, 0, st>>>((const unsigned int*)a->in0, (unsigned int*)a->out, d->m, d->n, d->ldi, d->ldo, count, si, so);
        else if (ts == 2) meltw_transpose_tiled_kernel<unsigned short, B><<<tg, 256, 0, st>>>((const unsigned short*)a->in0, (unsigned short*)a->out, d->m, d->n, d->ldi, d->ldo, count, si, so);
        else meltw_transpose_tiled_kernel<unsigned char, B><<<tg, 256, 0, st>>>((const unsigned char*)a->in0, (unsigned char*)a->out, d->m, d->n, d->ldi, d->ldo, count, si, so);
        return launch_done("meltw_transpose");
      }
      if (variant == 3) {
        const long long items = (long long)((d->n + (ts == 2 ? 2 : 4) - 1) / (ts == 2 ? 2 : 4)) * (d->ldo / (16 / ts));
        const dim3 vg = batch_grid((items + 255) / 256, count, 132 * 16);
        if (ts == 2) meltw_vnni_pack_vec_kernel<unsigned short, 2, B><<<vg, 256, 0, st>>>((const unsigned short*)a->in0, (unsigned short*)a->out, d->m, d->n, d->ldi, d->ldo, count, si, so);
        else meltw_vnni_pack_vec_kernel<unsigned char, 4, B><<<vg, 256, 0, st>>>((const unsigned char*)a->in0, (unsigned char*)a->out, d->m, d->n, d->ldi, d->ldo, count, si, so);
        return launch_done("meltw_vnni_pack_vec");
      }
      if (variant == 2) {
        const int V = (ts == 2) ? 2 : 4;
        const long long workp = (long long)((d->n + V - 1) / V) * ((d->ldo + 3) / 4);
        long long pg = (workp + 255) / 256; if (pg > 132 * 16) pg = 132 * 16;
        const dim3 g = batch_grid(pg, count, 132 * 16);
        if (ts == 2) meltw_vnni_pack_kernel<unsigned short, 2, B><<<g, 256, 0, st>>>((const unsigned short*)a->in0, (unsigned short*)a->out, d->m, d->n, d->ldi, d->ldo, count, si, so);
        else meltw_vnni_pack_kernel<unsigned char, 4, B><<<g, 256, 0, st>>>((const unsigned char*)a->in0, (unsigned char*)a->out, d->m, d->n, d->ldi, d->ldo, count, si, so);
        return launch_done("meltw_vnni_pack");
      }
      if (fam == FAM_TRANSFORM) {
        const dim3 g = batch_grid(grid, count, 132 * 16);
        if (ts == 8) meltw_transform_kernel<unsigned long long, B><<<g, 256, 0, st>>>(*d, ka, tl);
        else if (ts == 4) meltw_transform_kernel<unsigned int, B><<<g, 256, 0, st>>>(*d, ka, tl);
        else if (ts == 2) meltw_transform_kernel<unsigned short, B><<<g, 256, 0, st>>>(*d, ka, tl);
        else meltw_transform_kernel<unsigned char, B><<<g, 256, 0, st>>>(*d, ka, tl);
      } else {
        if (ts == 4) meltw_gs_kernel<unsigned int><<<(unsigned int)grid, 256, 0, st>>>(*d, ka);
        else if (ts == 2) meltw_gs_kernel<unsigned short><<<(unsigned int)grid, 256, 0, st>>>(*d, ka);
        else meltw_gs_kernel<unsigned char><<<(unsigned int)grid, 256, 0, st>>>(*d, ka);
      }
      return launch_done("meltw_move");
    }
    case FAM_QUANT: {
      long long grid = ((long long)d->m * d->n + 255) / 256; if (grid > 132 * 16) grid = 132 * 16;
      meltw_quant_kernel<B><<<batch_grid(grid, count, 132 * 16), 256, 0, st>>>(*d, ka, tl);
      return launch_done("meltw_quant");
    }
    case FAM_MXQUANT: {
      const int blk = (d->t_out == LIBXSMM_DATATYPE_NVFP4X2) ? 16 : 32;
      const long long items = (long long)(d->m / blk) * d->n;
      if (items <= 0) return 0;
      const dim3 g = batch_grid((items + 127) / 128, count, 132 * 16);
      const unsigned short* in = (const unsigned short*)a->in0; unsigned char* out = (unsigned char*)a->out; unsigned char* sc = (unsigned char*)a->out_aux;
      if (d->t_out == LIBXSMM_DATATYPE_MXFP4X2) meltw_mxquant_kernel<32, 0, B><<<g, 128, 0, st>>>(in, out, sc, d->m, d->n, d->ldi, d->ldo, count, a->s_in0, a->s_out, a->s_out_aux);
      else if (d->t_out == LIBXSMM_DATATYPE_NVFP4X2) meltw_mxquant_kernel<16, 1, B><<<g, 128, 0, st>>>(in, out, sc, d->m, d->n, d->ldi, d->ldo, count, a->s_in0, a->s_out, a->s_out_aux);
      else meltw_mxquant_kernel<32, 2, B><<<g, 128, 0, st>>>(in, out, sc, d->m, d->n, d->ldi, d->ldo, count, a->s_in0, a->s_out, a->s_out_aux);
      return launch_done("meltw_mxquant");
    }
    case FAM_DROPOUT: {
      const long long warps = (long long)((d->m + 31) / 32) * d->n;
      long long grid = (warps + 7) / 8; if (grid > 132 * 8) grid = 132 * 8; if (grid < 1) return 0;
      if (d->op == LIBXSMM_MELTW_TYPE_UNARY_DROPOUT) {
        meltw_rng_kernel<<<1, 32, 0, st>>>((unsigned int*)a->rng, a->rnd, (long long)((d->m + 15) / 16) * d->n);
        if (launch_done("meltw_rng") != 0) return 1;
      }
      meltw_dropout_kernel<B><<<batch_grid(grid, count, 132 * 8), 256, 0, st>>>(*d, ka, tl);
      return launch_done("meltw_dropout");
    }
    case FAM_SPLIT: {
      long long grid = ((long long)d->m * d->n + 255) / 256; if (grid > 132 * 16) grid = 132 * 16;
      meltw_split_kernel<<<(unsigned int)grid, 256, 0, st>>>(*d, ka);
      return launch_done("meltw_split");
    }
    default: return 1;
  }
  };
  return (count > 1) ? run(std::true_type()) : run(std::false_type());
}
