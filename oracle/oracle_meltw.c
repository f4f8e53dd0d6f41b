/* TEST INFRASTRUCTURE -- not part of the product; nothing under libxsmm_b200/ may call into this file.
 *
 * CPU restatement (plain C, written from the algorithm) of the reference's portable matrix-eltwise kernels,
 * src/generator_mateltwise_reference_impl.c, for the operations of SURVEY.md 8a (rows a5, a6) that the CUDA
 * library dispatches most: element-wise unary / binary / ternary maps with broadcast, the ReLU family with
 * bitmasks, compare / select / zip, row / column / to-scalar reductions (sum, sum of squares, max, min, absmax), all
 * layout transforms (incl. VNNI8 and the PAD forms), gather / scatter, quantise / dequantise (integer and the block-scaled MXFP4 / NVFP4 /
 * MXBF8 formats), dropout with the reference's 16-lane generator, unzip / decomp, BF8 / HF8 element types, stochastic rounding to BF8, DUMP.
 * Operations that are not restated return 2 and stay pinned by the reference itself (oracle/_ref). Pinned bit for bit -- outputs AND advanced
 * generator states -- against libxsmm_reference_elementwise in tests/test_oracle_meltw.py (transcendental ops: same libm calls, so equal on the
 * same host).
 *
 * Interface mirrors ref_meltw (oracle/ref_shim.c): desc = {op_class, op, flags, m, n, ldi, ldi2, ldi3, ldo,
 * t_in0, t_in1, t_in2, t_out, t_comp}, param = the reference's libxsmm_meltw_{unary,binary,ternary}_param.
 * All matrices are column-major: element (i, j) at i + j*ld.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>
#include "libxsmm_typedefs.h"      /* this repository's own ABI header: enumerators and argument structs */

#define ORACLE_API __attribute__((visibility("default")))

float oracle_bf16_to_f32(uint16_t h);
uint16_t oracle_f32_to_bf16(float f);
float oracle_f16_to_f32(uint16_t h);
uint16_t oracle_f32_to_f16(float f);

typedef struct mdesc { int op_class, op; unsigned int flags; int m, n; long long ldi, ldi2, ldi3, ldo; int t0, t1, t2, to, tc; } mdesc;

static int is_f(int t) { return t == LIBXSMM_DATATYPE_F32 || t == LIBXSMM_DATATYPE_BF16 || t == LIBXSMM_DATATYPE_F16 || t == LIBXSMM_DATATYPE_BF8 || t == LIBXSMM_DATATYPE_HF8; }
static float bf8_value(unsigned b);  static unsigned bf8_rne(float f);      /* 8-bit floats: defined with the block quantisers below */
static float e4m3_value(unsigned b); static unsigned e4m3_rne(float f);
static int tsz(int t) {
  switch (t) { case LIBXSMM_DATATYPE_F64: case LIBXSMM_DATATYPE_I64: case LIBXSMM_DATATYPE_U64: return 8;
               case LIBXSMM_DATATYPE_F32: case LIBXSMM_DATATYPE_I32: case LIBXSMM_DATATYPE_U32: return 4;
               case LIBXSMM_DATATYPE_BF16: case LIBXSMM_DATATYPE_F16: case LIBXSMM_DATATYPE_I16: case LIBXSMM_DATATYPE_U16: return 2;
               default: return 1; }
}
/* load to f32 / store with RNE: reference :2470-2498 (load via libxsmm_convert_*_to_f32, store via *_rne) */
static float ldf(const void* p, long long i, int t) {
  if (t == LIBXSMM_DATATYPE_F32) return ((const float*)p)[i];
  if (t == LIBXSMM_DATATYPE_BF16) return oracle_bf16_to_f32(((const uint16_t*)p)[i]);
  if (t == LIBXSMM_DATATYPE_BF8) return bf8_value(((const uint8_t*)p)[i]);
  if (t == LIBXSMM_DATATYPE_HF8) return e4m3_value(((const uint8_t*)p)[i]);
  return oracle_f16_to_f32(((const uint16_t*)p)[i]);
}
static void stf(void* p, long long i, int t, float v) {
  if (t == LIBXSMM_DATATYPE_F32) ((float*)p)[i] = v;
  else if (t == LIBXSMM_DATATYPE_BF16) ((uint16_t*)p)[i] = oracle_f32_to_bf16(v);
  else if (t == LIBXSMM_DATATYPE_BF8) ((uint8_t*)p)[i] = (uint8_t)bf8_rne(v);
  else if (t == LIBXSMM_DATATYPE_HF8) ((uint8_t*)p)[i] = (uint8_t)e4m3_rne(v);
  else ((uint16_t*)p)[i] = oracle_f32_to_f16(v);
}
/* store with optional stochastic rounding (libxsmm_elementwise_store_value :299-325): only a BF8 output uses the flag. Element number e
 * of the op (j-major, i inner) draws from generator e % 16 of the 4 x 16-word state (libxsmm_lsfr_i32, src/libxsmm_lpflt_quant.c:303-330:
 * one xoshiro128++ step); the top byte is added to the f16 image below the 8 kept bits; f16-subnormals round to nearest even instead,
 * Inf / NaN pass (src/libxsmm_lpflt_quant.c:332-368) */
static void stf_rnd(void* p, long long i, int t, float v, int stochastic, uint32_t* state, long long e) {
  if (stochastic && t == LIBXSMM_DATATYPE_BF8 && state != NULL) {
    uint32_t* s = state + (e % 16);
    const uint32_t sum = s[0] + s[48], draw = ((sum << 7) | (sum >> 25)) + s[0], t9 = s[16] << 9;
    unsigned h = oracle_f32_to_f16(v);
    s[32] ^= s[0]; s[48] ^= s[16]; s[16] ^= s[32]; s[0] ^= s[48]; s[32] ^= t9; s[48] = (s[48] << 11) | (s[48] >> 21);
    if ((h & 0x7c00u) == 0x7c00u) { if (h & 0x3ffu) h |= 0x200u; }
    else if ((h & 0x7c00u) == 0) h = (h + 0x7fu + ((h >> 8) & 1u)) & 0xffffu;
    else h = (h + (draw >> 24)) & 0xffffu;
    ((uint8_t*)p)[i] = (uint8_t)(h >> 8);
  } else stf(p, i, t, v);
}
/* operand index under the broadcast flags: reference :241-272 (row-bcast -> j*ld, col-bcast -> i, scalar -> 0) */
static long long bidx(const mdesc* d, int which, int i, int j, long long ld) {
  unsigned int row = 0, col = 0, sca = 0;
  if (d->op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    row = d->flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_ROW; col = d->flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_COL; sca = d->flags & LIBXSMM_MELTW_FLAG_UNARY_BCAST_SCALAR;
  } else if (d->op_class == LIBXSMM_MELTW_OPERATION_BINARY) {
    row = d->flags & (which == 0 ? LIBXSMM_MELTW_FLAG_BINARY_BCAST_ROW_IN_0 : LIBXSMM_MELTW_FLAG_BINARY_BCAST_ROW_IN_1);
    col = d->flags & (which == 0 ? LIBXSMM_MELTW_FLAG_BINARY_BCAST_COL_IN_0 : LIBXSMM_MELTW_FLAG_BINARY_BCAST_COL_IN_1);
    sca = d->flags & (which == 0 ? LIBXSMM_MELTW_FLAG_BINARY_BCAST_SCALAR_IN_0 : LIBXSMM_MELTW_FLAG_BINARY_BCAST_SCALAR_IN_1);
  } else {
    const unsigned int r[3] = { LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_0, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_1, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_ROW_IN_2 };
    const unsigned int c[3] = { LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_0, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_1, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_COL_IN_2 };
    const unsigned int s[3] = { LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_0, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_1, LIBXSMM_MELTW_FLAG_TERNARY_BCAST_SCALAR_IN_2 };
    row = d->flags & r[which]; col = d->flags & c[which]; sca = d->flags & s[which];
  }
  if (row) return (long long)j * ld;
  if (col) return i;
  if (sca) return 0;
  return i + (long long)j * ld;
}
/* bitmask addressing: bit (i, j) at byte i/8 + j*(mask_ld/8), mask_ld = UPDIV(ld,16)*16 bits (reference :2142) */
static long long mask_ld_of(long long ld) { return ((ld + 15) / 16) * 16; }
static int mask_get(const void* mask, int i, int j, long long mld) { return (((const uint8_t*)mask)[i / 8 + (long long)j * (mld / 8)] >> (i % 8)) & 1; }
static void mask_put(void* mask, int i, int j, long long mld, int bit) {
  uint8_t* b = (uint8_t*)mask + i / 8 + (long long)j * (mld / 8);
  *b = (uint8_t)((*b & ~(1u << (i % 8))) | ((unsigned int)(bit != 0) << (i % 8)));
}

/* generic f32 unary ops: reference :76-113 (sigmoid defined through tanh, gelu through erff: :18-40) */
static float sigm(float x) { return (tanhf(x / 2.0f) + 1.0f) / 2.0f; }
static float unary_f32(float x, int op) {
  switch (op) {
    case LIBXSMM_MELTW_TYPE_UNARY_NEGATE: return -1.0f * x;
    case LIBXSMM_MELTW_TYPE_UNARY_X2: return x * x;
    case LIBXSMM_MELTW_TYPE_UNARY_XOR: return 0.0f;
    case LIBXSMM_MELTW_TYPE_UNARY_TANH: return tanhf(x);
    case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID: return sigm(x);
    case LIBXSMM_MELTW_TYPE_UNARY_GELU: return (erff(x / sqrtf(2.0f)) + 1.0f) * 0.5f * x;
    case LIBXSMM_MELTW_TYPE_UNARY_GELU_INV: return 0.5f + 0.5f * erff(x / sqrtf(2.0f)) + x / sqrtf(2.0f * 3.14159265358979323846f) * expf(-0.5f * x * x);
    case LIBXSMM_MELTW_TYPE_UNARY_TANH_INV: { const float t = tanhf(x); return 1.0f - t * t; }
    case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID_INV: { const float s = sigm(x); return s * (1.0f - s); }
    case LIBXSMM_MELTW_TYPE_UNARY_SQRT: return sqrtf(x);
    case LIBXSMM_MELTW_TYPE_UNARY_INC: return x + 1.0f;
    case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL: return 1.0f / x;
    case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL_SQRT: return 1.0f / sqrtf(x);
    case LIBXSMM_MELTW_TYPE_UNARY_EXP: return expf(x);
    default: return x;
  }
}
static double unary_f64(double x, int op) {   /* reference :116-139 */
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

static int unary_map(const mdesc* d, const libxsmm_meltw_unary_param* p) {
  const int op = d->op, f64 = (d->t0 == LIBXSMM_DATATYPE_F64 && d->to == LIBXSMM_DATATYPE_F64);
  const int bitm = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) != 0;
  const float alpha = (p->op.primary != NULL && (op == LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU || op == LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU_INV
                       || op == LIBXSMM_MELTW_TYPE_UNARY_ELU || op == LIBXSMM_MELTW_TYPE_UNARY_ELU_INV)) ? *(const float*)p->op.primary : 0.0f;
  /* REPLICATE_COL_VAR copies the column in0[0..m) into N columns, N = *(unsigned long long*)op.primary at call time (:249, :2084) */
  const int rep = (op == LIBXSMM_MELTW_TYPE_UNARY_REPLICATE_COL_VAR);
  const long long n_eff = rep ? (p->op.primary != NULL ? (long long)*(const unsigned long long*)p->op.primary : -1) : d->n;
  mdesc dc = *d;
  int i, j;
  if (!f64 && !(is_f(d->t0) && is_f(d->to))) return 2;
  if (f64 && (op == LIBXSMM_MELTW_TYPE_UNARY_DUMP || rep)) return 2;      /* not in the reference's F64 op list (:116-138) */
  if (n_eff < 0) return 1;
  if (rep) { dc.flags |= LIBXSMM_MELTW_FLAG_UNARY_BCAST_COL; d = &dc; }
  for (j = 0; j < n_eff; ++j) for (i = 0; i < d->m; ++i) {
    const long long oi = i + (long long)j * d->ldo;
    if (f64) { ((double*)p->out.primary)[oi] = unary_f64(((const double*)p->in.primary)[bidx(d, 0, i, j, d->ldi)], op); continue; }
    {
      const float x = ldf(p->in.primary, bidx(d, 0, i, j, d->ldi), d->t0);
      switch (op) {
        case LIBXSMM_MELTW_TYPE_UNARY_RELU: case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU: case LIBXSMM_MELTW_TYPE_UNARY_ELU: {   /* :2138-2167: test is in <= 0 */
          float y = x;
          if (x <= 0.0f) y = (op == LIBXSMM_MELTW_TYPE_UNARY_RELU) ? 0.0f : ((op == LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU) ? alpha * x : alpha * (expf(x) - 1.0f));
          stf(p->out.primary, oi, d->to, y);
          if (bitm) mask_put(p->out.secondary, i, j, mask_ld_of(d->ldo), !(x <= 0.0f));
        } break;
        case LIBXSMM_MELTW_TYPE_UNARY_RELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU_INV: {                           /* :2168-2194 */
          const int bit = mask_get(p->in.secondary, i, j, bitm ? mask_ld_of(d->ldi) : d->ldi);
          stf(p->out.primary, oi, d->to, bit ? x : ((op == LIBXSMM_MELTW_TYPE_UNARY_RELU_INV) ? 0.0f : alpha * x));
        } break;
        case LIBXSMM_MELTW_TYPE_UNARY_ELU_INV: {
          const float fwd = ldf(p->in.secondary, i + (long long)j * d->ldi, d->t0);
          stf(p->out.primary, oi, d->to, (fwd > 0) ? x : x * (fwd + alpha));
        } break;
        default:
          stf_rnd(p->out.primary, oi, d->to, unary_f32(x, op), (d->flags & LIBXSMM_MELTW_FLAG_UNARY_STOCHASTIC_ROUND) != 0, (uint32_t*)p->op.secondary, (long long)j * d->m + i);
          if (op == LIBXSMM_MELTW_TYPE_UNARY_DUMP) {      /* :2478-2493: the value is stored a second time (the stochastic byte is copied) */
            if ((d->flags & LIBXSMM_MELTW_FLAG_UNARY_STOCHASTIC_ROUND) != 0 && d->to == LIBXSMM_DATATYPE_BF8) ((uint8_t*)p->out.secondary)[oi] = ((uint8_t*)p->out.primary)[oi];
            else stf(p->out.secondary, oi, d->to, x);
          }
      }
    }
  }
  return 0;
}

/* reductions: reference :1065-1443. REDUCE_ROWS collapses i (n results), otherwise j (m results, buffer pitch ldo);
 * X_X2 stores the sums, then the sums of squares at element offset result_size (:1073-1076); INIT_ACC adds the old output.
 * COLS_IDX_OP_* reduce the columns listed in in.secondary (*in.tertiary of them, 4- or 8-byte indices) and ignore INIT_ACC
 * (:1121-1138, :1347-1356). Max / min / absmax are the reference's sequential folds with its macros (include/libxsmm_macros.h:635-637):
 * MAX(A,B) = A < B ? B : A, MIN(A,B) = A < B ? A : B, ABS(A) = 0 <= A ? A : -A (so ABS(-0) = -0 and ABS flips a NaN's sign).
 *   rows (:1215-1224, :1360-1369): tmp = first element, then tmp = f(tmp, x) for EVERY element, the first included;
 *   cols (:1226-1284, :1371-1428): tmp = -FLT_MAX (max), 0 (absmax) or FLT_MAX (min), then tmp = f(x, tmp) -- operands swapped;
 *   RECORD_ARGOP, columns only: x >= tmp (max, absmax) / x <= tmp (min) takes x and records its column in out.secondary,
 *   an index that is never taken is not written. */
#define RMAX(A, B) ((A) < (B) ? (B) : (A))
#define RMIN(A, B) ((A) < (B) ? (A) : (B))
#define RABS(A) (0 <= (A) ? (A) : -(A))
static int unary_reduce(const mdesc* d, const libxsmm_meltw_unary_param* p) {
  const int op = d->op, rows = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_ROWS) != 0;
  const int by_idx = (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_ADD || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MAX
                   || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MIN);
  const int init = !by_idx && (d->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_INIT_ACC) != 0;
  const int argop = !rows && (d->flags & LIBXSMM_MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP) != 0;
  const int idx4 = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_IDX_SIZE_4BYTES) != 0;    /* the reference's default is 8 bytes (:1088) */
  const int f64 = (d->t0 == LIBXSMM_DATATYPE_F64 && d->to == LIBXSMM_DATATYPE_F64);
  const int kind = (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MAX || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MAX) ? 1
                 : ((op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MIN || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MIN) ? 2
                 : ((op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX) ? 3 : 0));
  const int want_x = (op != LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD), want_x2 = (op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD || op == LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD);
  const long long ncols = by_idx ? (p->in.tertiary != NULL ? (long long)*(const unsigned long long*)p->in.tertiary : -1) : d->n;
  const int nres = rows ? d->n : d->m;
  const long long len = rows ? d->m : ncols;
  const long long result_size = rows ? d->n : d->ldo;
  long long t;
  int o;
  if (!f64 && !(is_f(d->t0) && is_f(d->to))) return 2;
  if ((by_idx && (rows || ncols < 0 || p->in.secondary == NULL)) || (argop && kind != 0 && p->out.secondary == NULL)) return 1;
  for (o = 0; o < nres; ++o) {
    double sx = 0.0, sx2 = 0.0, best = 0.0; float fsx = 0.0f, fsx2 = 0.0f, fbest = 0.0f;
    long long arg = -1;
    if (kind != 0 && rows) { if (f64) best = ((const double*)p->in.primary)[(long long)o * d->ldi]; else fbest = ldf(p->in.primary, (long long)o * d->ldi, d->t0); }
    else if (kind != 0) { best = (kind == 1) ? -FLT_MAX : ((kind == 2) ? FLT_MAX : 0); fbest = (kind == 1) ? -FLT_MAX : ((kind == 2) ? FLT_MAX : 0); }
    for (t = 0; t < len; ++t) {
      const long long j = !by_idx ? t : (idx4 ? (long long)((const uint32_t*)p->in.secondary)[t] : (long long)((const uint64_t*)p->in.secondary)[t]);
      const long long idx = rows ? (t + (long long)o * d->ldi) : (o + j * d->ldi);
      if (f64) {
        double v = ((const double*)p->in.primary)[idx];
        if (kind == 0) { sx += v; sx2 += v * v; }
        else if (rows) best = (kind == 1) ? RMAX(best, v) : ((kind == 3) ? RMAX(RABS(best), RABS(v)) : RMIN(best, v));
        else {
          if (kind == 3) v = RABS(v);
          if (argop) { if (kind == 2 ? (v <= best) : (v >= best)) { best = v; arg = j; } }
          else best = (kind == 2) ? RMIN(v, best) : RMAX(v, best);
        }
      } else {
        float v = ldf(p->in.primary, idx, d->t0);
        if (kind == 0) { fsx += v; fsx2 += v * v; }
        else if (rows) fbest = (kind == 1) ? RMAX(fbest, v) : ((kind == 3) ? RMAX(RABS(fbest), RABS(v)) : RMIN(fbest, v));
        else {
          if (kind == 3) v = RABS(v);
          if (argop) { if (kind == 2 ? (v <= fbest) : (v >= fbest)) { fbest = v; arg = j; } }
          else fbest = (kind == 2) ? RMIN(v, fbest) : RMAX(v, fbest);
        }
      }
    }
    if (kind != 0) {
      if (f64) ((double*)p->out.primary)[o] = best; else stf(p->out.primary, o, d->to, fbest);
      if (argop && arg >= 0) { if (idx4) ((uint32_t*)p->out.secondary)[o] = (uint32_t)arg; else ((uint64_t*)p->out.secondary)[o] = (uint64_t)arg; }
    } else if (f64) {
      double* ox = (double*)p->out.primary; double* ox2 = want_x ? ox + result_size : ox;
      if (want_x) ox[o] = sx + (init ? ox[o] : 0.0);
      if (want_x2) ox2[o] = sx2 + (init ? ox2[o] : 0.0);
    } else {
      char* base2 = (char*)p->out.primary + (want_x ? (size_t)result_size * tsz(d->to) : 0);
      if (want_x) { float r = fsx; if (init) r += ldf(p->out.primary, o, d->to); stf(p->out.primary, o, d->to, r); }
      if (want_x2) { float r = fsx2; if (init) r += ldf(base2, o, d->to); stf(base2, o, d->to, r); }
    }
  }
  return 0;
}
#undef RMAX
#undef RMIN
#undef RABS

/* layout transforms, pure data movement: reference :377-1062. Formulas (elements, E = element of 1/2/4/8 bytes):
 *   NORM_TO_NORMT      out[j*ldo + i] = in[i*ldi + j]                      i < n, j < m               (:390-417)
 *   NORM_TO_VNNIv(_PAD) the WHOLE ldo x ceil(n/v)*v output is defined: zero, except
 *                      out[j*ldo*v + i*v + j2] = in[(j*v + j2)*ldi + i]     i < m, j*v + j2 < n        (:541-553, :690-759)
 *   NORM_TO_VNNIvT     out[i*ldo*v + j*v + i2] = in[j*ldi + i*v + i2]       i < m/v, j < n
 *   VNNIv_TO_VNNIvT    out[j*ldo*v + j2 + (i*v + i2)*v] = in[i*ldi*v + i2 + (j*v + j2)*v]   i < n/v, j < m/v (:433-441)
 *   VNNIvT_TO_NORM     roles of m and n swapped: out[j*ldo + i*v + i2] = in[i*ldi*v + j*v + i2]   i < n/v, j < m  (:620-660)
 *   VNNI4_TO_NORM      out[i*ldo + j] = in[(i/4)*ldi*4 + j*4 + i%4]         i < n, j < m               (:787-803) */
#define CP(dst_idx, src_idx) memcpy(out + (dst_idx) * ts, in + (src_idx) * ts, (size_t)ts)
static int unary_transform(const mdesc* d, const libxsmm_meltw_unary_param* p) {
  const int ts = tsz(d->t0), op = d->op;
  const char* in = (const char*)p->in.primary; char* out = (char*)p->out.primary;
  const long long M = d->m, N = d->n, ldi = d->ldi, ldo = d->ldo;
  long long i, j, i2, j2, v;
  switch (op) {
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT:
      for (j = 0; j < M; ++j) for (i = 0; i < N; ++i) CP(j * ldo + i, i * ldi + j);
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD:
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4_PAD: {
      long long e; const long long Nn = 0;
      v = (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD) ? 2 : 4;
      (void)Nn;
      for (e = 0; e < ldo * (((N + v - 1) / v) * v); ++e) {
        const long long jj = e / (ldo * v), rem = e % (ldo * v), col = jj * v + rem % v;
        i = rem / v;
        if (i < M && col < N) CP(e, col * ldi + i); else memset(out + e * ts, 0, (size_t)ts);
      }
      return 0;
    }
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4T:
      v = (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2T) ? 2 : 4;
      for (i = 0; i < M / v; ++i) for (j = 0; j < N; ++j) for (i2 = 0; i2 < v; ++i2) CP(i * ldo * v + j * v + i2, j * ldi + i * v + i2);
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2_TO_VNNI2T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI4T:
      v = (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2_TO_VNNI2T) ? 2 : 4;
      for (j = 0; j < M / v; ++j) for (i = 0; i < N / v; ++i) for (j2 = 0; j2 < v; ++j2) for (i2 = 0; i2 < v; ++i2)
        CP(j * ldo * v + j2 + (i * v + i2) * v, i * ldi * v + i2 + (j * v + j2) * v);
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2T_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4T_TO_NORM:
      v = (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2T_TO_NORM) ? 2 : 4;
      for (i = 0; i < N / v; ++i) for (j = 0; j < M; ++j) for (i2 = 0; i2 < v; ++i2) CP(j * ldo + i * v + i2, i * ldi * v + j * v + i2);
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_NORM:
      for (i = 0; i < N; ++i) for (j = 0; j < M; ++j) CP(i * ldo + j, (i / 4) * ldi * 4 + j * 4 + (i % 4));
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8_PAD: {   /* :712-786 */
      long long e;                       /* columns past N (only when N % 8 != 0, where the reference reads past its input) count as zero */
      for (e = 0; e < ldo * (((N + 7) / 8) * 8); ++e) {
        const long long jj = e / (ldo * 8), rem = e % (ldo * 8), col = jj * 8 + rem % 8;
        i = rem / 8;
        if (i < M && col < N) CP(e, col * ldi + i); else memset(out + e * ts, 0, (size_t)ts);
      }
      return 0;
    }
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8T:                                                                   /* :666-686 */
      for (i = 0; i < M / 8; ++i) for (j = 0; j < N; ++j) for (i2 = 0; i2 < 8; ++i2) CP(i * ldo * 8 + j * 8 + i2, j * ldi + i * 8 + i2);
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8_TO_VNNI8T:                                                                  /* :489-531 */
      for (j = 0; j < M / 8; ++j) for (i = 0; i < N / 8; ++i) for (j2 = 0; j2 < 8; ++j2) for (i2 = 0; i2 < 8; ++i2)
        CP(j * ldo * 8 + j2 + (i * 8 + i2) * 8, i * ldi * 8 + i2 + (j * 8 + j2) * 8);
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8T_TO_NORM:                                                                   /* :581-601, m/n swapped */
      for (i = 0; i < N / 8; ++i) for (j = 0; j < M; ++j) for (i2 = 0; i2 < 8; ++i2) CP(j * ldo + i * 8 + i2, i * ldi * 8 + j * 8 + i2);
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI2:                                                                   /* :806-823 */
      for (i = 0; i < N; ++i) for (j = 0; j < M; ++j) CP((i / 2) * ldo * 2 + j * 2 + (i % 2), (i / 4) * ldi * 4 + j * 4 + (i % 4));
      return 0;
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD2:
    case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD4: {
      const int mod4 = (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD4 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD4);
      const int padm_only = (op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD2 || op == LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4);
      const long long Nn = padm_only ? N : ((N + (mod4 ? 3 : 1)) / (mod4 ? 4 : 2)) * (mod4 ? 4 : 2);                          /* :825-960 */
      memset(out, 0, (size_t)(ldo * Nn) * ts);
      for (j = 0; j < N; ++j) for (i = 0; i < M; ++i) CP(j * ldo + i, j * ldi + i);
      return 0;
    }
    default: return 2;
  }
}
#undef CP

/* dropout forward / backward: reference :2361-2422 with the 16-lane generator step of :43-73 */
static void lsfr16(unsigned int* st, float* out) {
  int w;
  for (w = 0; w < 16; ++w) {
    unsigned int s0 = st[w], s1 = st[16 + w], s2 = st[32 + w], s3 = st[48 + w], t;
    union { unsigned int u; float f; } r;
    r.u = 0x3f800000u | ((s3 + s0) >> 9);
    out[w] = r.f - 1.0f;
    t = s1 << 9; s2 ^= s0; s3 ^= s1; s1 ^= s2; s0 ^= s3; s2 ^= t; s3 = (s3 << 11) | (s3 >> 21);
    st[w] = s0; st[16 + w] = s1; st[32 + w] = s2; st[48 + w] = s3;
  }
}
static void set_bit(unsigned char* m, long long i, long long j, long long ld, int on) {
  unsigned char* b = m + i / 8 + j * (ld / 8);
  if (on) *b = (unsigned char)(*b | (1u << (i % 8))); else *b = (unsigned char)(*b & ~(1u << (i % 8)));
}
static int unary_dropout(const mdesc* d, const libxsmm_meltw_unary_param* p) {
  const int bitm = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) != 0;
  const float prob = *(const float*)p->op.primary, pn = 1.0f - prob, pi = 1.0f / pn;
  int i, j;
  if (!(is_f(d->t0) && is_f(d->to))) return 2;
  if (d->op == LIBXSMM_MELTW_TYPE_UNARY_DROPOUT) {
    const long long mld = bitm ? ((d->ldo + 15) / 16) * 16 : d->ldo;
    float r[16];
    for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
      float x; int keep;
      if (i % 16 == 0) lsfr16((unsigned int*)p->op.secondary, r);       /* one draw per group of 16 rows, remainder groups included */
      x = ldf(p->in.primary, bidx(d, 0, i, j, d->ldi), d->t0);
      keep = r[i % 16] < pn;
      stf(p->out.primary, i + (long long)j * d->ldo, d->to, keep ? pi * x : 0.0f);
      if (bitm) set_bit((unsigned char*)p->out.secondary, i, j, mld, keep);
    }
  } else {
    const long long mld = bitm ? ((d->ldi + 15) / 16) * 16 : d->ldi;
    for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
      const float x = ldf(p->in.primary, bidx(d, 0, i, j, d->ldi), d->t0) * pi;
      const int bit = (((const unsigned char*)p->in.secondary)[i / 8 + (long long)j * (mld / 8)] >> (i % 8)) & 1;
      stf(p->out.primary, i + (long long)j * d->ldo, d->to, bit ? x : 0.0f);
    }
  }
  return 0;
}
/* f32 -> bf16 planes: reference :2423-2469 */
static int unary_split(const mdesc* d, const libxsmm_meltw_unary_param* p) {
  const unsigned long long* offs = (const unsigned long long*)p->out.secondary;
  uint16_t* out = (uint16_t*)p->out.primary;
  int i, j;
  if (d->t0 != LIBXSMM_DATATYPE_F32) return 2;
  for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
    union { float f; unsigned int u; } x, h, r1, h1;
    const long long o = i + (long long)j * d->ldo;
    x.f = ((const float*)p->in.primary)[bidx(d, 0, i, j, d->ldi)];
    if (d->op == LIBXSMM_MELTW_TYPE_UNARY_UNZIP) {
      out[o] = (uint16_t)(x.u & 0xffffu);
      ((uint16_t*)((char*)p->out.primary + offs[0]))[o] = (uint16_t)(x.u >> 16);
    } else {
      h.u = x.u & 0xffff0000u; r1.f = x.f - h.f;
      out[o] = (uint16_t)(x.u >> 16);
      if (d->op == LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X3) {
        h1.u = r1.u & 0xffff0000u;
        out[o + (long long)(offs[0] / 2)] = (uint16_t)(r1.u >> 16);
        out[o + (long long)(offs[1] / 2)] = oracle_f32_to_bf16(r1.f - h1.f);
      } else out[o + (long long)(offs[0] / 2)] = oracle_f32_to_bf16(r1.f);
    }
  }
  return 0;
}

/* ---- block-scaled quantisers (bf16 -> MXFP4 / NVFP4 / MXBF8): reference :1796-2073, :2247-2326 ------------------------------
 * one scale byte per block of consecutive rows of a column; data and scales have their own leading dimensions derived from ldo */
static float bits_f32(uint32_t u) { union { uint32_t u; float f; } x; x.u = u; return x.f; }
static uint32_t f32_bits(float f) { union { uint32_t u; float f; } x; x.f = f; return x.u; }
static float bf16_round(float f) { return bits_f32((uint32_t)oracle_f32_to_bf16(f) << 16); }    /* f32 -> bf16 (RNE) -> f32 */
/* |x| -> 3-bit E2M1 code {0, .5, 1, 1.5, 2, 3, 4, 6}: round to nearest, ties to the even code, NaN and overflow saturate (:1796-1808) */
static unsigned e2m1_code(float a) {
  static const float edge[7] = { 0.25f, 0.75f, 1.25f, 1.75f, 2.5f, 3.5f, 5.0f };   /* midpoints between neighbouring codes */
  unsigned c = 0;
  if (a != a) return 7;
  while (c < 7 && (a > edge[c] || (a == edge[c] && (c & 1u)))) ++c;                /* a tie goes up only out of an odd code */
  return c;
}
/* f32 -> E4M3 byte for the NVFP4 scale (:1812-1893): RNE, clamps to 448 (0x78) instead of NaN, flushes below 2^-10 */
static unsigned e4m3_scale_code(float v) {
  const uint32_t u = f32_bits(v), sign = (u >> 31) << 7, ef = (u >> 23) & 0xffu, mf = u & 0x7fffffu;
  int e = (int)ef - 127;
  uint32_t m;
  if (ef == 0xff && mf != 0) return sign | 0x7f;
  if (ef == 0xff || fabsf(v) > 448.0f || e > 8) return sign | 0x78;
  if (ef == 0 || e < -9) return sign;
  if (e >= -6) {                                          /* normal: keep 3 mantissa bits */
    m = mf >> 20;
    if (((mf >> 19) & 1u) && ((mf & 0x7ffffu) || (m & 1u))) ++m;
    if (m == 8) { m = 0; ++e; }
    return (e + 7 >= 15) ? (sign | 0x78) : (sign | ((uint32_t)(e + 7) << 3) | m);
  } else {                                                /* subnormal: 1.mmm shifted right by (-6 - e) in 1..3 */
    const int sh = -6 - e;
    const uint32_t full = 8u | (mf >> 20);
    uint32_t sticky = ((full & ((1u << (sh - 1)) - 1u)) != 0) || ((mf & 0xfffffu) != 0);
    m = full >> sh;
    if (((full >> (sh - 1)) & 1u) && (sticky || (m & 1u))) ++m;
    return (m >= 8) ? (sign | 0x08) : (sign | (m & 7u));
  }
}
static float e4m3_value(unsigned b) {                     /* libxsmm_convert_hf8_to_f32 (src/libxsmm_math.c): 0x7f/0xff are NaN */
  const unsigned e = (b >> 3) & 0xf, m = b & 7;
  float v;
  if (e == 0xf && m == 7) return bits_f32(((uint32_t)(b & 0x80) << 24) | 0x7fc00000u);
  v = (e == 0) ? ldexpf((float)m, -9) : ldexpf((float)(8 + m), (int)e - 10);
  return (b & 0x80) ? -v : v;
}
static unsigned bf8_rne(float f) {                        /* libxsmm_convert_f32_to_bf8_rne (src/libxsmm_math.c:731-746): via f16, RNE on the low byte */
  unsigned h = oracle_f32_to_f16(f);
  if ((h & 0x7c00u) == 0x7c00u) { if (h & 0x03ffu) h |= 0x0200u; }
  else h = (h + 0x7fu + ((h >> 8) & 1u)) & 0xffffu;
  return h >> 8;
}
static float bf8_value(unsigned b) { return oracle_f16_to_f32((uint16_t)(b << 8)); }        /* libxsmm_convert_bf8_to_f32 (:546-551) */
/* libxsmm_convert_f32_to_hf8_rne (src/libxsmm_math.c:749-822): through f16; RNE on the 7 dropped mantissa bits; results below 2^-6 are
 * sub-normal (sticky bit kept across the alignment shift); beyond 448 (+ half an ulp) and Inf/NaN all give the NaN code */
static unsigned e4m3_rne(float f) {
  const unsigned h = oracle_f32_to_f16(f), sign = (h & 0x8000u) >> 8, e16 = (h >> 10) & 0x1fu, m16 = h & 0x3ffu;
  unsigned e, m, r;
  if (e16 == 0x1f || e16 > 23 || (e16 == 23 && m16 > 0x340u)) return sign | 0x7fu;
  if (e16 < 5) return sign;
  if (e16 > 8) { r = (h & 0x7fffu) + 0x3fu + ((m16 >> 7) & 1u); e = ((r >> 10) & 0x1fu) - 8u; m = (r & 0x3ffu) >> 7; return sign | (e << 3) | m; }
  m = ((m16 | 0x400u) >> (9 - e16)) | (((m16 & 0x7fu) + 0x7fu) >> 7);
  m = (m + 0x3fu + ((m >> 7) & 1u)) >> 7;
  return sign | m;
}
/* E8M0 shared exponent of a block: biased exponent of the largest |x| (NaN sticks) minus the element format's emax (:1911-1921) */
static int mx_shared_exp(const float* x, int n, int emax, float* scale, int* special) {
  float amax = 0.0f; int i, e;
  for (i = 0; i < n; ++i) { const float a = fabsf(x[i]); if (a > amax || a != a) amax = a; }
  e = (int)((f32_bits(amax) >> 23) & 0xffu);
  *special = (e == 0xff);
  e = *special ? 0xff : (e - emax < 0 ? 0 : e - emax);
  *scale = bits_f32(((uint32_t)e << 23) | ((e == 0 || *special) ? 0x400000u : 0u));     /* 2^(e-127); e = 0 stands for 2^-127 */
  return e;
}
static int unary_mxquant(const mdesc* d, const libxsmm_meltw_unary_param* p) {
  const uint16_t* in = (const uint16_t*)p->in.primary;
  unsigned char* out = (unsigned char*)p->out.primary; unsigned char* scl = (unsigned char*)p->out.secondary;
  const int blk = (d->to == LIBXSMM_DATATYPE_NVFP4X2) ? 16 : 32;
  const long long ld_data = (d->to == LIBXSMM_DATATYPE_MXBF8) ? d->ldo : d->ldo / 2, ld_scl = d->ldo / blk;
  int j, b, k;
  if (d->t0 != LIBXSMM_DATATYPE_BF16 || scl == NULL) return 2;
  for (j = 0; j < d->n; ++j) for (b = 0; b < d->m / blk; ++b) {
    float x[32], scale; int special;
    unsigned char* o = out + (size_t)j * ld_data + (size_t)b * ((d->to == LIBXSMM_DATATYPE_MXBF8) ? blk : blk / 2);
    for (k = 0; k < blk; ++k) x[k] = bits_f32((uint32_t)in[(size_t)j * d->ldi + (size_t)b * blk + k] << 16);   /* no denormal flush here */
    if (d->to == LIBXSMM_DATATYPE_NVFP4X2) {              /* :1948-2025: E4M3 scale = amax/6 and the scaling itself in bf16 precision */
      float amax = 0.0f, sv = 0.0f, rcp; unsigned sc = 0;
      for (k = 0; k < blk; ++k) { const float a = fabsf(x[k]); if (a > amax || a != a) amax = a; }
      if (amax != 0.0f) { sc = e4m3_scale_code(bf16_round(bf16_round(amax) * bits_f32(0x3e2a0000u))); sv = e4m3_value(sc); }
      scl[(size_t)j * ld_scl + b] = (unsigned char)sc;
      if (sv == 0.0f) { memset(o, 0, 8); continue; }
      rcp = bf16_round(1.0f / bf16_round(sv));
      for (k = 0; k < 8; ++k) {
        const unsigned lo = ((f32_bits(x[2 * k]) >> 31) << 3) | e2m1_code(fabsf(bf16_round(x[2 * k] * rcp)));
        const unsigned hi = ((f32_bits(x[2 * k + 1]) >> 31) << 3) | e2m1_code(fabsf(bf16_round(x[2 * k + 1] * rcp)));
        o[k] = (unsigned char)((hi << 4) | lo);
      }
    } else if (d->to == LIBXSMM_DATATYPE_MXFP4X2) {       /* :1898-1945 */
      scl[(size_t)j * ld_scl + b] = (unsigned char)mx_shared_exp(x, 32, 2, &scale, &special);
      if (special) { memset(o, 0x77, 16); continue; }
      for (k = 0; k < 16; ++k) {
        const unsigned lo = ((f32_bits(x[2 * k]) >> 31) << 3) | e2m1_code(fabsf(x[2 * k] / scale));
        const unsigned hi = ((f32_bits(x[2 * k + 1]) >> 31) << 3) | e2m1_code(fabsf(x[2 * k + 1] / scale));
        o[k] = (unsigned char)((hi << 4) | lo);
      }
    } else {                                              /* MXBF8, :2030-2071 */
      scl[(size_t)j * ld_scl + b] = (unsigned char)mx_shared_exp(x, 32, 15, &scale, &special);
      if (special) { memset(o, 0x7b, 32); continue; }
      for (k = 0; k < 32; ++k) o[k] = (unsigned char)bf8_rne(x[k] / scale);
    }
  }
  return 0;
}

/* quantise / dequantise: reference :2195-2360 */
static int unary_quant(const mdesc* d, const libxsmm_meltw_unary_param* p) {
  int i, j;
  if (d->op == LIBXSMM_MELTW_TYPE_UNARY_QUANT && (d->to == LIBXSMM_DATATYPE_MXFP4X2 || d->to == LIBXSMM_DATATYPE_NVFP4X2 || d->to == LIBXSMM_DATATYPE_MXBF8))
    return unary_mxquant(d, p);
  if (d->op == LIBXSMM_MELTW_TYPE_UNARY_DEQUANT) {
    const float scf = *(const float*)p->in.secondary;
    if (d->to != LIBXSMM_DATATYPE_F32) return 2;
    for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
      const long long ii = i + (long long)j * d->ldi; float v;
      if (d->t0 == LIBXSMM_DATATYPE_I8) v = (float)((const int8_t*)p->in.primary)[ii];
      else if (d->t0 == LIBXSMM_DATATYPE_I16) v = (float)((const int16_t*)p->in.primary)[ii];
      else if (d->t0 == LIBXSMM_DATATYPE_I32) v = (float)((const int32_t*)p->in.primary)[ii];
      else return 2;
      ((float*)p->out.primary)[i + (long long)j * d->ldo] = v * scf;
    }
    return 0;
  }
  if (d->op == LIBXSMM_MELTW_TYPE_UNARY_QUANT && d->t0 == LIBXSMM_DATATYPE_F32 && p->in.secondary != NULL
      && (d->flags & LIBXSMM_MELTW_FLAG_UNARY_NO_SCF_QUANT) == 0) {
    /* :2206-2217: nearbyintf(x * scf), then wrap to the low bits or saturate (SIGN_SAT_QUANT) */
    const float scf = *(const float*)p->in.secondary;
    const int sat = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_SIGN_SAT_QUANT) != 0;
    if (!(d->to == LIBXSMM_DATATYPE_I8 || d->to == LIBXSMM_DATATYPE_I16 || d->to == LIBXSMM_DATATYPE_I32)) return 2;
    for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
      const float r = nearbyintf(((const float*)p->in.primary)[bidx(d, 0, i, j, d->ldi)] * scf);
      const long long oi = i + (long long)j * d->ldo;
      if (d->to == LIBXSMM_DATATYPE_I8) ((int8_t*)p->out.primary)[oi] = sat ? (int8_t)fminf(fmaxf(r, -128.f), 127.f) : (int8_t)(0xff & (int)r);
      else if (d->to == LIBXSMM_DATATYPE_I16) ((int16_t*)p->out.primary)[oi] = sat ? (int16_t)fminf(fmaxf(r, -32768.f), 32767.f) : (int16_t)(0xffff & (int)r);
      else ((int32_t*)p->out.primary)[oi] = (int32_t)r;
    }
    return 0;
  }
  return 2;
}

/* gather / scatter, pure data movement: reference :1444-1794. Index array in in.secondary (gather) or out.secondary
 * (scatter), 4-byte entries unless IDX_SIZE_8BYTES; GS_COLS moves whole columns, GS_ROWS whole rows, otherwise one
 * linear offset per element of the m x n index matrix */
static int unary_gs(const mdesc* d, const libxsmm_meltw_unary_param* p) {
  const int ts = tsz(d->t0), gather = (d->op == LIBXSMM_MELTW_TYPE_UNARY_GATHER);
  const int idx8 = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_IDX_SIZE_8BYTES) != 0;
  const int cols = (d->flags & LIBXSMM_MELTW_FLAG_UNARY_GS_COLS) != 0, rows = !cols && (d->flags & LIBXSMM_MELTW_FLAG_UNARY_GS_ROWS) != 0;
  const void* idxp = gather ? p->in.secondary : p->out.secondary;
  const char* in = (const char*)p->in.primary; char* out = (char*)p->out.primary;
  long long i, j;
  if (ts > 4 || idxp == NULL) return 2;
  for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
    const long long sel = cols ? j : (rows ? i : (i + j * d->m));
    const long long x = idx8 ? (long long)((const uint64_t*)idxp)[sel] : (long long)((const uint32_t*)idxp)[sel];
    long long src, dst;
    if (gather) { dst = i + j * d->ldo; src = cols ? (i + x * d->ldi) : (rows ? (x + j * d->ldi) : x); }
    else { src = i + j * d->ldi; dst = cols ? (i + x * d->ldo) : (rows ? (x + j * d->ldo) : x); }
    memcpy(out + dst * ts, in + src * ts, (size_t)ts);
  }
  return 0;
}

/* sum of all elements (unary) / of the element-wise product (binary) into one scalar, sequential over j then i in the
 * compute type: reference :2097-2117 and :2523-2546 */
static int reduce_to_scalar(const mdesc* d, const void* in0, const void* in1, void* out) {
  const int f64 = d->t0 == LIBXSMM_DATATYPE_F64 && d->to == LIBXSMM_DATATYPE_F64 && d->tc == LIBXSMM_DATATYPE_F64 && (in1 == NULL || d->t1 == LIBXSMM_DATATYPE_F64);
  float acc = 0.0f; double acc64 = 0.0;
  int i, j;
  if (!f64 && !(is_f(d->t0) && is_f(d->to) && (in1 == NULL || is_f(d->t1)))) return 2;
  for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
    if (f64) { double v = ((const double*)in0)[bidx(d, 0, i, j, d->ldi)]; if (in1 != NULL) v *= ((const double*)in1)[bidx(d, 1, i, j, d->ldi2)]; acc64 += v; }
    else { float v = ldf(in0, bidx(d, 0, i, j, d->ldi), d->t0); if (in1 != NULL) v = v * ldf(in1, bidx(d, 1, i, j, d->ldi2), d->t1); acc += v; }
  }
  if (f64) ((double*)out)[0] = acc64; else stf(out, 0, d->to, acc);
  return 0;
}

static int binary_map(const mdesc* d, const libxsmm_meltw_binary_param* p) {
  const int op = d->op;
  const int f64 = d->t0 == LIBXSMM_DATATYPE_F64 && d->t1 == LIBXSMM_DATATYPE_F64 && d->to == LIBXSMM_DATATYPE_F64;
  int i, j;
  if (op == LIBXSMM_MELTW_TYPE_BINARY_ZIP) {   /* :2547-2559: two 16-bit planes -> one 32-bit word (in1 is the high half) */
    for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i)
      ((uint32_t*)p->out.primary)[i + (long long)j * d->ldo] = (uint32_t)((const uint16_t*)p->in0.primary)[bidx(d, 0, i, j, d->ldi)]
                                                            | ((uint32_t)((const uint16_t*)p->in1.primary)[bidx(d, 1, i, j, d->ldi2)] << 16);
    return 0;
  }
  if (op == LIBXSMM_MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD) return reduce_to_scalar(d, p->in0.primary, p->in1.primary, p->out.primary);
  if (!f64 && !(is_f(d->t0) && is_f(d->t1))) return 2;
  for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
    const long long oi = i + (long long)j * d->ldo;
    if (f64) {
      const double a = ((const double*)p->in0.primary)[bidx(d, 0, i, j, d->ldi)], b = ((const double*)p->in1.primary)[bidx(d, 1, i, j, d->ldi2)];
      double* o = (double*)p->out.primary + oi;
      switch (op) {
        case LIBXSMM_MELTW_TYPE_BINARY_ADD: *o = a + b; break; case LIBXSMM_MELTW_TYPE_BINARY_SUB: *o = a - b; break;
        case LIBXSMM_MELTW_TYPE_BINARY_MUL: *o = a * b; break; case LIBXSMM_MELTW_TYPE_BINARY_DIV: *o = a / b; break;
        case LIBXSMM_MELTW_TYPE_BINARY_MULADD: *o = *o + a * b; break;
        case LIBXSMM_MELTW_TYPE_BINARY_MAX: *o = (a > b) ? a : b; break; case LIBXSMM_MELTW_TYPE_BINARY_MIN: *o = (a > b) ? b : a; break;
        default: return 2;
      }
    } else {
      const float a = ldf(p->in0.primary, bidx(d, 0, i, j, d->ldi), d->t0), b = ldf(p->in1.primary, bidx(d, 1, i, j, d->ldi2), d->t1);
      float r;
      switch (op) {
        case LIBXSMM_MELTW_TYPE_BINARY_ADD: r = a + b; break; case LIBXSMM_MELTW_TYPE_BINARY_SUB: r = a - b; break;
        case LIBXSMM_MELTW_TYPE_BINARY_MUL: r = a * b; break; case LIBXSMM_MELTW_TYPE_BINARY_DIV: r = a / b; break;
        case LIBXSMM_MELTW_TYPE_BINARY_MULADD: r = ldf(p->out.primary, oi, d->to) + a * b; break;       /* :2505-2593: out += a*b, reads out */
        case LIBXSMM_MELTW_TYPE_BINARY_MAX: r = (a > b) ? a : b; break; case LIBXSMM_MELTW_TYPE_BINARY_MIN: r = (a > b) ? b : a; break;
        case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GE: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LT:
        case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LE: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_EQ: case LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_NE: {   /* :2573-2581 */
          const int bit = (op == LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GT) ? (a > b) : (op == LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_GE) ? (a >= b)
                        : (op == LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LT) ? (a < b) : (op == LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_LE) ? (a <= b)
                        : (op == LIBXSMM_MELTW_TYPE_BINARY_CMP_OP_EQ) ? (a == b) : (a != b);
          mask_put(p->out.primary, i, j, mask_ld_of(d->ldo), bit);
          continue;
        }
        default: return 2;
      }
      if (!is_f(d->to)) return 2;
      stf_rnd(p->out.primary, oi, d->to, r, (d->flags & LIBXSMM_MELTW_FLAG_BINARY_STOCHASTIC_ROUND) != 0, (uint32_t*)p->op.secondary, (long long)j * d->m + i);
    }
  }
  return 0;
}

static int ternary_map(const mdesc* d, const libxsmm_meltw_ternary_param* p) {   /* reference :2596-2660 */
  const int f64 = d->t0 == LIBXSMM_DATATYPE_F64 && d->t1 == LIBXSMM_DATATYPE_F64 && d->to == LIBXSMM_DATATYPE_F64;
  int i, j;
  for (j = 0; j < d->n; ++j) for (i = 0; i < d->m; ++i) {
    const long long oi = i + (long long)j * d->ldo;
    if (d->op == LIBXSMM_MELTW_TYPE_TERNARY_SELECT) {          /* bit 0 -> in0, bit 1 -> in1; mask pitch rounded up to 16 bits (:2620) */
      const int bit = mask_get(p->in2.primary, i, j, mask_ld_of(d->ldi3));
      if (f64) ((double*)p->out.primary)[oi] = bit ? ((const double*)p->in1.primary)[bidx(d, 1, i, j, d->ldi2)] : ((const double*)p->in0.primary)[bidx(d, 0, i, j, d->ldi)];
      else if (is_f(d->t0) && is_f(d->t1) && is_f(d->to))
        stf_rnd(p->out.primary, oi, d->to, bit ? ldf(p->in1.primary, bidx(d, 1, i, j, d->ldi2), d->t1) : ldf(p->in0.primary, bidx(d, 0, i, j, d->ldi), d->t0),
                (d->flags & LIBXSMM_MELTW_FLAG_TERNARY_STOCHASTIC_ROUND) != 0, (uint32_t*)p->op.secondary, (long long)j * d->m + i);
      else return 2;
    } else if (d->op == LIBXSMM_MELTW_TYPE_TERNARY_MULADD || d->op == LIBXSMM_MELTW_TYPE_TERNARY_NMULADD) {
      float x, y, z;
      if (!(is_f(d->t0) && is_f(d->t1) && is_f(d->t2) && is_f(d->to))) return 2;
      x = ldf(p->in0.primary, bidx(d, 0, i, j, d->ldi), d->t0); y = ldf(p->in1.primary, bidx(d, 1, i, j, d->ldi2), d->t1);
      z = ldf(p->in2.primary, bidx(d, 2, i, j, d->ldi3), d->t2);
      stf_rnd(p->out.primary, oi, d->to, (d->op == LIBXSMM_MELTW_TYPE_TERNARY_MULADD) ? (z + x * y) : (y - x * z),   /* in2 + in0*in1 ; in1 - in0*in2 */
              (d->flags & LIBXSMM_MELTW_FLAG_TERNARY_STOCHASTIC_ROUND) != 0, (uint32_t*)p->op.secondary, (long long)j * d->m + i);
    } else return 2;
  }
  return 0;
}

/* returns 0 = computed, 2 = operation not restated here (use the reference), 1 = invalid */
ORACLE_API int oracle_meltw(const int* desc, void* param, int mode) {
  mdesc d;
  (void)mode;
  d.op_class = desc[0]; d.op = desc[1]; d.flags = (unsigned int)desc[2]; d.m = desc[3]; d.n = desc[4];
  d.ldi = desc[5]; d.ldi2 = desc[6]; d.ldi3 = desc[7]; d.ldo = desc[8]; d.t0 = desc[9]; d.t1 = desc[10]; d.t2 = desc[11]; d.to = desc[12]; d.tc = desc[13];
  if (d.m <= 0 || d.n <= 0 || param == NULL) return 1;
  if (d.op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    switch (d.op) {
      case LIBXSMM_MELTW_TYPE_UNARY_IDENTITY: case LIBXSMM_MELTW_TYPE_UNARY_XOR: case LIBXSMM_MELTW_TYPE_UNARY_X2: case LIBXSMM_MELTW_TYPE_UNARY_SQRT: case LIBXSMM_MELTW_TYPE_UNARY_DUMP:
      case LIBXSMM_MELTW_TYPE_UNARY_NEGATE: case LIBXSMM_MELTW_TYPE_UNARY_INC: case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL: case LIBXSMM_MELTW_TYPE_UNARY_RECIPROCAL_SQRT:
      case LIBXSMM_MELTW_TYPE_UNARY_TANH: case LIBXSMM_MELTW_TYPE_UNARY_TANH_INV: case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID: case LIBXSMM_MELTW_TYPE_UNARY_SIGMOID_INV:
      case LIBXSMM_MELTW_TYPE_UNARY_GELU: case LIBXSMM_MELTW_TYPE_UNARY_GELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_EXP:
      case LIBXSMM_MELTW_TYPE_UNARY_RELU: case LIBXSMM_MELTW_TYPE_UNARY_RELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU: case LIBXSMM_MELTW_TYPE_UNARY_LEAKY_RELU_INV:
      case LIBXSMM_MELTW_TYPE_UNARY_ELU: case LIBXSMM_MELTW_TYPE_UNARY_ELU_INV: case LIBXSMM_MELTW_TYPE_UNARY_REPLICATE_COL_VAR:
        return unary_map(&d, (const libxsmm_meltw_unary_param*)param);
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MAX: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_MIN: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX:
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_ADD: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MAX: case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_MIN:
        return unary_reduce(&d, (const libxsmm_meltw_unary_param*)param);
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4T:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2_TO_VNNI2T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI4T:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI2T_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4T_TO_NORM:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_NORM:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8_PAD:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI8T: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8_TO_VNNI8T:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI8T_TO_NORM: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_VNNI4_TO_VNNI2:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD2: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD2:
      case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADM_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADN_MOD4: case LIBXSMM_MELTW_TYPE_UNARY_TRANSFORM_PADNM_MOD4:
        return unary_transform(&d, (const libxsmm_meltw_unary_param*)param);
      case LIBXSMM_MELTW_TYPE_UNARY_DROPOUT: case LIBXSMM_MELTW_TYPE_UNARY_DROPOUT_INV:
        return unary_dropout(&d, (const libxsmm_meltw_unary_param*)param);
      case LIBXSMM_MELTW_TYPE_UNARY_UNZIP: case LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X2: case LIBXSMM_MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X3:
        return unary_split(&d, (const libxsmm_meltw_unary_param*)param);
      case LIBXSMM_MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD:
        return reduce_to_scalar(&d, ((const libxsmm_meltw_unary_param*)param)->in.primary, NULL, ((const libxsmm_meltw_unary_param*)param)->out.primary);
      case LIBXSMM_MELTW_TYPE_UNARY_DEQUANT: case LIBXSMM_MELTW_TYPE_UNARY_QUANT:
        return unary_quant(&d, (const libxsmm_meltw_unary_param*)param);
      case LIBXSMM_MELTW_TYPE_UNARY_GATHER: case LIBXSMM_MELTW_TYPE_UNARY_SCATTER:
        return unary_gs(&d, (const libxsmm_meltw_unary_param*)param);
      default: return 2;
    }
  }
  if (d.op_class == LIBXSMM_MELTW_OPERATION_BINARY) return binary_map(&d, (const libxsmm_meltw_binary_param*)param);
  if (d.op_class == LIBXSMM_MELTW_OPERATION_TERNARY) return ternary_map(&d, (const libxsmm_meltw_ternary_param*)param);
  return 1;
}
