/* TEST INFRASTRUCTURE -- not part of the product; nothing under libxsmm_b200/ may call into this file.
 *
 * CPU restatement (plain C, written from the algorithm, not copied) of the reference kernels that
 * define the semantics of the hot path. Each function cites the reference code it follows
 * (paths relative to /root/reference). The restatement is pinned in tests/test_oracle_vs_ref.py
 * against the reference itself (oracle/_ref/libxsmm_ref.so, built from the unmodified sources) on
 * seeded inputs, bit for bit, and against the committed fixtures under tests/golden/.
 *
 * Interface mirrors oracle/ref_shim.c (ref_* -> oracle_*), so a test can run either side.
 * Build: gcc -O2 -ffp-contract=off (separate multiply and add, like the reference built for baseline
 * x86-64: no FMA contraction). Where the reference's JIT emits a fused multiply-add (the EDGE/SeisSol
 * packed kernels and the f32 BCSC kernel, see there), the restatement says so with an explicit fma()/fmaf().
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

/* datatype enumerators: include/libxsmm_typedefs.h:218-246 */
enum { T_F64 = 0, T_F32 = 1, T_BF16 = 2, T_F16 = 3, T_BF8 = 4, T_HF8 = 5, T_I64 = 6, T_U64 = 7, T_I32 = 8, T_U32 = 9,
       T_I16 = 10, T_U16 = 11, T_I8 = 12, T_U8 = 13, T_BF32 = 24, T_IMPLICIT = 25 };
/* gemm flags: include/libxsmm_typedefs.h:468-529 */
enum { F_TRANS_A = 1, F_TRANS_B = 2, F_BETA_0 = 4, F_VNNI_A = 256, F_VNNI_B = 512 };

static int tsize(int t) {
  switch (t) { case T_F64: case T_I64: case T_U64: return 8; case T_F32: case T_I32: case T_U32: case T_BF32: return 4;
               case T_BF16: case T_F16: case T_I16: case T_U16: return 2; default: return 1; }
}

/* ---- conversions: src/libxsmm_math.c:587-703, 824-900 ------------------------------------------------ */
static float bits2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t f2bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

ORACLE_API float oracle_bf16_widen(uint16_t h) { return bits2f((uint32_t)h << 16); }     /* GEMM kernels: no flush */
ORACLE_API float oracle_bf16_to_f32(uint16_t h) {                                           /* :587-597 flushes denormals */
  if ((h & 0x7f80) == 0) h &= 0x8000;
  return bits2f((uint32_t)h << 16);
}
ORACLE_API uint16_t oracle_f32_to_bf16(float f) {                                            /* :684-703 */
  uint32_t u = f2bits(f);
  if ((u & 0x7f800000u) == 0) u &= 0x80000000u;
  if ((u & 0x7f800000u) == 0x7f800000u) { if (u & 0x007fffffu) u |= 0x00400000u; }
  else u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
ORACLE_API float oracle_f16_to_f32(uint16_t h) {                                             /* :600-640 */
  uint32_t s = ((uint32_t)h & 0x8000u) << 16, e = (h >> 10) & 0x1f, m = h & 0x3ff, r;
  if (e == 0x1f) { if (m) m |= 0x200; r = 0x7f800000u | (m << 13); }
  else if (e == 0) {
    if (m == 0) r = 0;
    else { int sh = 0; while (!(m & 0x400)) { m <<= 1; ++sh; } m &= 0x3ff; r = ((uint32_t)(113 - sh) << 23) | (m << 13); }
  } else r = ((e + 112) << 23) | (m << 13);
  return bits2f(r | s);
}
/* 8-bit floats: bf8 (E5M2) is the high byte of an f16 (src/libxsmm_math.c:546-551, :731-746); hf8 (E4M3, bias 7, 0x7f = NaN, no Inf)
 * converts through f16 with RNE on the 7 dropped mantissa bits (:554-584, :749-822) */
ORACLE_API float oracle_f16_to_f32(uint16_t h);
ORACLE_API uint16_t oracle_f32_to_f16(float f);
ORACLE_API float oracle_bf8_to_f32(uint8_t b) { return oracle_f16_to_f32((uint16_t)((uint16_t)b << 8)); }
ORACLE_API uint8_t oracle_f32_to_bf8(float f) {
  unsigned h = oracle_f32_to_f16(f);
  if ((h & 0x7c00u) == 0x7c00u) { if (h & 0x3ffu) h |= 0x200u; } else h = (h + 0x7fu + ((h >> 8) & 1u)) & 0xffffu;
  return (uint8_t)(h >> 8);
}
ORACLE_API float oracle_hf8_to_f32(uint8_t b) {
  const unsigned e = (b >> 3) & 0xfu, m = b & 7u;
  union { uint32_t u; float f; } x;
  float v;
  if (e == 0xf && m == 7) { x.u = ((uint32_t)(b & 0x80u) << 24) | 0x7fc00000u; return x.f; }
  v = (e == 0) ? ldexpf((float)m, -9) : ldexpf((float)(8 + m), (int)e - 10);
  return (b & 0x80u) ? -v : v;
}
ORACLE_API uint8_t oracle_f32_to_hf8(float f) {
  const unsigned h = oracle_f32_to_f16(f), sign = (h & 0x8000u) >> 8, e16 = (h >> 10) & 0x1fu, m16 = h & 0x3ffu;
  unsigned e, m, r;
  if (e16 == 0x1f || e16 > 23 || (e16 == 23 && m16 > 0x340u)) return (uint8_t)(sign | 0x7fu);
  if (e16 < 5) return (uint8_t)sign;
  if (e16 > 8) { r = (h & 0x7fffu) + 0x3fu + ((m16 >> 7) & 1u); e = ((r >> 10) & 0x1fu) - 8u; m = (r & 0x3ffu) >> 7; return (uint8_t)(sign | (e << 3) | m); }
  m = ((m16 | 0x400u) >> (9 - e16)) | (((m16 & 0x7fu) + 0x7fu) >> 7);
  m = (m + 0x3fu + ((m >> 7) & 1u)) >> 7;
  return (uint8_t)(sign | m);
}
ORACLE_API uint16_t oracle_f32_to_f16(float f) {                                             /* :824-900 */
  uint32_t u = f2bits(f), s = (u & 0x80000000u) >> 16, e32 = (u >> 23) & 0xff, m32 = u & 0x7fffff, e, m;
  if (e32 == 0xff) { e = 0x1f; m = m32 ? ((m32 >> 13) | 0x200) : 0; }
  else if (e32 > 142) { e = 0x1f; m = 0; }
  else if (e32 < 102) { e = 0; m = 0; }
  else if (e32 <= 112) {
    uint32_t mm = (m32 | 0x800000u) >> (113 - e32);
    mm |= ((m32 & 0x1fff) + 0x1fff) >> 13;
    mm += 0xfff + ((mm >> 13) & 1);
    return (uint16_t)(s | (mm >> 13));
  } else {
    uint32_t r = (u & 0x7fffffffu) + 0xfff + ((m32 >> 13) & 1);
    return (uint16_t)(s | ((((r >> 23) & 0xff) - 112) << 10) | ((r & 0x7fffff) >> 13));
  }
  return (uint16_t)(s | (e << 10) | m);
}

/* ---- dense GEMM / BRGEMM: src/generator_gemm_reference_impl.c:821-2800 (libxsmm_ref_matmul) ----------- */
typedef struct gemm_ctx {
  int m, n, k, lda, ldb, ldc, ta, tb, tcomp, tc, br_type;
  unsigned int flags;
  long long stride_a, stride_b;            /* bytes */
  unsigned long long br;
  const char *a, *b; char* c;
  const long long *offs_a, *offs_b;
  float scf;
} gemm_ctx;

/* operand bases of the r-th reduction step, :178-197 (byte offsets are truncated to whole elements) */
static void br_base(const gemm_ctx* g, unsigned long long r, const char** pa, const char** pb) {
  const int tsa = tsize(g->ta), tsb = tsize(g->tb);
  switch (g->br_type) {
    case 1: *pa = (const char*)((void* const*)g->a)[r]; *pb = (const char*)((void* const*)g->b)[r]; break;
    case 2: *pa = g->a + (g->offs_a[r] / tsa) * tsa; *pb = g->b + (g->offs_b[r] / tsb) * tsb; break;
    case 3: *pa = g->a + (long long)r * ((g->stride_a / tsa) * tsa); *pb = g->b + (long long)r * ((g->stride_b / tsb) * tsb); break;
    default: *pa = g->a; *pb = g->b;
  }
}

static int gemm_run(const gemm_ctx* g) {
  const int m = g->m, n = g->n, k = g->k;
  const long long lda = g->lda, ldb = g->ldb, ldc = g->ldc;
  const int beta0 = (g->flags & F_BETA_0) != 0, trans_a = (g->flags & F_TRANS_A) != 0, trans_b = (g->flags & F_TRANS_B) != 0;
  const int vnni_a = (g->flags & F_VNNI_A) != 0, vnni_b = (g->flags & F_VNNI_B) != 0;
  const unsigned long long br = (g->br_type == 0) ? 1 : g->br;
  const int a8 = (g->ta == T_I8 || g->ta == T_U8), b8 = (g->tb == T_I8 || g->tb == T_U8);
  int i, j, s, k2; unsigned long long r;
  const char *pa, *pb;

  for (j = 0; j < n; ++j) for (i = 0; i < m; ++i) {
    const long long ci = j * ldc + i;
    if (g->ta == T_F64 && g->tb == T_F64 && g->tc == T_F64 && g->tcomp == T_F64) {                    /* :1322-1358 */
      double* C = (double*)g->c;
      if (beta0) C[ci] = 0.0;
      for (r = 0; r < br; ++r) { br_base(g, r, &pa, &pb);
        for (s = 0; s < k; ++s) {
          const double av = ((const double*)pa)[trans_a ? (i * lda + s) : (s * lda + i)];
          const double bv = ((const double*)pb)[trans_b ? (s * ldb + j) : (j * ldb + s)];
          C[ci] += av * bv;
        } }
    } else if ((g->ta == T_F32 || g->ta == T_BF32) && (g->tb == T_F32 || g->tb == T_BF32) && g->tc == T_F32 && g->tcomp == T_F32) { /* :1359-1426 */
      float* C = (float*)g->c;
      if (beta0) C[ci] = 0.0f;
      for (r = 0; r < br; ++r) { br_base(g, r, &pa, &pb);
        for (s = 0; s < k; ++s) {
          float av = ((const float*)pa)[trans_a ? (i * lda + s) : (s * lda + i)];
          float bv = ((const float*)pb)[trans_b ? (s * ldb + j) : (j * ldb + s)];
          if (g->ta == T_BF32) { av = oracle_bf16_widen(oracle_f32_to_bf16(av)); bv = oracle_bf16_widen(oracle_f32_to_bf16(bv)); }
          C[ci] += av * bv;
        } }
    } else if (g->ta == T_I16 && g->tb == T_I16 && g->tc == T_I32 && g->tcomp == T_I32) {             /* :1427-1451 */
      const int kb = vnni_a ? 2 : 1; int* C = (int*)g->c;
      if (beta0) C[ci] = 0;
      for (r = 0; r < br; ++r) { br_base(g, r, &pa, &pb);
        for (s = 0; s < k / kb; ++s) for (k2 = 0; k2 < kb; ++k2)
          C[ci] += ((const short*)pa)[s * (lda * kb) + i * kb + k2] * ((const short*)pb)[j * ldb + s * kb + k2];
      }
    } else if (a8 && b8 && g->tcomp == T_I32 && (g->tc == T_I32 || g->tc == T_F32)) {                  /* :1452-1683 */
      const int kb = (g->tc == T_F32) ? 4 : (vnni_a ? 4 : 1);
      unsigned int acc = (g->tc == T_I32 && !beta0) ? (unsigned int)((int*)g->c)[ci] : 0u;
      for (r = 0; r < br; ++r) { br_base(g, r, &pa, &pb);
        for (s = 0; s < k / kb; ++s) for (k2 = 0; k2 < kb; ++k2) {
          const unsigned char ar = ((const unsigned char*)pa)[s * (lda * kb) + i * kb + k2];
          const unsigned char bw = ((const unsigned char*)pb)[j * ldb + s * kb + k2];
          const int av = (g->ta == T_U8) ? (int)ar : (int)(signed char)ar, bv = (g->tb == T_U8) ? (int)bw : (int)(signed char)bw;
          acc += (unsigned int)(av * bv);
        } }
      if (g->tc == T_I32) ((int*)g->c)[ci] = (int)acc;
      else { float f = (float)(int)acc; f *= g->scf; if (!beta0) f += ((float*)g->c)[ci]; ((float*)g->c)[ci] = f; }
    } else if (g->ta == T_F16 && g->tb == T_F16 && (g->tc == T_F16 || g->tc == T_F32)
            && (g->tcomp == T_F16 || g->tcomp == T_F32 || g->tcomp == T_IMPLICIT)) {                     /* :2025-2126 */
      const int kb = vnni_a ? 2 : 1;
      /* comp F16 (and IMPLICIT on an SPR-class host, which is what the x86 pack factors freeze) rounds per FMA */
      const int round_each = (g->tcomp == T_F16 || g->tcomp == T_IMPLICIT);
      float acc = 0.0f;
      for (r = 0; r < br; ++r) { br_base(g, r, &pa, &pb);
        for (s = 0; s < k / kb; ++s) for (k2 = 0; k2 < kb; ++k2) {
          const long long kk = (long long)s * kb + k2;
          const float av = oracle_f16_to_f32(((const uint16_t*)pa)[s * (lda * kb) + i * kb + k2]);
          const float bv = oracle_f16_to_f32(((const uint16_t*)pb)[trans_b ? (kk * ldb + j) : (j * ldb + kk)]);
          acc += av * bv;
          if (round_each) acc = oracle_f16_to_f32(oracle_f32_to_f16(acc));
        } }
      if (g->tc == T_F16) { if (!beta0) acc += oracle_f16_to_f32(((uint16_t*)g->c)[ci]); ((uint16_t*)g->c)[ci] = oracle_f32_to_f16(acc); }
      else { if (!beta0) acc += oracle_f16_to_f32(oracle_f32_to_f16(((float*)g->c)[ci])); ((float*)g->c)[ci] = acc; }
    } else if (g->ta == T_BF16 && g->tb == T_BF16 && (g->tc == T_F32 || g->tc == T_BF16) && g->tcomp == T_F32) { /* :2127-2170, :2367-2419 */
      const int kb = vnni_a ? 2 : 1;
      float acc;
      if (g->tc == T_F32) { if (beta0) ((float*)g->c)[ci] = 0.0f; acc = ((float*)g->c)[ci]; }
      else acc = beta0 ? 0.0f : oracle_bf16_widen(((uint16_t*)g->c)[ci]);
      for (r = 0; r < br; ++r) { br_base(g, r, &pa, &pb);
        for (s = 0; s < k / kb; ++s) for (k2 = kb - 1; k2 >= 0; --k2) {                                   /* high k of a pair first */
          const long long kk = (long long)s * kb + k2;
          uint16_t ar = 0, bw = 0;
          if (!trans_a) ar = ((const uint16_t*)pa)[s * (lda * kb) + i * kb + k2];
          else if (!vnni_a) ar = ((const uint16_t*)pa)[i * lda + kk];
          if (trans_b && vnni_b) bw = ((const uint16_t*)pb)[j * kb + s * (ldb * kb) + k2];
          else if (trans_b) bw = ((const uint16_t*)pb)[kk * ldb + j];
          else if (!vnni_b) bw = ((const uint16_t*)pb)[j * ldb + kk];
          acc += oracle_bf16_widen(ar) * oracle_bf16_widen(bw);
        } }
      if (g->tc == T_F32) ((float*)g->c)[ci] = acc; else ((uint16_t*)g->c)[ci] = oracle_f32_to_bf16(acc);
    } else if ((g->ta == T_BF8 || g->ta == T_HF8) && g->tcomp == T_F32 && !vnni_b
               && ((g->tb == g->ta && (g->tc == T_F32 || g->tc == g->ta)) || (g->tb == T_BF16 && (g->tc == T_F32 || g->tc == T_BF16)))) {
      /* 8-bit float A: :2420-2630 (B of the same type: VNNI factor 4, k ascending inside a group) and :2171-2366 (bf16 B: pairs, high k
       * first); f32 accumulation seeded from C unless beta = 0, one rounding into C's type at the end */
      const int b16 = (g->tb == T_BF16), hf = (g->ta == T_HF8), kb = vnni_a ? (b16 ? 2 : 4) : 1;
      int q;
      float acc = 0.0f;
      if (!beta0) acc = (g->tc == T_F32) ? ((float*)g->c)[ci] : (g->tc == T_BF16 ? oracle_bf16_widen(((uint16_t*)g->c)[ci])
                                         : (hf ? oracle_hf8_to_f32(((uint8_t*)g->c)[ci]) : oracle_bf8_to_f32(((uint8_t*)g->c)[ci])));
      for (r = 0; r < br; ++r) { br_base(g, r, &pa, &pb);
        for (s = 0; s < k / kb; ++s) for (q = 0; q < kb; ++q) {
          const int kq = b16 ? (kb - 1 - q) : q;
          const long long kk = (long long)s * kb + kq;
          uint8_t ar = 0; float bv;
          if (!trans_a) ar = ((const uint8_t*)pa)[s * (lda * kb) + i * kb + kq];
          else if (!vnni_a) ar = ((const uint8_t*)pa)[i * lda + kk];
          if (b16) bv = oracle_bf16_widen(((const uint16_t*)pb)[trans_b ? (kk * ldb + j) : (j * ldb + kk)]);
          else { const uint8_t bw = ((const uint8_t*)pb)[trans_b ? (kk * ldb + j) : (j * ldb + kk)]; bv = hf ? oracle_hf8_to_f32(bw) : oracle_bf8_to_f32(bw); }
          acc += (hf ? oracle_hf8_to_f32(ar) : oracle_bf8_to_f32(ar)) * bv;
        } }
      if (g->tc == T_F32) ((float*)g->c)[ci] = acc;
      else if (g->tc == T_BF16) ((uint16_t*)g->c)[ci] = oracle_f32_to_bf16(acc);
      else ((uint8_t*)g->c)[ci] = hf ? oracle_f32_to_hf8(acc) : oracle_f32_to_bf8(acc);
    } else return 1;
  }
  return 0;
}

/* dims = {m,n,k,lda,ldb,ldc}; types = {a,b,comp,c}; same calling convention as ref_gemm (mode ignored) */
ORACLE_API int oracle_gemm(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                           unsigned long long br, void* a, void* b, void* c, long long* offs_a, long long* offs_b, float scf, int mode)
{
  gemm_ctx g;
  (void)mode;
  g.m = dims[0]; g.n = dims[1]; g.k = dims[2]; g.lda = dims[3]; g.ldb = dims[4]; g.ldc = dims[5];
  g.ta = types[0]; g.tb = types[1]; g.tcomp = types[2]; g.tc = types[3]; g.flags = flags; g.br_type = br_type;
  g.stride_a = stride_a; g.stride_b = stride_b; g.br = br; g.a = (const char*)a; g.b = (const char*)b; g.c = (char*)c;
  g.offs_a = offs_a; g.offs_b = offs_b; g.scf = scf;
  return gemm_run(&g);
}

/* ---- packed DENSE GEMM: golds of samples/xgemm_packed/gemm_packed_kernel.c:36-66 (kind 0), samples/xgemm_norm_packed/
 * dense_packedacrm.c:37-49 (kind 1) and dense_packedbcrm.c (kind 2); k outermost. Every product-accumulate is ONE fused multiply-add:
 * on an FMA-capable x86 host the packed generators set vmul_instruction to VFMADD231PS/PD (generator_gemm_common.c), and the JIT's
 * loops keep k ascending per C element. This states that AVX2/AVX-512 path; a pre-FMA host would round twice. ----------------------- */
#define PKD_BODY(T, FMA) do { \
  const T* A = (const T*)a; const T* B = (const T*)b; T* C = (T*)c; long long mm, nn, kk, p; \
  if (kind == 0) { \
    if (beta0) for (nn = 0; nn < N; ++nn) for (mm = 0; mm < M; ++mm) for (p = 0; p < P; ++p) C[(nn * ldc + mm) * P + p] = 0; \
    for (kk = 0; kk < K; ++kk) for (mm = 0; mm < M; ++mm) for (nn = 0; nn < N; ++nn) for (p = 0; p < P; ++p) { \
      T* cp = &C[(nn * ldc + mm) * P + p]; *cp = FMA(A[(kk * lda + mm) * P + p], B[(nn * ldb + kk) * P + p], *cp); } \
  } else { \
    if (beta0) for (mm = 0; mm < M; ++mm) for (nn = 0; nn < N; ++nn) for (p = 0; p < P; ++p) C[(mm * ldc + nn) * P + p] = 0; \
    for (kk = 0; kk < K; ++kk) for (mm = 0; mm < M; ++mm) for (nn = 0; nn < N; ++nn) for (p = 0; p < P; ++p) { \
      T* cp = &C[(mm * ldc + nn) * P + p]; \
      *cp = (kind == 1) ? FMA(A[(mm * lda + kk) * P + p], B[kk * ldb + nn], *cp) : FMA(A[mm * lda + kk], B[(kk * ldb + nn) * P + p], *cp); } \
  } } while (0)
ORACLE_API int oracle_packed_dense(int kind, int dtype, const int* dims, unsigned int flags, int P, const void* a, const void* b, void* c)
{
  const long long M = dims[0], N = dims[1], K = dims[2], lda = dims[3], ldb = dims[4], ldc = dims[5];
  const int beta0 = (flags & F_BETA_0) != 0;
  if (kind < 0 || kind > 2) return 1;
  if (dtype == T_F64) PKD_BODY(double, fma); else if (dtype == T_F32) PKD_BODY(float, fmaf); else return 1;
  return 0;
}

/* ---- 4-bit A x 8-bit B -> I32 with zero points (U4_U8_I32_I32 of the reference's test matrix), reference :1273-1321.
 * A: VNNI_A | INTLV_A_FORMAT: byte [(k/8)*lda*4 + 4*m + q] holds k = 8*(k/8)+q in the low and k = 8*(k/8)+4+q in the high nibble;
 * the zero point of row m (one byte) is subtracted in 8-bit arithmetic (`char even_use = even - zpt`, :833-834, 1290-1291),
 * B is read as unsigned bytes. zpt: br_type 0: column vector [m]; stride mode: vector r at +(stride_a*2/k)*r (:240-252). */
ORACLE_API int oracle_gemm_i4(const int* dims, unsigned int flags, int br_type, long long stride_a, long long stride_b, unsigned long long br,
                              const unsigned char* a, const unsigned char* b, int* c, const unsigned char* zpt)
{
  const int m = dims[0], n = dims[1], k = dims[2]; const long long lda = dims[3], ldb = dims[4], ldc = dims[5];
  int i, j, s, q; unsigned long long r;
  if (br_type != 0 && br_type != 3) return 1;
  if (br_type == 0) br = 1;
  for (j = 0; j < n; ++j) for (i = 0; i < m; ++i) {
    int acc = (flags & F_BETA_0) ? 0 : c[j * ldc + i];
    for (r = 0; r < br; ++r) {
      const unsigned char* pa = a + (br_type == 3 ? (long long)r * stride_a : 0);
      const unsigned char* pb = b + (br_type == 3 ? (long long)r * stride_b : 0);
      const unsigned char z = (br_type == 3) ? zpt[((stride_a * 2) / k) * (long long)r + i] : zpt[i];
      for (s = 0; s < k / 8; ++s) for (q = 0; q < 4; ++q) {
        const unsigned char pk = pa[s * lda * 4 + 4 * i + q];
        const signed char ev = (signed char)((pk & 0x0f) - z), od = (signed char)(((pk >> 4) & 0x0f) - z);
        acc = (int)((unsigned int)acc + (unsigned int)(ev * (int)pb[j * ldb + s * 8 + q]));
        acc = (int)((unsigned int)acc + (unsigned int)(od * (int)pb[j * ldb + s * 8 + 4 + q]));
      }
    }
    c[j * ldc + i] = acc;
  }
  return 0;
}

/* ---- bitmap-compressed A ("spmm", DECOMPRESS_A_VIA_BITMASK), reference :857-948. A holds only the elements whose bit is set, in
 * bit order; bit (s, i, k2) = position s*(m*kb) + i*kb + k2 with kb = 1 for F32 A, else the pack factor of B's type (2). No batch
 * reduce. Non-F32 C accumulates in an f32 image (seeded from C when beta = 1) and is rounded once at the end. */
ORACLE_API int oracle_gemm_bitmap(const int* dims, const int* types, unsigned int flags, const void* a, const void* b, void* c, const unsigned char* bitmap)
{
  const int m = dims[0], n = dims[1], k = dims[2]; const long long ldb = dims[4], ldc = dims[5];
  const int ta = types[0], tb = types[1], tc = types[3];
  const int kb = (ta == T_F32) ? 1 : ((tsize(tb) == 2) ? 2 : (tsize(tb) == 1 ? 4 : 1));
  float* img = (tc == T_F32) ? NULL : (float*)malloc((size_t)m * n * 4);
  unsigned long long ci = 0; int s, i, j, k2;
  if ((ta != T_F32 && ta != T_BF16 && ta != T_F16) || (tb != T_F32 && tb != T_BF16 && tb != T_F16) || (tc != T_F32 && tc != T_BF16 && tc != T_F16)) { free(img); return 1; }
  for (s = 0; s < k / kb; ++s) for (i = 0; i < m; ++i) {
    if (s == 0) for (j = 0; j < n; ++j) {
      if (tc == T_F32) { if (flags & F_BETA_0) ((float*)c)[j * ldc + i] = 0.0f; }
      else img[(size_t)j * m + i] = (flags & F_BETA_0) ? 0.0f : (tc == T_BF16 ? oracle_bf16_widen(((uint16_t*)c)[j * ldc + i]) : oracle_f16_to_f32(((uint16_t*)c)[j * ldc + i]));
    }
    for (k2 = 0; k2 < kb; ++k2) {
      const long long bit = (long long)s * m * kb + (long long)i * kb + k2;
      if ((bitmap[bit / 8] >> (bit % 8)) & 1) {
        const float av = (ta == T_F32) ? ((const float*)a)[ci] : (ta == T_BF16 ? oracle_bf16_widen(((const uint16_t*)a)[ci]) : oracle_f16_to_f32(((const uint16_t*)a)[ci]));
        for (j = 0; j < n; ++j) {
          const long long bi = j * ldb + (long long)s * kb + k2;
          const float bv = (tb == T_F32) ? ((const float*)b)[bi] : (tb == T_BF16 ? oracle_bf16_widen(((const uint16_t*)b)[bi]) : oracle_f16_to_f32(((const uint16_t*)b)[bi]));
          if (tc == T_F32) ((float*)c)[j * ldc + i] += av * bv; else img[(size_t)j * m + i] += av * bv;
        }
        ++ci;
      }
    }
  }
  if (tc != T_F32) {
    for (i = 0; i < m; ++i) for (j = 0; j < n; ++j) {
      if (tc == T_BF16) ((uint16_t*)c)[j * ldc + i] = oracle_f32_to_bf16(img[(size_t)j * m + i]); else ((uint16_t*)c)[j * ldc + i] = oracle_f32_to_f16(img[(size_t)j * m + i]);
    }
    free(img);
  }
  return 0;
}

/* ---- fused form (libxsmm_dispatch_brgemm_ext): reference :255-372, 2803-2842 ------------------------------------------
 * fuse = {colbias (0/1), cp_op (0 none, 5 RELU, 9 SIGMOID), relu bitmask (0/1), vnni_c (0/1)}. With any of the first three and a
 * C type other than F32 the product is accumulated in an f32 image of C (bias column broadcast, plus the old C when beta=1),
 * the post-op reads that image and rounds ONCE into C. For F32 C everything happens in place. */
static float ld_c(const void* p, long long i, int t) {
  if (t == T_F32) return ((const float*)p)[i];
  if (t == T_BF16) return oracle_bf16_to_f32(((const uint16_t*)p)[i]);   /* the pre-ops are mateltwise kernels: their bf16 load */
  return oracle_f16_to_f32(((const uint16_t*)p)[i]);
}
static void st_c(void* p, long long i, int t, float v) {
  if (t == T_F32) ((float*)p)[i] = v;
  else if (t == T_BF16) ((uint16_t*)p)[i] = oracle_f32_to_bf16(v);
  else ((uint16_t*)p)[i] = oracle_f32_to_f16(v);
}
ORACLE_API int oracle_gemm_ext(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                               unsigned long long br, void* a, void* b, void* c, long long* offs_a, long long* offs_b, float scf,
                               const int* fuse, const void* colbias, unsigned char* relu_mask)
{
  const int m = dims[0], n = dims[1], ldc = dims[5], tc = types[3];
  const int f_bias = fuse[0], cp = fuse[1], f_mask = fuse[2], f_vnni = fuse[3];
  const int fused = f_bias || cp != 0, via = fused && tc != T_F32;
  float* img = via ? (float*)malloc((size_t)ldc * n * 4) : (float*)c;
  int tt[4], i, j, rc; unsigned int fl = flags;
  if (tc != T_F32 && tc != T_BF16 && tc != T_F16) return 1;
  if (fused) {
    if (f_bias) {                                          /* :296-317 */
      for (j = 0; j < n; ++j) for (i = 0; i < m; ++i) {
        const float bias = ld_c(colbias, i, tc);
        img[(size_t)j * ldc + i] = (flags & F_BETA_0) ? bias : bias + ld_c(c, (long long)j * ldc + i, tc);
      }
      fl &= ~(unsigned int)F_BETA_0;
    } else if (via && !(flags & F_BETA_0)) {               /* :319-328 */
      for (j = 0; j < n; ++j) for (i = 0; i < m; ++i) img[(size_t)j * ldc + i] = ld_c(c, (long long)j * ldc + i, tc);
    }
  }
  tt[0] = types[0]; tt[1] = types[1]; tt[2] = types[2]; tt[3] = via ? T_F32 : tc;
  rc = oracle_gemm(dims, tt, fl, br_type, stride_a, stride_b, br, a, b, via ? (void*)img : c, offs_a, offs_b, scf, 0);
  if (rc == 0 && fused) {                                  /* :336-371 */
    const long long mld = ((ldc + 15) / 16) * 16;
    for (j = 0; j < n; ++j) for (i = 0; i < m; ++i) {
      const float x = img[(size_t)j * ldc + i];
      float y = x;
      if (cp == 5) { y = (x <= 0.0f) ? 0.0f : x;
        if (f_mask) { unsigned char* bp = relu_mask + i / 8 + (long long)j * (mld / 8);
          if (x <= 0.0f) *bp = (unsigned char)(*bp & ~(1u << (i % 8))); else *bp = (unsigned char)(*bp | (1u << (i % 8))); } }
      else if (cp == 9) y = (tanhf(x / 2.0f) + 1.0f) / 2.0f;
      if (via || cp != 0) st_c(c, (long long)j * ldc + i, tc, y);
    }
  }
  if (via) free(img);
  if (rc == 0 && f_vnni) {                                 /* :2803-2815: C (16-bit) re-packed norm -> VNNI2 through a copy */
    const int ts = tsize(tc); const long long Nn = ((n + 1) / 2) * 2;
    char* copy = (char*)malloc((size_t)ldc * Nn * ts); long long e;
    if (ts != 2) { free(copy); return 1; }
    memset(copy, 0, (size_t)ldc * Nn * ts); memcpy(copy, c, (size_t)ldc * n * ts);
    for (e = 0; e < (long long)ldc * Nn; ++e) {
      const long long jj = e / (ldc * 2), rem = e % (ldc * 2), col = jj * 2 + rem % 2; i = (int)(rem / 2);
      ((uint16_t*)c)[e] = (i < m && col < n) ? ((const uint16_t*)copy)[col * ldc + i] : 0;
    }
    free(copy);
  }
  return rc;
}

/* strided batch of tiles = the caller's loop of the reference (samples/xgemm/gemm_kernel.c:3179-3259), OpenMP over tiles */
ORACLE_API int oracle_gemm_batch(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                                 unsigned long long br, char* a, char* b, char* c, long long ta, long long tb, long long tc, long long count)
{
  long long t; int rc = 0;
# pragma omp parallel for schedule(static)
  for (t = 0; t < count; ++t) {
    if (oracle_gemm(dims, types, flags, br_type, stride_a, stride_b, br, a + t * ta, b + t * tb, c + t * tc, NULL, NULL, 0.f, 0)) rc = 1;
  }
  return rc;
}

/* ---- fsspmdm: gold of samples/xgemm_sparse_Ainregs/pyfr_driver_asp_reg.c:350-374 with the create()
 * rules of src/libxsmm_fsspmdm.c:80-140, 190-238 (alpha folded in the operand type, exact zeros dropped) */
ORACLE_API int oracle_fsspmdm(int dtype, int M, int N, int K, int lda, int ldb, int ldc, const void* alpha, const void* beta,
                              const void* a_dense, const void* B, void* C)
{
  const int vl = 64 / tsize(dtype);
  int i, j, z, nnz = 0;
  if (a_dense == NULL || (dtype != T_F32 && dtype != T_F64)) return 1;
  if (dtype == T_F64) {
    const double fa = alpha ? *(const double*)alpha : 1.0, fb = beta ? *(const double*)beta : 1.0;
    const double* A = (const double*)a_dense; const double* Bm = (const double*)B; double* Cm = (double*)C;
    if ((N % vl) != 0 || !(fb == 1.0 || fb == 0.0) || lda < K || ldc < N || ldb < N) return 1;
    for (i = 0; i < M; ++i) for (z = 0; z < K; ++z) if (fa * A[(size_t)i * lda + z] != 0.0) ++nnz;
    if (nnz == 0) return 1;
    for (j = 0; j < N; ++j) for (i = 0; i < M; ++i) {
      if (fb == 0.0) Cm[(size_t)i * ldc + j] = 0;
      for (z = 0; z < K; ++z) { const double v = fa * A[(size_t)i * lda + z]; if (v != 0.0) Cm[(size_t)i * ldc + j] += v * Bm[(size_t)z * ldb + j]; }
    }
  } else {
    const float fa = alpha ? *(const float*)alpha : 1.0f, fb = beta ? *(const float*)beta : 1.0f;
    const float* A = (const float*)a_dense; const float* Bm = (const float*)B; float* Cm = (float*)C;
    if ((N % vl) != 0 || !(fb == 1.0f || fb == 0.0f) || lda < K || ldc < N || ldb < N) return 1;
    for (i = 0; i < M; ++i) for (z = 0; z < K; ++z) if (fa * A[(size_t)i * lda + z] != 0.0f) ++nnz;
    if (nnz == 0) return 1;
    for (j = 0; j < N; ++j) for (i = 0; i < M; ++i) {
      if (fb == 0.0f) Cm[(size_t)i * ldc + j] = 0;
      for (z = 0; z < K; ++z) { const float v = fa * A[(size_t)i * lda + z]; if (v != 0.0f) Cm[(size_t)i * ldc + j] += v * Bm[(size_t)z * ldb + j]; }
    }
  }
  return 0;
}

/* ---- BCSC: dense gold of samples/xgemm_sparse/spmm_kernel.c:74-217 evaluated on the kernel's own inputs
 * (A as handed to the kernel: VNNI [K/v][M][v] unless TRANS_A; B in BCSC, blocks [bn][bk], optionally
 * VNNI-T re-packed, :349-372). k runs 0..K-1 like the gold; absent blocks contribute exact zeros.
 * f32: one fmaf per product, like the x86 JIT (generator_packed_spgemm_bcsc_bsparse_avx_avx2_avx512_amx.c, VFMADD231PS per
 * k of each stored block, blocks in pattern order). bf16: the widened product is exact in f32 (8 x 8 significand bits), so a
 * fused and a separate multiply-add round the same way; that line keeps the plain form.
 * TRANS_A (the AT_CT kernel) reads A as [M][K] and writes C as [M][N] like the gold (spmm_kernel.c:92-101), but the JIT sums k
 * across vector lanes and reduces horizontally at the end; this restatement keeps k ascending, so there the two agree only to
 * rounding. */
ORACLE_API int oracle_bcsc(const int* types, const int* geo, unsigned int flags, void* A, void* Bvals, unsigned int* colptr,
                           unsigned int* rowidx, void* C)
{
  const int ta = types[0], tb = types[1], tc = types[3];
  const int mblocks = geo[0], M = geo[1], K = geo[2], N = geo[3], bk = geo[4], bn = geo[5];
  const int beta0 = (flags & F_BETA_0) != 0, trans_a = (flags & F_TRANS_A) != 0, vnni_a = (flags & F_VNNI_A) != 0;
  const int vnni_bt = (flags & F_VNNI_B) && (flags & F_TRANS_B);
  const int v = (ta == T_BF16) ? 2 : (ta == T_F32 ? 1 : 4);
  int mb, i, j, kk; unsigned int z;
  if (!((ta == T_F32 && tb == T_F32 && tc == T_F32) || (ta == T_BF16 && tb == T_BF16 && tc == T_BF16)
     || (((ta == T_U8 && tb == T_I8) || (ta == T_I8 && tb == T_U8)) && tc == T_I32))) return 1;
  for (mb = 0; mb < mblocks; ++mb) {
    const char* Ab = (const char*)A + (size_t)mb * K * M * tsize(ta);
    char* Cb = (char*)C + (size_t)mb * N * M * tsize(tc);
    for (j = 0; j < N; ++j) for (i = 0; i < M; ++i) {
      const size_t ci = trans_a ? ((size_t)i * N + j) : ((size_t)j * M + i);
      const int jb = j / bn, nl = j % bn;
      float facc = 0.f; int iacc = 0;
      if (!beta0) { if (tc == T_I32) iacc = ((int*)Cb)[ci]; else if (tc == T_F32) facc = ((float*)Cb)[ci]; else facc = oracle_bf16_widen(((uint16_t*)Cb)[ci]); }
      for (z = colptr[jb]; z < colptr[jb + 1]; ++z) for (kk = 0; kk < bk; ++kk) {
        const int k = (int)rowidx[z] * bk + kk;
        const size_t ai = trans_a ? ((size_t)i * K + k) : ((vnni_a && v > 1) ? ((size_t)(k / v) * M * v + (size_t)i * v + (k % v)) : ((size_t)k * M + i));
        const size_t bi = (size_t)z * bk * bn + (vnni_bt ? ((size_t)(kk / v) * bn * v + (size_t)nl * v + (kk % v)) : ((size_t)nl * bk + kk));
        if (tc == T_I32) {
          const unsigned char ar = ((const unsigned char*)Ab)[ai], bw = ((const unsigned char*)Bvals)[bi];
          iacc += ((ta == T_U8) ? (int)ar : (int)(signed char)ar) * ((tb == T_U8) ? (int)bw : (int)(signed char)bw);
        } else if (ta == T_F32) facc = fmaf(((const float*)Ab)[ai], ((const float*)Bvals)[bi], facc);
        else facc += oracle_bf16_widen(((const uint16_t*)Ab)[ai]) * oracle_bf16_widen(((const uint16_t*)Bvals)[bi]);
      }
      if (tc == T_I32) ((int*)Cb)[ci] = iacc; else if (tc == T_F32) ((float*)Cb)[ci] = facc; else ((uint16_t*)Cb)[ci] = oracle_f32_to_bf16(facc);
    }
  }
  return 0;
}

/* ---- packed sparse: golds of samples/xgemm_norm_packed/asparse_packed_csr.c:116-128,
 * bsparse_packed_csc.c:137-150, bsparse_packed_csr.c; BETA_0 per src/generator_packed_spgemm_cs*.c.
 * Every product-accumulate is ONE fused multiply-add (FMA = fma / fmaf), in the order below: on an FMA-capable x86 host the packed
 * generators' vmul_instruction is VFMADD231PS/PD (generator_gemm_common.c; generator_packed_spgemm_csr_asparse_avx_avx2_avx512.c:
 * 420-470), and the C-sparse generator hard-codes VFMADD231PS (generator_packed_spgemm_csc_csparse_avx_avx2_avx512.c:84-91). The
 * C-sparse schedule is the AVX-512 one: 16 accumulator lanes (lane p % 16), k outer, then the 8 / 4 / (0+2)+(1+3) fold. A host
 * without FMA, or an AVX2 host for C-sparse (8 lanes), would give other bits. --------------------------------------------------- */
#define PACKED_BODY(T, FMA) do { \
  const T* A = (const T*)a; const T* B = (const T*)b; T* C = (T*)c; int i, j, k, p; unsigned int z; \
  if (lda == 0) {                          /* A sparse, CSR over M rows */ \
    for (i = 0; i < M; ++i) { if (ptr[i + 1] == ptr[i]) continue;  /* empty rows are not even zeroed (..._csr_asparse_avx_avx2_avx512.c:347-348) */ \
     for (j = 0; j < N; ++j) for (p = 0; p < P; ++p) { \
      T acc = beta0 ? (T)0 : C[((size_t)i * ldc + j) * P + p]; \
      for (z = ptr[i]; z < ptr[i + 1]; ++z) acc = FMA(A[z], B[((size_t)idx[z] * ldb + j) * P + p], acc); \
      C[((size_t)i * ldc + j) * P + p] = acc; } } \
  } else if (ldb == 0 && is_csc) {        /* B sparse, CSC over N columns */ \
    for (i = 0; i < M; ++i) for (j = 0; j < N; ++j) for (p = 0; p < P; ++p) { \
      T acc = beta0 ? (T)0 : C[((size_t)i * ldc + j) * P + p]; \
      for (z = ptr[j]; z < ptr[j + 1]; ++z) acc = FMA(A[((size_t)i * lda + idx[z]) * P + p], B[z], acc); \
      C[((size_t)i * ldc + j) * P + p] = acc; } \
  } else if (ldb == 0) {                  /* B sparse, CSR over K rows; columns past the last populated one are left alone \
      (generator_packed_spgemm_csr_bsparse_avx_avx2_avx512.c:64-70) */ \
    int ncol = 0; for (z = 0; z < ptr[K]; ++z) ncol = ((int)idx[z] + 1 > ncol) ? (int)idx[z] + 1 : ncol; \
    for (i = 0; i < M; ++i) for (j = 0; j < ncol && j < N; ++j) for (p = 0; p < P; ++p) { \
      T acc = beta0 ? (T)0 : C[((size_t)i * ldc + j) * P + p]; \
      for (k = 0; k < K; ++k) for (z = ptr[k]; z < ptr[k + 1]; ++z) if ((int)idx[z] == j) acc = FMA(A[((size_t)i * lda + k) * P + p], B[z], acc); \
      C[((size_t)i * ldc + j) * P + p] = acc; } \
  } else if (ldc == 0 && is_csc) {        /* C sparse, CSC pattern: ONE scalar per non-zero, the packed dimension is summed \
      away; A is [K][lda][P], B is [K][ldb][P] (..._csc_csparse_avx_avx2_avx512.c:63-79, 123-191) */ \
    for (j = 0; j < N; ++j) for (z = ptr[j]; z < ptr[j + 1]; ++z) { \
      T lane[16], acc; int l; for (l = 0; l < 16; ++l) lane[l] = (T)0; \
      for (k = 0; k < K; ++k) for (p = 0; p < P; ++p) \
        lane[p % 16] = FMA(A[((size_t)k * lda + idx[z]) * P + p], B[((size_t)k * ldb + j) * P + p], lane[p % 16]); \
      for (l = 0; l < 8; ++l) lane[l] += lane[l + 8]; for (l = 0; l < 4; ++l) lane[l] += lane[l + 4]; \
      acc = (lane[0] + lane[2]) + (lane[1] + lane[3]); \
      C[z] = beta0 ? acc : acc + C[z]; } \
  } else return 1; } while (0)

ORACLE_API int oracle_packed_sp(int is_csc, int dtype, const int* dims, unsigned int flags, int P,
                                const unsigned int* ptr, const unsigned int* idx, const void* values, void* a, void* b, void* c)
{
  const int M = dims[0], N = dims[1], K = dims[2], lda = dims[3], ldb = dims[4], ldc = dims[5];
  const int beta0 = (flags & F_BETA_0) != 0;
  (void)values;
  if (ldc == 0 && (dtype != T_F32 || P % 16 != 0 || P <= 0)) return 1;  /* C-sparse exists for f32, full 16-lane vectors only */
  if (dtype == T_F64) PACKED_BODY(double, fma); else if (dtype == T_F32) PACKED_BODY(float, fmaf); else return 1;
  return 0;
}
