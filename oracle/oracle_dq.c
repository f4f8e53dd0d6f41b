/* TEST INFRASTRUCTURE -- not part of the product; nothing under libxsmm_b200/ may call into this file.
 *
 * CPU restatement (plain C, written from the algorithm, not copied) of the reference's dequantising GEMM branches of
 * libxsmm_ref_matmul, src/generator_gemm_reference_impl.c (operand slots :551-630, batch-reduce offsets :180-197):
 *   I8 x BF16 -> F32 / BF16, comp F32                    :1684-1730
 *   BF8 x F16 -> F16 / F32, comp F16 / F32 / IMPLICIT     :1731-1792
 *   I4 / U4 pairs x F16 -> F16 / F32, same comps          :1793-1880 (VNNI_A, no INTLV_A_FORMAT: :472-475)
 *   I8 x F16 -> F16                                       :1881-1952
 *   I8 x F16 -> F32                                       :1953-2024
 * Paths are relative to the reference tree. Comp IMPLICIT is resolved as on an SPR host (the "replacement FMA" of :1749).
 * Pinned against the reference itself (oracle/ref_dq_shim.c) in tests/test_dequant.py. The f16 / bf16 / bf8 conversions are
 * oracle.c's (liboracle.so). Build: `make oracle`, gcc -O2 -ffp-contract=off.
 */
#include <stdint.h>
#include <stdlib.h>

#define ORACLE_API __attribute__((visibility("default")))

enum { T_F32 = 1, T_BF16 = 2, T_F16 = 3, T_BF8 = 4, T_I8 = 12, T_I4X2 = 18, T_U4X2 = 19, T_IMPLICIT = 25 };
enum { F_TRANS_B = 2, F_BETA_0 = 4, F_VNNI_A = 256 };
enum { DQ_I8_BF16 = 1, DQ_I8_F16, DQ_I4_F16, DQ_BF8_F16 };

extern float oracle_f16_to_f32(uint16_t h);
extern uint16_t oracle_f32_to_f16(float f);
extern float oracle_bf8_to_f32(uint8_t b);
extern uint16_t oracle_f32_to_bf16(float f);
extern float oracle_bf16_widen(uint16_t h);

static float f16r(float v) { return oracle_f16_to_f32(oracle_f32_to_f16(v)); }

static int dq_form(const int* types) {
  const int ta = types[0], tb = types[1], tcomp = types[2], tc = types[3];
  const int f16comp = (tcomp == T_F16 || tcomp == T_F32 || tcomp == T_IMPLICIT), f16c = (tc == T_F16 || tc == T_F32);
  if (ta == T_I8 && tb == T_BF16) return (tcomp == T_F32 && (tc == T_F32 || tc == T_BF16)) ? DQ_I8_BF16 : 0;
  if (tb != T_F16 || !f16comp || !f16c) return 0;
  if (ta == T_I8) return DQ_I8_F16;
  if (ta == T_I4X2 || ta == T_U4X2) return DQ_I4_F16;
  if (ta == T_BF8) return DQ_BF8_F16;
  return 0;
}

/* dims = {m,n,k,lda,ldb,ldc}; types = {a,b,comp,c}; br_type 0 none, 1 address (a / b are arrays of br block pointers), 2 offset
 * (offs_a / offs_b: byte offsets per block), 3 stride (stride_a / stride_b: bytes). scf: the m row scales (f32 for I8 x BF16, else
 * f16), zpt: the m f16 zero points of an int4 A; the same for every r. Returns 1 for a tuple the reference has no branch for. */
ORACLE_API int oracle_gemm_dq(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                              unsigned long long br, const void* a, const void* b, void* c, const long long* offs_a, const long long* offs_b,
                              const void* scf, const void* zpt)
{
  const int m = dims[0], n = dims[1], k = dims[2];
  const long long lda = dims[3], ldb = dims[4], ldc = dims[5];
  const int form = dq_form(types), tc = types[3];
  const int beta0 = (flags & F_BETA_0) != 0, trans_b = (flags & F_TRANS_B) != 0;
  /* the replacement FMA: comp F16, or IMPLICIT on an SPR host (:1749, :1811, :1898, :1970) */
  const int rep = form != DQ_I8_BF16 && (types[2] == T_F16 || types[2] == T_IMPLICIT);
  const int kb = (form == DQ_I4_F16 || (form == DQ_BF8_F16 && (flags & F_VNNI_A) != 0)) ? 2 : 1;
  const unsigned long long nbr = (br_type == 0) ? 1 : br;
  int i, j, s, k2; unsigned long long r;
  if (form == 0) return 1;
  for (j = 0; j < n; ++j) for (i = 0; i < m; ++i) {
    float acc = 0.0f;
    for (r = 0; r < nbr; ++r) {
      const uint8_t* pa; const uint16_t* pb;
      if (br_type == 1) { pa = ((const uint8_t* const*)a)[r]; pb = ((const uint16_t* const*)b)[r]; }
      else if (br_type == 2) { pa = (const uint8_t*)a + offs_a[r]; pb = (const uint16_t*)b + offs_b[r] / 2; }
      else if (br_type == 3) { pa = (const uint8_t*)a + stride_a * (long long)r; pb = (const uint16_t*)b + (stride_b / 2) * (long long)r; }
      else { pa = (const uint8_t*)a; pb = (const uint16_t*)b; }
      for (s = 0; s < k / kb; ++s) for (k2 = 0; k2 < kb; ++k2) {
        const long long kk = (long long)s * kb + k2;
        const uint16_t bw = trans_b ? pb[kk * ldb + j] : pb[j * ldb + kk];
        float av, bv;
        if (form == DQ_BF8_F16) av = oracle_bf8_to_f32(pa[s * lda * kb + (long long)i * kb + k2]);
        else {
          const uint8_t by = pa[s * lda + i];
          int q;
          if (form != DQ_I4_F16) q = (int8_t)by;                              /* (char) of the byte: signed */
          else if (types[0] == T_U4X2) q = (k2 == 0) ? (by & 0x0f) : (by >> 4);
          else { const int nib = (k2 == 0) ? (by & 0x0f) : (by >> 4); q = (nib >= 8) ? nib - 16 : nib; }
          av = (float)q;                                                        /* exact in f16: the rounding of :1910-1913 is void */
          if (form == DQ_I8_BF16) av = oracle_bf16_widen(oracle_f32_to_bf16(av * ((const float*)scf)[i]));
          else {
            if (form == DQ_I4_F16) { av = av - oracle_f16_to_f32(((const uint16_t*)zpt)[i]); if (rep) av = f16r(av); }
            av = av * oracle_f16_to_f32(((const uint16_t*)scf)[i]);
            if (rep) av = f16r(av);
          }
        }
        bv = (form == DQ_I8_BF16) ? oracle_bf16_widen(bw) : oracle_f16_to_f32(bw);
        acc += av * bv;
        if (rep) acc = f16r(acc);
      }
    }
    if (tc == T_F32) {
      float* cp = (float*)c + j * ldc + i;
      if (!beta0) acc += (form == DQ_I8_BF16 || form == DQ_BF8_F16) ? *cp : f16r(*cp);   /* I8 / I4 x F16: old C through f16 */
      *cp = acc;
    } else if (form == DQ_I8_BF16) {
      uint16_t* cp = (uint16_t*)c + j * ldc + i;
      if (!beta0) acc += oracle_bf16_widen(*cp);
      *cp = oracle_f32_to_bf16(acc);
    } else {
      uint16_t* cp = (uint16_t*)c + j * ldc + i;
      if (!beta0) acc += oracle_f16_to_f32(*cp);
      *cp = oracle_f32_to_f16(acc);
    }
  }
  return 0;
}
