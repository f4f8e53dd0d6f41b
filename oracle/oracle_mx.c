/* TEST INFRASTRUCTURE -- not part of the product; nothing under libxsmm_b200/ may call into this file.
 *
 * CPU restatement (plain C, written from the algorithm, not copied) of the reference's MX fp8 GEMM: MXBF8 x MXBF8 and
 * MXHF8 x MXHF8 with E8M0 block scales, F32 comp, F32 C or (MXBF8 only) MXBF8 C -- libxsmm_ref_matmul,
 * src/generator_gemm_reference_impl.c:2620-2679 (operand slots :577-586), and the MXBF8 block quantiser it calls for C, :757-.
 * Paths are relative to the reference tree. Pinned against the reference itself (oracle/ref_mx_shim.c) in tests/test_mxfp8.py.
 * The 8-bit float and bf16 conversions are oracle.c's (liboracle.so). Build: `make oracle`, gcc -O2 -ffp-contract=off.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

enum { T_F32 = 1, T_MXBF8 = 14, T_MXHF8 = 15 };
enum { F_TRANS_A = 1, F_TRANS_B = 2, F_BETA_0 = 4, F_VNNI_A = 256, F_VNNI_B = 512 };

extern float oracle_bf8_to_f32(uint8_t b);
extern float oracle_hf8_to_f32(uint8_t b);
extern uint16_t oracle_f32_to_bf16(float f);
extern float oracle_bf16_widen(uint16_t h);
extern uint8_t oracle_f32_to_bf8(float f);

static float bits2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t f2bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static float bf16_rne(float f) { return oracle_bf16_widen(oracle_f32_to_bf16(f)); }   /* RNE, subnormals flushed */

/* E8M0 byte -> float as bits = s << 23: 0 gives +0 (not 2^-127), 0xFF gives +inf (not NaN) */
ORACLE_API float oracle_e8m0_to_f32(uint8_t s) { return bits2f((uint32_t)s << 23); }

/* 32 f32 values -> 32 MXBF8 bytes and one E8M0 scale byte, :757-: bf16 RNE of every value; amax of the block (a NaN wins);
 * shared exponent = biased exponent of amax - 15 (E5M2's emax), clamped to [0, 254], 0 for amax = 0; the scale 2^(e-127) (the
 * subnormal 2^-127 for e = 0) rounded to bf16, its reciprocal rounded to bf16; each value times it, rounded to bf16, then to bf8
 * nearest-even; an Inf / NaN byte is clamped to the largest normal of its sign (0x7B). */
ORACLE_API void oracle_f32_to_mxbf8_block(const float* in, uint8_t* out, uint8_t* scale) {
  float v[32], amax = 0.0f, sc, rcp;
  int i, e;
  for (i = 0; i < 32; ++i) { const float a = fabsf(v[i] = bf16_rne(in[i])); if (a > amax || a != a) amax = a; }
  e = (amax == 0.0f) ? 0 : (int)((f2bits(amax) >> 23) & 0xffu);
  e -= 15;
  if (e < 0) e = 0;
  if (e > 254) e = 254;
  *scale = (uint8_t)e;
  sc = bits2f(((uint32_t)e << 23) | (e == 0 ? 0x400000u : 0u));
  rcp = bf16_rne(1.0f / bf16_rne(sc));
  for (i = 0; i < 32; ++i) {
    uint8_t o = oracle_f32_to_bf8(bf16_rne(v[i] * rcp));
    if ((o & 0x7c) == 0x7c) o = (uint8_t)((o & 0x80) | 0x7b);
    out[i] = o;
  }
}

/* dims = {m,n,k,lda,ldb,ldc}; types = {a,b,comp,c}; br_type 0 (none) or 3 (stride); the stride hints are ignored like the
 * reference does (block r at r*lda*k / r*ldb*k). a_s: [br][k/32][lda], b_s: [br][k/32][ldb], c_s (MXBF8 C): [n][ldc/32].
 * A VNNI4 [k/4][lda][4], B VNNI4-transposed [k/4][ldb][4]. Returns 1 for a tuple or layout the reference does not define. */
ORACLE_API int oracle_gemm_mx(const int* dims, const int* types, unsigned int flags, int br_type, unsigned long long br,
                              const uint8_t* a, const uint8_t* b, void* c, const uint8_t* a_s, const uint8_t* b_s, uint8_t* c_s)
{
  const int m = dims[0], n = dims[1], k = dims[2];
  const long long lda = dims[3], ldb = dims[4], ldc = dims[5];
  const int ta = types[0], tb = types[1], tcomp = types[2], tc = types[3];
  const int hf = (ta == T_MXHF8), mx_c = (tc == T_MXBF8), beta0 = (flags & F_BETA_0) != 0;
  const unsigned long long nbr = (br_type == 0) ? 1 : br;
  float* img;
  int i, j, s, k2; unsigned long long r;
  if ((ta != T_MXBF8 && ta != T_MXHF8) || tb != ta || tcomp != T_F32 || !(tc == T_F32 || (mx_c && ta == T_MXBF8))) return 1;
  if (!((flags & F_VNNI_A) && (flags & F_VNNI_B) && (flags & F_TRANS_B)) || (k % 32) != 0 || (br_type != 0 && br_type != 3)) return 1;
  if (mx_c && (!beta0 || (m % 32) != 0 || (ldc % 32) != 0)) return 1;
  img = mx_c ? (float*)malloc((size_t)ldc * n * sizeof(float)) : (float*)c;
  for (j = 0; j < n; ++j) for (i = 0; i < m; ++i) {
    float acc = 0.0f;
    if (beta0) img[j * ldc + i] = 0.0f;
    for (r = 0; r < nbr; ++r) for (s = 0; s < k / 4; ++s) {
      float tmp = 0.0f, sa, sb;
      for (k2 = 3; k2 >= 0; --k2) {
        const uint8_t ab = a[(long long)r * lda * k + s * lda * 4 + i * 4 + k2], bb = b[(long long)r * ldb * k + s * ldb * 4 + j * 4 + k2];
        tmp += (hf ? oracle_hf8_to_f32(ab) : oracle_bf8_to_f32(ab)) * (hf ? oracle_hf8_to_f32(bb) : oracle_bf8_to_f32(bb));
      }
      sa = oracle_e8m0_to_f32(a_s[(long long)r * lda * (k / 32) + (s / 8) * lda + i]);
      sb = oracle_e8m0_to_f32(b_s[(long long)r * ldb * (k / 32) + (s / 8) * ldb + j]);
      acc += tmp * sa * sb;
    }
    img[j * ldc + i] += acc;
  }
  if (mx_c) {
    for (j = 0; j < n; ++j) for (i = 0; i < m; i += 32)
      oracle_f32_to_mxbf8_block(img + j * ldc + i, (uint8_t*)c + j * ldc + i, c_s + j * (ldc / 32) + i / 32);
    free(img);
  }
  return 0;
}
