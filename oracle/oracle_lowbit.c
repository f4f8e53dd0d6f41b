/* TEST INFRASTRUCTURE -- not part of the product; nothing under libxsmm_b200/ may call into this file.
 *
 * CPU restatement (plain C, written from the algorithm, not copied) of the reference's low-bit weight GEMM branches of
 * libxsmm_ref_matmul, src/generator_gemm_reference_impl.c (set-up :457-490 and :560-620, batch-reduce offsets :180-197):
 *   MXFP4X2 x I8 -> F32 / BF16, comp I32     :1009-1088 (nibble table :67, block scales :200-236)
 *   I2X4 x I8 / U8 -> I32, comp I32          :1089-1198 (2-bit codes :19-57)
 *   I1X8 x I8 / U8 -> I32, comp I32          :1199-1272
 * Paths are relative to the reference tree. Pinned against the reference itself (oracle/ref_lowbit_shim.c) in tests/test_lowbit.py.
 * The bf16 conversions are oracle.c's (liboracle.so). Build: `make oracle`, gcc -O2 -ffp-contract=off.
 */
#include <stdint.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

enum { T_F32 = 1, T_BF16 = 2, T_I32 = 8, T_I8 = 12, T_U8 = 13, T_MXFP4 = 20, T_I2 = 22, T_I1 = 23 };
enum { F_BETA_0 = 4 };

extern uint16_t oracle_f32_to_bf16(float f);
extern float oracle_bf16_widen(uint16_t h);

static const int8_t fp4_int[16] = { 0, 11, 21, 32, 42, 64, 85, 127, 0, -11, -21, -32, -42, -64, -85, -127 };

static int i2_value(int code) { return code == 0 ? 0 : (code == 1 ? 1 : -1); }   /* 2 and 3 both mean -1 */

static float e8m0(uint8_t s) { const uint32_t u = (uint32_t)s << 23; float f; memcpy(&f, &u, 4); return f; }

/* dims = {m,n,k,lda,ldb,ldc}; types = {a,b,comp,c}; br_type 0 none, 1 address (a / b and scf_a / scf_b are arrays of br pointers),
 * 2 offset (offs_a / offs_b: byte offsets per block), 3 stride (stride_a / stride_b: bytes). scf_a: E8M0 bytes [k/32][lda]; scf_b: f32
 * [n][ldb/32], both of block 0 and moved per block as the reference does. Returns 1 for a tuple the reference has no branch for. */
ORACLE_API int oracle_gemm_lowbit(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                                  unsigned long long br, const void* a, const void* b, void* c, const long long* offs_a, const long long* offs_b,
                                  const void* scf_a, const void* scf_b)
{
  const int m = dims[0], n = dims[1], k = dims[2];
  const long long lda = dims[3], ldb = dims[4], ldc = dims[5];
  const int ta = types[0], tb = types[1], tc = types[3];
  const int beta0 = (flags & F_BETA_0) != 0, ub = (tb == T_U8);
  const unsigned long long nbr = (br_type == 0) ? 1 : br;
  int i, j, s, q; unsigned long long r;
  if (types[2] != T_I32 || (tb != T_I8 && tb != T_U8)) return 1;
  if (ta == T_MXFP4 && !(tb == T_I8 && (tc == T_F32 || tc == T_BF16))) return 1;
  if ((ta == T_I2 || ta == T_I1) && tc != T_I32) return 1;
  if (ta != T_MXFP4 && ta != T_I2 && ta != T_I1) return 1;
  for (j = 0; j < n; ++j) for (i = 0; i < m; ++i) {
    int32_t isum = 0;                  /* I2 / I1: wraps like the reference's int += */
    float acc = 0.0f;                  /* MXFP4 */
    for (r = 0; r < nbr; ++r) {
      const uint8_t* pa; const uint8_t* pb; const uint8_t* psa = NULL; const float* psb = NULL;
      if (br_type == 1) { pa = ((const uint8_t* const*)a)[r]; pb = ((const uint8_t* const*)b)[r]; }
      else if (br_type == 2) { pa = (const uint8_t*)a + offs_a[r]; pb = (const uint8_t*)b + offs_b[r]; }
      else if (br_type == 3) { pa = (const uint8_t*)a + stride_a * (long long)r; pb = (const uint8_t*)b + stride_b * (long long)r; }
      else { pa = (const uint8_t*)a; pb = (const uint8_t*)b; }
      if (ta == T_MXFP4) {             /* :207-235: the scales of block r */
        if (br_type == 1) { psa = ((const uint8_t* const*)scf_a)[r]; psb = ((const float* const*)scf_b)[r]; }
        else if (br_type == 2) { psa = (const uint8_t*)scf_a + (offs_a[r] * 2) / 32; psb = (const float*)scf_b + offs_b[r] / 32; }
        else if (br_type == 3) { psa = (const uint8_t*)scf_a + ((stride_a * 2) / 32) * (long long)r; psb = (const float*)scf_b + (stride_b / 32) * (long long)r; }
        else { psa = (const uint8_t*)scf_a; psb = (const float*)scf_b; }
        for (s = 0; s < k / 32; ++s) {
          int32_t t = 0;
          for (q = 0; q < 32; ++q) {   /* the sum is exact: its order does not matter */
            const uint8_t byte = pa[((long long)(s * 32 + q) / 8) * lda * 4 + (long long)i * 4 + (q % 4)];
            const int code = ((q % 8) < 4) ? (byte & 0x0f) : (byte >> 4);
            t += (int32_t)fp4_int[code] * (int8_t)pb[(long long)j * ldb + s * 32 + q];
          }
          acc += ((float)t * e8m0(psa[(long long)s * lda + i])) * psb[(long long)j * (ldb / 32) + s];
        }
      } else if (ta == T_I2) {
        const int m4 = m / 4, pair = i / m4;
        for (s = 0; s < k / 4; ++s) for (q = 0; q < 4; ++q) {
          const int code = (pa[(long long)s * lda + (long long)(i % m4) * 4 + q] >> (2 * pair)) & 3;
          const int bv = ub ? (int)pb[(long long)j * ldb + s * 4 + q] : (int)(int8_t)pb[(long long)j * ldb + s * 4 + q];
          isum = (int32_t)((uint32_t)isum + (uint32_t)(i2_value(code) * bv));
        }
      } else {
        for (s = 0; s < k / 4; ++s) for (q = 0; q < 4; ++q) {
          const int bit = (pa[((long long)s * lda) / 2 + i / 2] >> (4 * (i & 1) + q)) & 1;
          const int bv = ub ? (int)pb[(long long)j * ldb + s * 4 + q] : (int)(int8_t)pb[(long long)j * ldb + s * 4 + q];
          isum = (int32_t)((uint32_t)isum + (uint32_t)(bit ? -bv : bv));
        }
      }
    }
    if (ta != T_MXFP4) {
      int32_t* cp = (int32_t*)c + (long long)j * ldc + i;
      *cp = (int32_t)((beta0 ? 0u : (uint32_t)*cp) + (uint32_t)isum);
    } else if (tc == T_F32) {
      float* cp = (float*)c + (long long)j * ldc + i;
      *cp = (beta0 ? 0.0f : *cp) + acc;
    } else {
      uint16_t* cp = (uint16_t*)c + (long long)j * ldc + i;
      *cp = oracle_f32_to_bf16((beta0 ? 0.0f : oracle_bf16_widen(*cp)) + acc);
    }
  }
  return 0;
}
