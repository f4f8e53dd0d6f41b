// libxsmm_b200 -- sparse kernels of the hot path (sm_90a):
//   * sreg_kernel      : fsspmdm -- fixed sparse A (CSR, alpha folded in) times dense row-major B,
//                        N streamed through shared memory in 512-byte column strips with
//                        TMA 2D tensor copies into a ring of 1 to 3 mbarrier-guarded stages. HBM-bound.
//                        Replaces src/generator_spgemm_csr_asparse_reg.c (A kept in registers on x86).
//   * packed_sp_kernel : SOA-packed sparse x dense with `packed_width` innermost
//                        (src/generator_packed_spgemm_cs*.c; golds in samples/xgemm_norm_packed/*.c)
//   * bcsc_simt_kernel : block-sparse B (BCSC) exact-order kernel, every datatype of the reference's
//                        spmm driver (samples/xgemm_sparse/spmm_kernel.c:74-217); the tensor-core
//                        version lives in bcsc_tc.cu.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include "xb_internal.h"
#include "xb_device.cuh"
#include "xb_tma.cuh"

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  } while (!done);
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// ------------------------------------------------------------------------------------------------------
// fsspmdm: C[M x N] (row-major, ldc) = beta*C + A_csr * B[K x N] (row-major, ldb)
// T = float (V = float4) or double (V = double2): a strip is 32 vectors = 512 bytes of every B row.
template <typename T> struct Vec;
template <> struct Vec<float> { typedef float4 type; enum { N = 4 }; };
template <> struct Vec<double> { typedef double2 type; enum { N = 2 }; };

__device__ __forceinline__ void vfma(float4& acc, float a, const float4& b) {
  acc.x = fmaf(a, b.x, acc.x); acc.y = fmaf(a, b.y, acc.y); acc.z = fmaf(a, b.z, acc.z); acc.w = fmaf(a, b.w, acc.w);
}
__device__ __forceinline__ void vfma(double2& acc, double a, const double2& b) { acc.x = fma(a, b.x, acc.x); acc.y = fma(a, b.y, acc.y); }
__device__ __forceinline__ void vadd(float4& a, const float4& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ void vadd(double2& a, const double2& b) { a.x += b.x; a.y += b.y; }
__device__ __forceinline__ void vzero(float4& a) { a = make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void vzero(double2& a) { a = make_double2(0.0, 0.0); }

struct SregParams {
  int M, K; long long N, ldb, ldc;
  unsigned int nnz;
  const unsigned int* rowptr; const void* entries;      // entries: packed {value, byte offset of the B row in a stage}
  const void* b; void* c;
  int beta0; int stages;
};

template <typename T> struct SregEntry;
template <> struct SregEntry<float> { float v; unsigned int off; };
template <> struct SregEntry<double> { double v; unsigned int off; unsigned int pad; };

// shared memory: [barriers 1 KB][stages x K x 512 B of B][nnz entries][M+1 row pointers]
template <typename T>
__global__ void __launch_bounds__(1024, 1) sreg_kernel(const __grid_constant__ CUtensorMap map_b, const SregParams P) {
  typedef typename Vec<T>::type V;
  typedef SregEntry<T> E;
  constexpr int VN = Vec<T>::N;
  constexpr int STRIP = 32 * VN;                // elements per strip row (512 bytes)
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);
  unsigned char* sB = smem_raw + 1024;       // TMA tensor destinations: keep stage bases 1 KB aligned
  const size_t stage_bytes = (size_t)P.K * 512;
  E* s_ent = reinterpret_cast<E*>(sB + (size_t)P.stages * stage_bytes);
  unsigned int* s_rowptr = reinterpret_cast<unsigned int*>(s_ent + P.nnz);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;
  for (int i = tid; i <= P.M; i += blockDim.x) s_rowptr[i] = P.rowptr[i];
  for (unsigned int i = tid; i < P.nnz; i += blockDim.x) s_ent[i] = reinterpret_cast<const E*>(P.entries)[i];
  if (tid == 0) {
    for (int s = 0; s < P.stages; ++s) mbar_init(smem_u32(&bars[s]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const long long nstrips = (P.N + STRIP - 1) / STRIP;
  const long long first = blockIdx.x, step = gridDim.x;
  T* Cg = (T*)P.c;
  const int S = P.stages;

  // producer: one TMA tensor copy per strip (box = 512 bytes x K rows, K <= 256; columns past N are zero-filled)
  auto issue = [&](long long strip, int stage) {
    if (lane == 0) {
      const uint32_t bar = smem_u32(&bars[stage]);
      mbar_expect_tx(bar, (uint32_t)stage_bytes);
      asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                   :: "r"(smem_u32(sB + (size_t)stage * stage_bytes)), "l"(&map_b), "r"((int)(strip * STRIP)), "r"(0), "r"(bar) : "memory");
    }
  };

  // prologue: fill S-1 stages
  if (warp == 0) {
    if (S == 1) { if (first < nstrips) issue(first, 0); }
    else for (int s = 0; s < S - 1; ++s) if (first + (long long)s * step < nstrips) issue(first + (long long)s * step, s);
  }
  long long it = 0;
  for (long long strip = first; strip < nstrips; strip += step, ++it) {
    const int stage = (int)(it % S);
    if (S > 1 && warp == 0) {             // keep S-1 strips in flight: the stage being refilled was released by the barrier below
      const long long nxt = strip + (long long)(S - 1) * step;
      if (nxt < nstrips) issue(nxt, (int)((it + S - 1) % S));
    }
    mbar_wait(smem_u32(&bars[stage]), (uint32_t)((it / S) & 1));
    const unsigned char* Bs = sB + (size_t)stage * stage_bytes + (size_t)lane * sizeof(V);
    const long long n0 = strip * STRIP;
    const bool in = (n0 + (long long)lane * VN) < P.N;        // N % VN == 0 is guaranteed by create()
    for (int row = warp; row < P.M; row += nwarps) {
      V acc0, acc1; vzero(acc0); vzero(acc1);
      unsigned int e = s_rowptr[row];
      const unsigned int e1 = s_rowptr[row + 1];
      for (; e + 4 <= e1; e += 4) {                           // 4 independent B loads in flight
        const E t0 = s_ent[e], t1 = s_ent[e + 1], t2 = s_ent[e + 2], t3 = s_ent[e + 3];
        const V b0 = *reinterpret_cast<const V*>(Bs + t0.off), b1 = *reinterpret_cast<const V*>(Bs + t1.off);
        const V b2 = *reinterpret_cast<const V*>(Bs + t2.off), b3 = *reinterpret_cast<const V*>(Bs + t3.off);
        vfma(acc0, t0.v, b0); vfma(acc1, t1.v, b1); vfma(acc0, t2.v, b2); vfma(acc1, t3.v, b3);
      }
      for (; e < e1; ++e) { const E t = s_ent[e]; vfma(acc0, t.v, *reinterpret_cast<const V*>(Bs + t.off)); }
      vadd(acc0, acc1);
      if (in) {
        V* dst = reinterpret_cast<V*>(Cg + (size_t)row * P.ldc + n0) + lane;
        if (!P.beta0) { const V old = *dst; vadd(acc0, old); }
        *dst = acc0;
      }
    }
    __syncthreads();                                          // strip consumed: its stage may be refilled
    if (S == 1 && warp == 0 && strip + step < nstrips) issue(strip + step, 0);
  }
}

// fallback without shared-memory staging (very large K, or unaligned leading dimensions)
template <typename T>
__global__ void __launch_bounds__(256) sreg_direct_kernel(const SregParams P) {
  const T* Bg = (const T*)P.b; T* Cg = (T*)P.c; const SregEntry<T>* ent = (const SregEntry<T>*)P.entries;
  const long long total = (long long)P.M * P.N;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(e / P.N); const long long col = e % P.N;
    T acc = 0;
    for (unsigned int z = P.rowptr[row]; z < P.rowptr[row + 1]; ++z) acc += ent[z].v * Bg[(size_t)(ent[z].off >> 9) * P.ldb + col];
    T* dst = Cg + (size_t)row * P.ldc + col;
    *dst = P.beta0 ? acc : (*dst + acc);
  }
}

// ------------------------------------------------------------------------------------------------------
// packed sparse: one CTA per batch item, threads over (n, p). The call axis (count, strides) of every packed kernel runs through
// blockIdx.y: a single call launches its own grid in x with one row of CTAs, a batch stacks up to 65,535 rows of calls and loops
// over the rest.
struct PackedParams {
  int kind, M, N, K, P, lda, ldb, ldc, beta0, is_f64;
  const unsigned int* ptr; const unsigned int* idx;
  const char* a; const char* b; char* c;
  long long stride_a, stride_b, stride_c, count;
};

template <typename T>
__global__ void __launch_bounds__(256) packed_sp_kernel(const PackedParams Q) {
  const int P = Q.P;
  for (long long item = blockIdx.y; item < Q.count; item += gridDim.y) {
    const T* A = (const T*)(Q.a + item * Q.stride_a); const T* B = (const T*)(Q.b + item * Q.stride_b);
    T* C = (T*)(Q.c + item * Q.stride_c);
    const int work = Q.M * Q.N * P;
    for (int e = threadIdx.x; e < work; e += blockDim.x) {
      const int p = e % P, j = (e / P) % Q.N, i = e / (P * Q.N);
      if (Q.kind == XB_KIND_SP_A_CSR) {           // C[i][j][p] (+)= sum_z a[z] * B[col[z]][j][p]
        if (Q.ptr[i] == Q.ptr[i + 1]) continue;    // the reference emits nothing for an empty row, not even the BETA_0 zeroing
        T acc = Q.beta0 ? (T)0 : C[((size_t)i * Q.ldc + j) * P + p];
        for (unsigned int z = Q.ptr[i]; z < Q.ptr[i + 1]; ++z) acc += A[z] * B[((size_t)Q.idx[z] * Q.ldb + j) * P + p];
        C[((size_t)i * Q.ldc + j) * P + p] = acc;
      } else if (Q.kind == XB_KIND_SP_B_CSC) {    // C[i][j][p] (+)= sum_{z in col j} A[i][row[z]][p] * b[z]
        T acc = Q.beta0 ? (T)0 : C[((size_t)i * Q.ldc + j) * P + p];
        for (unsigned int z = Q.ptr[j]; z < Q.ptr[j + 1]; ++z) acc += A[((size_t)i * Q.lda + Q.idx[z]) * P + p] * B[z];
        C[((size_t)i * Q.ldc + j) * P + p] = acc;
      } else if (Q.kind == XB_KIND_SP_B_CSR) {    // rows of B are k; scan each row for column j
        T acc = Q.beta0 ? (T)0 : C[((size_t)i * Q.ldc + j) * P + p];
        for (int k = 0; k < Q.K; ++k) {
          for (unsigned int z = Q.ptr[k]; z < Q.ptr[k + 1]; ++z) {
            if ((int)Q.idx[z] == j) acc += A[((size_t)i * Q.lda + k) * P + p] * B[z];
          }
        }
        C[((size_t)i * Q.ldc + j) * P + p] = acc;
      }
    }
  }
}

// C sparse (CSC pattern): c[z][p] (+)= sum_k A[row[z]][k][p] * B[k][col][p]
// C sparse (CSC pattern, ldc == 0): ONE scalar per non-zero, the packed dimension is summed away:
//   C[z] (+)= sum_k sum_p A[k][row(z)][p] * B[k][col(z)][p],   A = [K][lda][P], B = [K][ldb][P]
// (src/generator_packed_spgemm_csc_csparse_avx_avx2_avx512.c:63-191). One warp per non-zero: lanes stride the packed
// dimension (coalesced 128-byte rows of A and B), shuffle reduction at the end.
template <typename T>
__global__ void __launch_bounds__(256) packed_csparse_kernel(const PackedParams Q) {
  const int P = Q.P, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const unsigned int nnz = Q.ptr[Q.N];
  for (long long item = blockIdx.y; item < Q.count; item += gridDim.y) {
    const T* A = (const T*)(Q.a + item * Q.stride_a); const T* B = (const T*)(Q.b + item * Q.stride_b);
    T* C = (T*)(Q.c + item * Q.stride_c);
    for (unsigned int z = blockIdx.x * nwarps + warp; z < nnz; z += gridDim.x * nwarps) {
      int lo = 0, hi = Q.N;                               // column of z: last j with ptr[j] <= z
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (Q.ptr[mid] <= z) lo = mid; else hi = mid; }
      const int j = lo, i = (int)Q.idx[z];
      T acc = 0;
      for (int k = 0; k < Q.K; ++k) {
        const T* ar = A + ((size_t)k * Q.lda + i) * P; const T* br = B + ((size_t)k * Q.ldb + j) * P;
        for (int p = lane; p < P; p += 32) acc += ar[p] * br[p];
      }
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) C[z] = Q.beta0 ? acc : acc + C[z];
    }
  }
}

// ------------------------------------------------------------------------------------------------------
// packed DENSE GEMM (EDGE/SeisSol, src/generator_packed_gemm*.c): the packed dimension P (a vector of independent problems)
// is innermost in every packed operand, so consecutive lanes take consecutive p: every access is a coalesced row.
//   PK_GEMM   C[n][m][p] (+)= sum_k A[k][m][p] * B[n][k][p]          (gold: samples/xgemm_packed/gemm_packed_kernel.c:36-66)
//   PK_AC_RM  C[m][n][p] (+)= sum_k A[m][k][p] * B[k][n]             (gold: samples/xgemm_norm_packed/dense_packedacrm.c:37-49)
//   PK_BC_RM  C[m][n][p] (+)= sum_k A[m][k]    * B[k][n][p]          (gold: samples/xgemm_norm_packed/dense_packedbcrm.c)
// k ascending with fused multiply-add like the reference's FMA kernels; one thread per C element.
template <typename T>
__global__ void __launch_bounds__(256) packed_dense_kernel(const PackedParams Q) {
  const long long P = Q.P, total = (long long)Q.M * Q.N * P;
  for (long long item = blockIdx.y; item < Q.count; item += gridDim.y) {
    const T* A = (const T*)(Q.a + item * Q.stride_a); const T* B = (const T*)(Q.b + item * Q.stride_b);
    T* C = (T*)(Q.c + item * Q.stride_c);
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
      const long long p = e % P, rest = e / P;
      long long ci; T acc;
      if (Q.kind == XB_KIND_PK_GEMM) {
        const long long mm = rest % Q.M, nn = rest / Q.M;
        ci = (nn * Q.ldc + mm) * P + p; acc = Q.beta0 ? (T)0 : C[ci];
        for (int k = 0; k < Q.K; ++k) acc = fma(A[((long long)k * Q.lda + mm) * P + p], B[(nn * Q.ldb + k) * P + p], acc);
      } else {
        const long long nn = rest % Q.N, mm = rest / Q.N;
        ci = (mm * Q.ldc + nn) * P + p; acc = Q.beta0 ? (T)0 : C[ci];
        if (Q.kind == XB_KIND_PK_AC_RM) { for (int k = 0; k < Q.K; ++k) acc = fma(A[(mm * Q.lda + k) * P + p], B[(long long)k * Q.ldb + nn], acc); }
        else { for (int k = 0; k < Q.K; ++k) acc = fma(A[mm * Q.lda + k], B[((long long)k * Q.ldb + nn) * P + p], acc); }
      }
      C[ci] = acc;
    }
  }
}

// ------------------------------------------------------------------------------------------------------
// BCSC exact-order kernel. One CTA per (m_block, block-column); thread per (m, n_local) element.
// Call axis (a strided batch, xb_sparse_calls): the template flag B. A single call launches B = false, whose loop over the calls is
// the one iteration t = 0 and folds away at compile time, so its code is that of the kernel without the axis. A batch launches
// B = true: blockIdx.x keeps the single call's split of the (m_block, block-column) items, blockIdx.y strides the calls, and call t
// reads A and the block values and writes C at its bases advanced by t times their byte strides. The pattern is shared.
struct BcscParams {
  int M, K, bk, bn, ta, tb, tc, beta0, trans_a, vnni_a, vnni_b_t;
  long long N;                  // total columns = n_blocks * bn
  long long m_blocks;
  const char* a; const char* bvals; const unsigned int* colptr; const unsigned int* rowidx; char* c;
};

__device__ __forceinline__ float bcsc_load_f(const char* base, size_t idx, int t) {
  return (t == LIBXSMM_DATATYPE_F32) ? ((const float*)base)[idx] : xb_bf16_to_f32(((const unsigned short*)base)[idx]);
}

template <bool B>
__global__ void __launch_bounds__(256) bcsc_simt_kernel(const BcscParams Q, const xb_sparse_calls tl) {
  const long long nbc = Q.N / Q.bn;
  const size_t tsa = xb_dev_typesize(Q.ta), tsc = xb_dev_typesize(Q.tc);
  const bool is_int = (Q.tc == LIBXSMM_DATATYPE_I32);
  const int v = (Q.ta == LIBXSMM_DATATYPE_BF16) ? 2 : ((Q.ta == LIBXSMM_DATATYPE_F32) ? 1 : 4);
#pragma unroll 1
  for (long long t = B ? blockIdx.y : 0; t < (B ? tl.count : 1); t += B ? gridDim.y : 1) {
  const char* const a0 = B ? Q.a + t * tl.s_a : Q.a;
  const char* const bvals = B ? Q.bvals + t * tl.s_b : Q.bvals;
  char* const c0 = B ? Q.c + t * tl.s_c : Q.c;
  for (long long w = blockIdx.x; w < Q.m_blocks * nbc; w += gridDim.x) {
    const long long mb = w / nbc, jb = w % nbc;
    const char* A = a0 + (size_t)mb * Q.K * Q.M * tsa;
    char* C = c0 + (size_t)mb * Q.N * Q.M * tsc;
    for (int e = threadIdx.x; e < Q.M * Q.bn; e += blockDim.x) {
      const int i = e % Q.M, nl = e / Q.M;
      const long long j = jb * Q.bn + nl;
      const size_t ci = Q.trans_a ? ((size_t)i * Q.N + j) : ((size_t)j * Q.M + i);
      float facc = 0.f; int iacc = 0;
      if (!Q.beta0) {
        if (is_int) iacc = ((const int*)C)[ci];
        else facc = (Q.tc == LIBXSMM_DATATYPE_F32) ? ((const float*)C)[ci] : xb_bf16_to_f32(((const unsigned short*)C)[ci]);
      }
      for (unsigned int z = Q.colptr[jb]; z < Q.colptr[jb + 1]; ++z) {
        const int kb = (int)Q.rowidx[z];
        if (kb >= Q.K / Q.bk) continue;            // block-row outside A: ignored, like the tensor-core kernel
        for (int kk = 0; kk < Q.bk; ++kk) {
          const int k = kb * Q.bk + kk;
          size_t ai;
          if (Q.trans_a) ai = (size_t)i * Q.K + k;
          else if (Q.vnni_a && v > 1) ai = (size_t)(k / v) * Q.M * v + (size_t)i * v + (k % v);
          else ai = (size_t)k * Q.M + i;
          size_t bi;
          if (Q.vnni_b_t) bi = (size_t)z * Q.bk * Q.bn + (size_t)(kk / v) * Q.bn * v + (size_t)nl * v + (kk % v);
          else bi = (size_t)z * Q.bk * Q.bn + (size_t)nl * Q.bk + kk;
          if (is_int) {
            const unsigned char ar = ((const unsigned char*)A)[ai], br = ((const unsigned char*)bvals)[bi];
            const int av = (Q.ta == LIBXSMM_DATATYPE_U8) ? (int)ar : (int)(signed char)ar;
            const int bv = (Q.tb == LIBXSMM_DATATYPE_U8) ? (int)br : (int)(signed char)br;
            iacc += av * bv;
          } else {
            facc = __fadd_rn(facc, __fmul_rn(bcsc_load_f(A, ai, Q.ta), bcsc_load_f(bvals, bi, Q.tb)));
          }
        }
      }
      if (is_int) ((int*)C)[ci] = iacc;
      else if (Q.tc == LIBXSMM_DATATYPE_F32) ((float*)C)[ci] = facc;
      else ((unsigned short*)C)[ci] = xb_f32_to_bf16_rne(facc);
    }
  }
  }
}

int g_sms = 0;
int num_sms() {
  if (g_sms == 0) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev); if (g_sms <= 0) g_sms = 132; }
  return g_sms;
}
int check_launch(const char* where, int backend = LIBXSMM_B200_BACKEND_STREAM) {
  xb_rt_count_launch_backend(backend);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { xb_rt_note_error((int)e, where); return (int)e; }
  return 0;
}
unsigned long long g_sreg_attr[2] = {0ull, 0ull};   // one bit per device ordinal

}  // namespace

// shared memory sreg_kernel needs besides its stages: barriers, the entries of A, the row pointers
static size_t sreg_meta_bytes(const xb_sparse_desc* d) {
  const size_t es = (d->ta == LIBXSMM_DATATYPE_F64) ? 16 : 8;
  return 1024 + (size_t)d->nnz * es + (size_t)(d->m + 1) * 4 + 16;
}

// The one decision of which kernel an fsspmdm call runs: 0 = sreg_direct_kernel, S = 1..3 = sreg_kernel with S stages. The staged
// kernel needs 16-byte aligned B, C and rows (TMA), one TMA box per strip (K <= 256 rows) and S stages of K x 512 bytes plus the
// pattern within 226 KB of shared memory; it takes as many stages up to 3 as fit.
static int xb_sreg_variant(const xb_sparse_desc* d, const void* b, const void* c, long long n_total) {
  const size_t ts = (d->ta == LIBXSMM_DATATYPE_F64) ? 8 : 4;
  const size_t limit = 226 * 1024;
  const bool aligned = ((uintptr_t)b % 16 == 0) && ((uintptr_t)c % 16 == 0) && ((d->ldb * ts) % 16 == 0) && ((d->ldc * ts) % 16 == 0)
                    && ((n_total * ts) % 16 == 0);
  if (!aligned || d->k > 256 || xb_tma_encoder() == nullptr) return 0;
  int stages = 3;
  while (stages > 0 && (size_t)stages * d->k * 512 + sreg_meta_bytes(d) > limit) --stages;
  return stages;
}

// the same answer for a handle and the operands of a call (include/libxsmm_b200.h). Defined here, next to the decision, so that the
// host objects need nothing new from the CUDA side.
LIBXSMM_API int libxsmm_b200_fsspmdm_variant(const libxsmm_fsspmdm* handle, const void* B, const void* C) {
  const xb_sparse_desc* d = xb_fsspmdm_desc(handle);
  const void* staged = (const void*)(uintptr_t)256;   // pageable operands travel through the scratch arena, 256-byte aligned
  if (d == nullptr) return -1;
  if (B == nullptr || xb_rt_ptr_kind(B) == 0) B = staged;
  if (C == nullptr || xb_rt_ptr_kind(C) == 0) C = staged;
  return xb_sreg_variant(d, B, C, d->max_n);
}

extern "C" int xb_sreg_launch(const xb_sparse_desc* d, const void* b, void* c, long long n_total) {
  if (n_total <= 0) return 0;
  SregParams P;
  P.M = d->m; P.K = d->k; P.N = n_total; P.ldb = d->ldb; P.ldc = d->ldc; P.nnz = d->nnz;
  P.rowptr = d->d_ptr; P.entries = d->d_val; P.b = b; P.c = c; P.beta0 = d->beta0;
  P.stages = xb_sreg_variant(d, b, c, n_total);
  const bool f64 = (d->ta == LIBXSMM_DATATYPE_F64);
  const size_t ts = f64 ? 8 : 4;
  cudaStream_t stream = (cudaStream_t)xb_rt_stream();
  if (P.stages == 0) {
    const long long total = (long long)d->m * n_total;
    long long grid = (total + 255) / 256; if (grid > num_sms() * 16) grid = num_sms() * 16;
    if (f64) sreg_direct_kernel<double><<<(unsigned int)grid, 256, 0, stream>>>(P);
    else sreg_direct_kernel<float><<<(unsigned int)grid, 256, 0, stream>>>(P);
    return check_launch("sreg_direct");
  }
  const size_t smem = (size_t)P.stages * d->k * 512 + sreg_meta_bytes(d);
  const long long strip = f64 ? 64 : 128;
  long long grid = (n_total + strip - 1) / strip; if (grid > num_sms()) grid = num_sms();
  const int warps = d->m < 4 ? 4 : (d->m > 32 ? 32 : d->m);      // one row per warp and pass
  const int threads = warps * 32;
  // the encoder is a driver-API call and needs the device's context current on this thread. The runtime binds it lazily, so in a
  // thread whose first CUDA work is this call (an OpenMP worker on managed B and C) encoding fails unless it is bound here first.
  { int dev = 0; if (cudaGetDevice(&dev) == cudaSuccess) cudaSetDevice(dev); }
  CUtensorMap map_b;
  {
    const cuuint64_t dims[2] = {(cuuint64_t)n_total, (cuuint64_t)d->k};
    const cuuint64_t strides[1] = {(cuuint64_t)d->ldb * ts};
    const cuuint32_t box[2] = {(cuuint32_t)strip, (cuuint32_t)d->k};
    const cuuint32_t estr[2] = {1, 1};
    // xb_sreg_variant accepted these operands: a tensor map that still cannot be encoded is a bug, not a reason to fall back
    const CUresult r = xb_tma_encoder()(&map_b, f64 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT64 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)b,
          dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { xb_rt_note_error((int)r, "sreg: TMA tensor map"); return (int)r; }
  }
  if (f64) {
    if (xb_rt_first_use_on_device(&g_sreg_attr[1])) cudaFuncSetAttribute(sreg_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    sreg_kernel<double><<<(unsigned int)grid, threads, smem, stream>>>(map_b, P);
  } else {
    if (xb_rt_first_use_on_device(&g_sreg_attr[0])) cudaFuncSetAttribute(sreg_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    sreg_kernel<float><<<(unsigned int)grid, threads, smem, stream>>>(map_b, P);
  }
  return check_launch("sreg");
}

extern "C" int xb_packed_sp_launch(const xb_sparse_desc* d, const void* a, const void* b, void* c, long long count,
                                   long long stride_a, long long stride_b, long long stride_c)
{
  PackedParams Q;
  Q.kind = d->kind; Q.M = d->m; Q.N = (d->kind == XB_KIND_SP_B_CSR) ? d->max_n : d->n; Q.K = d->k; Q.P = d->packed_width; Q.lda = d->lda; Q.ldb = d->ldb; Q.ldc = d->ldc;
  Q.beta0 = d->beta0; Q.is_f64 = (d->ta == LIBXSMM_DATATYPE_F64); Q.ptr = d->d_ptr; Q.idx = d->d_idx;
  Q.a = (const char*)a; Q.b = (const char*)b; Q.c = (char*)c; Q.stride_a = stride_a; Q.stride_b = stride_b; Q.stride_c = stride_c; Q.count = count;
  if (count <= 0) return 0;
  cudaStream_t stream = (cudaStream_t)xb_rt_stream();
  const unsigned int grid = (unsigned int)(count < 65535 ? count : 65535);
  if (d->kind == XB_KIND_PK_GEMM || d->kind == XB_KIND_PK_AC_RM || d->kind == XB_KIND_PK_BC_RM) {
    const long long total = (long long)Q.M * Q.N * Q.P;
    long long gx = (total + 255) / 256; if (gx > 132 * 8) gx = 132 * 8; if (gx < 1) gx = 1;
    const dim3 g2((unsigned int)gx, grid);
    if (Q.is_f64) packed_dense_kernel<double><<<g2, 256, 0, stream>>>(Q); else packed_dense_kernel<float><<<g2, 256, 0, stream>>>(Q);
    return check_launch("packed_dense");
  }
  if (d->kind == XB_KIND_SP_C_CSC) {
    const unsigned int gx = (d->nnz + 7) / 8 > 0 ? (d->nnz + 7) / 8 : 1;
    const dim3 g2(gx < 1024 ? gx : 1024, grid);
    if (Q.is_f64) packed_csparse_kernel<double><<<g2, 256, 0, stream>>>(Q); else packed_csparse_kernel<float><<<g2, 256, 0, stream>>>(Q);
  } else {
    const dim3 g2(1, grid);
    if (Q.is_f64) packed_sp_kernel<double><<<g2, 256, 0, stream>>>(Q); else packed_sp_kernel<float><<<g2, 256, 0, stream>>>(Q);
  }
  return check_launch("packed_sp");
}

extern "C" int xb_bcsc_tc_launch(const xb_sparse_desc* d, void** work, const void* a, const void* b_vals, const unsigned int* colptr,
                                 const unsigned int* rowidx, unsigned long long n_blocks, unsigned int nnzb, void* c);

extern "C" int xb_bcsc_launch(xb_sparse_desc* d, const void* a, const void* b_vals, const unsigned int* colptr,
                              const unsigned int* rowidx, unsigned long long n_blocks, unsigned int nnzb, void* c)
{
  if (d->m > 0 && n_blocks > 0) {   // tensor-core kernel for the bf16 VNNI case; everything else: exact-order kernel below
    const int rc = xb_bcsc_tc_launch(d, &d->work, a, b_vals, colptr, rowidx, n_blocks, nnzb, c);
    if (rc >= 0) return rc;
  }
  BcscParams Q;
  Q.M = d->packed_width; Q.K = d->k; Q.bk = d->bk; Q.bn = d->bn; Q.ta = d->ta; Q.tb = d->tb; Q.tc = d->tc;
  Q.beta0 = d->beta0; Q.trans_a = (d->flags & LIBXSMM_GEMM_FLAG_TRANS_A) != 0; Q.vnni_a = (d->flags & LIBXSMM_GEMM_FLAG_VNNI_A) != 0;
  Q.vnni_b_t = ((d->flags & LIBXSMM_GEMM_FLAG_VNNI_B) != 0) && ((d->flags & LIBXSMM_GEMM_FLAG_TRANS_B) != 0);
  Q.N = (long long)n_blocks * d->bn; Q.m_blocks = d->m;
  Q.a = (const char*)a; Q.bvals = (const char*)b_vals; Q.colptr = colptr; Q.rowidx = rowidx; Q.c = (char*)c;
  if (Q.m_blocks <= 0 || n_blocks == 0) return 0;
  const long long work = Q.m_blocks * (long long)n_blocks;
  const unsigned int grid = (unsigned int)(work < (1 << 20) ? work : (1 << 20));
  cudaStream_t stream = (cudaStream_t)xb_rt_stream();
  if (d->calls.count > 1) {
    const dim3 g2(grid, (unsigned int)(d->calls.count < 65535 ? d->calls.count : 65535));
    bcsc_simt_kernel<true><<<g2, 256, 0, stream>>>(Q, d->calls);
  } else {
    bcsc_simt_kernel<false><<<grid, 256, 0, stream>>>(Q, d->calls);
  }
  return check_launch("bcsc_simt", LIBXSMM_B200_BACKEND_SIMT);
}
