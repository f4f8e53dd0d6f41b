// libxsmm_b200 -- packed block-sparse (BCSC) B x dense A on the Hopper tensor cores (sm_90a, wgmma.mma_async), bf16.
//
// For every m_block mb:  C_mb[N][M] = beta * C_mb + A_mb(M x K) * B(K x N),  B given as BCSC blocks [bn][bk].
// Replaces src/generator_packed_spgemm_bcsc_bsparse_avx_avx2_avx512_amx.c (AMX/AVX-512 per block);
// semantics are those of the driver's dense gold (samples/xgemm_sparse/spmm_kernel.c:74-217) with f32
// accumulation in registers (tolerance 5e-3 for bf16 like spmm_kernel.c:1019-1029).
//
// Mapping. The m_blocks are M rows each and stacked, so 64 consecutive rows of the stacked A form one wgmma M=64 operand
// ("group"). A work item is (group, block-column j); one warpgroup per CTA walks the items round-robin. For every non-zero
// block (kb, j) of the column:
//   D[:, 0 : bn] += A_grp[:, kb*bk : (kb+1)*bk] * B_blk^T          (bk/16 instructions m64 x bn x k16)
// A is VNNI2-packed (A[K/2][M][2]): a 32-bit word holds two consecutive k of one row, which is exactly one register of the
// wgmma A fragment, so A goes from global memory (L2-resident across the columns of a group) straight into registers.
// B blocks ([bn][bk], k contiguous: the K-major operand) are copied into the canonical no-swizzle shared-memory layout
// (8 x 16-byte core matrices), two buffers so that the copy of the next block overlaps the MMAs of the current one.
// The pattern (colptr, rowidx) and the values arrive with the call and are read directly: no preparation kernel.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "xb_internal.h"
#include "xb_device.cuh"
#include "xb_wgmma.cuh"
#include "xb_epilogue.cuh"

namespace {

struct BcscParams {
  int M, K, bk, bn, nbc;                  // packed width, depth, block shape, block-columns
  long long m_blocks, ngroups, items;     // items = ngroups * nbc
  const uint32_t* a;                      // VNNI2 words, m_block mb at a + mb * (K/2) * M
  const uint4* b_vals;                    // [nnzb][bn][bk] bf16
  const unsigned int* colptr; const unsigned int* rowidx;
  unsigned short* c; int beta0;
};


// element (n, k) of a block in shared memory: core matrix (n / 8, k / 8) at (n / 8) * sbo + (k / 8) * 128, row n % 8 at 16 bytes
__device__ __forceinline__ void stage_block(uint8_t* dst, const uint4* src, int bn, int bk) {
  const int kc = bk / 8, sbo = kc * 128, chunks = bn * kc;
  for (int i = threadIdx.x; i < chunks; i += blockDim.x) {
    const int n = i / kc, k8 = i - n * kc;
    *reinterpret_cast<uint4*>(dst + (n >> 3) * sbo + k8 * 128 + (n & 7) * 16) = src[i];
  }
}

template <int NC>
__device__ __forceinline__ void mma_rs(float (&d)[NC / 2], const uint32_t (&a)[4], uint64_t b, int scale_d) {
  if (NC == 16) xb_wgmma_rs_bf16_n16(*reinterpret_cast<float(*)[8]>(&d), a, b, scale_d);
  if (NC == 32) xb_wgmma_rs_bf16_n32(*reinterpret_cast<float(*)[16]>(&d), a, b, scale_d);
  if (NC == 64) xb_wgmma_rs_bf16_n64(*reinterpret_cast<float(*)[32]>(&d), a, b, scale_d);
}

// NC: columns per instruction, NCH: instructions side by side (NC * NCH >= bn)
template <int NC, int NCH>
__global__ void __launch_bounds__(128, (NCH >= 4) ? 2 : 4)
bcsc_wg_kernel(const BcscParams P) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int buf_bytes = NC * NCH * P.bk * 2;                 // the instructions read NC * NCH rows of a block
  uint8_t* sbuf[2] = {smem_raw, smem_raw + buf_bytes};
  const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5, q = lane & 3;
  const int sbo = (P.bk / 8) * 128, ksteps = P.bk / 16;
  const long long KW = P.K / 2;
  float acc[NCH][NC / 2];
  int buf = 0;
  for (long long item = blockIdx.x; item < P.items; item += gridDim.x) {
    const long long grp = item / P.nbc;
    const int j = (int)(item - grp * P.nbc);
    // fragment rows r0, r0 + 8 of the group: stacked row R = 64 grp + r is row R % M of m_block R / M
    const uint32_t* arow[2]; bool avalid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long R = grp * 64 + 16 * wq + (lane >> 2) + 8 * h, mb = R / P.M;
      avalid[h] = mb < P.m_blocks;
      arow[h] = P.a + (avalid[h] ? mb * KW * P.M + (R - mb * P.M) : 0);
    }
    const unsigned int z0 = P.colptr[j], z1 = P.colptr[j + 1];
    bool started = false;
    for (unsigned int z = z0; z < z1; ++z) {
      const unsigned int kb = P.rowidx[z];
      if (kb >= (unsigned int)(P.K / P.bk)) continue;     // block-row outside A: ignored (uniform over the CTA)
      // every warp has passed its wait_group after the MMAs that read this buffer two blocks ago (or the previous item's
      // wait_group 0): only then may any warp overwrite it
      __syncthreads();
      stage_block(sbuf[buf], P.b_vals + (size_t)z * (P.bn * P.bk / 8), P.bn, P.bk);
      xb_fence_proxy_async();
      __syncthreads();
      const long long kw0 = (long long)kb * (P.bk / 2);
      const uint32_t sb = xb_smem_u32(sbuf[buf]);
      xb_wgmma_fence();
      for (int ks = 0; ks < ksteps; ++ks) {
        uint32_t a[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) a[r] = avalid[r & 1] ? __ldg(arow[r & 1] + (kw0 + 8 * ks + q + 4 * (r >> 1)) * P.M) : 0u;
        const int scale_d = (started || ks > 0) ? 1 : 0;
#pragma unroll
        for (int c = 0; c < NCH; ++c)
          mma_rs<NC>(acc[c], a, xb_wg_desc(sb + (uint32_t)((c * NC / 8) * sbo + ks * 256), 128, (uint32_t)sbo, 0), scale_d);
      }
      xb_wgmma_commit();
      xb_wgmma_wait<1>();             // this thread's previous group (the other buffer) retired
      started = true;
      buf ^= 1;
    }
    xb_wgmma_wait<0>();
    if (!started) {
#pragma unroll
      for (int c = 0; c < NCH; ++c)
#pragma unroll
        for (int i = 0; i < NC / 2; ++i) acc[c][i] = 0.0f;
    }
    // C_mb[n][m]: the group's rows are not one column-major tile when M < 64, so every fragment row is resolved to its m_block
    const long long ncols = (long long)P.nbc * P.bn;
    const int r0 = 16 * wq + (lane >> 2), c0 = 2 * q;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
#pragma unroll
      for (int i = 0; i < NC / 2; ++i) {
        const int col = c * NC + c0 + 8 * (i >> 2) + (i & 1), h = (i >> 1) & 1;
        if (col >= P.bn || !avalid[h]) continue;
        const long long R = grp * 64 + r0 + 8 * h, mb = R / P.M;
        char* p = reinterpret_cast<char*>(P.c + (mb * ncols + (long long)j * P.bn + col) * P.M + (R - mb * P.M));
        if (P.beta0) xb_ep_store_one<XB_EP_BF16, true>(__float_as_uint(acc[c][i]), p, 0.0f);
        else xb_ep_store_one<XB_EP_BF16, false>(__float_as_uint(acc[c][i]), p, 0.0f);
      }
    }
  }
}

int device_sms() {
  static int sms[64] = {0};
  int dev = 0; cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 132;
  if (sms[dev] == 0) { int n = 0; cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); sms[dev] = (n > 0) ? n : 132; }
  return sms[dev];
}

// MaxDynamicSharedMemorySize is a per-device function attribute: set it once per (instantiation, device)
template <int NC, int NCH>
cudaError_t launch(long long grid, size_t smem, cudaStream_t stream, const BcscParams& P) {
  static unsigned long long done = 0ull;
  if (xb_rt_first_use_on_device(&done)) cudaFuncSetAttribute(bcsc_wg_kernel<NC, NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * NC * NCH * 64 * 2);
  bcsc_wg_kernel<NC, NCH><<<(unsigned int)grid, 128, smem, stream>>>(P);
  return cudaGetLastError();
}

}  // namespace

// the kernel keeps no per-handle state: pattern and values are read as they arrive with every call
extern "C" void xb_bcsc_state_free(void* work) { (void)work; }

// which kernel a call with this geometry takes: 0 none (caller falls back to the exact-order kernel), 1 the wgmma kernel
extern "C" int xb_bcsc_tc_variant(const xb_sparse_desc* d, unsigned long long n_blocks) {
  const unsigned int bad = LIBXSMM_GEMM_FLAG_TRANS_A | LIBXSMM_GEMM_FLAG_TRANS_B | LIBXSMM_GEMM_FLAG_VNNI_B;
  const int M = d->packed_width, K = d->k, bk = d->bk, bn = d->bn;
  if (getenv("LIBXSMM_B200_BCSC_SIMT") != nullptr) return 0;
  if (d->ta != LIBXSMM_DATATYPE_BF16 || d->tb != LIBXSMM_DATATYPE_BF16 || d->tc != LIBXSMM_DATATYPE_BF16) return 0;
  if ((d->flags & bad) != 0 || (d->flags & LIBXSMM_GEMM_FLAG_VNNI_A) == 0) return 0;
  if (!(M == 16 || M == 32 || M == 64 || M == 128)) return 0;
  if (!(bk == 16 || bk == 32 || bk == 64) || (bn % 16) != 0 || bn > 256 || bn < 16 || K < 64 || (K % bk) != 0) return 0;
  if (n_blocks == 0 || n_blocks > 0x7fffffffull) return 0;
  return 1;
}

// returns 0 if launched, <0 if this descriptor/problem is not served by the tensor-core kernel (caller falls back)
extern "C" int xb_bcsc_tc_launch(const xb_sparse_desc* d, void** work, const void* a, const void* b_vals, const unsigned int* colptr,
                                 const unsigned int* rowidx, unsigned long long n_blocks, unsigned int nnzb, void* c)
{
  (void)work; (void)nnzb;
  if (xb_bcsc_tc_variant(d, n_blocks) == 0) return -1;
  if ((((uintptr_t)a | (uintptr_t)b_vals | (uintptr_t)c) & 15) != 0) return -1;
  BcscParams P; memset(&P, 0, sizeof(P));
  P.M = d->packed_width; P.K = d->k; P.bk = d->bk; P.bn = d->bn; P.nbc = (int)n_blocks;
  P.m_blocks = d->m; P.ngroups = (d->m * (long long)P.M + 63) / 64; P.items = P.ngroups * P.nbc;
  P.a = (const uint32_t*)a; P.b_vals = (const uint4*)b_vals; P.colptr = colptr; P.rowidx = rowidx;
  P.c = (unsigned short*)c; P.beta0 = d->beta0;
  const int nt = P.bn <= 16 ? 16 : (P.bn <= 32 ? 32 : (P.bn <= 64 ? 64 : (P.bn <= 128 ? 128 : 256)));
  long long grid = P.items; const long long cap = (long long)device_sms() * 8; if (grid > cap) grid = cap; if (grid < 1) grid = 1;
  const size_t smem = 2 * (size_t)nt * P.bk * 2;
  cudaStream_t stream = (cudaStream_t)xb_rt_stream();
  cudaError_t e;
  switch (nt) {
    case 16:  e = launch<16, 1>(grid, smem, stream, P); break;
    case 32:  e = launch<32, 1>(grid, smem, stream, P); break;
    case 64:  e = launch<64, 1>(grid, smem, stream, P); break;
    case 128: e = launch<64, 2>(grid, smem, stream, P); break;
    default:  e = launch<64, 4>(grid, smem, stream, P); break;
  }
  xb_rt_count_launch_backend(LIBXSMM_B200_BACKEND_TCGEN05);
  if (e != cudaSuccess) { xb_rt_note_error((int)e, "bcsc_tc"); return (int)e; }
  return 0;
}
