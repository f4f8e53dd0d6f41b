// libxsmm_b200 -- batched small-tile GEMM/BRGEMM on the Hopper tensor cores (sm_90a, wgmma.mma_async).
//
//   C_t(m x n) = beta * C_t + sum_{r < br} A_{t,r}(m x k) * B_{t,r}(k x n)      for t < count tiles
//
// Replaces the reference's per-ISA GEMM micro-kernels (src/generator_gemm_amx*.c,
// src/generator_gemm_avx512_microkernel.c) for the 16-bit floating-point and 8-bit integer dense paths; semantics are those
// of libxsmm_ref_matmul (src/generator_gemm_reference_impl.c:2025-2170, 2367-2419, 1452-1683) with f32 accumulation in
// registers instead of a sequential scalar loop (tolerance, not bit-exact); integer sums are exact in any order, so the
// 8-bit path is bit-identical to the reference.
//
// One kernel, `gemm_wg_kernel<AMODE, NC, NCH, WG, GRID>`, persistent, tiles assigned round-robin over the CTAs:
//   warps 0 .. 4*WG-1   WG consumer warpgroups; warpgroup g owns rows 64g .. 64g+63 of the tile (m <= 64: one warpgroup;
//                       pooled pair mode: warpgroup g owns the item's tile g) and issues wgmma m64 x (NC*NCH) x k16/k32
//   warp 4*WG           TMA producer: cp.async.bulk.tensor.4d of the A and B boxes of one (tile, r, k-chunk) per stage,
//                       ring of `stages` stages guarded by full/empty mbarriers
// A operand forms (AMODE):
//   XB_WG_SS16  A[k*lda+m] is M-contiguous: the box lands in the SWIZZLE_128B MN-major layout and wgmma reads it through a
//               descriptor with the transpose bit set (bf16 / f16)
//   XB_WG_RS16, XB_WG_RS8  VNNI-packed A (the reference's canonical low-precision layouts, A[(k/v)*lda*v + m*v + k%v], v = 2
//               for 16-bit, 4 for 8-bit): one 32-bit word holds v consecutive k of one row, which is exactly one register of
//               a wgmma A fragment, so the words go from the raw TMA stage straight into registers
// B[n*ldb+k] is K-contiguous: the K-major operand, SWIZZLE_128B boxes of 128 bytes of k x (NC*NCH) rows, rows beyond n and
// k beyond the matrix are zero-filled by TMA. A stage is released (empty barrier) once the wgmma group that read it retired.
// The code keeps one group in flight while the next stage is issued, but ptxas serializes the wgmma of every instantiation
// (C7520: the run-time bf16/f16 and int8-signedness selection around each instruction), so in the binary a stage's MMAs finish
// before the next are issued. Several CTAs share an SM, so one CTA's MMAs and epilogue (direct stores of the accumulator
// fragments, xb_epilogue.cuh) overlap the others' loads; the HBM-bound shapes are limited by the loads, not by that.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "xb_internal.h"
#include "xb_device.cuh"
#include "xb_tma.cuh"
#include "xb_wgmma.cuh"
#include "xb_epilogue.cuh"

namespace {

enum { XB_WG_SS16 = 0, XB_WG_RS16 = 1, XB_WG_RS8 = 2 };

struct WgParams {
  int m, n, k;
  int kchunks, kc_elems, kinst;       // k per stage (64 for 16-bit, 128 for 8-bit), k per instruction (16 or 32)
  int stages, stage_bytes, a_bytes, tx_bytes;
  int bf16;                           // 16-bit forms: bf16 (1) or f16 (0)
  int sgn;                            // 8-bit form: bit 1 A signed, bit 0 B signed
  unsigned long long br;
  long long count;                    // items the CTAs walk (tiles; pooled pair mode: pairs of tiles)
  char* c; long long tile_stride_c, ldc;
  int ep_mode, c_esz, beta0;
  float scf;
  // pooled address mode (libxsmm_b200_gemm_plan over ADDRESS/OFFSET batch-reduce): item p reads block-set sets[p].x of A (pair
  // mode: sets[p].y for its second tile) and sets[p].z of B (4th tensor-map coordinate) and writes cptrs[p] (pair mode:
  // cptrs[2p], cptrs[2p+1], the second may be null)
  // grid (libxsmm_b200_gemm_batch_grid, the GRID instantiations, which are never pooled): tile t is (i, j) = (t % grid_m, t / grid_m),
  // reads row block i of A and column block j of B (4th tensor-map coordinates) and writes c + i * tile_stride_c + j * tile_stride_c_n.
  // The two share storage, so that the flat and pooled instantiations see the struct they always had and compile to the same code.
  union {
    struct { const int4* sets; char* const* cptrs; int pair; };
    struct { long long grid_m, tile_stride_c_n; };
  };
};

template <int NC>
__device__ __forceinline__ void wg_mma16(int bf16, float (&d)[NC / 2], uint64_t a, uint64_t b, int scale_d) {
  if (NC == 16) { if (bf16) xb_wgmma_ss_bf16_n16<1>(*reinterpret_cast<float(*)[8]>(&d), a, b, scale_d); else xb_wgmma_ss_f16_n16<1>(*reinterpret_cast<float(*)[8]>(&d), a, b, scale_d); }
  if (NC == 32) { if (bf16) xb_wgmma_ss_bf16_n32<1>(*reinterpret_cast<float(*)[16]>(&d), a, b, scale_d); else xb_wgmma_ss_f16_n32<1>(*reinterpret_cast<float(*)[16]>(&d), a, b, scale_d); }
  if (NC == 64) { if (bf16) xb_wgmma_ss_bf16_n64<1>(*reinterpret_cast<float(*)[32]>(&d), a, b, scale_d); else xb_wgmma_ss_f16_n64<1>(*reinterpret_cast<float(*)[32]>(&d), a, b, scale_d); }
}
template <int NC>
__device__ __forceinline__ void wg_mma16_rs(int bf16, float (&d)[NC / 2], const uint32_t (&a)[4], uint64_t b, int scale_d) {
  if (NC == 16) { if (bf16) xb_wgmma_rs_bf16_n16(*reinterpret_cast<float(*)[8]>(&d), a, b, scale_d); else xb_wgmma_rs_f16_n16(*reinterpret_cast<float(*)[8]>(&d), a, b, scale_d); }
  if (NC == 32) { if (bf16) xb_wgmma_rs_bf16_n32(*reinterpret_cast<float(*)[16]>(&d), a, b, scale_d); else xb_wgmma_rs_f16_n32(*reinterpret_cast<float(*)[16]>(&d), a, b, scale_d); }
  if (NC == 64) { if (bf16) xb_wgmma_rs_bf16_n64(*reinterpret_cast<float(*)[32]>(&d), a, b, scale_d); else xb_wgmma_rs_f16_n64(*reinterpret_cast<float(*)[32]>(&d), a, b, scale_d); }
}
#define XB_WG_I8(N) \
  switch (sgn) { case 0: xb_wgmma_rs_u8u8_n##N(*reinterpret_cast<int(*)[N / 2]>(&d), a, b, scale_d); break; \
                 case 1: xb_wgmma_rs_u8s8_n##N(*reinterpret_cast<int(*)[N / 2]>(&d), a, b, scale_d); break; \
                 case 2: xb_wgmma_rs_s8u8_n##N(*reinterpret_cast<int(*)[N / 2]>(&d), a, b, scale_d); break; \
                 default: xb_wgmma_rs_s8s8_n##N(*reinterpret_cast<int(*)[N / 2]>(&d), a, b, scale_d); break; }
template <int NC>
__device__ __forceinline__ void wg_mma8_rs(int sgn, float (&d)[NC / 2], const uint32_t (&a)[4], uint64_t b, int scale_d) {
  if (NC == 16) { XB_WG_I8(16) }
  if (NC == 32) { XB_WG_I8(32) }
  if (NC == 64) { XB_WG_I8(64) }
}
#undef XB_WG_I8

// NC: columns per instruction, NCH: instructions side by side (N = NC * NCH), WG: consumer warpgroups, GRID: a grid launch (the flat
// and pooled instantiations carry no grid arithmetic)
template <int AMODE, int NC, int NCH, int WG, bool GRID>
__global__ void __launch_bounds__(WG * 128 + 32, (NCH == 1 && WG == 1) ? 3 : 1)
gemm_wg_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const WgParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t smem_base = xb_smem_u32(smem);
  const int S = P.stages;
  const uint32_t full0 = xb_smem_u32(smem + (size_t)S * P.stage_bytes), empty0 = full0 + 8 * S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long G = gridDim.x, b = blockIdx.x;
  const long long n_local = (b < P.count) ? (P.count - b + G - 1) / G : 0;
  const bool pooled = !GRID && P.sets != nullptr;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" :: "l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" :: "l"(&map_b) : "memory");
    for (int i = 0; i < S; ++i) { xb_mbar_init(full0 + 8 * i, 1); xb_mbar_init(empty0 + 8 * i, 4 * WG); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 4 * WG) {
    // ===================================== TMA producer =====================================
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (long long i = 0; i < n_local; ++i) {
        const long long t = b + i * G;
        int ta0 = (int)t, ta1 = (int)t, tb = (int)t, m1 = 64;            // warpgroup 1: rows 64.. of the same tile
        if (pooled) {
          const int4 st = P.sets[t];
          ta0 = st.x; ta1 = P.pair ? st.y : st.x; tb = st.z; m1 = P.pair ? 0 : 64;
        } else if (GRID) {
          ta0 = ta1 = (int)t % (int)P.grid_m; tb = (int)t / (int)P.grid_m;
        }
        for (unsigned long long r = 0; r < P.br; ++r) {
          for (int kc = 0; kc < P.kchunks; ++kc) {
            xb_mbar_wait(empty0 + 8 * stage, phase ^ 1);
            const uint32_t full = full0 + 8 * stage, sa = smem_base + stage * P.stage_bytes, sb = sa + P.a_bytes;
            xb_mbar_expect_tx(full, (uint32_t)P.tx_bytes);
            if (AMODE == XB_WG_SS16) {
              xb_tma_load_4d(sa, &map_a, full, 0, kc * 64, (int)r, ta0);
              if (WG == 2) xb_tma_load_4d(sa + 8192, &map_a, full, m1, kc * 64, (int)r, ta1);
            } else {
              xb_tma_load_4d(sa, &map_a, full, 0, kc * 32, (int)r, ta0);       // m words x 32 word-rows
            }
            xb_tma_load_4d(sb, &map_b, full, kc * P.kc_elems, 0, (int)r, tb);
            if (++stage == S) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===================================== consumer warpgroups =====================================
  const int g = warp >> 2, wq = warp & 3;
  const int row_a = 64 * g + 16 * wq + (lane >> 2), q = lane & 3;      // RS forms: fragment rows row_a, row_a + 8 of the tile
  const int loads = (int)P.br * P.kchunks;
  float acc[NCH][NC / 2];
  int stage = 0; uint32_t phase = 0;
  for (long long i = 0; i < n_local; ++i) {
    const long long t = b + i * G;
    int kc = 0, prev = -1;
    for (int l = 0; l < loads; ++l) {
      xb_mbar_wait(full0 + 8 * stage, phase);
      const uint32_t sa = smem_base + stage * P.stage_bytes, sb = sa + P.a_bytes;
      const int krem = P.k - kc * P.kc_elems;
      const int ksteps = (krem >= P.kc_elems) ? P.kc_elems / P.kinst : (krem + P.kinst - 1) / P.kinst;
      xb_wgmma_fence();
      for (int ks = 0; ks < ksteps; ++ks) {
        const int scale_d = (l > 0 || ks > 0) ? 1 : 0;
        if (AMODE == XB_WG_SS16) {
          // A: MN-major SWIZZLE_128B, 128-byte rows of 64 m per k, 8-row atoms 1024 bytes apart, 16 k = 2048 bytes per step
          const uint64_t ad = xb_wg_desc(sa + 8192u * g + 2048u * ks, 8192, 1024, 1);
#pragma unroll
          for (int c = 0; c < NCH; ++c) wg_mma16<NC>(P.bf16, acc[c], ad, xb_wg_desc(sb + (uint32_t)(c * NC * 128) + 32u * ks, 16, 1024, 1), scale_d);
        } else {
          // raw stage: [32 word-rows][m words]; register j of the fragment is word-row 8*ks + q + 4*(j >> 1), row row_a + 8*(j & 1)
          const uint32_t* w = reinterpret_cast<const uint32_t*>(smem + (size_t)stage * P.stage_bytes);
          uint32_t a[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int rr = row_a + 8 * (j & 1), kw = 8 * ks + q + 4 * (j >> 1);
            a[j] = (rr < P.m) ? w[kw * P.m + rr] : 0u;
          }
#pragma unroll
          for (int c = 0; c < NCH; ++c) {
            const uint64_t bd = xb_wg_desc(sb + (uint32_t)(c * NC * 128) + 32u * ks, 16, 1024, 1);
            if (AMODE == XB_WG_RS16) wg_mma16_rs<NC>(P.bf16, acc[c], a, bd, scale_d);
            else wg_mma8_rs<NC>(P.sgn, acc[c], a, bd, scale_d);
          }
        }
      }
      xb_wgmma_commit();
      xb_wgmma_wait<1>();                      // the previous stage's group retired: hand that stage back to the producer
      if (prev >= 0) { __syncwarp(); if (lane == 0) xb_mbar_arrive(empty0 + 8 * prev); }
      prev = stage;
      if (++kc == P.kchunks) kc = 0;
      if (++stage == S) { stage = 0; phase ^= 1; }
    }
    xb_wgmma_wait<0>();
    if (prev >= 0) { __syncwarp(); if (lane == 0) xb_mbar_arrive(empty0 + 8 * prev); }
    // epilogue
    char* ctile; int row0 = 64 * g;
    if (GRID) ctile = P.c + ((int)t % (int)P.grid_m) * P.tile_stride_c + ((int)t / (int)P.grid_m) * P.tile_stride_c_n;
    else if (!pooled) ctile = P.c + t * P.tile_stride_c;
    else if (P.pair) { ctile = P.cptrs[2 * t + g]; row0 = 0; }
    else ctile = P.cptrs[t];
    if (ctile == nullptr) continue;
    // ctile - row0 rows: the fragment store adds 64g + 16*warp + ...; in pair mode warpgroup g's rows start at row 0 of its tile
    char* cbase = ctile - (long long)(64 * g - row0) * P.c_esz;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      if (c * NC >= P.n) break;
      xb_ep_store_frag<NC / 2>(P.ep_mode, P.beta0, *reinterpret_cast<const uint32_t(*)[NC / 2]>(&acc[c]), cbase, 64 * g, c * NC,
                               P.m + (64 * g - row0), P.n, P.ldc * P.c_esz, P.c_esz, P.scf);
    }
  }
}

int g_num_sms = 0;

int env_int(const char* name, int fallback) {
  const char* e = getenv(name);
  return (e != nullptr && *e != 0) ? atoi(e) : fallback;
}

int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0; cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

// MaxDynamicSharedMemorySize is a per-device function attribute: one bit per (instantiation, device)
template <int AMODE, int NC, int NCH, int WG, bool GRID>
cudaError_t launch_one(long long grid, size_t smem, cudaStream_t stream, const CUtensorMap& ma, const CUtensorMap& mb, const WgParams& P) {
  static unsigned long long done = 0ull;
  if (xb_rt_first_use_on_device(&done)) cudaFuncSetAttribute(gemm_wg_kernel<AMODE, NC, NCH, WG, GRID>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  gemm_wg_kernel<AMODE, NC, NCH, WG, GRID><<<(unsigned int)grid, WG * 128 + 32, smem, stream>>>(ma, mb, P);
  return cudaGetLastError();
}

template <int AMODE, int WG, bool GRID>
cudaError_t launch_n(int nt, long long grid, size_t smem, cudaStream_t stream, const CUtensorMap& ma, const CUtensorMap& mb, const WgParams& P) {
  switch (nt) {
    case 16:  return launch_one<AMODE, 16, 1, WG, GRID>(grid, smem, stream, ma, mb, P);
    case 32:  return launch_one<AMODE, 32, 1, WG, GRID>(grid, smem, stream, ma, mb, P);
    case 64:  return launch_one<AMODE, 64, 1, WG, GRID>(grid, smem, stream, ma, mb, P);
    case 128: return launch_one<AMODE, 64, 2, WG, GRID>(grid, smem, stream, ma, mb, P);
    default:  return launch_one<AMODE, 64, 4, WG, GRID>(grid, smem, stream, ma, mb, P);
  }
}

template <int AMODE>
cudaError_t launch_a(int wg, int nt, bool is_grid, long long grid, size_t smem, cudaStream_t stream, const CUtensorMap& ma, const CUtensorMap& mb,
                     const WgParams& P) {
  if (is_grid) return (wg == 2) ? launch_n<AMODE, 2, true>(nt, grid, smem, stream, ma, mb, P) : launch_n<AMODE, 1, true>(nt, grid, smem, stream, ma, mb, P);
  return (wg == 2) ? launch_n<AMODE, 2, false>(nt, grid, smem, stream, ma, mb, P) : launch_n<AMODE, 1, false>(nt, grid, smem, stream, ma, mb, P);
}

// columns of the instruction: n rounded up to 16, 32, 64, 128 or 256
int n_tile(int n) { return n <= 16 ? 16 : (n <= 32 ? 32 : (n <= 64 ? 64 : (n <= 128 ? 128 : 256))); }

// ring size and co-resident CTAs: several CTAs per SM hide each other's epilogues; the ring takes what shared memory is left
void plan_stages(WgParams& P, int nt, int wg, int* ctas) {
  int c = (nt == 64 && wg == 1) || nt < 64 ? 3 : 1;
  while (c > 1 && 2 * P.stage_bytes + 2048 > (227 * 1024) / c) --c;
  int st = ((227 * 1024) / c - 2048) / P.stage_bytes; if (st > 8) st = 8; if (st < 2) st = 2;
  P.stages = st; *ctas = c;
}

int wg_launch(int amode, int wg, int nt, bool is_grid, const WgParams& P, int ctas, const CUtensorMap& ma, const CUtensorMap& mb,
              const char* where) {
  const size_t smem = (size_t)P.stages * P.stage_bytes + 1024 /*align slack*/ + 2 * 8 * P.stages;
  long long grid = P.count; if (grid > (long long)num_sms() * ctas) grid = (long long)num_sms() * ctas; if (grid < 1) grid = 1;
  cudaStream_t stream = (cudaStream_t)xb_rt_stream();
  cudaError_t e;
  if (amode == XB_WG_SS16) e = launch_a<XB_WG_SS16>(wg, nt, is_grid, grid, smem, stream, ma, mb, P);
  else if (amode == XB_WG_RS16) e = launch_a<XB_WG_RS16>(wg, nt, is_grid, grid, smem, stream, ma, mb, P);
  else e = launch_a<XB_WG_RS8>(wg, nt, is_grid, grid, smem, stream, ma, mb, P);
  xb_rt_count_launch_backend(LIBXSMM_B200_BACKEND_TCGEN05);
  if (e != cudaSuccess) { xb_rt_note_error((int)e, where); return (int)e; }
  return 0;
}

// the extents of the 4th tensor-map dimension of A and of B (a flat batch: count each; a grid: grid_m row blocks of A and grid_n
// column blocks of B), and whether TMA can walk them: 16-byte aligned bases and strides, and a nonzero stride wherever the extent is
// above 1. A launch that fails this runs on the exact-order kernel.
bool tile_maps_ok(const xb_gemm_launch* L, const char* a, const char* b, long long sa, long long sb, long long* na, long long* nb) {
  *na = (L->grid_m > 0) ? L->grid_m : L->count;
  *nb = (L->grid_m > 0) ? L->count / L->grid_m : L->count;
  return (((uintptr_t)a | (uintptr_t)b) & 15) == 0 && (sa % 16) == 0 && (sb % 16) == 0 && (*na == 1 || sa > 0) && (*nb == 1 || sb > 0);
}

}  // namespace

extern "C" int xb_gemm_tc_supported(const xb_gemm_desc* d);
extern "C" int xb_gemm_tc_shape_ok(const xb_gemm_desc* d) {
  xb_gemm_desc t = *d;
  t.br_type = 0;
  return xb_gemm_tc_supported(&t);
}

extern "C" int xb_gemm_tc_supported(const xb_gemm_desc* d) {
  const unsigned int bad = LIBXSMM_GEMM_FLAG_TRANS_A | LIBXSMM_GEMM_FLAG_TRANS_B | LIBXSMM_GEMM_FLAG_VNNI_A
                         | LIBXSMM_GEMM_FLAG_VNNI_B | LIBXSMM_GEMM_FLAG_VNNI_C | LIBXSMM_GEMM_FLAG_DECOMPRESS_A_VIA_BITMASK;
  if ((d->flags & bad) != 0) return 0;
  if (!(d->ta == d->tb && (d->ta == LIBXSMM_DATATYPE_BF16 || d->ta == LIBXSMM_DATATYPE_F16))) return 0;
  if (d->tcomp != LIBXSMM_DATATYPE_F32) return 0;
  if (d->ta == LIBXSMM_DATATYPE_BF16 && !(d->tc == LIBXSMM_DATATYPE_F32 || d->tc == LIBXSMM_DATATYPE_BF16)) return 0;
  if (d->ta == LIBXSMM_DATATYPE_F16 && !(d->tc == LIBXSMM_DATATYPE_F32 || d->tc == LIBXSMM_DATATYPE_F16)) return 0;
  if (d->m < 16 || d->n < 16 || d->k < 16 || d->m > 128 || d->n > 256 || d->k > 4096) return 0;
  if ((d->lda % 8) != 0 || (d->ldb % 8) != 0) return 0;                 // TMA: 16-byte global strides
  if (!(d->br_type == 0 || d->br_type == 3)) return 0;                  // address/offset modes: SIMT kernel
  if (d->br_type == 3 && ((d->br_stride_a % 16) != 0 || (d->br_stride_b % 16) != 0 || d->br_stride_a <= 0 || d->br_stride_b <= 0)) return 0;
  return 1;
}

static int tc_launch_common(const xb_gemm_launch* L, const xb_tc_pool* pool);
extern "C" int xb_gemm_tc_launch(const xb_gemm_launch* L) { return tc_launch_common(L, nullptr); }
extern "C" int xb_gemm_tc_launch_pooled(const xb_gemm_desc* d, const xb_tc_pool* pool, unsigned long long br, long long count) {
  xb_gemm_launch L; memset(&L, 0, sizeof(L));
  L.d = *d; L.count = count; L.br = br;
  L.a = pool->base_a; L.b = pool->base_b; L.c = (void*)pool->cptrs;        // non-null markers; the pool carries the real addressing
  L.tile_stride_a = pool->set_a; L.tile_stride_b = pool->set_b; L.tile_stride_c = 16;
  return tc_launch_common(&L, pool);
}

static int tc_launch_common(const xb_gemm_launch* L, const xb_tc_pool* pool) {
  const xb_gemm_desc& d = L->d;
  // resolve the uniform strided form (count==1 by-value record included)
  const char* a = (const char*)L->a; const char* b = (const char*)L->b; char* c = (char*)L->c;
  long long sa = L->tile_stride_a, sb = L->tile_stride_b, sc = L->tile_stride_c;
  unsigned long long br = L->br;
  if (L->recs != nullptr) return xb_gemm_simt_launch(L);
  if (a == nullptr && c == nullptr) { a = (const char*)L->one.a; b = (const char*)L->one.b; c = (char*)L->one.c; br = L->one.br; sa = sb = sc = 0; }
  if (d.br_type == 0 && pool == nullptr) br = 1;
  const int es = 2;
  long long na, nb;
  const bool aligned = tile_maps_ok(L, a, b, sa, sb, &na, &nb);
  xb_encode_tiled_fn enc = xb_tma_encoder();
  if (br == 0 || !aligned || L->count <= 0 || br > 0x7fffffffull || L->count > 0x7fffffffll || enc == nullptr) {
    return (pool != nullptr) ? 1 : xb_gemm_simt_launch(L);
  }

  const int wg = (d.m <= 64 && !(pool != nullptr && pool->pair)) ? 1 : 2;
  const int nt = n_tile(d.n);
  WgParams P; memset(&P, 0, sizeof(P));
  P.m = d.m; P.n = d.n; P.k = d.k;
  P.kc_elems = 64; P.kinst = 16; P.kchunks = (d.k + 63) / 64;
  P.a_bytes = wg * 8192; P.stage_bytes = P.a_bytes + nt * 128; P.tx_bytes = P.stage_bytes;
  P.bf16 = (d.ta == LIBXSMM_DATATYPE_BF16) ? 1 : 0;
  P.br = br; P.count = L->count; P.c = c; P.tile_stride_c = sc; P.ldc = d.ldc;
  if (L->grid_m > 0) { P.grid_m = L->grid_m; P.tile_stride_c_n = L->tile_stride_c_n; }
  if (pool != nullptr) { P.sets = (const int4*)pool->sets; P.cptrs = (char* const*)pool->cptrs; P.pair = pool->pair; }
  P.beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) ? 1 : 0;
  P.ep_mode = xb_ep_mode(d.ta, d.tc, &P.c_esz);
  int ctas = 1;
  plan_stages(P, nt, wg, &ctas);

  const CUtensorMapDataType dt = P.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const size_t ext_a = ((size_t)(d.k - 1) * d.lda + d.m) * es, ext_b = ((size_t)(d.n - 1) * d.ldb + d.k) * es;
  const cuuint64_t pad_a = (ext_a + 15) & ~(size_t)15, pad_b = (ext_b + 15) & ~(size_t)15;
  CUtensorMap map_a, map_b;
  {
    const cuuint64_t dims[4] = {(cuuint64_t)d.m, (cuuint64_t)d.k, (cuuint64_t)br, (cuuint64_t)(pool ? pool->nsets_a : na)};
    const cuuint64_t strides[3] = {(cuuint64_t)d.lda * es, pool ? (cuuint64_t)pool->blk_a : ((d.br_type == 3) ? (cuuint64_t)d.br_stride_a : pad_a),
                                   pool ? (cuuint64_t)pool->set_a : ((na > 1) ? (cuuint64_t)sa : pad_a)};
    const cuuint32_t box[4] = {64, 64, 1, 1};
    if (CUDA_SUCCESS != enc(&map_a, dt, 4, (void*)a, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE))
      return (pool != nullptr) ? 1 : xb_gemm_simt_launch(L);
  }
  {
    const cuuint64_t dims[4] = {(cuuint64_t)d.k, (cuuint64_t)d.n, (cuuint64_t)br, (cuuint64_t)(pool ? pool->nsets_b : nb)};
    const cuuint64_t strides[3] = {(cuuint64_t)d.ldb * es, pool ? (cuuint64_t)pool->blk_b : ((d.br_type == 3) ? (cuuint64_t)d.br_stride_b : pad_b),
                                   pool ? (cuuint64_t)pool->set_b : ((nb > 1) ? (cuuint64_t)sb : pad_b)};
    const cuuint32_t box[4] = {64, (cuuint32_t)nt, 1, 1};
    if (CUDA_SUCCESS != enc(&map_b, dt, 4, (void*)b, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE))
      return (pool != nullptr) ? 1 : xb_gemm_simt_launch(L);
  }
  return wg_launch(XB_WG_SS16, wg, nt, L->grid_m > 0, P, ctas, map_a, map_b, "gemm_tc");
}

// ---- VNNI-packed A (register-fragment form) ----------------------------------------------------------------------------
extern "C" int xb_gemm_ts_supported(const xb_gemm_desc* d) {
  const unsigned int bad = LIBXSMM_GEMM_FLAG_TRANS_A | LIBXSMM_GEMM_FLAG_TRANS_B | LIBXSMM_GEMM_FLAG_VNNI_B | LIBXSMM_GEMM_FLAG_VNNI_C
                         | LIBXSMM_GEMM_FLAG_DECOMPRESS_A_VIA_BITMASK | LIBXSMM_GEMM_FLAG_INTLV_A_FORMAT;
  const int a8 = (d->ta == LIBXSMM_DATATYPE_I8 || d->ta == LIBXSMM_DATATYPE_U8), b8 = (d->tb == LIBXSMM_DATATYPE_I8 || d->tb == LIBXSMM_DATATYPE_U8);
  static int enabled = -1;
  if (enabled < 0) enabled = env_int("LIBXSMM_B200_TS", 1) != 0 ? 1 : 0;
  if (!enabled || (d->flags & bad) != 0 || d->fuse_colbias != 0 || d->cp_op != 0) return 0;
  if (a8 && b8) {
    if (d->tcomp != LIBXSMM_DATATYPE_I32 || !(d->tc == LIBXSMM_DATATYPE_I32 || d->tc == LIBXSMM_DATATYPE_F32)) return 0;
    if ((d->flags & LIBXSMM_GEMM_FLAG_VNNI_A) == 0 && d->tc != LIBXSMM_DATATYPE_F32) return 0;   // flat int8 A: exact-order kernel (the F32-out path is always VNNI4)
    if ((d->k % 4) != 0 || (d->ldb % 16) != 0) return 0;
  } else if (d->ta == d->tb && (d->ta == LIBXSMM_DATATYPE_BF16 || d->ta == LIBXSMM_DATATYPE_F16)) {
    if ((d->flags & LIBXSMM_GEMM_FLAG_VNNI_A) == 0 || d->tcomp != LIBXSMM_DATATYPE_F32) return 0;
    if (d->ta == LIBXSMM_DATATYPE_BF16 && !(d->tc == LIBXSMM_DATATYPE_F32 || d->tc == LIBXSMM_DATATYPE_BF16)) return 0;
    if (d->ta == LIBXSMM_DATATYPE_F16 && !(d->tc == LIBXSMM_DATATYPE_F32 || d->tc == LIBXSMM_DATATYPE_F16)) return 0;
    if ((d->k % 2) != 0 || (d->ldb % 8) != 0) return 0;
  } else return 0;
  if (d->m < 4 || d->m > 128 || (d->m % 4) != 0 || (d->lda % 4) != 0 || d->n < 1 || d->n > 128 || d->k > 8192) return 0;
  if (!(d->br_type == 0 || d->br_type == 3)) return 0;
  if (d->br_type == 3 && ((d->br_stride_a % 16) != 0 || (d->br_stride_b % 16) != 0 || d->br_stride_a <= 0 || d->br_stride_b <= 0)) return 0;
  return 1;
}

extern "C" int xb_gemm_ts_launch(const xb_gemm_launch* L) {
  const xb_gemm_desc& d = L->d;
  const char* a = (const char*)L->a; const char* b = (const char*)L->b; char* c = (char*)L->c;
  long long sa = L->tile_stride_a, sb = L->tile_stride_b, sc = L->tile_stride_c;
  unsigned long long br = L->br;
  if (L->recs != nullptr) return xb_gemm_simt_launch(L);
  if (a == nullptr && c == nullptr) { a = (const char*)L->one.a; b = (const char*)L->one.b; c = (char*)L->one.c; br = L->one.br; sa = sb = sc = 0; }
  if (d.br_type == 0) br = 1;
  long long na, nb;
  const bool aligned = tile_maps_ok(L, a, b, sa, sb, &na, &nb);
  xb_encode_tiled_fn enc = xb_tma_encoder();
  if (br == 0 || !aligned || L->count <= 0 || br > 0x7fffffffull || L->count > 0x7fffffffll || enc == nullptr) return xb_gemm_simt_launch(L);

  const int is_i8 = (d.ta == LIBXSMM_DATATYPE_I8 || d.ta == LIBXSMM_DATATYPE_U8);
  const int v = is_i8 ? 4 : 2, es = is_i8 ? 1 : 2;
  const int wg = (d.m <= 64) ? 1 : 2, nt = n_tile(d.n);
  WgParams P; memset(&P, 0, sizeof(P));
  P.m = d.m; P.n = d.n; P.k = d.k;
  P.kc_elems = 128 / es; P.kinst = is_i8 ? 32 : 16; P.kchunks = (d.k + P.kc_elems - 1) / P.kc_elems;
  P.a_bytes = (d.m * 128 + 1023) & ~1023;                        // m words x 32 word-rows; B starts 1024-byte aligned (SWIZZLE_128B atom)
  P.stage_bytes = P.a_bytes + nt * 128; P.tx_bytes = d.m * 128 + nt * 128;
  P.bf16 = (d.ta == LIBXSMM_DATATYPE_BF16) ? 1 : 0;
  P.sgn = ((d.ta == LIBXSMM_DATATYPE_I8) ? 2 : 0) | ((d.tb == LIBXSMM_DATATYPE_I8) ? 1 : 0);
  P.br = br; P.count = L->count; P.c = c; P.tile_stride_c = sc; P.ldc = d.ldc;
  if (L->grid_m > 0) { P.grid_m = L->grid_m; P.tile_stride_c_n = L->tile_stride_c_n; }
  P.beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) ? 1 : 0; P.scf = L->one.scf;
  P.ep_mode = xb_ep_mode(d.ta, d.tc, &P.c_esz);
  int ctas = 1;
  plan_stages(P, nt, wg, &ctas);

  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const size_t ext_a = ((size_t)(d.k / v - 1) * d.lda + d.m) * 4, ext_b = ((size_t)(d.n - 1) * d.ldb + d.k) * es;
  const cuuint64_t pad_a = (ext_a + 15) & ~(size_t)15, pad_b = (ext_b + 15) & ~(size_t)15;
  CUtensorMap map_a, map_b;
  {
    const cuuint64_t dims[4] = {(cuuint64_t)d.m, (cuuint64_t)(d.k / v), (cuuint64_t)br, (cuuint64_t)na};
    const cuuint64_t strides[3] = {(cuuint64_t)d.lda * 4, (d.br_type == 3) ? (cuuint64_t)d.br_stride_a : pad_a, (na > 1) ? (cuuint64_t)sa : pad_a};
    const cuuint32_t box[4] = {(cuuint32_t)d.m, 32, 1, 1};
    if (CUDA_SUCCESS != enc(&map_a, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4, (void*)a, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE)) return xb_gemm_simt_launch(L);
  }
  {
    const CUtensorMapDataType dt = is_i8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : (P.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
    const cuuint64_t dims[4] = {(cuuint64_t)d.k, (cuuint64_t)d.n, (cuuint64_t)br, (cuuint64_t)nb};
    const cuuint64_t strides[3] = {(cuuint64_t)d.ldb * es, (d.br_type == 3) ? (cuuint64_t)d.br_stride_b : pad_b, (nb > 1) ? (cuuint64_t)sb : pad_b};
    const cuuint32_t box[4] = {(cuuint32_t)P.kc_elems, (cuuint32_t)nt, 1, 1};
    if (CUDA_SUCCESS != enc(&map_b, dt, 4, (void*)b, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE)) return xb_gemm_simt_launch(L);
  }
  return wg_launch(is_i8 ? XB_WG_RS8 : XB_WG_RS16, wg, nt, L->grid_m > 0, P, ctas, map_a, map_b, "gemm_ts");
}
