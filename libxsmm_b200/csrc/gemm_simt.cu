// libxsmm_b200 -- exact-order dense GEMM/BRGEMM on CUDA cores (sm_90a).
//
// This is the "every datatype, every layout flag" kernel: one CTA per tile, one thread per C element,
// and for each element the SAME sequence of multiply/add operations the reference's C kernel performs
// (src/generator_gemm_reference_impl.c:821-2800, libxsmm_ref_matmul). Because the order and the
// rounding points are identical (separate multiply and add, no contraction), results are bit-identical
// to the reference for integer AND floating-point types. The tensor-core kernel (gemm_tc.cu) is the
// fast path for the shapes it supports; this kernel is what every other descriptor launches.
//
// Layout formulas (elements), from the reference (file above, lines cited per branch):
//   A flat    A[k*lda + m]            A trans   A[m*lda + k]
//   A VNNI-v  A[(k/v)*lda*v + m*v + k%v]   (v = 2 for 16-bit, 4 for 8-bit; x86 pack factors)
//   B flat    B[n*ldb + k]            B trans   B[k*ldb + n]       B VNNI-T  B[(k/v)*ldb*v + n*v + k%v]
//   C         C[n*ldc + m]
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdlib.h>
#include "xb_internal.h"
#include "xb_device.cuh"

namespace {

struct TileCtx {
  const char* a0; const char* b0; char* c;       // tile bases
  const void* const* a_addr; const void* const* b_addr;   // address mode
  const long long* a_offs; const long long* b_offs;       // offset mode
  unsigned long long br;
  float scf;
  const void* colbias; unsigned char* relu_mask;          // fused form (libxsmm_dispatch_brgemm_ext)
  const unsigned char* a_q;                                // int4: zero points; bitmap-compressed A: the bitmap
  const unsigned char* a_s; const unsigned char* b_s; unsigned char* c_s;   // scales of A, B and C (xb_gemm_sides)
};

// GRID: the instantiation that runs grids (libxsmm_b200_gemm_batch_grid); the others carry no grid arithmetic
template <bool GRID> __device__ inline void resolve_tile(const xb_gemm_launch& L, long long t, TileCtx& x) {
  const xb_gemm_rec r = xb_gemm_tile_at(&L, t, GRID ? L.grid_m : 0);
  x.a0 = (const char*)r.a; x.b0 = (const char*)r.b; x.c = (char*)r.c;
  x.a_addr = (const void* const*)r.a; x.b_addr = (const void* const*)r.b;
  x.a_offs = (const long long*)r.a_aux; x.b_offs = (const long long*)r.b_aux;
  x.br = (L.d.br_type == 0) ? 1ull : r.br; x.scf = r.scf;
  x.colbias = r.d; x.relu_mask = (unsigned char*)r.c_aux; x.a_q = (const unsigned char*)r.a_q;
  x.a_s = (const unsigned char*)r.a_s; x.b_s = (const unsigned char*)r.b_s; x.c_s = (unsigned char*)r.c_s;
}

// base pointers of the r-th batch-reduce operand pair; mirrors libxsmm_calculate_brgemm_offsets
// (generator_gemm_reference_impl.c:178-197): byte offsets/strides are truncated to whole elements.
__device__ inline void br_ptrs(const xb_gemm_desc& d, const TileCtx& x, unsigned long long r, int tsa, int tsb,
                               const char*& pa, const char*& pb) {
  switch (d.br_type) {
    case 1: pa = (const char*)x.a_addr[r]; pb = (const char*)x.b_addr[r]; break;
    case 2: pa = x.a0 + (x.a_offs[r] / tsa) * tsa; pb = x.b0 + (x.b_offs[r] / tsb) * tsb; break;
    case 3: pa = x.a0 + (long long)r * ((d.br_stride_a / tsa) * tsa); pb = x.b0 + (long long)r * ((d.br_stride_b / tsb) * tsb); break;
    default: pa = x.a0; pb = x.b0;
  }
}

template <typename T> __device__ inline T ldg_as(const char* base, long long idx) {
  return reinterpret_cast<const T*>(base)[idx];
}

// Loop invariants of the dot_* loops, read from the descriptor once at kernel entry. Derived from `d` inside the loops instead,
// they are reloaded and recomputed per element: the fused kernel then needs more registers and ran up to 1.9x slower (H100 SXM,
// 400 W power limit).
struct DotGeom {
  int k; long long lda, ldb;
  bool trans_a, trans_b, vnni_a, vnni_b, ua, ub;
};
__device__ __forceinline__ DotGeom dot_geom(const xb_gemm_desc& d) {
  DotGeom g;
  g.k = d.k; g.lda = d.lda; g.ldb = d.ldb;
  g.trans_a = (d.flags & LIBXSMM_GEMM_FLAG_TRANS_A) != 0; g.trans_b = (d.flags & LIBXSMM_GEMM_FLAG_TRANS_B) != 0;
  g.vnni_a = (d.flags & LIBXSMM_GEMM_FLAG_VNNI_A) != 0; g.vnni_b = (d.flags & LIBXSMM_GEMM_FLAG_VNNI_B) != 0;
  g.ua = (d.ta == LIBXSMM_DATATYPE_U8); g.ub = (d.tb == LIBXSMM_DATATYPE_U8);
  return g;
}

// ---- the reference's accumulation loops, shared by gemm_simt_kernel and gemm_fused_kernel --------------------------------
// Each returns `acc` after the batch-reduce and k loops of element (i, j), in the reference's order and rounding points; the
// seed, the scale, the epilogue and the store stay with the caller. `x` is the operand source: a TileCtx is the tile in global
// memory (every batch-reduce block, the k of `g`); a Staged source is one k-chunk of one block that gemm_fused_kernel copied into
// shared memory in the operand's own layout, described by the leading dimensions and the k of `g`.
struct Staged {
  const char* a; const char* b;
  static constexpr unsigned long long br = 1;
};
__device__ __forceinline__ void br_ptrs(const xb_gemm_desc&, const Staged& x, unsigned long long, int, int, const char*& pa, const char*& pb) {
  pa = x.a; pb = x.b;
}

template <class S> __device__ __forceinline__ float dot_f32(const xb_gemm_desc& d, const DotGeom& g, const S& x, int i, int j, float acc) {   // reference :1359-1426
  const int k = g.k;
  const long long lda = g.lda, ldb = g.ldb;
  const bool trans_a = g.trans_a, trans_b = g.trans_b;
  const bool cvt = (d.ta == LIBXSMM_DATATYPE_BF32);   // BF32: operands rounded to bf16 first
  for (unsigned long long r = 0; r < x.br; ++r) {
    const char *pa, *pb; br_ptrs(d, x, r, 4, 4, pa, pb);
    for (int s = 0; s < k; ++s) {
      float av = ldg_as<float>(pa, trans_a ? (i * lda + s) : (s * lda + i));
      float bv = ldg_as<float>(pb, trans_b ? (s * ldb + j) : (j * ldb + s));
      if (cvt) { av = xb_bf16_to_f32(xb_f32_to_bf16_rne(av)); bv = xb_bf16_to_f32(xb_f32_to_bf16_rne(bv)); }
      acc = __fadd_rn(acc, __fmul_rn(av, bv));
    }
  }
  return acc;
}

// reference :1452-1683 (four sign combinations); an f32 C always reads A as VNNI4
template <class S> __device__ __forceinline__ unsigned int dot_i8(const xb_gemm_desc& d, const DotGeom& g, const S& x, int i, int j, unsigned int acc) {
  const int k = g.k;
  const long long lda = g.lda, ldb = g.ldb;
  const bool ua = g.ua, ub = g.ub;
  const int kb = (d.tc == LIBXSMM_DATATYPE_F32 || g.vnni_a) ? 4 : 1;
  for (unsigned long long r = 0; r < x.br; ++r) {
    const char *pa, *pb; br_ptrs(d, x, r, 1, 1, pa, pb);
    for (int s = 0; s < k / kb; ++s) for (int k2 = 0; k2 < kb; ++k2) {
      const unsigned char ar = ldg_as<unsigned char>(pa, s * (lda * kb) + (long long)i * kb + k2);
      const unsigned char brw = ldg_as<unsigned char>(pb, j * ldb + (long long)s * kb + k2);
      const int av = ua ? (int)ar : (int)(signed char)ar;
      const int bv = ub ? (int)brw : (int)(signed char)brw;
      acc += (unsigned int)(av * bv);      // wrap-around like the reference's int accumulator
    }
  }
  return acc;
}

template <class S> __device__ __forceinline__ float dot_f16(const xb_gemm_desc& d, const DotGeom& g, const S& x, int i, int j, float acc) {   // reference :2025-2126
  const int k = g.k;
  const long long lda = g.lda, ldb = g.ldb;
  const bool trans_b = g.trans_b;
  const int kb = g.vnni_a ? 2 : 1;
  // comp F16 (or IMPLICIT, resolved like an SPR host) rounds the accumulator to f16 per FMA
  const bool round_each = (d.tcomp == LIBXSMM_DATATYPE_F16 || d.tcomp == LIBXSMM_DATATYPE_IMPLICIT);
  for (unsigned long long r = 0; r < x.br; ++r) {
    const char *pa, *pb; br_ptrs(d, x, r, 2, 2, pa, pb);
    for (int s = 0; s < k / kb; ++s) for (int k2 = 0; k2 < kb; ++k2) {
      const float av = xb_f16_to_f32(ldg_as<unsigned short>(pa, s * (lda * kb) + (long long)i * kb + k2));
      const long long kk = (long long)s * kb + k2;
      const float bv = xb_f16_to_f32(ldg_as<unsigned short>(pb, trans_b ? (kk * ldb + j) : (j * ldb + kk)));
      acc = __fadd_rn(acc, __fmul_rn(av, bv));
      if (round_each) acc = xb_f16_to_f32(xb_f32_to_f16(acc));
    }
  }
  return acc;
}

template <class S> __device__ __forceinline__ float dot_bf16(const xb_gemm_desc& d, const DotGeom& g, const S& x, int i, int j, float acc) {   // reference :2127-2170 and :2367-2419
  const int k = g.k;
  const long long lda = g.lda, ldb = g.ldb;
  const bool trans_a = g.trans_a, trans_b = g.trans_b;
  const bool vnni_a = g.vnni_a, vnni_b = g.vnni_b;
  const int kb = vnni_a ? 2 : 1;
  for (unsigned long long r = 0; r < x.br; ++r) {
    const char *pa, *pb; br_ptrs(d, x, r, 2, 2, pa, pb);
    for (int s = 0; s < k / kb; ++s) for (int k2 = kb - 1; k2 >= 0; --k2) {   // high k of a pair first
      const long long kk = (long long)s * kb + k2;
      unsigned short ar = 0, brw = 0;
      if (!trans_a) ar = ldg_as<unsigned short>(pa, s * (lda * kb) + (long long)i * kb + k2);
      else if (!vnni_a) ar = ldg_as<unsigned short>(pa, i * lda + kk);
      if (trans_b && vnni_b) brw = ldg_as<unsigned short>(pb, (long long)j * kb + s * (ldb * kb) + k2);
      else if (trans_b) brw = ldg_as<unsigned short>(pb, kk * ldb + j);
      else if (!vnni_b) brw = ldg_as<unsigned short>(pb, j * ldb + kk);
      acc = __fadd_rn(acc, __fmul_rn(xb_bf16_to_f32(ar), xb_bf16_to_f32(brw)));
    }
  }
  return acc;
}

// ---- fused form: column-bias pre-op, ReLU (+bitmask) / sigmoid post-op (reference :255-372) -----------------------------
// The reference builds an f32 image of C (bias column broadcast, + old C when beta = 1), lets the GEMM accumulate into it
// with beta = 1 and C type F32, applies the post-op and rounds ONCE into C. Per element that is: seed -> the precision path's
// dot_* loop, as gemm_simt_kernel runs it for an F32 C -> activation -> one conversion. The pre-ops are mateltwise kernels,
// hence their bf16 load (flushes bf16 subnormals).
__device__ __forceinline__ float fuse_ld(const void* p, long long i, int t) {
  if (t == LIBXSMM_DATATYPE_F32) return ((const float*)p)[i];
  if (t == LIBXSMM_DATATYPE_BF16) { unsigned short h = ((const unsigned short*)p)[i]; if ((h & 0x7f80) == 0) h &= 0x8000; return xb_bf16_to_f32(h); }
  return xb_f16_to_f32(((const unsigned short*)p)[i]);
}
__device__ __forceinline__ void fuse_st(void* p, long long i, int t, float v) {
  if (t == LIBXSMM_DATATYPE_F32) ((float*)p)[i] = v;
  else if (t == LIBXSMM_DATATYPE_BF16) ((unsigned short*)p)[i] = xb_f32_to_bf16_rne(v);
  else ((unsigned short*)p)[i] = xb_f32_to_f16(v);
}
// the f32 image of element (i, j) before the product: the bias, plus the old C when beta = 1
__device__ __forceinline__ float fuse_seed(const xb_gemm_desc& d, const TileCtx& x, bool bias, bool beta0, int i, long long ci) {
  if (bias) { const float bv = fuse_ld(x.colbias, i, d.tc); return beta0 ? bv : __fadd_rn(bv, fuse_ld(x.c, ci, d.tc)); }
  if (!beta0) return (d.tc == LIBXSMM_DATATYPE_F32) ? ((const float*)x.c)[ci] : fuse_ld(x.c, ci, d.tc);
  return 0.0f;
}

// gemm_fused_kernel: a CTA computes one block of C of 32*wm rows x FB_COLS/wm columns (wm = 1 for m <= 32, else 2), the blocks of
// every tile taken in a grid-stride loop. For each batch-reduce block and each k-chunk of FB_K, the CTA copies the block's rows of A
// and columns of B into shared memory once, in the operand's own layout (FuseLay); every thread then runs the path's dot_* loop over
// the staged chunk for FB_NC columns of its row, carrying their accumulators in registers from chunk to chunk, so that each
// element sees the operations of one uninterrupted loop. A warp owns 32 consecutive rows: the ReLU bitmask is one ballot per warp
// and column. Chunks start at multiples of FB_K, a multiple of every VNNI factor, and the last one is k % FB_K long.
constexpr int FB_THREADS = 256, FB_K = 32, FB_NC = 4, FB_COLS = (FB_THREADS / 32) * FB_NC, FB_MAX_CTAS = 4096;

__host__ __device__ inline void fuse_blocks(int m, int n, int& bm, int& bn, int& per_tile) {
  const int wm = (m > 32) ? 2 : 1;
  bm = 32 * wm; bn = FB_COLS / wm;
  per_tile = ((m + bm - 1) / bm) * ((n + bn - 1) / bn);
}

// how a path reads an operand at row (A) / column (B) p and k index kk: in packed groups of v k (v = 1: kk*ld + p), p-major
// (p*ld + kk), or not at all (the reference's zero operand); es: bytes per element
enum { FUSE_PK = 0, FUSE_PM, FUSE_ZERO };
struct FuseLay { int form, v, es; };
__device__ __forceinline__ void fuse_layouts(const DotGeom& g, int path, FuseLay& la, FuseLay& lb) {
  switch (path) {
    case P_F32: la = { g.trans_a ? FUSE_PM : FUSE_PK, 1, 4 }; lb = { g.trans_b ? FUSE_PK : FUSE_PM, 1, 4 }; break;
    case P_I8_F32: la = { FUSE_PK, 4, 1 }; lb = { FUSE_PM, 1, 1 }; break;
    case P_F16_F16: case P_F16_F32: la = { FUSE_PK, g.vnni_a ? 2 : 1, 2 }; lb = { g.trans_b ? FUSE_PK : FUSE_PM, 1, 2 }; break;
    default: {   // P_BF16_F32 / P_BF16_BF16, as dot_bf16 reads them
      const int kb = g.vnni_a ? 2 : 1;
      la = { !g.trans_a ? FUSE_PK : (!g.vnni_a ? FUSE_PM : FUSE_ZERO), kb, 2 };
      if (g.trans_b) lb = { FUSE_PK, g.vnni_b ? kb : 1, 2 };
      else lb = { !g.vnni_b ? FUSE_PM : FUSE_ZERO, 1, 2 };
    }
  }
}
// local leading dimension of a staged operand with a p-extent of np
__device__ __forceinline__ int fuse_ld_local(const FuseLay& l, int np) { return (l.form == FUSE_PK) ? np : FB_K + 1; }

// copies rows / columns [p0, p0 + np) x k [k0, k0 + kc) of an operand (global leading dimension ld) into dst, laid out as in global
// memory with the local leading dimension; p past np_ok lies outside the matrix and is staged as zero
template <typename T>
__device__ __forceinline__ void fuse_stage(char* dst, const char* src, const FuseLay& l, long long ld, int p0, int np, int np_ok, int k0, int kc) {
  if (l.form == FUSE_ZERO) return;
  const T* s = reinterpret_cast<const T*>(src);
  T* o = reinterpret_cast<T*>(dst);
  const int v = l.v, lv = (v == 4) ? 2 : (v == 2 ? 1 : 0), ldl = fuse_ld_local(l, np);   // v is 1, 2 or 4: shifts, no divisions
  for (int e = threadIdx.x; e < np * kc; e += FB_THREADS) {
    int p, kl;
    if (l.form == FUSE_PK) { const int q = e / (np * v), w = e - q * (np * v); p = w >> lv; kl = q * v + (w & (v - 1)); }   // consecutive threads: consecutive bytes
    else { p = e / kc; kl = e - p * kc; }
    const int kk = k0 + kl;
    T val = T(0);
    if (p < np_ok) val = (l.form == FUSE_PK) ? s[(long long)(kk >> lv) * ld * v + (long long)(p0 + p) * v + (kk & (v - 1))] : s[(long long)(p0 + p) * ld + kk];
    o[(l.form == FUSE_PK) ? (kl >> lv) * ldl * v + p * v + (kl & (v - 1)) : p * ldl + kl] = val;
  }
}
__device__ __forceinline__ void fuse_stage_any(char* dst, const char* src, const FuseLay& l, long long ld, int p0, int np, int np_ok, int k0, int kc) {
  if (l.es == 4) fuse_stage<unsigned int>(dst, src, l, ld, p0, np, np_ok, k0, kc);
  else if (l.es == 2) fuse_stage<unsigned short>(dst, src, l, ld, p0, np, np_ok, k0, kc);
  else fuse_stage<unsigned char>(dst, src, l, ld, p0, np, np_ok, k0, kc);
}

// the path's loop over one staged chunk for the thread's columns jl0 .. jl0 + nc - 1; an int8 sum travels in acc as its bits
template <int PATH>
__device__ __forceinline__ void fuse_dots(const xb_gemm_desc& d, const DotGeom& gs, const Staged& st, int il, int jl0, int nc, float (&acc)[FB_NC]) {
#pragma unroll
  for (int c = 0; c < FB_NC; ++c) {
    if (c >= nc) break;
    if (PATH == P_F32) acc[c] = dot_f32(d, gs, st, il, jl0 + c, acc[c]);
    else if (PATH == P_I8_F32) acc[c] = __uint_as_float(dot_i8(d, gs, st, il, jl0 + c, __float_as_uint(acc[c])));
    else if (PATH == P_F16_F16) acc[c] = dot_f16(d, gs, st, il, jl0 + c, acc[c]);
    else acc[c] = dot_bf16(d, gs, st, il, jl0 + c, acc[c]);
  }
}

__global__ void __launch_bounds__(FB_THREADS) gemm_fused_kernel(const xb_gemm_launch L, const int path) {
  __shared__ __align__(16) char smem_a[64 * (FB_K + 1) * 4];
  __shared__ __align__(16) char smem_b[FB_COLS * (FB_K + 1) * 4];
  const xb_gemm_desc& d = L.d;
  const DotGeom g = dot_geom(d);
  const int m = d.m, n = d.n;
  const long long ldc = d.ldc;
  const bool bias = d.fuse_colbias != 0, relu = d.cp_op == LIBXSMM_MELTW_TYPE_UNARY_RELU, sigm = d.cp_op == LIBXSMM_MELTW_TYPE_UNARY_SIGMOID;
  const bool bitm_desc = relu && (d.cp_flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) != 0;
  const bool beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) != 0, beta0_eff = beta0 && !bias;
  const bool seeded = (path == P_F32 || path == P_BF16_F32 || path == P_BF16_BF16);   // the seed is the loop's starting value
  const long long mask_ld = ((ldc + 15) / 16) * 16;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int bm, bn, per_tile; fuse_blocks(m, n, bm, bn, per_tile);
  const int wm = bm / 32, blocks_m = (m + bm - 1) / bm;
  const int il = (warp % wm) * 32 + lane, jl0 = (warp / wm) * FB_NC;   // the thread's row and first column in the block
  FuseLay la, lb; fuse_layouts(g, path, la, lb);
  DotGeom gs = g; gs.lda = fuse_ld_local(la, bm); gs.ldb = fuse_ld_local(lb, bn);
  const Staged st = { smem_a, smem_b };
  for (long long item = blockIdx.x; item < L.count * per_tile; item += gridDim.x) {
    const long long t = item / per_tile;
    const int blk = (int)(item - t * per_tile), i0 = (blk % blocks_m) * bm, j0 = (blk / blocks_m) * bn;
    const int i = i0 + il, nc = min(FB_NC, max(0, n - j0 - jl0));   // nc is warp-uniform
    const bool act = i < m;
    TileCtx x; resolve_tile<false>(L, t, x);
    float acc[FB_NC];
#pragma unroll
    for (int c = 0; c < FB_NC; ++c) acc[c] = (seeded && act && c < nc) ? fuse_seed(d, x, bias, beta0, i, (long long)(j0 + jl0 + c) * ldc + i) : 0.0f;
    for (unsigned long long r = 0; r < x.br; ++r) {
      const char *pa, *pb; br_ptrs(d, x, r, la.es, lb.es, pa, pb);
      for (int k0 = 0; k0 < g.k; k0 += FB_K) {
        const int kc = min(FB_K, g.k - k0);
        __syncthreads();                                       // the previous chunk is consumed
        fuse_stage_any(smem_a, pa, la, g.lda, i0, bm, min(bm, m - i0), k0, kc);
        fuse_stage_any(smem_b, pb, lb, g.ldb, j0, bn, min(bn, n - j0), k0, kc);
        __syncthreads();
        gs.k = kc;
        switch (path) {
          case P_F32: fuse_dots<P_F32>(d, gs, st, il, jl0, nc, acc); break;
          case P_I8_F32: fuse_dots<P_I8_F32>(d, gs, st, il, jl0, nc, acc); break;
          case P_F16_F16: case P_F16_F32: fuse_dots<P_F16_F16>(d, gs, st, il, jl0, nc, acc); break;
          default: fuse_dots<P_BF16_F32>(d, gs, st, il, jl0, nc, acc); break;
        }
      }
    }
    const bool bitm = bitm_desc && x.relu_mask != nullptr;
#pragma unroll
    for (int c = 0; c < FB_NC; ++c) {
      if (c >= nc) break;
      const int j = j0 + jl0 + c;
      const long long ci = (long long)j * ldc + i;
      float a = acc[c];
      if (act) {
        if (path == P_I8_F32) {
          a = __fmul_rn((float)(int)__float_as_uint(acc[c]), x.scf);
          if (!beta0_eff) a = __fadd_rn(a, fuse_seed(d, x, bias, beta0, i, ci));
        } else if (path == P_F16_F16 || path == P_F16_F32) {   // the F32-C variant rounds the old C through f16 (:2118-2124)
          if (!beta0_eff) a = __fadd_rn(a, xb_f16_to_f32(xb_f32_to_f16(fuse_seed(d, x, bias, beta0, i, ci))));
        }
        fuse_st(x.c, ci, d.tc, relu ? ((a <= 0.0f) ? 0.0f : a) : (sigm ? (tanhf(a / 2.0f) + 1.0f) / 2.0f : a));
      }
      if (bitm) {
        const unsigned int word = __ballot_sync(0xffffffffu, act && !(a <= 0.0f));
        const int iw = i0 + (il & ~31);
        if (lane < 4) {
          const int ib = iw + lane * 8;
          if (ib < m) {
            unsigned char* dst = x.relu_mask + ib / 8 + (long long)j * (mask_ld / 8);
            const unsigned int valid = (m - ib >= 8) ? 0xffu : ((1u << (m - ib)) - 1u);
            const unsigned int nb = (word >> (lane * 8)) & 0xffu;
            *dst = (unsigned char)((valid == 0xffu) ? nb : ((*dst & ~valid) | (nb & valid)));
          }
        }
      }
    }
  }
}

template <bool GRID>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const xb_gemm_launch L, const int path) {
  const xb_gemm_desc& d = L.d;
  const DotGeom g = dot_geom(d);
  const int m = d.m, n = d.n, k = d.k;
  const long long lda = d.lda, ldb = d.ldb, ldc = d.ldc;
  const bool beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) != 0;
  const bool trans_a = (d.flags & LIBXSMM_GEMM_FLAG_TRANS_A) != 0;
  const bool trans_b = (d.flags & LIBXSMM_GEMM_FLAG_TRANS_B) != 0;
  const bool vnni_a = (d.flags & LIBXSMM_GEMM_FLAG_VNNI_A) != 0;

  for (long long t = blockIdx.x; t < L.count; t += gridDim.x) {
    TileCtx x; resolve_tile<GRID>(L, t, x);
    for (int e = threadIdx.x; e < m * n; e += blockDim.x) {
      const int i = e % m, j = e / m;
      const long long ci = (long long)j * ldc + i;
      switch (path) {
        case P_F64: {   // reference :1322-1358, accumulates in place in C
          double acc = beta0 ? 0.0 : ldg_as<double>(x.c, ci);
          for (unsigned long long r = 0; r < x.br; ++r) {
            const char *pa, *pb; br_ptrs(d, x, r, 8, 8, pa, pb);
            for (int s = 0; s < k; ++s) {
              const double av = ldg_as<double>(pa, trans_a ? (i * lda + s) : (s * lda + i));
              const double bv = ldg_as<double>(pb, trans_b ? (s * ldb + j) : (j * ldb + s));
              acc = __dadd_rn(acc, __dmul_rn(av, bv));
            }
          }
          reinterpret_cast<double*>(x.c)[ci] = acc;
        } break;
        case P_F32:
          reinterpret_cast<float*>(x.c)[ci] = dot_f32(d, g, x, i, j, beta0 ? 0.0f : ldg_as<float>(x.c, ci));
          break;
        case P_I16: {   // reference :1427-1451 (trans flags ignored, VNNI2 A optional)
          const int kb = vnni_a ? 2 : 1;
          int acc = beta0 ? 0 : ldg_as<int>(x.c, ci);
          for (unsigned long long r = 0; r < x.br; ++r) {
            const char *pa, *pb; br_ptrs(d, x, r, 2, 2, pa, pb);
            for (int s = 0; s < k / kb; ++s) for (int k2 = 0; k2 < kb; ++k2) {
              const int av = ldg_as<short>(pa, s * (lda * kb) + (long long)i * kb + k2);
              const int bv = ldg_as<short>(pb, j * ldb + (long long)s * kb + k2);
              acc += av * bv;
            }
          }
          reinterpret_cast<int*>(x.c)[ci] = acc;
        } break;
        case P_I8_I32: case P_I8_F32: {
          const unsigned int acc = dot_i8(d, g, x, i, j, (path == P_I8_I32 && !beta0) ? (unsigned int)ldg_as<int>(x.c, ci) : 0u);
          if (path == P_I8_I32) reinterpret_cast<int*>(x.c)[ci] = (int)acc;
          else {
            float f = __fmul_rn((float)(int)acc, x.scf);
            if (!beta0) f = __fadd_rn(f, ldg_as<float>(x.c, ci));
            reinterpret_cast<float*>(x.c)[ci] = f;
          }
        } break;
        case P_F16_F16: case P_F16_F32: {
          float acc = dot_f16(d, g, x, i, j, 0.0f);
          if (path == P_F16_F16) {
            if (!beta0) acc = __fadd_rn(acc, xb_f16_to_f32(ldg_as<unsigned short>(x.c, ci)));
            reinterpret_cast<unsigned short*>(x.c)[ci] = xb_f32_to_f16(acc);
          } else {
            if (!beta0) acc = __fadd_rn(acc, xb_f16_to_f32(xb_f32_to_f16(ldg_as<float>(x.c, ci))));
            reinterpret_cast<float*>(x.c)[ci] = acc;
          }
        } break;
        case P_BF16_F32: case P_BF16_BF16: {
          float acc;
          if (path == P_BF16_F32) acc = beta0 ? 0.0f : ldg_as<float>(x.c, ci);
          else acc = beta0 ? 0.0f : xb_bf16_to_f32(ldg_as<unsigned short>(x.c, ci));
          acc = dot_bf16(d, g, x, i, j, acc);
          if (path == P_BF16_F32) reinterpret_cast<float*>(x.c)[ci] = acc;
          else reinterpret_cast<unsigned short*>(x.c)[ci] = xb_f32_to_bf16_rne(acc);
        } break;
        case P_FP8: {   // reference :2420-2630 (B of A's 8-bit type: k ascending, VNNI factor 4) and :2171-2366 (bf16 B: pairs, high k first)
          const bool b16 = (d.tb == LIBXSMM_DATATYPE_BF16), hf = (d.ta == LIBXSMM_DATATYPE_HF8);
          const int kb = vnni_a ? (b16 ? 2 : 4) : 1;
          float acc = 0.0f;
          if (!beta0) {
            if (d.tc == LIBXSMM_DATATYPE_F32) acc = ldg_as<float>(x.c, ci);
            else if (d.tc == LIBXSMM_DATATYPE_BF16) acc = xb_bf16_to_f32(ldg_as<unsigned short>(x.c, ci));
            else acc = hf ? xb_hf8_to_f32(ldg_as<unsigned char>(x.c, ci)) : xb_bf8_to_f32(ldg_as<unsigned char>(x.c, ci));
          }
          for (unsigned long long r = 0; r < x.br; ++r) {
            const char *pa, *pb; br_ptrs(d, x, r, 1, b16 ? 2 : 1, pa, pb);
            for (int s = 0; s < k / kb; ++s) for (int q = 0; q < kb; ++q) {
              const int k2 = b16 ? (kb - 1 - q) : q;
              const long long kk = (long long)s * kb + k2;
              unsigned char ar = 0;
              if (!trans_a) ar = ldg_as<unsigned char>(pa, s * (lda * kb) + (long long)i * kb + k2);
              else if (!vnni_a) ar = ldg_as<unsigned char>(pa, i * lda + kk);
              float bv;
              if (b16) bv = xb_bf16_to_f32(trans_b ? ldg_as<unsigned short>(pb, kk * ldb + j) : ldg_as<unsigned short>(pb, j * ldb + kk));
              else { const unsigned char bw = trans_b ? ldg_as<unsigned char>(pb, kk * ldb + j) : ldg_as<unsigned char>(pb, j * ldb + kk); bv = hf ? xb_hf8_to_f32(bw) : xb_bf8_to_f32(bw); }
              acc = __fadd_rn(acc, __fmul_rn(hf ? xb_hf8_to_f32(ar) : xb_bf8_to_f32(ar), bv));
            }
          }
          if (d.tc == LIBXSMM_DATATYPE_F32) reinterpret_cast<float*>(x.c)[ci] = acc;
          else if (d.tc == LIBXSMM_DATATYPE_BF16) reinterpret_cast<unsigned short*>(x.c)[ci] = xb_f32_to_bf16_rne(acc);
          else reinterpret_cast<unsigned char*>(x.c)[ci] = hf ? xb_f32_to_hf8(acc) : xb_f32_to_bf8(acc);
        } break;
        case P_I4_I32: {   // reference :1273-1321; zero point subtracted in 8-bit arithmetic, B read as unsigned bytes
          unsigned int acc = beta0 ? 0u : (unsigned int)ldg_as<int>(x.c, ci);
          for (unsigned long long r = 0; r < x.br; ++r) {
            const char *pa, *pb; br_ptrs(d, x, r, 1, 1, pa, pb);
            const unsigned char z = (d.br_type == 3) ? x.a_q[((d.br_stride_a * 2) / k) * (long long)r + i] : x.a_q[i];
            for (int s = 0; s < k / 8; ++s) for (int q = 0; q < 4; ++q) {
              const unsigned char pk = ldg_as<unsigned char>(pa, s * lda * 4 + 4 * (long long)i + q);
              const int ev = (int)(signed char)((pk & 0x0f) - z), od = (int)(signed char)(((pk >> 4) & 0x0f) - z);
              acc += (unsigned int)(ev * (int)ldg_as<unsigned char>(pb, j * ldb + (long long)s * 8 + q));
              acc += (unsigned int)(od * (int)ldg_as<unsigned char>(pb, j * ldb + (long long)s * 8 + 4 + q));
            }
          }
          reinterpret_cast<int*>(x.c)[ci] = (int)acc;
        } break;
        default: break;
      }
    }
  }
}

// ---- bitmap-compressed A (DECOMPRESS_A_VIA_BITMASK, reference :857-948) ---------------------------------------------------
// A stores only the elements whose bit is set, in bit order; bit (s, i, k2) sits at position s*(m*kb) + i*kb + k2. The index
// of an element in the compressed array is the number of set bits in front of it: phase 1 scans the bitmap once (per-word
// population counts -> exclusive prefix in `prefix`), phase 2 is the exact-order element loop of the reference with
// idx = prefix[word] + popc(bits below). One CTA per call (the flag excludes batch reduce; single-tile launches only).
__device__ __forceinline__ unsigned int bitmap_word(const unsigned char* bm, long long w, long long nbytes) {
  unsigned int v = 0;
  for (int q = 0; q < 4; ++q) { const long long bi = w * 4 + q; if (bi < nbytes) v |= (unsigned int)bm[bi] << (8 * q); }
  return v;
}
__global__ void __launch_bounds__(1024) gemm_bitmap_kernel(const xb_gemm_launch L, unsigned int* __restrict__ prefix) {
  const xb_gemm_desc& d = L.d;
  const int m = d.m, n = d.n, k = d.k;
  const long long ldb = d.ldb, ldc = d.ldc;
  const bool beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) != 0;
  const int kb = (d.ta == LIBXSMM_DATATYPE_F32) ? 1 : ((d.tb == LIBXSMM_DATATYPE_F32) ? 1 : 2);
  const long long nbits = (long long)m * k, nbytes = (nbits + 7) / 8, nwords = (nbits + 31) / 32;
  const unsigned char* bm = (const unsigned char*)L.one.a_q;
  const char* a = (const char*)L.one.a; const char* b = (const char*)L.one.b; char* c = (char*)L.one.c;
  __shared__ unsigned int seg_total[1024];
  // phase 1: thread t owns a contiguous range of words
  const long long per = (nwords + blockDim.x - 1) / blockDim.x, w0 = (long long)threadIdx.x * per, w1 = (w0 + per < nwords) ? w0 + per : nwords;
  unsigned int run = 0;
  for (long long w = w0; w < w1; ++w) { prefix[w] = run; run += __popc(bitmap_word(bm, w, nbytes)); }
  seg_total[threadIdx.x] = run;
  __syncthreads();
  if (threadIdx.x == 0) { unsigned int acc = 0; for (unsigned int t = 0; t < blockDim.x; ++t) { const unsigned int v = seg_total[t]; seg_total[t] = acc; acc += v; } }
  __syncthreads();
  { const unsigned int base = seg_total[threadIdx.x]; for (long long w = w0; w < w1; ++w) prefix[w] += base; }
  __syncthreads();
  // phase 2
  for (int e = threadIdx.x; e < m * n; e += blockDim.x) {
    const int i = e % m, j = e / m;
    const long long ci = (long long)j * ldc + i;
    float acc;
    if (d.tc == LIBXSMM_DATATYPE_F32) acc = beta0 ? 0.0f : ((const float*)c)[ci];
    else acc = beta0 ? 0.0f : ((d.tc == LIBXSMM_DATATYPE_BF16) ? xb_bf16_to_f32(((const unsigned short*)c)[ci]) : xb_f16_to_f32(((const unsigned short*)c)[ci]));
    for (int s = 0; s < k / kb; ++s) for (int k2 = 0; k2 < kb; ++k2) {
      const long long bit = (long long)s * m * kb + (long long)i * kb + k2, w = bit >> 5;
      const unsigned int word = bitmap_word(bm, w, nbytes), sh = (unsigned int)(bit & 31);
      if ((word >> sh) & 1u) {
        const long long idx = (long long)prefix[w] + __popc(word & ((1u << sh) - 1u));
        const float av = (d.ta == LIBXSMM_DATATYPE_F32) ? ((const float*)a)[idx]
                       : ((d.ta == LIBXSMM_DATATYPE_BF16) ? xb_bf16_to_f32(((const unsigned short*)a)[idx]) : xb_f16_to_f32(((const unsigned short*)a)[idx]));
        const long long bi = j * ldb + (long long)s * kb + k2;
        const float bv = (d.tb == LIBXSMM_DATATYPE_F32) ? ((const float*)b)[bi]
                       : ((d.tb == LIBXSMM_DATATYPE_BF16) ? xb_bf16_to_f32(((const unsigned short*)b)[bi]) : xb_f16_to_f32(((const unsigned short*)b)[bi]));
        acc = __fadd_rn(acc, __fmul_rn(av, bv));
      }
    }
    if (d.tc == LIBXSMM_DATATYPE_F32) ((float*)c)[ci] = acc;
    else if (d.tc == LIBXSMM_DATATYPE_BF16) ((unsigned short*)c)[ci] = xb_f32_to_bf16_rne(acc);
    else ((unsigned short*)c)[ci] = xb_f32_to_f16(acc);
  }
}


// ---- MX fp8: MXBF8 x MXBF8 / MXHF8 x MXHF8 with E8M0 block scales (reference :2620-2679) -------------------------------
// A is VNNI4 [k/4][lda][4], B is VNNI4-transposed [k/4][ldb][4]; one scale byte per (row, 32 k): A's [r][k/32][lda], B's
// [r][k/32][ldb]. A scale byte widens as bits = s << 23 (0 -> +0, 0xFF -> +inf). Per element and 4-k group: tmp = sum of a*b
// over k2 = 3..0 from 0, then acc += (tmp * sa) * sb; acc runs over (r, group) from 0 and C = (beta0 ? 0 : C) + acc. Block r of
// a batch-reduce sits at r*lda*k (A) and r*ldb*k (B): the reference ignores the stride hints, dispatch accepts stride mode only
// where they agree with that.
__device__ __forceinline__ float mx_scale(unsigned char s) { return __uint_as_float((unsigned int)s << 23); }

__device__ __forceinline__ float dot_mx8(const xb_gemm_desc& d, const TileCtx& x, int i, int j) {
  const int k = d.k, groups = d.k / 4;
  const long long lda = d.lda, ldb = d.ldb;
  const bool hf = (d.ta == LIBXSMM_DATATYPE_MXHF8);
  float acc = 0.0f;
  for (unsigned long long r = 0; r < x.br; ++r) {
    const unsigned char* pa = (const unsigned char*)x.a0 + (long long)r * lda * k + (long long)i * 4;
    const unsigned char* pb = (const unsigned char*)x.b0 + (long long)r * ldb * k + (long long)j * 4;
    const unsigned char* psa = x.a_s + (long long)r * lda * (k / 32) + i;
    const unsigned char* psb = x.b_s + (long long)r * ldb * (k / 32) + j;
    for (int s = 0; s < groups; ++s) {
      float tmp = 0.0f;
      for (int k2 = 3; k2 >= 0; --k2) {
        const unsigned char ab = pa[(long long)s * lda * 4 + k2], bb = pb[(long long)s * ldb * 4 + k2];
        tmp = __fadd_rn(tmp, __fmul_rn(hf ? xb_hf8_to_f32(ab) : xb_bf8_to_f32(ab), hf ? xb_hf8_to_f32(bb) : xb_bf8_to_f32(bb)));
      }
      acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(tmp, mx_scale(psa[(long long)(s / 8) * lda])), mx_scale(psb[(long long)(s / 8) * ldb])));
    }
  }
  return acc;
}

// F32 C: written in place. MXBF8 C: the f32 image (0 + acc, BETA_0 only) goes to img [tile][n][m] for gemm_mx8_quant_kernel.
__global__ void __launch_bounds__(256) gemm_mx8_kernel(const xb_gemm_launch L, float* __restrict__ img) {
  const xb_gemm_desc& d = L.d;
  const int m = d.m, n = d.n;
  const long long ldc = d.ldc;
  const bool beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) != 0;
  for (long long t = blockIdx.x; t < L.count; t += gridDim.x) {
    TileCtx x; resolve_tile<false>(L, t, x);
    for (int e = threadIdx.x; e < m * n; e += blockDim.x) {
      const int i = e % m, j = e / m;
      const float acc = dot_mx8(d, x, i, j);
      if (img != nullptr) img[(t * n + j) * (long long)m + i] = __fadd_rn(0.0f, acc);
      else { float* c = reinterpret_cast<float*>(x.c) + (long long)j * ldc + i; *c = __fadd_rn(beta0 ? 0.0f : *c, acc); }
    }
  }
}

// MXBF8 C (reference :757-, one 32-row block of one column per thread): each value rounded to bf16 (nearest-even, subnormals
// flushed); the block's amax (NaN wins); shared exponent e = biased exponent of amax - 15, clamped to [0, 254], 0 for amax = 0,
// stored as the scale byte; the scale 2^(e-127) (2^-127 for e = 0) rounded to bf16 and its reciprocal rounded to bf16; each value
// times that reciprocal, rounded to bf16, then to bf8 (E5M2) nearest-even, Inf and NaN bytes clamped to +-0x7B. The flushes
// matter: e = 0 gives a zero scale and an infinite reciprocal, e = 254 a zero reciprocal. The elementwise MXBF8 quantiser
// (meltw.cu) divides by the unrounded scale and writes a NaN block as 0x7B with scale 0xFF, so it does not give these bytes.
__device__ __forceinline__ float mx_bf16_rne(float f) { return xb_bf16_to_f32(xb_f32_to_bf16_rne(f)); }
// the reference runs on x86: an invalid product (0 * inf) is the negative default NaN there, and a NaN operand passes through
__device__ __forceinline__ float mx_x86_mul(float a, float b) {
  if (a != a) return __uint_as_float(__float_as_uint(a) | 0x400000u);
  const float p = __fmul_rn(a, b);
  return (p != p) ? __uint_as_float(0xffc00000u) : p;
}
__global__ void __launch_bounds__(128) gemm_mx8_quant_kernel(const xb_gemm_launch L, const float* __restrict__ img) {
  const int m = L.d.m, n = L.d.n, bm = L.d.m / 32;
  const long long ldc = L.d.ldc, per_tile = (long long)n * bm;
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= L.count * per_tile) return;
  const long long t = e / per_tile;
  const int j = (int)((e % per_tile) / bm), b = (int)(e % bm);
  TileCtx x; resolve_tile<false>(L, t, x);
  const float* src = img + (t * n + j) * (long long)m + b * 32;
  float v[32], amax = 0.0f;
#pragma unroll
  for (int q = 0; q < 32; ++q) { v[q] = mx_bf16_rne(src[q]); const float a = fabsf(v[q]); if (a > amax || a != a) amax = a; }
  int se = (amax == 0.0f) ? 0 : (int)((__float_as_uint(amax) >> 23) & 0xffu);
  se = (se - 15 < 0) ? 0 : ((se - 15 > 254) ? 254 : se - 15);
  x.c_s[(long long)j * (ldc / 32) + b] = (unsigned char)se;
  const float scale = __uint_as_float(((unsigned int)se << 23) | (se == 0 ? 0x400000u : 0u));
  const float rcp = mx_bf16_rne(__fdiv_rn(1.0f, mx_bf16_rne(scale)));
  unsigned char* dst = reinterpret_cast<unsigned char*>(x.c) + (long long)j * ldc + b * 32;
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    unsigned char o = xb_f32_to_bf8(mx_bf16_rne(mx_x86_mul(v[q], rcp)));
    if ((o & 0x7c) == 0x7c) o = (unsigned char)((o & 0x80) | 0x7b);
    dst[q] = o;
  }
}


// ---- dequantising A: I8 x BF16, I8 / I4 / U4 / BF8 x F16 with per-row scales and zero points (reference :1684-2024) -----------
// One thread per C element, the reference's order: acc runs from 0 over (r, k) with acc += a * b, where a is A's element widened
// and dequantised with row i's scale sc (a.tertiary) and zero point zp (a.quaternary):
//   I8 x BF16 (:1684-1730)  a = bf16_rne((float)int8 * sc), sc f32      A flat [k][lda], B [n][ldb]
//   I8 x F16  (:1881-2024)  a = (float)int8 * sc, sc f16                 A flat; no zero point (the reference's fuse_zpt_sub is 0)
//   I4 x F16  (:1793-1880)  a = ((float)nibble - zp) * sc, both f16       A bytes [k/2][lda]: low nibble even k, high nibble odd k,
//                                                                          sign-extended unless U4
//   BF8 x F16 (:1731-1792)  a = bf8 widened through f16                  A flat, or VNNI2 [k/2][lda][2]
// An F16 B honours TRANS_B. Comp F16, or IMPLICIT resolved like an SPR host (as dot_f16), is the reference's "replacement FMA":
// a is rounded to f16 after the subtraction and after the scaling, and acc after every add (the integer itself is exact in f16).
// Then C: a 16-bit C adds its old value widened (beta = 1) and rounds once; an F32 C adds the old value as is, except next to an
// I8 / I4 A and an F16 B, where the old value is first rounded to f16 (:1871-1876, :2016-2021).
__device__ __forceinline__ float dq_f16r(float v) { return xb_f16_to_f32(xb_f32_to_f16(v)); }

template <bool GRID>
__global__ void __launch_bounds__(256) gemm_dq_kernel(const xb_gemm_launch L) {
  const xb_gemm_desc& d = L.d;
  const int form = xb_dq_form(&d);
  const int m = d.m, n = d.n, k = d.k;
  const long long lda = d.lda, ldb = d.ldb, ldc = d.ldc;
  const bool beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) != 0, trans_b = (d.flags & LIBXSMM_GEMM_FLAG_TRANS_B) != 0;
  const bool round_each = form != XB_DQ_I8_BF16 && (d.tcomp == LIBXSMM_DATATYPE_F16 || d.tcomp == LIBXSMM_DATATYPE_IMPLICIT);
  const bool u4 = (d.ta == LIBXSMM_DATATYPE_U4X2), i4 = (form == XB_DQ_I4_F16), b16 = (form == XB_DQ_I8_BF16);
  const int kb = (i4 || (form == XB_DQ_BF8_F16 && (d.flags & LIBXSMM_GEMM_FLAG_VNNI_A) != 0)) ? 2 : 1;
  for (long long t = blockIdx.x; t < L.count; t += gridDim.x) {
    TileCtx x; resolve_tile<GRID>(L, t, x);
    for (int e = threadIdx.x; e < m * n; e += blockDim.x) {
      const int i = e % m, j = e / m;
      const long long ci = (long long)j * ldc + i;
      float sc = 1.0f, zp = 0.0f;
      if (b16) sc = reinterpret_cast<const float*>(x.a_s)[i];
      else if (form != XB_DQ_BF8_F16) sc = xb_f16_to_f32(reinterpret_cast<const unsigned short*>(x.a_s)[i]);
      if (i4) zp = xb_f16_to_f32(reinterpret_cast<const unsigned short*>(x.a_q)[i]);
      float acc = 0.0f;
      for (unsigned long long r = 0; r < x.br; ++r) {
        const char *pa, *pb; br_ptrs(d, x, r, 1, 2, pa, pb);
        for (int s = 0; s < k / kb; ++s) for (int k2 = 0; k2 < kb; ++k2) {
          const long long kk = (long long)s * kb + k2;
          float av;
          if (form == XB_DQ_BF8_F16) av = xb_bf8_to_f32(ldg_as<unsigned char>(pa, s * (lda * kb) + (long long)i * kb + k2));
          else {
            const unsigned char by = ldg_as<unsigned char>(pa, s * lda + i);
            int q;
            if (!i4) q = (signed char)by;
            else if (u4) q = (k2 == 0) ? (by & 0x0f) : (by >> 4);
            else q = (k2 == 0) ? ((signed char)(by << 4)) >> 4 : ((signed char)by) >> 4;
            av = (float)q;
            if (b16) av = xb_bf16_to_f32(xb_f32_to_bf16_rne(__fmul_rn(av, sc)));
            else {
              if (i4) { av = __fsub_rn(av, zp); if (round_each) av = dq_f16r(av); }
              av = __fmul_rn(av, sc);
              if (round_each) av = dq_f16r(av);
            }
          }
          const unsigned short bw = trans_b ? ldg_as<unsigned short>(pb, kk * ldb + j) : ldg_as<unsigned short>(pb, j * ldb + kk);
          acc = __fadd_rn(acc, __fmul_rn(av, b16 ? xb_bf16_to_f32(bw) : xb_f16_to_f32(bw)));
          if (round_each) acc = dq_f16r(acc);
        }
      }
      if (d.tc == LIBXSMM_DATATYPE_F32) {
        if (!beta0) { const float old = ldg_as<float>(x.c, ci); acc = __fadd_rn(acc, (b16 || form == XB_DQ_BF8_F16) ? old : dq_f16r(old)); }
        reinterpret_cast<float*>(x.c)[ci] = acc;
      } else if (b16) {
        if (!beta0) acc = __fadd_rn(acc, xb_bf16_to_f32(ldg_as<unsigned short>(x.c, ci)));
        reinterpret_cast<unsigned short*>(x.c)[ci] = xb_f32_to_bf16_rne(acc);
      } else {
        if (!beta0) acc = __fadd_rn(acc, xb_f16_to_f32(ldg_as<unsigned short>(x.c, ci)));
        reinterpret_cast<unsigned short*>(x.c)[ci] = xb_f32_to_f16(acc);
      }
    }
  }
}


// ---- 8-bit integer tiles: dp4a kernel ------------------------------------------------------------------------------
// Integer sums wrap modulo 2^32 and are therefore exact in ANY order: the int8 paths need not follow the reference's
// loop order to stay bit-identical (reference :1452-1683). One WARP per tile: the VNNI4 A words [k/4][m] and the
// k-contiguous B words [n][k/4] of a 64-wide k chunk are staged in shared memory with coalesced 4-byte loads, every
// lane keeps a TM x TN block of accumulators and issues one dp4a per (m, n, 4 k). HBM-bound by construction
// (m*k + k*n + 4*m*n bytes per tile); 8 warps per CTA and several CTAs per SM hide the load latency.
template <bool UA, bool UB> __device__ __forceinline__ unsigned int dp4a_x(unsigned int a, unsigned int b, unsigned int c) {
  unsigned int d;
  if (UA && UB) asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  else if (UA && !UB) asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  else if (!UA && UB) asm("dp4a.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  else asm("dp4a.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

constexpr int I8_WARPS = 16, I8_KC = 64;   // warps per CTA, k bytes per staged chunk

__device__ __forceinline__ void group_sync(int wpt, int group) {
  if (wpt == 1) __syncwarp();
  else asm volatile("bar.sync %0, %1;" :: "r"(group + 1), "r"(wpt * 32) : "memory");
}

// WPT warps share one tile: each owns one (LM*TM) x (LN*TN) block of C and keeps it in registers over the whole k loop;
// the group stages the operand chunk once. 16/WPT tiles are in flight per CTA.
template <int TM, int TN, bool UA, bool UB, bool GRID>
__global__ void __launch_bounds__(I8_WARPS * 32, 2) gemm_i8_kernel(const xb_gemm_launch L, const int to_f32, const int wpt, const int smem_words_per_group) {
  constexpr int LM = 8, LN = 4;                       // lanes along m and n
  extern __shared__ unsigned int smem_i8[];
  const xb_gemm_desc& d = L.d;
  const int m = d.m, n = d.n, kq_all = d.k >> 2;
  const long long lda = d.lda, ldb = d.ldb, ldc = d.ldc;
  const bool beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) != 0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = I8_WARPS / wpt, group = warp / wpt, wg = warp % wpt, gtid = wg * 32 + lane, gsize = wpt * 32;
  const int lm = lane % LM, ln = lane / LM;
  const int passes_m = (m + LM * TM - 1) / (LM * TM);
  const int m0 = (wg % passes_m) * (LM * TM), n0 = (wg / passes_m) * (LN * TN);   // this warp's block (may be empty: n0 >= n)
  const int kcq = (kq_all < I8_KC / 4) ? kq_all : I8_KC / 4;      // words of k per chunk
  // both panels are stored k-group-major ([q][m] and [q][n]) so that a lane's TM / TN operands are contiguous (128-bit shared
  // loads); row strides are 4 * odd words: 16-byte aligned, and the transposing B fill spreads over the banks
  const int ms = (((m + 3) >> 2) | 1) << 2, ns = (((n + 3) >> 2) | 1) << 2;
  unsigned int* sa = smem_i8 + (size_t)group * smem_words_per_group;   // [kcq][ms]
  unsigned int* sb = sa + (size_t)kcq * ms;                            // [kcq][ns]
  const long long ntiles_rounded = ((L.count + (long long)gridDim.x * groups - 1) / ((long long)gridDim.x * groups)) * ((long long)gridDim.x * groups);
  for (long long t = (long long)blockIdx.x * groups + group; t < ntiles_rounded; t += (long long)gridDim.x * groups) {
    const bool live = t < L.count;                    // dead iterations only keep the group barriers balanced
    TileCtx x; if (live) resolve_tile<GRID>(L, t, x); else { x.br = 0; }
    unsigned int acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = 0u;
    if (live) for (unsigned long long r = 0; r < x.br; ++r) {
      const char *pa, *pb; br_ptrs(d, x, r, 1, 1, pa, pb);
      for (int q0 = 0; q0 < kq_all; q0 += kcq) {
        const int qn = (kq_all - q0 < kcq) ? (kq_all - q0) : kcq;
        group_sync(wpt, group);                        // previous chunk fully consumed
        for (int e = gtid; e < qn * m; e += gsize) {   // A words: rows of m contiguous words
          const int q = e / m, i = e - q * m;
          sa[q * ms + i] = reinterpret_cast<const unsigned int*>(pa + ((long long)(q0 + q) * lda) * 4)[i];
        }
        for (int e = gtid; e < n * qn; e += gsize) {   // B words: rows of qn contiguous words
          const int jn = e / qn, q = e - jn * qn;
          sb[q * ns + jn] = reinterpret_cast<const unsigned int*>(pb + (long long)jn * ldb + (long long)q0 * 4)[q];
        }
        group_sync(wpt, group);
        if (n0 < n) for (int q = 0; q < qn; ++q) {
          unsigned int av[TM], bv[TN];
          if (TM == 4) {   // operands beyond m / n are padding words of the row (never stored to C)
            const uint4 a4 = *reinterpret_cast<const uint4*>(sa + q * ms + m0 + lm * 4);
            const uint4 b0 = *reinterpret_cast<const uint4*>(sb + q * ns + n0 + ln * 8), b1 = *reinterpret_cast<const uint4*>(sb + q * ns + n0 + ln * 8 + 4);
            av[0] = a4.x; av[1] = a4.y; av[2] = a4.z; av[3 % TM] = a4.w;
            bv[0] = b0.x; bv[1] = b0.y; bv[2 % TN] = b0.z; bv[3 % TN] = b0.w; bv[4 % TN] = b1.x; bv[5 % TN] = b1.y; bv[6 % TN] = b1.z; bv[7 % TN] = b1.w;
          } else {
#pragma unroll
            for (int i = 0; i < TM; ++i) { const int mi = m0 + lm * TM + i; av[i] = (mi < m) ? sa[q * ms + mi] : 0u; }
#pragma unroll
            for (int j = 0; j < TN; ++j) { const int nj = n0 + ln * TN + j; bv[j] = (nj < n) ? sb[q * ns + nj] : 0u; }
          }
#pragma unroll
          for (int i = 0; i < TM; ++i)
#pragma unroll
            for (int j = 0; j < TN; ++j) acc[i][j] = dp4a_x<UA, UB>(av[i], bv[j], acc[i][j]);
        }
      }
    }
    if (live && TM == 4 && (ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(x.c) & 15) == 0 && m0 + lm * 4 + 3 < m) {
      // four consecutive rows per lane: 16-byte accesses, 8 lanes cover 128 contiguous bytes of a C column
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int nj = n0 + ln * TN + j;
        if (nj < n) {
          const long long ci = (long long)nj * ldc + m0 + lm * 4;
          if (!to_f32) {
            uint4 v = make_uint4(acc[0][j], acc[1 % TM][j], acc[2 % TM][j], acc[3 % TM][j]);
            if (!beta0) { const uint4 o = *reinterpret_cast<const uint4*>(reinterpret_cast<const int*>(x.c) + ci); v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
            *reinterpret_cast<uint4*>(reinterpret_cast<int*>(x.c) + ci) = v;
          } else {
            float4 f = make_float4(__fmul_rn((float)(int)acc[0][j], x.scf), __fmul_rn((float)(int)acc[1 % TM][j], x.scf),
                                   __fmul_rn((float)(int)acc[2 % TM][j], x.scf), __fmul_rn((float)(int)acc[3 % TM][j], x.scf));
            if (!beta0) { const float4 o = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x.c) + ci);
                          f.x = __fadd_rn(f.x, o.x); f.y = __fadd_rn(f.y, o.y); f.z = __fadd_rn(f.z, o.z); f.w = __fadd_rn(f.w, o.w); }
            *reinterpret_cast<float4*>(reinterpret_cast<float*>(x.c) + ci) = f;
          }
        }
      }
    } else if (live) {
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int nj = n0 + ln * TN + j;
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          const int mi = m0 + lm * TM + i;
          if (mi < m && nj < n) {
            const long long ci = (long long)nj * ldc + mi;
            if (!to_f32) {
              unsigned int v = acc[i][j];
              if (!beta0) v += (unsigned int)reinterpret_cast<const int*>(x.c)[ci];
              reinterpret_cast<int*>(x.c)[ci] = (int)v;
            } else {                                               // reference :1579-1585
              float f = __fmul_rn((float)(int)acc[i][j], x.scf);
              if (!beta0) f = __fadd_rn(f, reinterpret_cast<const float*>(x.c)[ci]);
              reinterpret_cast<float*>(x.c)[ci] = f;
            }
          }
        }
      }
    }
  }
}

// host side: is the dp4a kernel applicable? (VNNI4 A, whole words everywhere, strided or single-tile launch)
bool i8_fast_ok(const xb_gemm_launch& L, int path) {
  const xb_gemm_desc& d = L.d;
  if (path != P_I8_I32 && path != P_I8_F32) return false;
  if (path == P_I8_I32 && (d.flags & LIBXSMM_GEMM_FLAG_VNNI_A) == 0) return false;    // flat A: bytes of 4 different rows per word
  if ((d.k & 3) != 0 || (d.ldb & 3) != 0 || d.m > 1024 || d.n > 1024) return false;
  if (L.recs != nullptr || d.br_type == 1 || d.br_type == 2) return false;            // per-tile pointers are not checkable on the host
  const bool single = (L.a == nullptr && L.c == nullptr);
  const uintptr_t a = (uintptr_t)(single ? L.one.a : L.a), b = (uintptr_t)(single ? L.one.b : L.b), c = (uintptr_t)(single ? L.one.c : L.c);
  if (((a | b | c) & 3) != 0) return false;
  if (!single && (((L.tile_stride_a | L.tile_stride_b | L.tile_stride_c | L.tile_stride_c_n) & 3) != 0)) return false;
  if (d.br_type == 3 && (((d.br_stride_a | d.br_stride_b) & 3) != 0)) return false;
  return true;
}

template <int TM, int TN>
void launch_i8(const xb_gemm_launch& L, int path, int wpt, int words_per_group, size_t smem, unsigned int grid, cudaStream_t st) {
  const bool ua = (L.d.ta == LIBXSMM_DATATYPE_U8), ub = (L.d.tb == LIBXSMM_DATATYPE_U8);
  const int to_f32 = (path == P_I8_F32);
#define XB_I8_CASE(A, B, G) do { \
    static unsigned long long attr_set = 0ull; \
    if (xb_rt_first_use_on_device(&attr_set)) cudaFuncSetAttribute(gemm_i8_kernel<TM, TN, A, B, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
    gemm_i8_kernel<TM, TN, A, B, G><<<grid, I8_WARPS * 32, smem, st>>>(L, to_f32, wpt, words_per_group); } while (0)
  if (L.grid_m > 0) {
    if (ua && ub) XB_I8_CASE(true, true, true); else if (ua) XB_I8_CASE(true, false, true); else if (ub) XB_I8_CASE(false, true, true); else XB_I8_CASE(false, false, true);
  } else {
    if (ua && ub) XB_I8_CASE(true, true, false); else if (ua) XB_I8_CASE(true, false, false); else if (ub) XB_I8_CASE(false, true, false); else XB_I8_CASE(false, false, false);
  }
#undef XB_I8_CASE
}


// ---- low-bit A x 8-bit B: ternary I2X4 / binary I1X8 x I8 / U8 -> I32, MXFP4X2 x I8 -> F32 / BF16 (reference :1009-1272) -------
// Every product is a small integer times an 8-bit one: A is expanded to four int8 per word in registers and multiplied by four k of
// B with dp4a (B unsigned for a U8 B). Integer sums wrap modulo 2^32 like the reference's int += and are exact in any order, so I2 / I1
// need not follow the reference's loop order. MXFP4 keeps it where it matters: one exact int32 sum t per (element, r, 32-k block),
// then acc += (t * sa) * sb over (r, block) from 0, and C = (beta0 ? 0 : C) + acc (F32) or bf16_rne(bf16(C or 0) + acc) (BF16).
// A layouts (bytes; s = k/4, g = k/8, q = k%4):
//   I2X4   A[s*lda + (i % (m/4))*4 + q], the 2-bit code of row i in bit pair i / (m/4); codes 0, 1, 2, 3 -> 0, +1, -1, -1 (:19-57)
//   I1X8   A[s*lda/2 + i/2], bit q of the low nibble (even i) or of the high nibble (odd i); clear -> +1, set -> -1
//   MXFP4  A[g*lda*4 + i*4 + q], low nibble k = 8g+q, high nibble k = 8g+q+4, widened by the integer table of :67 (not e2m1)
// B is [n][ldb] bytes. MXFP4 scales: A's E8M0 bytes [k/32][lda] widened as s << 23, B's f32 [n][ldb/32]; block r of a batch-reduce
// moves them as :200-236 does (address: arrays of br pointers; offset: + offs_a*2/32 bytes and + offs_b/32 floats; stride likewise).
// One CTA per tile. A thread owns one row and LB_E consecutive columns, so each A word is expanded once and used LB_E times. B goes
// through shared memory in panels of LB_NB columns x LB_KC k: the CTA reads B once per pass over its rows.
constexpr int LB_E = 16, LB_KC = 128, LB_NB = 256, LB_THREADS = 256, LB_SW = LB_KC / 4 + 1;   // LB_SW: panel row stride in words

__device__ __forceinline__ unsigned int lb_ld4(const unsigned char* p, bool aligned) {
  if (aligned) return *reinterpret_cast<const unsigned int*>(p);
  return (unsigned int)p[0] | ((unsigned int)p[1] << 8) | ((unsigned int)p[2] << 16) | ((unsigned int)p[3] << 24);
}
// byte q of w holds a 2-bit code in its low bits -> int8 0, +1, -1, -1 for codes 0, 1, 2, 3
__device__ __forceinline__ unsigned int lb_expand_i2(unsigned int w) {
  return (((w >> 1) & 0x01010101u) * 0xffu) | (w & 0x01010101u);
}
// bit q of x -> int8 +1 (clear) or -1 (set) in byte q
__device__ __forceinline__ unsigned int lb_expand_i1(unsigned int x) {
  const unsigned int w = (x & 1u) | ((x & 2u) << 7) | ((x & 4u) << 14) | ((x & 8u) << 21);
  return 0x01010101u | (w * 0xfeu);
}
// byte q of w holds an fp4 code in its low nibble -> int8 of {0, 11, 21, 32, 42, 64, 85, 127}, negated when bit 3 is set
__device__ __forceinline__ unsigned int lb_expand_fp4(unsigned int w) {
  unsigned int sel = w & 0x07070707u;
  sel = (sel | (sel >> 4)) & 0x00ff00ffu;
  sel = (sel | (sel >> 8)) & 0x0000ffffu;                        // one prmt selector nibble per byte
  const unsigned int mag = __byte_perm(0x20150b00u, 0x7f55402au, sel);
  const unsigned int neg = ((w >> 3) & 0x01010101u) * 0xffu;
  return (__vneg4(mag) & neg) | (mag & ~neg);
}

template <int FORM, bool UB, bool GRID>
__global__ void __launch_bounds__(LB_THREADS) gemm_lowbit_kernel(const xb_gemm_launch L) {
  __shared__ unsigned int sb[LB_NB * LB_SW];
  const xb_gemm_desc& d = L.d;
  const int m = d.m, n = d.n, k = d.k, m4 = d.m / 4;
  const long long lda = d.lda, ldb = d.ldb, ldc = d.ldc;
  const bool beta0 = (d.flags & LIBXSMM_GEMM_FLAG_BETA_0) != 0;
  for (long long t = blockIdx.x; t < L.count; t += gridDim.x) {
    TileCtx x; resolve_tile<GRID>(L, t, x);
    const unsigned char* as = x.a_s; const float* bs = (const float*)x.b_s;   // MXFP4 block scales (address mode: arrays of br pointers)
    for (int j0 = 0; j0 < n; j0 += LB_NB) {
      const int nb = (n - j0 < LB_NB) ? n - j0 : LB_NB;
      const int items = m * ((nb + LB_E - 1) / LB_E);
      for (int w0 = 0; w0 < items; w0 += LB_THREADS) {
        const int w = w0 + (int)threadIdx.x;
        const bool live = w < items;
        const int i = live ? w % m : 0, jg = live ? (w / m) * LB_E : 0;   // row; first column of the group within the panel
        unsigned int acc[LB_E];                                          // I2 / I1: the sums; MXFP4: the block sums
        float facc[LB_E];
#pragma unroll
        for (int p = 0; p < LB_E; ++p) { acc[p] = 0u; facc[p] = 0.0f; }
        for (unsigned long long r = 0; r < x.br; ++r) {
          const char *pa, *pb; br_ptrs(d, x, r, 1, 1, pa, pb);
          const unsigned char* ua = (const unsigned char*)pa;
          const unsigned char* psa = nullptr; const float* psb = nullptr;
          if (FORM == XB_LB_MXFP4) {
            switch (d.br_type) {
              case 1: psa = ((const unsigned char* const*)as)[r]; psb = ((const float* const*)bs)[r]; break;
              case 2: psa = as + (x.a_offs[r] * 2) / 32; psb = bs + x.b_offs[r] / 32; break;
              case 3: psa = as + ((d.br_stride_a * 2) / 32) * (long long)r; psb = bs + (d.br_stride_b / 32) * (long long)r; break;
              default: psa = as; psb = bs;
            }
          }
          const bool b_al = (((uintptr_t)pb | (uintptr_t)ldb) & 3) == 0;
          const bool a_al = (FORM == XB_LB_MXFP4) ? (((uintptr_t)ua & 3) == 0) : ((((uintptr_t)ua | (uintptr_t)lda) & 3) == 0);
          for (int k0 = 0; k0 < k; k0 += LB_KC) {
            const int kw = ((k - k0 < LB_KC) ? k - k0 : LB_KC) / 4;       // words of k in this panel
            __syncthreads();                                              // the previous panel is consumed
            for (int e = threadIdx.x; e < nb * kw; e += LB_THREADS) {
              const int jj = e / kw, q = e - jj * kw;
              sb[jj * LB_SW + q] = lb_ld4((const unsigned char*)pb + (long long)(j0 + jj) * ldb + k0 + 4 * q, b_al);
            }
            __syncthreads();
            if (!live) continue;
            const unsigned int* sbj = sb + jg * LB_SW;                    // columns past nb read stale words that are never stored
            if (FORM == XB_LB_MXFP4) {
              for (int bl = 0; bl < kw / 8; ++bl) {
                const long long sblk = k0 / 32 + bl;
#pragma unroll
                for (int p = 0; p < LB_E; ++p) acc[p] = 0u;
#pragma unroll
                for (int g8 = 0; g8 < 4; ++g8) {
                  const unsigned int word = lb_ld4(ua + (sblk * 4 + g8) * lda * 4 + (long long)i * 4, a_al);
                  const unsigned int lo = lb_expand_fp4(word & 0x0f0f0f0fu), hi = lb_expand_fp4((word >> 4) & 0x0f0f0f0fu);
                  const int qw = bl * 8 + g8 * 2;
#pragma unroll
                  for (int p = 0; p < LB_E; ++p) {
                    acc[p] = dp4a_x<false, false>(lo, sbj[p * LB_SW + qw], acc[p]);
                    acc[p] = dp4a_x<false, false>(hi, sbj[p * LB_SW + qw + 1], acc[p]);
                  }
                }
                const float sa = mx_scale(psa[sblk * lda + i]);
#pragma unroll
                for (int p = 0; p < LB_E; ++p) {
                  const int j = j0 + jg + p;
                  if (j < n) facc[p] = __fadd_rn(facc[p], __fmul_rn(__fmul_rn((float)(int)acc[p], sa), psb[(long long)j * (ldb / 32) + sblk]));
                }
              }
            } else {
              for (int q = 0; q < kw; ++q) {
                const long long s = k0 / 4 + q;
                unsigned int av;
                if (FORM == XB_LB_I2) av = lb_expand_i2((lb_ld4(ua + s * lda + (long long)(i % m4) * 4, a_al) >> (2 * (i / m4))) & 0x03030303u);
                else av = lb_expand_i1((unsigned int)(ua[(s * lda) / 2 + i / 2] >> (4 * (i & 1))) & 0xfu);
#pragma unroll
                for (int p = 0; p < LB_E; ++p) acc[p] = dp4a_x<false, UB>(av, sbj[p * LB_SW + q], acc[p]);
              }
            }
          }
        }
        if (!live) continue;
#pragma unroll
        for (int p = 0; p < LB_E; ++p) {
          const int j = j0 + jg + p;
          if (j >= n) break;
          const long long ci = (long long)j * ldc + i;
          if (FORM != XB_LB_MXFP4) {
            unsigned int v = acc[p];
            if (!beta0) v += (unsigned int)reinterpret_cast<const int*>(x.c)[ci];
            reinterpret_cast<int*>(x.c)[ci] = (int)v;
          } else if (d.tc == LIBXSMM_DATATYPE_F32) {
            float* c = reinterpret_cast<float*>(x.c) + ci;
            *c = __fadd_rn(beta0 ? 0.0f : *c, facc[p]);
          } else {
            unsigned short* c = reinterpret_cast<unsigned short*>(x.c) + ci;
            *c = xb_f32_to_bf16_rne(__fadd_rn(beta0 ? 0.0f : xb_bf16_to_f32(*c), facc[p]));
          }
        }
      }
    }
  }
}

template <bool GRID>
void launch_lowbit_g(const xb_gemm_launch& L, unsigned int grid, cudaStream_t st) {
  const int form = xb_lowbit_form(&L.d);
  const bool ub = (L.d.tb == LIBXSMM_DATATYPE_U8);
  if (form == XB_LB_I2 && ub) gemm_lowbit_kernel<XB_LB_I2, true, GRID><<<grid, LB_THREADS, 0, st>>>(L);
  else if (form == XB_LB_I2) gemm_lowbit_kernel<XB_LB_I2, false, GRID><<<grid, LB_THREADS, 0, st>>>(L);
  else if (form == XB_LB_I1 && ub) gemm_lowbit_kernel<XB_LB_I1, true, GRID><<<grid, LB_THREADS, 0, st>>>(L);
  else if (form == XB_LB_I1) gemm_lowbit_kernel<XB_LB_I1, false, GRID><<<grid, LB_THREADS, 0, st>>>(L);
  else gemm_lowbit_kernel<XB_LB_MXFP4, false, false><<<grid, LB_THREADS, 0, st>>>(L);   // side operands: never a grid
}

void launch_lowbit(const xb_gemm_launch& L, unsigned int grid, cudaStream_t st) {
  if (L.grid_m > 0) launch_lowbit_g<true>(L, grid, st); else launch_lowbit_g<false>(L, grid, st);
}

// after a launch: counts it and notes a launch error
int launched(const char* what) {
  xb_rt_count_launch_backend(LIBXSMM_B200_BACKEND_SIMT);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { xb_rt_note_error((int)e, what); return (int)e; }
  return 0;
}
}  // namespace

extern "C" int xb_gemm_simt_launch(const xb_gemm_launch* L) {
  const int path = L->d.path;
  if (path == XB_PATH_NONE) return 1;
  if (L->count <= 0) return 0;
  if (L->recs == nullptr && xb_gemm_rec_lacks(&L->one, xb_gemm_sides(&L->d))) {
    xb_rt_note_error(1, "GEMM: side operand missing (scales in a/b/c.tertiary, zero points in a.quaternary)"); return 1;
  }
  cudaStream_t st = (cudaStream_t)xb_rt_stream();
  const unsigned int grid = (unsigned int)(L->count < (1 << 20) ? L->count : (1 << 20));   // one CTA per tile, grid-stride beyond
  if (path == P_BITMAP) {
    if (L->count != 1 || L->recs != nullptr || L->one.a_q == nullptr) { xb_rt_note_error(1, "bitmap-compressed A: single calls only"); return 1; }
    unsigned int* prefix = (unsigned int*)xb_rt_scratch((size_t)(((long long)L->d.m * L->d.k + 31) / 32) * 4 + 16);
    if (prefix == nullptr) return 2;
    gemm_bitmap_kernel<<<1, 1024, 0, st>>>(*L, prefix);
    return launched("gemm_bitmap");
  }
  if (path == P_MX8) {
    float* img = nullptr;                        // MXBF8 C: f32 image in the caller's scratch arena (reset after the sync)
    if (L->d.tc == LIBXSMM_DATATYPE_MXBF8 && nullptr == (img = (float*)xb_rt_scratch((size_t)L->count * L->d.m * L->d.n * 4))) return 2;
    gemm_mx8_kernel<<<grid, 256, 0, st>>>(*L, img);
    const int rc = launched("gemm_mx8");
    if (rc != 0 || img == nullptr) return rc;
    const long long blocks = L->count * L->d.n * (L->d.m / 32);
    gemm_mx8_quant_kernel<<<(unsigned int)((blocks + 127) / 128), 128, 0, st>>>(*L, img);
    return launched("gemm_mx8_quant");
  }
  if (path == P_DQ) {
    if (L->grid_m > 0) gemm_dq_kernel<true><<<grid, 256, 0, st>>>(*L); else gemm_dq_kernel<false><<<grid, 256, 0, st>>>(*L);
    return launched("gemm_dq");
  }
  if (path == P_LOWBIT) {
    launch_lowbit(*L, grid, st);
    return launched("gemm_lowbit");
  }
  if (L->d.fuse_colbias != 0 || L->d.cp_op != 0) {
    int bm, bn, per_tile; fuse_blocks(L->d.m, L->d.n, bm, bn, per_tile);
    const long long blocks = L->count * per_tile;
    gemm_fused_kernel<<<(unsigned int)(blocks < FB_MAX_CTAS ? blocks : FB_MAX_CTAS), FB_THREADS, 0, st>>>(*L, path);
    return launched("gemm_fused");
  }
  if (i8_fast_ok(*L, path) && getenv("LIBXSMM_B200_I8_EXACT_ORDER") == nullptr) {
    const int small = (L->d.m < L->d.n) ? L->d.m : L->d.n;
    const int tm = (small >= 32) ? 4 : ((small >= 16) ? 2 : 1), tn = 2 * tm;           // lane block; a warp covers 8*tm x 4*tn of C
    const int passes = ((L->d.m + 8 * tm - 1) / (8 * tm)) * ((L->d.n + 4 * tn - 1) / (4 * tn));
    int wpt = 1; while (wpt < passes) wpt *= 2;                                        // warps per tile: 1, 2, 4, 8 or 16
    const int kcq = (L->d.k / 4 < I8_KC / 4) ? L->d.k / 4 : I8_KC / 4;
    // panels [kcq][ms] + [kcq][ns] (+ slack: a 4x8 lane block may read up to 31 padding words past the last row)
    const int words = kcq * (((((L->d.m + 3) >> 2) | 1) << 2) + ((((L->d.n + 3) >> 2) | 1) << 2)) + 64;
    const int groups = I8_WARPS / (wpt > I8_WARPS ? I8_WARPS : wpt);
    const size_t smem = (size_t)words * 4 * groups;
    if (wpt <= I8_WARPS && smem <= 200 * 1024) {
      static int sms = 0;
      if (sms == 0) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms <= 0) sms = 132; }
      const long long ctas_needed = (L->count + groups - 1) / groups;
      long long per_sm = (long long)((220 * 1024) / (smem + 1024)); if (per_sm < 1) per_sm = 1; if (per_sm > 2) per_sm = 2;   // 64 registers x 512 threads: two CTAs per SM
      long long i8_grid = (long long)sms * per_sm;
      if (i8_grid > ctas_needed) i8_grid = ctas_needed;
      if (tm == 4) launch_i8<4, 8>(*L, path, wpt, words, smem, (unsigned int)i8_grid, st);
      else if (tm == 2) launch_i8<2, 4>(*L, path, wpt, words, smem, (unsigned int)i8_grid, st);
      else launch_i8<1, 2>(*L, path, wpt, words, smem, (unsigned int)i8_grid, st);
      return launched("gemm_i8");
    }
  }
  if (L->grid_m > 0) gemm_simt_kernel<true><<<grid, 256, 0, st>>>(*L, path); else gemm_simt_kernel<false><<<grid, 256, 0, st>>>(*L, path);
  return launched("gemm_simt");
}
