// libxsmm_b200 -- accumulator write-back shared by the tensor-core GEMM kernels (gemm_tc.cu, bcsc_tc.cu).
// A thread holds its wgmma accumulator fragment; eight lanes cover eight consecutive rows of a column, so each store
// instruction of a warp writes full 32-byte sectors of the column-major C. Output type and beta are template parameters.
// Semantics per type follow libxsmm_ref_matmul (src/generator_gemm_reference_impl.c): f32 accumulate, one rounding at
// the end (:2367-2419 bf16, :2025-2126 f16), beta = 1 adds the old C in f32 (f16 inputs with f32 C round the old value
// through f16 first, :2118-2123), int32 wraps (:1452-1555), int8 -> f32 scales by scf (:1556-1683).
#ifndef XB_EPILOGUE_CUH
#define XB_EPILOGUE_CUH
#include "xb_device.cuh"

enum { XB_EP_F32 = 0, XB_EP_F32_FROM_F16 = 1, XB_EP_BF16 = 2, XB_EP_F16 = 3, XB_EP_I32 = 4, XB_EP_I32_TO_F32 = 5 };

template <int MODE, bool BETA0>
__device__ __forceinline__ void xb_ep_store_one(uint32_t raw, char* p, float scf) {
  if (MODE == XB_EP_F32 || MODE == XB_EP_F32_FROM_F16) {
    float acc = __uint_as_float(raw);
    float* d = reinterpret_cast<float*>(p);
    if (!BETA0) { float old = *d; if (MODE == XB_EP_F32_FROM_F16) old = xb_f16_to_f32(xb_f32_to_f16(old)); acc += old; }
    *d = acc;
  } else if (MODE == XB_EP_BF16) {
    float acc = __uint_as_float(raw);
    unsigned short* d = reinterpret_cast<unsigned short*>(p);
    if (!BETA0) acc += xb_bf16_to_f32(*d);
    *d = xb_f32_to_bf16_rne(acc);
  } else if (MODE == XB_EP_F16) {
    float acc = __uint_as_float(raw);
    unsigned short* d = reinterpret_cast<unsigned short*>(p);
    if (!BETA0) acc += xb_f16_to_f32(*d);
    *d = xb_f32_to_f16(acc);
  } else if (MODE == XB_EP_I32) {
    unsigned int* d = reinterpret_cast<unsigned int*>(p);
    *d = BETA0 ? raw : raw + *d;
  } else {
    float* d = reinterpret_cast<float*>(p);
    float f = __fmul_rn((float)(int)raw, scf);
    if (!BETA0) f = __fadd_rn(f, *d);
    *d = f;
  }
}

// one warpgroup's m64 x NC accumulator fragment (xb_wgmma.cuh layout) -> C tile. ctile: column-major C of the tile, rows
// row0 .. row0 + 63 of it are this warpgroup's, col0 is the fragment's first column; only rows < m and columns < n are stored.
template <int MODE, bool BETA0, int R>
__device__ __forceinline__ void xb_ep_store_frag_t(const uint32_t (&v)[R], char* ctile, int row0, int col0, int m, int n, long long ldc_bytes, int esz, float scf) {
  const int lane = threadIdx.x & 31, r = row0 + 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2), c = col0 + 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < R; ++i) {
    const int row = r + 8 * ((i >> 1) & 1), col = c + 8 * (i >> 2) + (i & 1);
    if (row < m && col < n) xb_ep_store_one<MODE, BETA0>(v[i], ctile + (long long)col * ldc_bytes + (long long)row * esz, scf);
  }
}

template <int R>
__device__ __forceinline__ void xb_ep_store_frag(int mode, int beta0, const uint32_t (&v)[R], char* ctile, int row0, int col0, int m, int n, long long ldc_bytes, int esz, float scf) {
  switch (mode * 2 + (beta0 ? 1 : 0)) {
    case XB_EP_F32 * 2 + 0:          xb_ep_store_frag_t<XB_EP_F32, false>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_F32 * 2 + 1:          xb_ep_store_frag_t<XB_EP_F32, true>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_F32_FROM_F16 * 2 + 0: xb_ep_store_frag_t<XB_EP_F32_FROM_F16, false>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_F32_FROM_F16 * 2 + 1: xb_ep_store_frag_t<XB_EP_F32, true>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_BF16 * 2 + 0:         xb_ep_store_frag_t<XB_EP_BF16, false>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_BF16 * 2 + 1:         xb_ep_store_frag_t<XB_EP_BF16, true>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_F16 * 2 + 0:          xb_ep_store_frag_t<XB_EP_F16, false>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_F16 * 2 + 1:          xb_ep_store_frag_t<XB_EP_F16, true>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_I32 * 2 + 0:          xb_ep_store_frag_t<XB_EP_I32, false>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_I32 * 2 + 1:          xb_ep_store_frag_t<XB_EP_I32, true>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    case XB_EP_I32_TO_F32 * 2 + 0:   xb_ep_store_frag_t<XB_EP_I32_TO_F32, false>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
    default:                         xb_ep_store_frag_t<XB_EP_I32_TO_F32, true>(v, ctile, row0, col0, m, n, ldc_bytes, esz, scf); break;
  }
}

// host side: epilogue mode and C element size of a GEMM descriptor's (a type, c type) pair
static inline int xb_ep_mode(int a_type, int c_type, int* esz) {
  const int a8 = (a_type == LIBXSMM_DATATYPE_I8 || a_type == LIBXSMM_DATATYPE_U8);
  if (a8) { *esz = 4; return (c_type == LIBXSMM_DATATYPE_I32) ? XB_EP_I32 : XB_EP_I32_TO_F32; }
  if (c_type == LIBXSMM_DATATYPE_F32) { *esz = 4; return (a_type == LIBXSMM_DATATYPE_F16) ? XB_EP_F32_FROM_F16 : XB_EP_F32; }
  *esz = 2;
  return (c_type == LIBXSMM_DATATYPE_BF16) ? XB_EP_BF16 : XB_EP_F16;
}
#endif  // XB_EPILOGUE_CUH
