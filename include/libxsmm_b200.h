/* libxsmm_b200 -- additive GPU entry points (not part of the reference API).
 *
 * The reference invokes one tile per function-pointer call from a host loop
 * (samples/xgemm/gemm_kernel.c:3179-3259, samples/magazine/magazine_xsmm.c:110-140). On a GPU one
 * launch per 64^3 tile cannot approach any roofline, so the batch loop itself becomes ONE launch.
 * Nothing here changes the meaning of a reference symbol.
 *
 * Pointer rules: every matrix pointer may be a device pointer, a managed pointer
 * (libxsmm_aligned_malloc) or a plain host pointer. Host pointers are staged through device scratch
 * inside the call (H2D, kernel, D2H), which is what the "e2e" number of bench.py measures.
 * Argument structs, batch-reduce counts and address/offset arrays are always read on the host.
 */
#ifndef LIBXSMM_B200_H
#define LIBXSMM_B200_H

#include "libxsmm_typedefs.h"
#include "libxsmm_fsspmdm.h"

#if defined(__cplusplus)
extern "C" {
#endif

/* kernel families a handle can be bound to (libxsmm_b200_kernel_backend) */
typedef enum libxsmm_b200_backend {
  LIBXSMM_B200_BACKEND_NONE = 0,
  LIBXSMM_B200_BACKEND_SIMT = 1,        /* exact-order CUDA-core kernel (all dtypes/layouts) */
  LIBXSMM_B200_BACKEND_TCGEN05 = 2,     /* tensor-core tile kernel: TMA -> SMEM -> wgmma.mma_async -> registers (sm_90a) */
  LIBXSMM_B200_BACKEND_STREAM = 3,      /* HBM-streaming kernels (fsspmdm, packed sparse, meltw) */
  LIBXSMM_B200_BACKEND_NOOP = 4         /* tile-config handles */
} libxsmm_b200_backend;

/* ---- device, stream, synchronisation ---------------------------------------------------------- */
LIBXSMM_API int libxsmm_b200_device_count(void);
LIBXSMM_API int libxsmm_b200_set_device(int ordinal);          /* calling thread; 0 on success */
LIBXSMM_API void libxsmm_b200_set_stream(void* cuda_stream);   /* calling thread; NULL = default stream */
/* 1 (default): a handle returns after its kernel completed (reference semantics);
 * 0: stream ordered, caller synchronises with libxsmm_b200_sync(). */
LIBXSMM_API void libxsmm_b200_set_blocking(int blocking);
LIBXSMM_API int libxsmm_b200_sync(void);                       /* 0, or the sticky CUDA error */
LIBXSMM_API int libxsmm_b200_last_error(void);
LIBXSMM_API const char* libxsmm_b200_last_error_string(void);
LIBXSMM_API unsigned long long libxsmm_b200_launch_count(void); /* kernels launched by this library */
/* the same, counted per kernel family: TCGEN05 (wgmma GEMM and BCSC kernels), SIMT (exact-order GEMM, int8 dp4a, bitmap-A and
 * BCSC kernels), STREAM (everything else); tells which kernel a call really ran, after any launch-time fallback */
LIBXSMM_API unsigned long long libxsmm_b200_launch_count_backend(int backend);
LIBXSMM_API int libxsmm_b200_kernel_backend(const void* kernel);
/* BCSC handles (libxsmm_create_packed_spgemm_bcsc): the kernel a call with `n_block_columns` (= *b.quaternary) takes:
 * 0 exact-order CUDA-core kernel, 1 wgmma tensor-core kernel; -1: not BCSC */
LIBXSMM_API int libxsmm_b200_bcsc_variant(const void* kernel, unsigned long long n_block_columns);
/* fsspmdm handles: the kernel libxsmm_fsspmdm_execute(handle, B, C) takes: 0 direct kernel (no shared-memory staging), S = 1..3 the
 * TMA-staged kernel with S shared-memory stages; -1: NULL handle. Pageable host B / C are answered for the device buffers they are
 * staged through. */
LIBXSMM_API int libxsmm_b200_fsspmdm_variant(const libxsmm_fsspmdm* handle, const void* B, const void* C);
/* matrix-eltwise handles: the kernel a call with this libxsmm_meltw_unary_param (NULL: aligned device operands) runs. 0 generic
 * transform, 1 tiled transpose, 2 VNNI pack, 3 VNNI pack with 16-byte accesses, 4 warp reduction, 5 two-phase column reduction,
 * 6 two-phase column reduction with the float4 partial pass, 7 any other kernel (map, to-scalar, gather / scatter, quantisers,
 * dropout, unzip / decomp); -1: not a matrix-eltwise handle. Pageable operands are answered for the buffers they are staged through. */
LIBXSMM_API int libxsmm_b200_meltw_variant(const void* kernel, const void* param);
/* force the SIMT kernel for dense GEMM handles dispatched afterwards (debug / parity checking) */
LIBXSMM_API void libxsmm_b200_set_force_simt(int on);

/* ---- memory ----------------------------------------------------------------------------------- */
LIBXSMM_API void* libxsmm_b200_device_malloc(size_t size);
LIBXSMM_API void libxsmm_b200_device_free(void* ptr);
LIBXSMM_API void* libxsmm_b200_host_malloc(size_t size);       /* pinned */
LIBXSMM_API void libxsmm_b200_host_free(void* ptr);
LIBXSMM_API int libxsmm_b200_memcpy(void* dst, const void* src, size_t size); /* any direction, blocking */

/* ---- batched dense GEMM / BRGEMM ---------------------------------------------------------------
 * count independent invocations of `kernel` in one launch. Tile t uses
 *   A + t*stride_a, B + t*stride_b, C + t*stride_c          (strides in BYTES)
 * and, inside a tile, the handle's own batch-reduce addressing (stride mode: the dispatch-time
 * br_stride hints; br_count as given). Returns 0 on success. */
/* returned by every batch form (and a NULL plan) for a handle a batch cannot run like a single call: a fused column bias or ReLU
 * bit mask (libxsmm_dispatch_brgemm_ext), VNNI-packed C, MX handles (their block scales travel per call: use
 * libxsmm_b200_gemm_batch_strided_scaled), and for the strided forms int8 -> f32 (the scale travels in c.tertiary of a call) and
 * a dequantising A with row scales (I8 x BF16, I8 / I4 / U4 x F16: use libxsmm_b200_gemm_batch_strided_scaled or
 * libxsmm_b200_gemm_batch; BF8 x F16 has no scales and batches in every form); nothing is launched and C is left untouched */
#define LIBXSMM_B200_ERROR_NOT_BATCHABLE (-6)
LIBXSMM_API int libxsmm_b200_gemm_batch_strided(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  unsigned long long br_count, long long count);
/* the same batch spread over the first `ndevices` GPUs of this process (contiguous ranges, one worker thread and one PCIe link per
 * device, no exchange between devices); operands must be host memory (pageable or pinned). Returns 0 or the first error. */
LIBXSMM_API int libxsmm_b200_gemm_batch_strided_multi(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  unsigned long long br_count, long long count, int ndevices);
/* MX GEMM (MXBF8 / MXHF8 handles) over a strided batch: the E8M0 block scales of tile t are scf_a + t*stride_scf_a (a.tertiary
 * of a single call), scf_b + t*stride_scf_b (b.tertiary) and, for an MXBF8 C, scf_c + t*stride_scf_c (c.tertiary); strides in
 * BYTES. Also I8 x BF16 and I8 x F16 handles (dequantising A): the m row scales of tile t are scf_a + t*stride_scf_a (f32 next to
 * a bf16 B, f16 next to an f16 B); stride 0 shares one set of scales, as a batch over one quantised weight does; scf_b / scf_c are
 * not read; -2 for address / offset batch-reduce. An int4 A also needs zero points per tile: use libxsmm_b200_gemm_batch.
 * Every operand must be device-accessible (-4 for pageable host memory); -1 for a handle without per-call scales.
 * An MXBF8 C is quantised from an f32 image in device scratch: the batch then runs in chunks of at most 64 MiB of image and the
 * call returns after the device has finished. */
LIBXSMM_API int libxsmm_b200_gemm_batch_strided_scaled(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  const void* scf_a, const void* scf_b, void* scf_c, long long stride_scf_a, long long stride_scf_b, long long stride_scf_c,
  unsigned long long br_count, long long count);
/* general form: one reference argument struct per tile (address/offset batch-reduce modes, scale
 * factors...). All matrix pointers must be device-accessible. A dequantising A reads each tile's a.tertiary (row scales) and,
 * for I4 / U4, a.quaternary (f16 zero points); -1 if one is missing. */
LIBXSMM_API int libxsmm_b200_gemm_batch(libxsmm_gemmfunction kernel, const libxsmm_gemm_param* params, long long count);
/* prepared form of the above: resolve and upload once, replay many times (NULL for handles with per-call row scales) */
typedef struct libxsmm_b200_gemm_plan libxsmm_b200_gemm_plan;
LIBXSMM_API libxsmm_b200_gemm_plan* libxsmm_b200_gemm_plan_create(libxsmm_gemmfunction kernel,
  const libxsmm_gemm_param* params, long long count);
LIBXSMM_API int libxsmm_b200_gemm_plan_run(const libxsmm_b200_gemm_plan* plan);
/* 1 if the plan walks a regular pool of block-sets on the tensor-core kernel (address batch-reduce, see DESIGN.md 3.1), else 0 */
LIBXSMM_API int libxsmm_b200_gemm_plan_is_pooled(const libxsmm_b200_gemm_plan* plan);
LIBXSMM_API void libxsmm_b200_gemm_plan_destroy(libxsmm_b200_gemm_plan* plan);

#if defined(__cplusplus)
}
#endif
#endif /* LIBXSMM_B200_H */
