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
 * bit mask (libxsmm_dispatch_brgemm_ext), VNNI-packed C, and for the strided forms int8 -> f32 (the scale travels in c.tertiary
 * of a call); nothing is launched and C is left untouched */
#define LIBXSMM_B200_ERROR_NOT_BATCHABLE (-6)
LIBXSMM_API int libxsmm_b200_gemm_batch_strided(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  unsigned long long br_count, long long count);
/* the same batch spread over the first `ndevices` GPUs of this process (contiguous ranges, one worker thread and one PCIe link per
 * device, no exchange between devices); operands must be host memory (pageable or pinned). Returns 0 or the first error. */
LIBXSMM_API int libxsmm_b200_gemm_batch_strided_multi(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  unsigned long long br_count, long long count, int ndevices);
/* general form: one reference argument struct per tile (address/offset batch-reduce modes, scale
 * factors...). All matrix pointers must be device-accessible. */
LIBXSMM_API int libxsmm_b200_gemm_batch(libxsmm_gemmfunction kernel, const libxsmm_gemm_param* params, long long count);
/* prepared form of the above: resolve and upload once, replay many times */
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
