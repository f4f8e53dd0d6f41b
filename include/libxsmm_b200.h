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
/* Side operands: besides A, B and C, a call of some handles reads
 *   scales:      a.tertiary, b.tertiary, c.tertiary -- MXBF8 / MXHF8: E8M0 block scales of A and B, and of an MXBF8 C;
 *                I8 x BF16, I8 / I4 / U4 x F16 (dequantising A): A's m row scales; MXFP4 x I8: A's E8M0 and B's f32 block scales
 *   zero points: a.quaternary -- I4 / U4 x F16 (f16, one per row) and I4 / U4 x I8 / U8 -> I32 (one byte per row and reduce step)
 * BF8 x F16 and I2 / I1 x I8 / U8 have none. Batch rules:
 *   - libxsmm_b200_gemm_batch_strided and _multi take no side operands: such a handle is not batchable there.
 *   - libxsmm_b200_gemm_batch_strided_scaled takes the scales of handles without zero points: scf_a, scf_b and scf_c stand for
 *     a.tertiary, b.tertiary and c.tertiary of tile 0, and tile t's are scf_x + t*stride_scf_x (BYTES; stride 0 shares one set, as
 *     a batch over one quantised weight does). It needs exactly the pointers the handle's scales name and reads no other.
 *   - libxsmm_b200_gemm_batch reads each tile's side operands from its argument struct, MX handles excepted (not batchable).
 *   - a plan (libxsmm_b200_gemm_plan_create) is NULL for a handle with side operands: they are per-call operands.
 * LIBXSMM_B200_ERROR_NOT_BATCHABLE is returned by every batch form (and a NULL plan) for a handle a batch cannot run like a single
 * call: a fused column bias or ReLU bit mask (libxsmm_dispatch_brgemm_ext), VNNI-packed C, side operands where the form takes none
 * (see above), and for the strided forms int8 -> f32 (the scale travels in c.tertiary of a call); nothing is launched and C is left
 * untouched */
#define LIBXSMM_B200_ERROR_NOT_BATCHABLE (-6)
LIBXSMM_API int libxsmm_b200_gemm_batch_strided(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  unsigned long long br_count, long long count);
/* the same batch spread over the first `ndevices` GPUs of this process (contiguous ranges, one worker thread and one PCIe link per
 * device, no exchange between devices); operands must be host memory (pageable or pinned). Returns 0 or the first error. */
LIBXSMM_API int libxsmm_b200_gemm_batch_strided_multi(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  unsigned long long br_count, long long count, int ndevices);
/* the strided batch of a handle with scales (see "Side operands" above). -1 for a handle without scales or with zero points, or a
 * NULL operand or scale pointer the handle needs; -2 for address / offset batch-reduce (per-tile arrays: libxsmm_b200_gemm_batch);
 * -4 if an operand or scale is pageable host memory (device-accessible only). An MXBF8 C is quantised from an f32 image in device
 * scratch: the batch then runs in chunks of at most 64 MiB of image and the call returns after the device has finished. */
LIBXSMM_API int libxsmm_b200_gemm_batch_strided_scaled(libxsmm_gemmfunction kernel,
  const void* a, const void* b, void* c, long long stride_a, long long stride_b, long long stride_c,
  const void* scf_a, const void* scf_b, void* scf_c, long long stride_scf_a, long long stride_scf_b, long long stride_scf_c,
  unsigned long long br_count, long long count);
/* general form: one reference argument struct per tile (address/offset batch-reduce modes, scale
 * factors, side operands; MXFP4 x I8 in address mode: arrays of br scale pointers). All matrix pointers must be device-accessible.
 * -1 if a tile lacks a side operand of the handle. */
LIBXSMM_API int libxsmm_b200_gemm_batch(libxsmm_gemmfunction kernel, const libxsmm_gemm_param* params, long long count);
/* prepared form of the above: resolve and upload once, replay many times (NULL for handles with side operands) */
typedef struct libxsmm_b200_gemm_plan libxsmm_b200_gemm_plan;
LIBXSMM_API libxsmm_b200_gemm_plan* libxsmm_b200_gemm_plan_create(libxsmm_gemmfunction kernel,
  const libxsmm_gemm_param* params, long long count);
LIBXSMM_API int libxsmm_b200_gemm_plan_run(const libxsmm_b200_gemm_plan* plan);
/* 1 if the plan walks a regular pool of block-sets on the tensor-core kernel (address batch-reduce, see DESIGN.md 3.1), else 0 */
LIBXSMM_API int libxsmm_b200_gemm_plan_is_pooled(const libxsmm_b200_gemm_plan* plan);
LIBXSMM_API void libxsmm_b200_gemm_plan_destroy(libxsmm_b200_gemm_plan* plan);

/* ---- batched matrix-eltwise and matrix equations -----------------------------------------------
 * count calls of one handle in one launch (an equation: one launch per node). Call t is the single call with every pointer of
 * *param advanced by t times its stride (BYTES; 0 = one operand shared by every call). Values a single call reads by value are
 * read once, from call 0: op.primary (alpha, drop probability) and the QUANT / DEQUANT scale in in.secondary. Returns 0; -1 for a
 * NULL or foreign handle, count < 0, a negative stride, or an output stride smaller than the bytes one call writes through that
 * pointer; -4 if an operand is pageable host memory (device, managed or pinned only); LIBXSMM_B200_ERROR_NOT_BATCHABLE for calls
 * with per-call state or run-time extents: DROPOUT forward, STOCHASTIC_ROUND, REPLICATE_COL_VAR, GATHER / SCATTER, the COLS_IDX
 * reductions, UNZIP and DECOMP_FP32_TO_BF16X2 / X3 (and an equation holding one); the positive CUDA error (2: out of device
 * scratch) if a launch fails. count == 0 does nothing. The meltw form honours
 * libxsmm_b200_set_blocking; the equation form returns after the device has finished, like a single equation call. */
typedef struct libxsmm_b200_meltw_strides {
  long long in0, in1, in2;   /* in.primary (unary) / in0, in1, in2 .primary */
  long long in_aux;          /* unary in.secondary: bit mask (RELU_INV, LEAKY_RELU_INV, DROPOUT_INV), forward output (ELU_INV) */
  long long out, out_aux;    /* out.primary; unary out.secondary: bit mask, argop indices, MX block scales, DUMP copy */
} libxsmm_b200_meltw_strides;
LIBXSMM_API int libxsmm_b200_meltw_batch_strided(const void* kernel, const void* param,
  const libxsmm_b200_meltw_strides* strides, long long count);
/* input_strides[i] applies to inputs[i], ops_strides[pos] to the ops_args[pos].primary a DUMP writes (NULL without DUMP),
 * output_aux_stride to the relu bit mask of the head (output.secondary); an argument a DUMP writes must have the DUMP's stride (-1
 * otherwise), and a NULL input is -1. Temporaries live in one device scratch block per chunk; past 64 MiB of them
 * the calls run in chunks, each one launch per node. */
LIBXSMM_API int libxsmm_b200_meqn_batch_strided(libxsmm_meqn_function kernel, const libxsmm_meqn_param* param,
  const long long* input_strides, long long output_stride, long long output_aux_stride,
  const long long* ops_strides, long long count);

/* ---- batched packed-sparse, packed-dense and BCSC calls ----------------------------------------
 * count calls of one libxsmm_create_packed_spgemm_csr / _csc, libxsmm_create_packed_gemm / _ac_rm / _bc_rm or
 * libxsmm_create_packed_spgemm_bcsc handle in one launch. Call t is kernel(param) with a.primary, b.primary (BCSC: the block
 * values) and c.primary advanced by t times their stride (BYTES; 0 = one operand shared by every call). Everything else in *param
 * is read once, from call 0, and shared: for BCSC the pattern (b.secondary colptr, b.tertiary rowidx, b.quaternary block-column
 * count), which may be device-resident or host memory (then staged once). Returns 0; -1 for a NULL or foreign handle, count < 0,
 * a NULL operand or pattern, a negative stride, a stride that is not a multiple of its operand's element size, or a C stride
 * smaller than the bytes one call writes through C (outputs of consecutive calls would overlap); -4 if A, B or C is pageable host
 * memory (device, managed or pinned only); LIBXSMM_B200_ERROR_NOT_BATCHABLE for fsspmdm handles
 * (libxsmm_create_spgemm_csr_areg), whose single call already covers every column of B; the positive CUDA error if a launch fails.
 * count == 0 does nothing. Honours libxsmm_b200_set_blocking. A BCSC batch takes the kernel libxsmm_b200_bcsc_variant names for
 * its call 0 when its strides are multiples of 16 bytes; otherwise the exact-order kernel (libxsmm_b200_launch_count_backend
 * tells which ran). */
typedef struct libxsmm_b200_spgemm_strides { long long a, b, c; } libxsmm_b200_spgemm_strides;
LIBXSMM_API int libxsmm_b200_spgemm_batch_strided(libxsmm_gemmfunction kernel, const libxsmm_gemm_param* param,
  const libxsmm_b200_spgemm_strides* strides, long long count);

#if defined(__cplusplus)
}
#endif
#endif /* LIBXSMM_B200_H */
