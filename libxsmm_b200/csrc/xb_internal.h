/* libxsmm_b200 internal interface between the plain-C host runtime (host_*.c) and the CUDA
 * translation units (*.cu). Everything crossing this boundary is C: plain structs and pointers.
 * The host side never includes a CUDA header; the .cu side never touches the registry. */
#ifndef XB_INTERNAL_H
#define XB_INTERNAL_H

#include "../../include/libxsmm.h"

#if defined(__cplusplus)
extern "C" {
#endif

#define XB_HIDDEN __attribute__((visibility("hidden")))

/* ---- kernel kinds held by a slot --------------------------------------------------------------- */
enum {
  XB_KIND_FREE = 0,
  XB_KIND_GEMM,          /* dense GEMM/BRGEMM (libxsmm_gemm_param) */
  XB_KIND_GEMM_EXT,      /* dense GEMM/BRGEMM with fused pre/post ops (libxsmm_gemm_ext_param) */
  XB_KIND_TILECFG,       /* callable no-op */
  XB_KIND_MELTW,         /* unary/binary/ternary eltwise */
  XB_KIND_SP_A_CSR,      /* packed: C[M][N][P] += A_csr * B[K][N][P] */
  XB_KIND_SP_B_CSR,      /* packed: C[M][N][P] += A[M][K][P] * B_csr */
  XB_KIND_SP_B_CSC,      /* packed: C[M][N][P] += A[M][K][P] * B_csc */
  XB_KIND_SP_C_CSC,      /* packed: C_csc pattern only */
  XB_KIND_BCSC,          /* packed block-sparse B */
  XB_KIND_SREG,          /* fsspmdm kernel: sparse A fixed at create time, row-major B/C */
  XB_KIND_PK_GEMM,       /* packed dense: C[N][M][P] += A[K][M][P] * B[N][K][P] */
  XB_KIND_PK_AC_RM,      /* packed dense: C[M][N][P] += A[M][K][P] * B[K][N] */
  XB_KIND_PK_BC_RM,      /* packed dense: C[M][N][P] += A[M][K] * B[K][N][P] */
  XB_KIND_MEQN           /* matrix equation: tree of mateltwise nodes (host_meqn.c), plan in u.sp.work */
};

/* normalised dense-GEMM descriptor == registry key for GEMM kinds (memcmp'd, so zero-filled) */
typedef struct xb_gemm_desc {
  int m, n, k, lda, ldb, ldc;
  int ta, tb, tc, tcomp;              /* libxsmm_datatype incl. signedness (I8 vs U8) */
  unsigned int flags;                 /* libxsmm_gemm_flags as completed by the init functions */
  int prefetch;
  int br_type;                        /* 0 none, 1 address, 2 offset, 3 stride */
  int br_unroll;
  long long br_stride_a, br_stride_b; /* bytes (stride mode) */
  /* fused ops (ext ABI): reference src/libxsmm_generator.c:297-321 */
  int fuse_colbias, d_type, ldd;      /* C += colbias (binary ADD with BCAST_COL) */
  int cp_op, cp_flags, ldcp;          /* unary on C: RELU (+bitmask) or SIGMOID */
  int backend;                        /* libxsmm_b200_backend chosen at dispatch */
  int pad_;
} xb_gemm_desc;

typedef struct xb_meltw_desc {
  int op_class;                       /* libxsmm_meltw_operation */
  int op;                             /* unary/binary/ternary type */
  unsigned int flags;
  int m, n, ldi, ldi2, ldi3, ldo;
  int t_in0, t_in1, t_in2, t_out, t_comp;
} xb_meltw_desc;

/* sparse kernels: pattern lives in device memory owned by the slot */
typedef struct xb_sparse_desc {
  int kind;                           /* XB_KIND_SP_* / BCSC / SREG */
  int m, n, k, lda, ldb, ldc;
  int ta, tb, tc, tcomp;
  unsigned int flags;
  int packed_width, bk, bn;
  int max_n;                          /* SREG: loop bound on N */
  unsigned int nnz, nrows;            /* rows of the pointer array (CSR: rows, CSC: cols) */
  /* device copies */
  unsigned int* d_ptr;                /* row_ptr / col_ptr  [nrows+1] */
  unsigned int* d_idx;                /* column / row indices [nnz] */
  void* d_val;                        /* SREG: values as the compute type [nnz] */
  int beta0;
  /* BCSC: per-(device, stream) scratch owned by the handle (pattern cache, re-packed B); created on first call, never
   * touched by the descriptor's readers (bcsc_tc.cu: BcscState) */
  void* work;
} xb_sparse_desc;

typedef struct xb_slot {
  int kind;                           /* XB_KIND_* (FREE when unused) */
  int registered;                     /* 1: owned by the registry, 0: caller-owned (create_*) */
  unsigned int nflops;
  union { xb_gemm_desc gemm; xb_meltw_desc meltw; xb_sparse_desc sp; } u;
} xb_slot;

/* ---- resolved per-tile record for dense GEMM kernels (device memory when count > 1) ------------ */
typedef struct xb_gemm_rec {
  const void* a;        /* base of A (addr mode: device array of br pointers) */
  const void* b;
  void* c;
  const void* a_aux;    /* offset mode: device array of br byte offsets (long long) */
  const void* b_aux;
  const void* d;        /* ext: colbias */
  void* c_aux;          /* ext: relu bitmask out */
  const void* a_q;      /* int4 A: zero points (a.quaternary); bitmap-compressed A: the bitmap (a.secondary) */
  unsigned long long br;
  float scf;            /* I8 x I8 -> F32 scalar scale */
  int pad_;
} xb_gemm_rec;

/* launch description handed to the CUDA side */
typedef struct xb_gemm_launch {
  xb_gemm_desc d;
  long long count;
  /* mode 0: uniform strided batch */
  const void* a; const void* b; void* c;
  long long tile_stride_a, tile_stride_b, tile_stride_c;   /* bytes */
  unsigned long long br;
  /* mode 1: per-tile records (device array of xb_gemm_rec[count]) */
  const xb_gemm_rec* recs;
  xb_gemm_rec one;      /* count==1 && !recs: passed by value */
} xb_gemm_launch;

/* ---- CUDA runtime layer (runtime.cu) ----------------------------------------------------------- */
int xb_rt_device_count(void);
int xb_rt_set_device(int ordinal);
void xb_rt_set_stream(void* stream);
void* xb_rt_stream(void);
void xb_rt_set_blocking(int on);
int xb_rt_blocking(void);
int xb_rt_sync(void);
int xb_rt_last_error(void);
const char* xb_rt_last_error_string(void);
void xb_rt_note_error(int code, const char* where);
unsigned long long xb_rt_launch_count(void);
void xb_rt_count_launch(void);
/* xb_rt_count_launch() plus one in the count of the kernel's family `backend` (libxsmm_b200_backend); the per-family counts and
 * libxsmm_b200_launch_count_backend live in runtime.cu next to the launchers that feed them */
void xb_rt_count_launch_backend(int backend);
void* xb_rt_device_malloc(size_t size);
void xb_rt_device_free(void* p);
void* xb_rt_host_malloc(size_t size);
void xb_rt_host_free(void* p);
void* xb_rt_managed_malloc(size_t size);
void xb_rt_managed_free(void* p);
int xb_rt_memcpy(void* dst, const void* src, size_t size);           /* blocking, any direction */
int xb_rt_memcpy_async(void* dst, const void* src, size_t size);     /* on the thread's stream */
int xb_rt_memcpy2d_async(void* dst, const void* src, size_t pitch, size_t width, size_t rows);   /* same pitch on both sides, any direction */
/* chunked host<->device pipeline (three streams, two staging slots); `launch` runs with the thread's stream switched
 * to the pipeline's compute stream and must only enqueue work */
typedef struct xb_pipe_chunk {
  const void* host_a; const void* host_b; void* host_c;
  size_t bytes_a, bytes_b, bytes_c;
  int copy_c_in;               /* C is read by the kernel (beta = 1, or gaps between tiles that must survive) */
  long long first, count;      /* units of the batch in this chunk */
} xb_pipe_chunk;
typedef void (*xb_pipe_describe_fn)(void* ctx, long long index, xb_pipe_chunk* out);
typedef int (*xb_pipe_launch_fn)(void* ctx, const xb_pipe_chunk* chunk, void* dev_a, void* dev_b, void* dev_c);
int xb_rt_pipeline(long long nchunks, size_t max_a, size_t max_b, size_t max_c, xb_pipe_describe_fn describe, xb_pipe_launch_fn launch, void* ctx);
int xb_rt_upload(void* dst_dev, const void* src_host, size_t size);  /* stream ordered from pageable */
/* 0: host (unregistered / pageable), 1: device, 2: managed, 3: pinned host */
int xb_rt_ptr_kind(const void* p);
int xb_rt_have_gpu(void);
/* scratch arena on the device, grown on demand, reset by the caller after sync */
void* xb_rt_scratch(size_t bytes);
int xb_rt_current_device(void);
int xb_rt_first_use_on_device(unsigned long long* mask);   /* 1 once per device ordinal */
void xb_rt_scratch_reset(void);

/* ---- kernel launchers (one per .cu file) ------------------------------------------------------- */
int xb_gemm_simt_launch(const xb_gemm_launch* L);
int xb_gemm_tc_supported(const xb_gemm_desc* d);          /* pure host logic, no CUDA call */
int xb_gemm_tc_launch(const xb_gemm_launch* L);
/* pooled address mode (gemm plan): block r of tile p is base + set[p]*set_stride + r*blk_stride; see gemm_tc.cu */
typedef struct xb_tc_pool {
  const void* base_a; const void* base_b; long long blk_a, blk_b, set_a, set_b, nsets_a, nsets_b;
  const void* sets;          /* device int4[items] {set of A, set of A of the second tile, set of B, 0}, sorted */
  const void* cptrs;         /* device char*[items] (pair: [2*items], second may be NULL): C tile(s) of every item */
  int pair;                  /* 1: an item is two tiles (m <= 64) sharing B, stacked into one M=128 instruction */
} xb_tc_pool;
int xb_gemm_tc_shape_ok(const xb_gemm_desc* d);           /* everything xb_gemm_tc_supported checks except the batch-reduce mode */
int xb_gemm_tc_launch_pooled(const xb_gemm_desc* d, const xb_tc_pool* pool, unsigned long long br, long long count);
int xb_gemm_ts_supported(const xb_gemm_desc* d);          /* VNNI-packed A as wgmma register fragments (gemm_tc.cu); pure host logic */
int xb_gemm_ts_launch(const xb_gemm_launch* L);
typedef struct xb_meltw_args {
  const void* in0; const void* in1; const void* in2; void* out;
  const void* in_aux;        /* unary in.secondary: bitmask in / index array / fwd output (ELU_INV) */
  void* out_aux;             /* unary out.secondary: bitmask out / argop indices / scatter index array */
  float alpha;               /* LEAKY_RELU/ELU alpha, QUANT/DEQUANT scale */
  unsigned long long n_rt;   /* REPLICATE_COL_VAR: run-time N; COLS_IDX reductions: number of indices */
  unsigned long long off[2]; /* UNZIP: byte offset of the high halves; DECOMP_FP32_TO_BF16X2/X3: byte strides of planes 2, 3 */
  void* rng;                 /* DROPOUT: 4 x 16 words of generator state (device copy, updated by the kernel) */
  float* rnd;                /* DROPOUT: scratch for the uniform numbers, 16 per group of rows */
  unsigned char* rnd8;       /* STOCHASTIC_ROUND to BF8: one random byte per element in the reference's visiting order (NULL: round to nearest) */
} xb_meltw_args;
void xb_invoke_meqn(const struct xb_slot* s, const void* param);
void xb_meqn_release(void* work);
int xb_meltw_supported(const xb_meltw_desc* d);                          /* pure host logic */
int xb_meltw_launch(const xb_meltw_desc* d, const xb_meltw_args* a);
int xb_sreg_launch(const xb_sparse_desc* d, const void* b, void* c, long long n_total);
int xb_packed_sp_launch(const xb_sparse_desc* d, const void* a, const void* b, void* c, long long count,
                        long long stride_a, long long stride_b, long long stride_c);
int xb_bcsc_launch(xb_sparse_desc* d, const void* a, const void* b_vals, const unsigned int* colptr,
                   const unsigned int* rowidx, unsigned long long n_blocks, unsigned int nnzb, void* c);
/* 0: exact-order CUDA-core kernel, 1: wgmma tensor-core kernel (bcsc_tc.cu) */
int xb_bcsc_tc_variant(const xb_sparse_desc* d, unsigned long long n_blocks);
void xb_bcsc_state_free(void* work);

/* ---- host runtime (host_core.c) ---------------------------------------------------------------- */
xb_slot* xb_slot_of(const void* fnptr);    /* NULL if not one of our thunks */
void xb_invoke(int slot, const void* param);
const void* xb_thunk(int slot);
#define XB_NTHUNKS 8192

#if defined(__cplusplus)
}
#endif
#endif /* XB_INTERNAL_H */
