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
  int path;                           /* exact-order path (xb_gemm_path of the fields above), computed at dispatch */
} xb_gemm_desc;

/* the exact-order paths (gemm_simt.cu): the kernels take the path as a run-time argument and switch on it */
enum { P_F64 = 0, P_F32, P_I16, P_I8_I32, P_I8_F32, P_F16_F16, P_F16_F32, P_BF16_F32, P_BF16_BF16, P_I4_I32, P_BITMAP, P_FP8, P_MX8, P_DQ,
       XB_PATH_NONE, P_LOWBIT };

typedef struct xb_meltw_desc {
  int op_class;                       /* libxsmm_meltw_operation */
  int op;                             /* unary/binary/ternary type */
  unsigned int flags;
  int m, n, ldi, ldi2, ldi3, ldo;
  int t_in0, t_in1, t_in2, t_out, t_comp;
} xb_meltw_desc;

/* call axis of a strided batch of sparse calls (libxsmm_b200_spgemm_batch_strided): `count` calls, call t with A, the B values and C
 * advanced by t times their byte strides; 0 or 1 is a single call. The pattern and everything else are shared by the calls. */
typedef struct xb_sparse_calls { long long count, s_a, s_b, s_c; } xb_sparse_calls;

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
  /* BCSC: zero in a handle; a batch hands xb_bcsc_launch a copy of the descriptor with its call axis here, so the handle itself
   * is never written and stays re-entrant */
  xb_sparse_calls calls;
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
  const void* a_q;      /* int4 A: zero points (a.quaternary: bytes next to an 8-bit B, m f16 next to an f16 B); bitmap-compressed A:
                         * the bitmap (a.secondary) */
  unsigned long long br;
  float scf;            /* I8 x I8 -> F32 scalar scale */
  int pad_;
  /* MXBF8 / MXHF8: E8M0 block scales, one byte per (row, 32 k); a.tertiary [br][k/32][lda], b.tertiary [br][k/32][ldb],
   * and for an MXBF8 C c.tertiary [n][ldc/32]. Dequantising A (xb_dq_form): a_s holds the m row scales of a.tertiary. MXFP4 x I8
   * (xb_lowbit_form): a_s the E8M0 bytes of a.tertiary, b_s the f32 scales of b.tertiary (address mode: device arrays of br pointers). */
  const void* a_s; const void* b_s; void* c_s;
} xb_gemm_rec;

/* dequantising GEMM: a narrow A widened to B's 16-bit float type inside the kernel, with per-row scales (and, for int4, zero
 * points) of the call (reference src/generator_gemm_reference_impl.c:1684-2024). The form of a descriptor by its types, or 0.
 * U8 A is not a form: the reference reads those bytes as signed char (:1703, :1907, :1979), so a U8 caller would get the
 * results of the I8 bytes; dispatch declines it instead. */
enum { XB_DQ_NONE = 0, XB_DQ_I8_BF16, XB_DQ_I8_F16, XB_DQ_I4_F16, XB_DQ_BF8_F16 };
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline int xb_dq_form(const xb_gemm_desc* d) {
  const int f16comp = (d->tcomp == LIBXSMM_DATATYPE_F16 || d->tcomp == LIBXSMM_DATATYPE_F32 || d->tcomp == LIBXSMM_DATATYPE_IMPLICIT);
  if (d->ta == LIBXSMM_DATATYPE_I8 && d->tb == LIBXSMM_DATATYPE_BF16) {            /* :1684-1730, comp F32 */
    return (d->tcomp == LIBXSMM_DATATYPE_F32 && (d->tc == LIBXSMM_DATATYPE_F32 || d->tc == LIBXSMM_DATATYPE_BF16)) ? XB_DQ_I8_BF16 : XB_DQ_NONE;
  }
  if (d->tb != LIBXSMM_DATATYPE_F16 || !f16comp || (d->tc != LIBXSMM_DATATYPE_F16 && d->tc != LIBXSMM_DATATYPE_F32)) return XB_DQ_NONE;
  if (d->ta == LIBXSMM_DATATYPE_I8) return XB_DQ_I8_F16;                                                 /* :1881-2024 */
  if (d->ta == LIBXSMM_DATATYPE_I4X2 || d->ta == LIBXSMM_DATATYPE_U4X2) return XB_DQ_I4_F16;             /* :1793-1880 */
  if (d->ta == LIBXSMM_DATATYPE_BF8) return XB_DQ_BF8_F16;                                               /* :1731-1792 */
  return XB_DQ_NONE;
}

/* low-bit weights x 8-bit activations with an int32 comp (reference src/generator_gemm_reference_impl.c:1009-1272): ternary I2X4 and
 * binary I1X8 A next to an I8 or U8 B -> I32, and MXFP4X2 A (E8M0 block scales in a.tertiary) next to an I8 B (f32 block scales in
 * b.tertiary) -> F32 or BF16. The form of a descriptor by its types, or 0. MXFP4 x U8 is not a form: the reference reads those bytes
 * as signed char (:1011) under a B type it calls unsigned, so dispatch declines it. */
enum { XB_LB_NONE = 0, XB_LB_I2, XB_LB_I1, XB_LB_MXFP4 };
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline int xb_lowbit_form(const xb_gemm_desc* d) {
  const int b8 = (d->tb == LIBXSMM_DATATYPE_I8 || d->tb == LIBXSMM_DATATYPE_U8);
  if (d->tcomp != LIBXSMM_DATATYPE_I32) return XB_LB_NONE;
  if (d->ta == LIBXSMM_DATATYPE_I2X4 && b8 && d->tc == LIBXSMM_DATATYPE_I32) return XB_LB_I2;                  /* :1089-1198 */
  if (d->ta == LIBXSMM_DATATYPE_I1X8 && b8 && d->tc == LIBXSMM_DATATYPE_I32) return XB_LB_I1;                  /* :1199-1272 */
  if (d->ta == LIBXSMM_DATATYPE_MXFP4X2 && d->tb == LIBXSMM_DATATYPE_I8
      && (d->tc == LIBXSMM_DATATYPE_F32 || d->tc == LIBXSMM_DATATYPE_BF16)) return XB_LB_MXFP4;                    /* :1009-1088 */
  return XB_LB_NONE;
}

/* side operands: what a call of a GEMM descriptor reads next to A, B and C, one bit each. A's scales (a.tertiary) are the row scales of
 * a dequantising A or the E8M0 block scales of MX fp8 / MXFP4 A; B's (b.tertiary) the block scales of MX fp8 / MXFP4 x I8; C's
 * (c.tertiary) those of an MXBF8 C; A's zero points (a.quaternary) those of an int4 A. In a record: a_s, b_s, c_s and a_q. */
enum { XB_SIDE_A_S = 1, XB_SIDE_B_S = 2, XB_SIDE_C_S = 4, XB_SIDE_A_Q = 8 };
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline int xb_gemm_sides(const xb_gemm_desc* d) {
  switch (d->path) {
    case P_MX8: return XB_SIDE_A_S | XB_SIDE_B_S | (d->tc == LIBXSMM_DATATYPE_MXBF8 ? XB_SIDE_C_S : 0);
    case P_DQ: return (xb_dq_form(d) == XB_DQ_BF8_F16) ? 0 : XB_SIDE_A_S | (xb_dq_form(d) == XB_DQ_I4_F16 ? XB_SIDE_A_Q : 0);
    case P_LOWBIT: return (xb_lowbit_form(d) == XB_LB_MXFP4) ? XB_SIDE_A_S | XB_SIDE_B_S : 0;
    case P_I4_I32: return XB_SIDE_A_Q;
    default: return 0;
  }
}

/* 1 if a side operand of `sides` is NULL in r */
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline int xb_gemm_rec_lacks(const xb_gemm_rec* r, int sides) {
  return ((sides & XB_SIDE_A_S) && r->a_s == NULL) || ((sides & XB_SIDE_B_S) && r->b_s == NULL)
      || ((sides & XB_SIDE_C_S) && r->c_s == NULL) || ((sides & XB_SIDE_A_Q) && r->a_q == NULL);
}

/* launch description handed to the CUDA side */
typedef struct xb_gemm_launch {
  xb_gemm_desc d;
  long long count;
  /* mode 0: uniform strided batch */
  const void* a; const void* b; void* c;
  long long tile_stride_a, tile_stride_b, tile_stride_c;   /* bytes */
  long long tile_stride_as, tile_stride_bs, tile_stride_cs; /* MX block scales, dequantising A's row scales (bases in one.a_s / b_s / c_s), bytes */
  unsigned long long br;
  /* mode 1: per-tile records (device array of xb_gemm_rec[count]) */
  const xb_gemm_rec* recs;
  xb_gemm_rec one;      /* count==1 && !recs: passed by value */
} xb_gemm_launch;

/* the complete record of tile t: the per-tile record, the single call, or a strided batch's bases advanced by t tile strides (a side
 * operand the launch lacks is NULL with a tile stride of 0). A strided batch shares `one`'s scale factor, bias column and zero
 * points, has offset arrays in offset mode only and no masks. */
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline xb_gemm_rec xb_gemm_tile(const xb_gemm_launch* L, long long t) {
  xb_gemm_rec r;
  if (L->recs != NULL) r = L->recs[t];
  else if (L->a == NULL && L->c == NULL) r = L->one;
  else {
    r.a = (const char*)L->a + t * L->tile_stride_a; r.b = (const char*)L->b + t * L->tile_stride_b; r.c = (char*)L->c + t * L->tile_stride_c;
    r.a_aux = NULL; r.b_aux = NULL; r.br = L->br; r.scf = L->one.scf; r.d = L->one.d; r.c_aux = NULL; r.a_q = L->one.a_q;
    if (L->d.br_type == 2) { r.a_aux = L->one.a_aux; r.b_aux = L->one.b_aux; }
    r.a_s = (const char*)L->one.a_s + t * L->tile_stride_as; r.b_s = (const char*)L->one.b_s + t * L->tile_stride_bs;
    r.c_s = (L->one.c_s != NULL) ? (char*)L->one.c_s + t * L->tile_stride_cs : NULL;
  }
  return r;
}

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
  /* tile axis: `count` calls of the handle in one launch, call t with every pointer above (in0 .. out_aux) advanced by t times its
   * byte stride; 0 or 1 is a single call. Generator state, scratch and the by-value fields are shared by the calls. */
  long long count;
  long long s_in0, s_in1, s_in2, s_in_aux, s_out, s_out_aux;
} xb_meltw_args;
void xb_invoke_meqn(const struct xb_slot* s, const void* param);
void xb_meqn_release(void* work);
int xb_meltw_launch(const xb_meltw_desc* d, const xb_meltw_args* a);
/* the matrix-eltwise rules (host_meltw.c), pure host logic. The kernel family that serves a descriptor, or XB_FAM_NONE: whether it
 * dispatches; meltw.cu launches by it. */
enum { XB_FAM_NONE = 0, XB_FAM_MAP, XB_FAM_REDUCE, XB_FAM_SCALAR, XB_FAM_TRANSFORM, XB_FAM_GS, XB_FAM_QUANT, XB_FAM_DROPOUT, XB_FAM_SPLIT,
       XB_FAM_MXQUANT };
int xb_meltw_family(const xb_meltw_desc* d);
/* side operands: what a call of a served descriptor reads or writes next to its inputs and its output, one bit each */
enum {
  XB_MSIDE_IN_AUX = 1,      /* in.secondary: a bit mask, an index array, the forward output or the quantiser scale */
  XB_MSIDE_MASK_OUT = 2,    /* out.secondary: a bit mask */
  XB_MSIDE_ARGOP = 4,       /* out.secondary: the argop indices of a column reduction */
  XB_MSIDE_COPY_OUT = 8,    /* out.secondary: the DUMP copy */
  XB_MSIDE_OUT_AUX = 16,    /* out.secondary: MX block scales, scatter indices or plane offsets */
  XB_MSIDE_ALPHA = 32,      /* op.primary: a float (alpha, the drop probability) */
  XB_MSIDE_STATE = 64,      /* op.secondary: generator state, read and advanced */
  XB_MSIDE_COUNT = 128,     /* a run-time count: the columns (op.primary) or the indices (in.tertiary) */
  XB_MSIDE_RUNTIME = 256    /* run-time indices or plane offsets: no extent to stage, the operands must be device-accessible */
};
int xb_meltw_sides(const xb_meltw_desc* d);
int xb_meltw_batchable(const xb_meltw_desc* d);   /* 0 if a call carries per-call state or run-time extents */
float xb_meltw_scalar(const void* p);             /* a float in host or device memory */
/* bytes of a bit mask of n columns whose rows are ld bits rounded up to 16 */
static inline size_t xb_meltw_mask_bytes(long long ld, long long n) { return (size_t)LIBXSMM_UP(ld, 16) / 8 * (size_t)n; }
int xb_sreg_launch(const xb_sparse_desc* d, const void* b, void* c, long long n_total);
int xb_packed_sp_launch(const xb_sparse_desc* d, const void* a, const void* b, void* c, long long count,
                        long long stride_a, long long stride_b, long long stride_c);
int xb_bcsc_launch(xb_sparse_desc* d, const void* a, const void* b_vals, const unsigned int* colptr,
                   const unsigned int* rowidx, unsigned long long n_blocks, unsigned int nnzb, void* c);
/* 0: exact-order CUDA-core kernel, 1: wgmma tensor-core kernel (bcsc_tc.cu) */
int xb_bcsc_tc_variant(const xb_sparse_desc* d, unsigned long long n_blocks);
void xb_bcsc_state_free(void* work);

/* ---- host runtime (host_core.c) ---------------------------------------------------------------- */
int xb_gemm_path(const xb_gemm_desc* d);   /* the exact-order path that serves d, or XB_PATH_NONE: whether d dispatches */
xb_slot* xb_slot_of(const void* fnptr);    /* NULL if not one of our thunks */
const xb_sparse_desc* xb_fsspmdm_desc(const libxsmm_fsspmdm* handle);   /* host_sparse.c: the descriptor of an fsspmdm handle, or NULL */
void xb_invoke(int slot, const void* param);
const void* xb_thunk(int slot);
#define XB_NTHUNKS 8192

#if defined(__cplusplus)
}
#endif
#endif /* XB_INTERNAL_H */
