/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * A stand-in for the CUDA side of the library (runtime.cu and the kernel launchers) so that the HOST logic above the kernels --
 * equation trees (host_meqn.c), operand staging, dispatch rules (the mateltwise family rule of host_meltw.c included, unstubbed) --
 * can be exercised in the GPU-less build container:
 * "device" memory is plain host memory, every elementwise launch and every dense GEMM tile is answered by the oracle
 * (oracle/liboracle.so), fsspmdm runs the library's own direct loop on the host, the tensor-core and packed / block-sparse launchers refuse. tests/test_hostsim.py links the host_*.o objects with this file into tests/c/_hostsim/libxsmm.so and
 * runs the reference's unmodified equation drivers against it; what that validates is the order of evaluation, the shapes and
 * leading dimensions handed to each node, and where secondary outputs land -- not any kernel. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../libxsmm_b200/csrc/xb_internal.h"
#include "../../include/libxsmm.h"

extern int oracle_meltw(const int* desc, void* param, int mode);

/* ---- runtime ------------------------------------------------------------------------------------------------------------- */
static __thread void* g_blocks[4096]; static __thread int g_nblocks = 0;
static __thread int g_err = 0; static __thread char g_errs[256];
static unsigned long long g_launches = 0, g_launches_by[LIBXSMM_B200_BACKEND_NOOP + 1];   /* all, and per kernel family */

int xb_rt_device_count(void) { return 1; }
int xb_rt_set_device(int ordinal) { return ordinal == 0 ? 0 : 1; }
void xb_rt_set_stream(void* stream) { (void)stream; }
void* xb_rt_stream(void) { return NULL; }
void xb_rt_set_blocking(int on) { (void)on; }
int xb_rt_blocking(void) { return 1; }
int xb_rt_sync(void) { return 0; }
int xb_rt_last_error(void) { const int e = g_err; g_err = 0; return e; }
const char* xb_rt_last_error_string(void) { return g_errs; }
void xb_rt_note_error(int code, const char* where) { g_err = code; snprintf(g_errs, sizeof(g_errs), "%s", where); fprintf(stderr, "hostsim: error %d: %s\n", code, where); }
unsigned long long xb_rt_launch_count(void) { return g_launches; }
void xb_rt_count_launch(void) { ++g_launches; }
/* the library defines this next to its launchers (runtime.cu); here every GEMM tile is an exact-order launch, everything else streams */
LIBXSMM_API unsigned long long libxsmm_b200_launch_count_backend(int backend) {
  return (backend >= 0 && backend <= LIBXSMM_B200_BACKEND_NOOP) ? g_launches_by[backend] : 0ull;
}
void* xb_rt_device_malloc(size_t size) { return malloc(size); }
void xb_rt_device_free(void* p) { free(p); }
void* xb_rt_host_malloc(size_t size) { return malloc(size); }
void xb_rt_host_free(void* p) { free(p); }
void* xb_rt_managed_malloc(size_t size) { return malloc(size); }
void xb_rt_managed_free(void* p) { free(p); }
int xb_rt_memcpy(void* dst, const void* src, size_t size) { memmove(dst, src, size); return 0; }
int xb_rt_memcpy_async(void* dst, const void* src, size_t size) { memmove(dst, src, size); return 0; }
int xb_rt_memcpy2d_async(void* dst, const void* src, size_t pitch, size_t width, size_t rows) {
  size_t r; for (r = 0; r < rows; ++r) memmove((char*)dst + r * pitch, (const char*)src + r * pitch, width); return 0;
}
int xb_rt_upload(void* dst_dev, const void* src_host, size_t size) { memmove(dst_dev, src_host, size); return 0; }
/* the chunked host<->device pipeline, serialised: describe a chunk, copy its operands in (C only when the kernel reads it), launch,
 * copy C out -- the staging buffers are poisoned first so that a chunk that relies on bytes it did not ask for shows up */
int xb_rt_pipeline(long long nchunks, size_t max_a, size_t max_b, size_t max_c, xb_pipe_describe_fn describe, xb_pipe_launch_fn launch, void* ctx) {
  char *da = (char*)malloc(max_a ? max_a : 1), *db = (char*)malloc(max_b ? max_b : 1), *dc = (char*)malloc(max_c ? max_c : 1);
  long long i; int rc = 0;
  if (da == NULL || db == NULL || dc == NULL) { free(da); free(db); free(dc); return 2; }
  for (i = 0; i < nchunks && rc == 0; ++i) {
    xb_pipe_chunk ch; memset(&ch, 0, sizeof(ch));
    describe(ctx, i, &ch);
    if (ch.bytes_a > max_a || ch.bytes_b > max_b || ch.bytes_c > max_c) { rc = 3; break; }
    memset(da, 0xa5, max_a); memset(db, 0xa5, max_b); memset(dc, 0xa5, max_c);
    if (ch.bytes_a) memcpy(da, ch.host_a, ch.bytes_a);
    if (ch.bytes_b) memcpy(db, ch.host_b, ch.bytes_b);
    if (ch.copy_c_in && ch.bytes_c) memcpy(dc, ch.host_c, ch.bytes_c);
    rc = launch(ctx, &ch, da, db, dc);
    if (rc == 0 && ch.bytes_c) memcpy(ch.host_c, dc, ch.bytes_c);
  }
  free(da); free(db); free(dc);
  return rc;
}
/* every caller pointer is "pageable host" so that the staging paths run; XB_HOSTSIM_PTR_KIND=3 ("pinned") lets the operations
 * that insist on device-accessible operands (gather / scatter, index reductions) through */
int xb_rt_ptr_kind(const void* p) { const char* e = getenv("XB_HOSTSIM_PTR_KIND"); (void)p; return (e != NULL) ? atoi(e) : 0; }
int xb_rt_have_gpu(void) { return 1; }
void* xb_rt_scratch(size_t bytes) {
  void* p;
  if (g_nblocks >= 4096) return NULL;
  p = calloc(1, bytes ? bytes : 1);
  if (p != NULL) g_blocks[g_nblocks++] = p;
  return p;
}
void xb_rt_scratch_reset(void) { while (g_nblocks > 0) free(g_blocks[--g_nblocks]); }
int xb_rt_current_device(void) { return 0; }
int xb_rt_first_use_on_device(unsigned long long* mask) { const int first = (*mask & 1ull) == 0; *mask |= 1ull; return first; }

/* ---- launchers ----------------------------------------------------------------------------------------------------------- */
/* dense GEMM: the "exact-order" backend is answered by the oracle tile by tile (strided batches, per-tile records, single calls;
 * plain, fused colbias / relu / sigmoid, bitmap-compressed A, 4-bit A); the tensor-core backends below refuse, so a dispatch in the
 * simulation always lands here. C re-packing (VNNI_C) is a separate elementwise pass of host_core.c, so the flag is masked. */
extern int oracle_gemm(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                       unsigned long long br, void* a, void* b, void* c, long long* offs_a, long long* offs_b, float scf, int mode);
extern int oracle_gemm_ext(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                           unsigned long long br, void* a, void* b, void* c, long long* offs_a, long long* offs_b, float scf,
                           const int* fuse, const void* colbias, unsigned char* relu_mask);
extern int oracle_gemm_i4(const int* dims, unsigned int flags, int br_type, long long stride_a, long long stride_b, unsigned long long br,
                          const unsigned char* a, const unsigned char* b, int* c, const unsigned char* zpt);
extern int oracle_gemm_bitmap(const int* dims, const int* types, unsigned int flags, const void* a, const void* b, void* c, const unsigned char* bitmap);

static int sim_gemm_tile(const xb_gemm_desc* d, const xb_gemm_rec* r) {
  const int dims[6] = { d->m, d->n, d->k, d->lda, d->ldb, d->ldc }, types[4] = { d->ta, d->tb, d->tcomp, d->tc };
  const unsigned int flags = d->flags & ~(unsigned int)LIBXSMM_GEMM_FLAG_VNNI_C;
  ++g_launches; ++g_launches_by[LIBXSMM_B200_BACKEND_SIMT];
  if (d->path == P_BITMAP) return oracle_gemm_bitmap(dims, types, flags, r->a, r->b, r->c, (const unsigned char*)r->a_q);
  if (d->path == P_I4_I32) {
    return oracle_gemm_i4(dims, flags, d->br_type, d->br_stride_a, d->br_stride_b, r->br, (const unsigned char*)r->a, (const unsigned char*)r->b, (int*)r->c, (const unsigned char*)r->a_q);
  }
  if (d->fuse_colbias != 0 || d->cp_op != 0) {
    const int fuse[4] = { d->fuse_colbias, d->cp_op, (d->cp_flags & LIBXSMM_MELTW_FLAG_UNARY_BITMASK_2BYTEMULT) != 0 && r->c_aux != NULL, 0 };
    return oracle_gemm_ext(dims, types, flags, d->br_type, d->br_stride_a, d->br_stride_b, r->br, (void*)(uintptr_t)r->a, (void*)(uintptr_t)r->b, r->c,
                           (long long*)(uintptr_t)r->a_aux, (long long*)(uintptr_t)r->b_aux, r->scf, fuse, r->d, (unsigned char*)r->c_aux);
  }
  return oracle_gemm(dims, types, flags, d->br_type, d->br_stride_a, d->br_stride_b, r->br, (void*)(uintptr_t)r->a, (void*)(uintptr_t)r->b, r->c,
                     (long long*)(uintptr_t)r->a_aux, (long long*)(uintptr_t)r->b_aux, r->scf, 0);
}
int xb_gemm_simt_launch(const xb_gemm_launch* L) {
  long long t; int rc = 0;
  for (t = 0; t < L->count && rc == 0; ++t) { const xb_gemm_rec r = xb_gemm_tile(L, t); rc = sim_gemm_tile(&L->d, &r); }
  if (rc != 0) fprintf(stderr, "hostsim: the oracle refused a GEMM tile (rc %d)\n", rc);
  return rc;
}
int xb_gemm_tc_supported(const xb_gemm_desc* d) { (void)d; return 0; }
int xb_gemm_tc_shape_ok(const xb_gemm_desc* d) { (void)d; return 0; }
int xb_gemm_tc_launch(const xb_gemm_launch* L) { (void)L; return 1; }
int xb_gemm_tc_launch_pooled(const xb_gemm_desc* d, const xb_tc_pool* pool, unsigned long long br, long long count) { (void)d; (void)pool; (void)br; (void)count; return 1; }
int xb_gemm_ts_supported(const xb_gemm_desc* d) { (void)d; return 0; }
int xb_gemm_ts_launch(const xb_gemm_launch* L) { (void)L; return 1; }
/* fsspmdm: C[row][col] (= or +=) sum over the row's non-zeros of value * B[column][col], entries as host_sparse.c stores them
 * ({value, 512 * column}); the accumulation order per element is the row order, like the library's direct kernel */
int xb_sreg_launch(const xb_sparse_desc* d, const void* b, void* c, long long n_total) {
  const int f64 = (d->ta == LIBXSMM_DATATYPE_F64); int row; long long col; unsigned int z;
  ++g_launches; ++g_launches_by[LIBXSMM_B200_BACKEND_STREAM];
  for (row = 0; row < d->m; ++row) for (col = 0; col < n_total; ++col) {
    if (f64) {
      double acc = 0, *dst = (double*)c + (size_t)row * d->ldc + col;
      for (z = d->d_ptr[row]; z < d->d_ptr[row + 1]; ++z) {
        const char* e = (const char*)d->d_val + (size_t)z * 16;
        acc += *(const double*)e * ((const double*)b)[(size_t)(*(const unsigned int*)(e + 8) >> 9) * d->ldb + col];
      }
      *dst = d->beta0 ? acc : (*dst + acc);
    } else {
      float acc = 0, *dst = (float*)c + (size_t)row * d->ldc + col;
      for (z = d->d_ptr[row]; z < d->d_ptr[row + 1]; ++z) {
        const char* e = (const char*)d->d_val + (size_t)z * 8;
        acc += *(const float*)e * ((const float*)b)[(size_t)(*(const unsigned int*)(e + 4) >> 9) * d->ldb + col];
      }
      *dst = d->beta0 ? acc : (*dst + acc);
    }
  }
  return 0;
}
int xb_packed_sp_launch(const xb_sparse_desc* d, const void* a, const void* b, void* c, long long count, long long sa, long long sb, long long sc) {
  (void)d; (void)a; (void)b; (void)c; (void)count; (void)sa; (void)sb; (void)sc; return 1;
}
int xb_bcsc_launch(xb_sparse_desc* d, const void* a, const void* b_vals, const unsigned int* colptr, const unsigned int* rowidx,
                   unsigned long long n_blocks, unsigned int nnzb, void* c) {
  (void)d; (void)a; (void)b_vals; (void)colptr; (void)rowidx; (void)n_blocks; (void)nnzb; (void)c; return 1;
}
int xb_bcsc_tc_variant(const xb_sparse_desc* d, unsigned long long n_blocks) { (void)d; (void)n_blocks; return 0; }
void xb_bcsc_state_free(void* work) { (void)work; }

/* elementwise: the oracle answers. The arguments are mapped back to a parameter struct by the descriptor's side operands (operands,
 * output, the two secondaries, the scalar of LEAKY_RELU/ELU/DROPOUT or the scale of QUANT/DEQUANT, the generator state); run-time
 * extents are refused */
int xb_meltw_launch(const xb_meltw_desc* d, const xb_meltw_args* a) {
  int desc[14]; int rc; float alpha = a->alpha;
  desc[0] = d->op_class; desc[1] = d->op; desc[2] = (int)d->flags; desc[3] = d->m; desc[4] = d->n; desc[5] = d->ldi; desc[6] = d->ldi2; desc[7] = d->ldi3;
  desc[8] = d->ldo; desc[9] = d->t_in0; desc[10] = d->t_in1; desc[11] = d->t_in2; desc[12] = d->t_out; desc[13] = d->t_comp;
  if (a->n_rt != 0) return 1;
  ++g_launches; ++g_launches_by[LIBXSMM_B200_BACKEND_STREAM];
  if (d->op_class == LIBXSMM_MELTW_OPERATION_UNARY) {
    libxsmm_meltw_unary_param p; memset(&p, 0, sizeof(p));
    p.in.primary = (void*)(uintptr_t)a->in0; p.in.secondary = (void*)(uintptr_t)a->in_aux; p.out.primary = a->out; p.out.secondary = a->out_aux; p.op.primary = &alpha;
    p.op.secondary = a->rng;                 /* dropout / stochastic rounding: the staged generator state, advanced in place */
    if ((xb_meltw_sides(d) & XB_MSIDE_IN_AUX) && a->in_aux == NULL) p.in.secondary = &alpha;   /* the quantiser's scale, read on the host */
    rc = oracle_meltw(desc, &p, 0);
  } else if (d->op_class == LIBXSMM_MELTW_OPERATION_BINARY) {
    libxsmm_meltw_binary_param p; memset(&p, 0, sizeof(p));
    p.in0.primary = (void*)(uintptr_t)a->in0; p.in1.primary = (void*)(uintptr_t)a->in1; p.out.primary = a->out; p.op.secondary = a->rng;
    rc = oracle_meltw(desc, &p, 0);
  } else {
    libxsmm_meltw_ternary_param p; memset(&p, 0, sizeof(p));
    p.in0.primary = (void*)(uintptr_t)a->in0; p.in1.primary = (void*)(uintptr_t)a->in1; p.in2.primary = (void*)(uintptr_t)a->in2; p.out.primary = a->out;
    p.op.secondary = a->rng;
    rc = oracle_meltw(desc, &p, 0);
  }
  if (rc != 0) fprintf(stderr, "hostsim: the oracle does not restate class %d op %d (rc %d)\n", d->op_class, d->op, rc);
  return rc;
}
