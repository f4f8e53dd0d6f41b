/* libxsmm_b200 -- host side of the sparse kernels: packed CSR/CSC/BCSC creation, the sparse-A "areg"
 * kernel and the fsspmdm front-end.
 *
 * Reference roles: src/libxsmm_main.c:3553-3883 (create_* entry points; caller-owned, not registered),
 * src/generator_packed_spgemm.c:19-126 (which operand is sparse is told by the zero leading
 * dimension), src/libxsmm_fsspmdm.c:24-560 (dense->CSR with alpha folded in, validity rules).
 * Sparsity patterns are copied to device memory at create time; packed CSR/CSC VALUES are read at
 * call time from the argument struct exactly like the reference kernels do.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "xb_internal.h"

extern int xb_host_slot_alloc(int kind, unsigned int nflops);
extern xb_slot* xb_host_slot(int i);

static int xb_is_fp(int t) { return t == LIBXSMM_DATATYPE_F32 || t == LIBXSMM_DATATYPE_F64; }

static int xb_upload_pattern(xb_sparse_desc* sp, const unsigned int* ptr, unsigned int nrows, const unsigned int* idx, unsigned int nnz) {
  sp->nrows = nrows; sp->nnz = nnz;
  sp->d_ptr = (unsigned int*)xb_rt_device_malloc(((size_t)nrows + 1) * sizeof(unsigned int));
  sp->d_idx = (unsigned int*)xb_rt_device_malloc(((size_t)nnz + 1) * sizeof(unsigned int));
  if (sp->d_ptr == NULL || sp->d_idx == NULL) return 1;
  if (0 != xb_rt_memcpy(sp->d_ptr, ptr, ((size_t)nrows + 1) * sizeof(unsigned int))) return 1;
  if (nnz > 0 && 0 != xb_rt_memcpy(sp->d_idx, idx, (size_t)nnz * sizeof(unsigned int))) return 1;
  return 0;
}

static void xb_fill_sparse_common(xb_sparse_desc* sp, int kind, const libxsmm_gemm_shape* s, unsigned int flags) {
  memset(sp, 0, sizeof(*sp));
  sp->kind = kind; sp->m = s->m; sp->n = s->n; sp->k = s->k; sp->lda = s->lda; sp->ldb = s->ldb; sp->ldc = s->ldc;
  sp->ta = (int)s->a_in_type; sp->tb = (int)s->b_in_type; sp->tc = (int)s->out_type; sp->tcomp = (int)s->comp_type;
  sp->flags = flags | LIBXSMM_GEMM_FLAG_USE_XGEMM_ABI;
  sp->beta0 = (flags & LIBXSMM_GEMM_FLAG_BETA_0) ? 1 : 0;
}

static libxsmm_gemmfunction xb_finish_sparse(int slot, int failed) {
  xb_slot* s = xb_host_slot(slot);
  if (failed) { libxsmm_release_kernel(xb_thunk(slot)); return NULL; }
  (void)s;
  return (libxsmm_gemmfunction)xb_thunk(slot);
}

/* ---- packed CSR: A sparse (lda==0) or B sparse (ldb==0) ------------------------------------------- */
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_spgemm_csr(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width,
  const unsigned int* row_ptr, const unsigned int* column_idx, const void* values)
{
  int slot, kind; unsigned int nrows, nnz;
  xb_slot* s;
  (void)prefetch_flags;
  LIBXSMM_INIT
  if (row_ptr == NULL || column_idx == NULL || values == NULL || packed_width <= 0) return NULL;
  if (gemm_shape.a_in_type != gemm_shape.b_in_type || !xb_is_fp((int)gemm_shape.a_in_type)
   || gemm_shape.out_type != gemm_shape.a_in_type) return NULL;           /* F32/F64 only (libxsmm_main.c:2353) */
  if (gemm_shape.m <= 0 || gemm_shape.n <= 0 || gemm_shape.k <= 0) return NULL;
  if (gemm_shape.lda == 0 && gemm_shape.ldb > 0 && gemm_shape.ldc > 0) { kind = XB_KIND_SP_A_CSR; nrows = (unsigned int)gemm_shape.m; }
  else if (gemm_shape.ldb == 0 && gemm_shape.lda > 0 && gemm_shape.ldc > 0) { kind = XB_KIND_SP_B_CSR; nrows = (unsigned int)gemm_shape.k; }
  else return NULL;                                                       /* generator_packed_spgemm.c:27-57 */
  if (!xb_rt_have_gpu()) return NULL;
  nnz = row_ptr[nrows];
  slot = xb_host_slot_alloc(kind, 2u * nnz * (unsigned int)(kind == XB_KIND_SP_A_CSR ? gemm_shape.n : gemm_shape.m) * (unsigned int)packed_width);
  if (slot < 0) return NULL;
  s = xb_host_slot(slot);
  xb_fill_sparse_common(&s->u.sp, kind, &gemm_shape, gemm_flags);
  s->u.sp.packed_width = packed_width;
  s->u.sp.max_n = gemm_shape.n;
  if (kind == XB_KIND_SP_B_CSR) {   /* only the columns up to the last one that holds a non-zero are computed -- the rest of C is
                                     * not even zeroed under BETA_0 (generator_packed_spgemm_csr_bsparse_avx_avx2_avx512.c:64-70) */
    unsigned int z, maxc = 0;
    for (z = 0; z < nnz; ++z) maxc = (column_idx[z] > maxc) ? column_idx[z] : maxc;
    s->u.sp.max_n = (nnz > 0 && (int)(maxc + 1) < gemm_shape.n) ? (int)(maxc + 1) : gemm_shape.n;
  }
  return xb_finish_sparse(slot, xb_upload_pattern(&s->u.sp, row_ptr, nrows, column_idx, nnz));
}

/* ---- packed CSC: B sparse (ldb==0) or C sparse (ldc==0) ------------------------------------------- */
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_spgemm_csc(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width,
  const unsigned int* column_ptr, const unsigned int* row_idx, const void* values)
{
  int slot, kind; unsigned int nnz;
  xb_slot* s;
  (void)prefetch_flags;
  LIBXSMM_INIT
  if (column_ptr == NULL || row_idx == NULL || values == NULL || packed_width <= 0) return NULL;
  if (gemm_shape.a_in_type != gemm_shape.b_in_type || !xb_is_fp((int)gemm_shape.a_in_type)
   || gemm_shape.out_type != gemm_shape.a_in_type) return NULL;
  if (gemm_shape.m <= 0 || gemm_shape.n <= 0 || gemm_shape.k <= 0) return NULL;
  if (gemm_shape.ldb == 0 && gemm_shape.lda > 0 && gemm_shape.ldc > 0) kind = XB_KIND_SP_B_CSC;
  else if (gemm_shape.ldc == 0 && gemm_shape.lda > 0 && gemm_shape.ldb > 0) kind = XB_KIND_SP_C_CSC;
  else return NULL;                                                       /* generator_packed_spgemm.c:68-99 */
  /* C-sparse: f32 and whole 16-lane vectors only (generator_packed_spgemm_csc_csparse_avx_avx2_avx512.c:607-622) */
  if (kind == XB_KIND_SP_C_CSC && (gemm_shape.a_in_type != LIBXSMM_DATATYPE_F32 || (packed_width % 16) != 0)) return NULL;
  if (!xb_rt_have_gpu()) return NULL;
  nnz = column_ptr[gemm_shape.n];
  slot = xb_host_slot_alloc(kind, 2u * nnz * (unsigned int)(kind == XB_KIND_SP_B_CSC ? gemm_shape.m : gemm_shape.k) * (unsigned int)packed_width);
  if (slot < 0) return NULL;
  s = xb_host_slot(slot);
  xb_fill_sparse_common(&s->u.sp, kind, &gemm_shape, gemm_flags);
  s->u.sp.packed_width = packed_width;
  return xb_finish_sparse(slot, xb_upload_pattern(&s->u.sp, column_ptr, (unsigned int)gemm_shape.n, row_idx, nnz));
}

/* ---- packed dense GEMM (include/libxsmm.h:195-214; src/libxsmm_main.c:3733-3840): F32/F64, caller-owned handles ------------ */
static libxsmm_gemmfunction xb_create_packed_dense(int kind, const libxsmm_gemm_shape* sh, unsigned int flags, libxsmm_blasint packed_width) {
  int slot; xb_slot* s;
  LIBXSMM_INIT
  if (packed_width <= 0 || sh->m <= 0 || sh->n <= 0 || sh->k <= 0) return NULL;
  if (sh->a_in_type != sh->b_in_type || !xb_is_fp((int)sh->a_in_type) || sh->out_type != sh->a_in_type) return NULL;
  if ((flags & (LIBXSMM_GEMM_FLAG_TRANS_A | LIBXSMM_GEMM_FLAG_TRANS_B)) != 0) return NULL;
  /* leading dimensions in units of packed vectors, as the golds index them */
  if (kind == XB_KIND_PK_GEMM) { if (sh->lda < sh->m || sh->ldb < sh->k || sh->ldc < sh->m) return NULL; }
  else if (sh->lda < sh->k || sh->ldb < sh->n || sh->ldc < sh->n) return NULL;
  if (!xb_rt_have_gpu()) return NULL;
  slot = xb_host_slot_alloc(kind, 2u * (unsigned int)sh->m * (unsigned int)sh->n * (unsigned int)sh->k * (unsigned int)packed_width);
  if (slot < 0) return NULL;
  s = xb_host_slot(slot);
  xb_fill_sparse_common(&s->u.sp, kind, sh, flags);
  s->u.sp.packed_width = packed_width;
  return (libxsmm_gemmfunction)xb_thunk(slot);
}
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_gemm(const libxsmm_gemm_shape gemm_shape, const libxsmm_bitfield gemm_flags,
  const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width)
{ (void)prefetch_flags; return xb_create_packed_dense(XB_KIND_PK_GEMM, &gemm_shape, gemm_flags, packed_width); }
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_gemm_ac_rm(const libxsmm_gemm_shape gemm_shape, const libxsmm_bitfield gemm_flags,
  const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width)
{ (void)prefetch_flags; return xb_create_packed_dense(XB_KIND_PK_AC_RM, &gemm_shape, gemm_flags, packed_width); }
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_gemm_bc_rm(const libxsmm_gemm_shape gemm_shape, const libxsmm_bitfield gemm_flags,
  const libxsmm_bitfield prefetch_flags, const libxsmm_blasint packed_width)
{ (void)prefetch_flags; return xb_create_packed_dense(XB_KIND_PK_BC_RM, &gemm_shape, gemm_flags, packed_width); }

/* ---- BCSC block-sparse B ------------------------------------------------------------------------------ */
static int xb_bcsc_types_ok(const libxsmm_gemm_shape* s) {
  const int a = (int)s->a_in_type, b = (int)s->b_in_type, c = (int)s->out_type, comp = (int)s->comp_type;
  if (a == LIBXSMM_DATATYPE_F32 && b == a && c == a && comp == a) return 1;
  if (a == LIBXSMM_DATATYPE_BF16 && b == a && c == a && comp == LIBXSMM_DATATYPE_F32) return 1;
  if ((a == LIBXSMM_DATATYPE_U8 && b == LIBXSMM_DATATYPE_I8) || (a == LIBXSMM_DATATYPE_I8 && b == LIBXSMM_DATATYPE_U8)) {
    return c == LIBXSMM_DATATYPE_I32 && comp == LIBXSMM_DATATYPE_I32;      /* spmm_kernel.c:851-856 */
  }
  return 0;
}

LIBXSMM_API libxsmm_gemmfunction libxsmm_create_packed_spgemm_bcsc(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_spgemm_config spgemm_config)
{
  int slot; xb_slot* s;
  const int nr = (gemm_flags & LIBXSMM_GEMM_FLAG_NO_RESET_TILECONFIG) != 0, ns = (gemm_flags & LIBXSMM_GEMM_FLAG_NO_SETUP_TILECONFIG) != 0;
  (void)prefetch_flags;
  LIBXSMM_INIT
  if (nr != ns) return NULL;                                               /* tile-config request, not a kernel */
  if (!xb_bcsc_types_ok(&gemm_shape)) return NULL;
  if (gemm_shape.m <= 0 || gemm_shape.k <= 0 || spgemm_config.packed_width <= 0 || spgemm_config.bk <= 0 || spgemm_config.bn <= 0) return NULL;
  if ((gemm_shape.k % spgemm_config.bk) != 0) return NULL;
  /* TRANS_B alone is unsupported by the reference emitter (bcsc generator :268-271); VNNI_B+TRANS_B is the VNNI-T re-pack */
  if ((gemm_flags & LIBXSMM_GEMM_FLAG_TRANS_B) != 0 && (gemm_flags & LIBXSMM_GEMM_FLAG_VNNI_B) == 0) return NULL;
  if (gemm_shape.a_in_type == LIBXSMM_DATATYPE_BF16 && (spgemm_config.bk % 2) != 0) return NULL;
  if (libxsmm_typesize(gemm_shape.a_in_type) == 1 && (spgemm_config.bk % 4) != 0) return NULL;
  slot = xb_host_slot_alloc(XB_KIND_BCSC, 0);
  if (slot < 0) return NULL;
  s = xb_host_slot(slot);
  xb_fill_sparse_common(&s->u.sp, XB_KIND_BCSC, &gemm_shape, gemm_flags);
  s->u.sp.packed_width = spgemm_config.packed_width; s->u.sp.bk = spgemm_config.bk; s->u.sp.bn = spgemm_config.bn;
  return (libxsmm_gemmfunction)xb_thunk(slot);
}

LIBXSMM_API libxsmm_tilecfgfunction libxsmm_create_tilecfg_packed_spgemm_bcsc(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_spgemm_config spgemm_config)
{
  int slot;
  const int nr = (gemm_flags & LIBXSMM_GEMM_FLAG_NO_RESET_TILECONFIG) != 0, ns = (gemm_flags & LIBXSMM_GEMM_FLAG_NO_SETUP_TILECONFIG) != 0;
  (void)gemm_shape; (void)spgemm_config;
  LIBXSMM_INIT
  if (nr == ns) return NULL;
  slot = xb_host_slot_alloc(XB_KIND_TILECFG, 0);
  return (slot < 0) ? NULL : (libxsmm_tilecfgfunction)xb_thunk(slot);
}

/* ---- sparse A fixed at create time (fsspmdm kernel) --------------------------------------------------- */
LIBXSMM_API libxsmm_gemmfunction libxsmm_create_spgemm_csr_areg(const libxsmm_gemm_shape gemm_shape,
  const libxsmm_bitfield gemm_flags, const libxsmm_bitfield prefetch_flags, const libxsmm_blasint max_N,
  const unsigned int* row_ptr, const unsigned int* column_idx, const double* values)
{
  int slot, failed; unsigned int nnz, i; xb_slot* s; size_t ts; void* tmp;
  (void)prefetch_flags;
  LIBXSMM_INIT
  if (row_ptr == NULL || column_idx == NULL || values == NULL) return NULL;
  if (!xb_is_fp((int)gemm_shape.a_in_type) || gemm_shape.b_in_type != gemm_shape.a_in_type || gemm_shape.out_type != gemm_shape.a_in_type) return NULL;
  if (gemm_shape.m <= 0 || gemm_shape.k <= 0 || gemm_shape.n <= 0 || max_N <= 0) return NULL;
  if (gemm_shape.ldb < max_N && gemm_shape.ldb < gemm_shape.n) return NULL;
  if (!xb_rt_have_gpu()) return NULL;
  nnz = row_ptr[gemm_shape.m];
  if (nnz == 0) return NULL;
  ts = libxsmm_typesize(gemm_shape.a_in_type);
  slot = xb_host_slot_alloc(XB_KIND_SREG, 2u * nnz * (unsigned int)gemm_shape.n);
  if (slot < 0) return NULL;
  s = xb_host_slot(slot);
  xb_fill_sparse_common(&s->u.sp, XB_KIND_SREG, &gemm_shape, gemm_flags);
  s->u.sp.max_n = max_N;
  failed = xb_upload_pattern(&s->u.sp, row_ptr, (unsigned int)gemm_shape.m, column_idx, nnz);
  /* values arrive as double (reference src/libxsmm_fsspmdm.c:163,225) and are narrowed to the compute type; each
   * non-zero is stored as {value, byte offset of its B row inside a shared-memory stage} for the streaming kernel */
  ts = (ts == 8) ? 16 : 8;
  tmp = malloc((size_t)nnz * ts);
  s->u.sp.d_val = xb_rt_device_malloc((size_t)nnz * ts);
  if (tmp == NULL || s->u.sp.d_val == NULL) failed = 1;
  else {
    memset(tmp, 0, (size_t)nnz * ts);
    for (i = 0; i < nnz; ++i) {
      if (ts == 16) { *(double*)((char*)tmp + (size_t)i * 16) = values[i]; *(unsigned int*)((char*)tmp + (size_t)i * 16 + 8) = column_idx[i] * 512u; }
      else { *(float*)((char*)tmp + (size_t)i * 8) = (float)values[i]; *(unsigned int*)((char*)tmp + (size_t)i * 8 + 4) = column_idx[i] * 512u; }
    }
    if (0 != xb_rt_memcpy(s->u.sp.d_val, tmp, (size_t)nnz * ts)) failed = 1;
  }
  free(tmp);
  return xb_finish_sparse(slot, failed);
}

/* ---- invocation ------------------------------------------------------------------------------------------ */
static const void* xb_dev_in(const void* p, size_t bytes, int* staged) {
  if (p == NULL || xb_rt_ptr_kind(p) != 0) return p;
  else { void* d = xb_rt_scratch(bytes); if (d != NULL) { xb_rt_upload(d, p, bytes); *staged = 1; } return d; }
}

/* the bytes one call reads through A and B and writes through C. BCSC: B is the block values (nnzb blocks; 0 while the count is
 * unknown on the host) and C covers n_blocks block-columns. Single calls stage by these extents, batches check their C stride
 * against them. */
static void xb_sparse_extents(const xb_sparse_desc* d, unsigned long long n_blocks, unsigned int nnzb, size_t* ab, size_t* bb, size_t* cb) {
  const size_t ts = libxsmm_typesize((libxsmm_datatype)d->ta), tsc = libxsmm_typesize((libxsmm_datatype)d->tc);
  const size_t P = (size_t)d->packed_width;
  switch (d->kind) {
    case XB_KIND_SREG:     /* a=NULL, b=B, c=C covering max_N columns (src/libxsmm_fsspmdm.c:491-515) */
      *ab = 0; *bb = ((size_t)(d->k - 1) * d->ldb + d->max_n) * ts; *cb = ((size_t)(d->m - 1) * d->ldc + d->max_n) * ts; break;
    case XB_KIND_SP_A_CSR: case XB_KIND_SP_B_CSR: case XB_KIND_SP_B_CSC: case XB_KIND_SP_C_CSC:
      *ab = (d->kind == XB_KIND_SP_A_CSR) ? (size_t)d->nnz * ts
          : (d->kind == XB_KIND_SP_C_CSC) ? (size_t)d->k * d->lda * P * ts   /* A is [K][lda][P] there */ : (size_t)d->m * d->lda * P * ts;
      *bb = (d->kind == XB_KIND_SP_B_CSR || d->kind == XB_KIND_SP_B_CSC) ? (size_t)d->nnz * ts : (size_t)d->k * d->ldb * P * ts;
      *cb = (d->kind == XB_KIND_SP_C_CSC) ? (size_t)d->nnz * ts /* one scalar per non-zero */ : (size_t)d->m * d->ldc * P * ts;
      break;
    case XB_KIND_PK_GEMM: case XB_KIND_PK_AC_RM: case XB_KIND_PK_BC_RM:
      *ab = (d->kind == XB_KIND_PK_GEMM) ? (size_t)d->k * d->lda * P * ts : ((d->kind == XB_KIND_PK_AC_RM) ? (size_t)d->m * d->lda * P * ts : (size_t)d->m * d->lda * ts);
      *bb = (d->kind == XB_KIND_PK_GEMM) ? (size_t)d->n * d->ldb * P * ts : ((d->kind == XB_KIND_PK_AC_RM) ? (size_t)d->k * d->ldb * ts : (size_t)d->k * d->ldb * P * ts);
      *cb = ((d->kind == XB_KIND_PK_GEMM) ? (size_t)d->n : (size_t)d->m) * d->ldc * P * ts;
      break;
    case XB_KIND_BCSC:     /* slots: samples/xgemm_sparse/spmm_kernel.c:451-466 */
      *ab = (size_t)d->m * d->k * P * ts; *bb = (size_t)nnzb * d->bk * d->bn * libxsmm_typesize((libxsmm_datatype)d->tb);
      *cb = (size_t)d->m * n_blocks * d->bn * P * tsc;
      break;
    default: *ab = *bb = *cb = 0; break;
  }
}

/* the BCSC pattern of a call: block-column count (b.quaternary, read on the host), colptr (b.secondary) and rowidx (b.tertiary);
 * a host-readable pattern is staged and its block count read, a device-resident one passes as is with nnzb 0 (unknown).
 * Returns 1 if there is nothing to run (no pattern or no block-columns). */
static int xb_bcsc_pattern(const libxsmm_gemm_param* p, unsigned long long* nbc, unsigned int* nnzb, const void** cp, const void** ri, int* staged) {
  const unsigned int* colptr_h = (const unsigned int*)p->b.secondary;
  *nbc = (p->b.quaternary != NULL) ? *(const unsigned long long*)p->b.quaternary : 0ull;
  *nnzb = 0;
  if (*nbc == 0 || colptr_h == NULL) return 1;
  if (xb_rt_ptr_kind(colptr_h) != 1) *nnzb = colptr_h[*nbc];   /* device-resident pattern: count stays on the device (0 = unknown) */
  *cp = xb_dev_in(colptr_h, (size_t)(*nbc + 1) * sizeof(unsigned int), staged);
  *ri = (*nnzb == 0) ? p->b.tertiary : xb_dev_in(p->b.tertiary, (size_t)*nnzb * sizeof(unsigned int), staged);
  return 0;
}

void xb_invoke_sparse(const xb_slot* s, const libxsmm_gemm_param* p) {
  const xb_sparse_desc* d = &s->u.sp;
  const size_t ts = libxsmm_typesize((libxsmm_datatype)d->ta);
  int staged = 0, rc = 0;
  void* c_host = NULL; void* c_dev = NULL; size_t ab = 0, bb = 0, c_bytes = 0;
  size_t c_pitch = 0, c_width = 0, c_rows = 0;   /* non-zero: the staged C is a column block of a wider matrix (see XB_KIND_SREG) */
  switch (d->kind) {
    case XB_KIND_SREG: {
      const void* b;
      xb_sparse_extents(d, 0, 0, &ab, &bb, &c_bytes);
      b = xb_dev_in(p->b.primary, bb, &staged);
      c_dev = p->c.primary;
      if (xb_rt_ptr_kind(p->c.primary) == 0) {
        c_host = p->c.primary; c_dev = xb_rt_scratch(c_bytes); staged = 1;
        /* A handle narrower than the rows of C (max_N < ldc) owns a column block, and callers run the blocks of one C concurrently
         * (samples/xgemm_sparse_Ainregs/pyfr_driver_asp_reg.c:381-392, omp parallel for over l_n_block): only the m x max_N block may
         * travel -- the contiguous span would carry the neighbours' columns out stale and back over their results */
        if (d->max_n < d->ldc) { c_pitch = (size_t)d->ldc * ts; c_width = (size_t)d->max_n * ts; c_rows = (size_t)d->m; }
        if (c_dev != NULL) { if (c_rows != 0) xb_rt_memcpy2d_async(c_dev, c_host, c_pitch, c_width, c_rows); else xb_rt_upload(c_dev, c_host, c_bytes); }
      }
      if (b == NULL || c_dev == NULL) { rc = 2; break; }
      rc = xb_sreg_launch(d, b, c_dev, d->max_n);
    } break;
    case XB_KIND_SP_A_CSR: case XB_KIND_SP_B_CSR: case XB_KIND_SP_B_CSC: case XB_KIND_SP_C_CSC:
    case XB_KIND_PK_GEMM: case XB_KIND_PK_AC_RM: case XB_KIND_PK_BC_RM: {
      const void *a, *b;
      xb_sparse_extents(d, 0, 0, &ab, &bb, &c_bytes);
      a = xb_dev_in(p->a.primary, ab, &staged); b = xb_dev_in(p->b.primary, bb, &staged);
      c_dev = p->c.primary;
      if (xb_rt_ptr_kind(p->c.primary) == 0) { c_host = p->c.primary; c_dev = xb_rt_scratch(c_bytes); if (c_dev) xb_rt_upload(c_dev, c_host, c_bytes); staged = 1; }
      if (a == NULL || b == NULL || c_dev == NULL) { rc = 2; break; }
      rc = xb_packed_sp_launch(d, a, b, c_dev, 1, 0, 0, 0);
    } break;
    case XB_KIND_BCSC: {
      unsigned long long nbc; unsigned int nnzb;
      const void *a, *bv, *cp = NULL, *ri = NULL;
      if (xb_bcsc_pattern(p, &nbc, &nnzb, &cp, &ri, &staged)) break;
      xb_sparse_extents(d, nbc, nnzb, &ab, &bb, &c_bytes);
      a = xb_dev_in(p->a.primary, ab, &staged);
      bv = (nnzb == 0) ? p->b.primary : xb_dev_in(p->b.primary, bb, &staged);
      c_dev = p->c.primary;
      if (xb_rt_ptr_kind(p->c.primary) == 0) { c_host = p->c.primary; c_dev = xb_rt_scratch(c_bytes); if (c_dev && !d->beta0) xb_rt_upload(c_dev, c_host, c_bytes); staged = 1; }
      if (a == NULL || bv == NULL || cp == NULL || ri == NULL || c_dev == NULL) { rc = 2; break; }
      rc = xb_bcsc_launch((xb_sparse_desc*)(uintptr_t)d /* only the handle's scratch cache (d->work) is touched, under its own lock */, a, bv, (const unsigned int*)cp, (const unsigned int*)ri, nbc, nnzb, c_dev);
    } break;
    default: break;
  }
  if (rc != 0) { xb_rt_note_error(rc, "invoke_sparse"); xb_rt_scratch_reset(); return; }
  if (c_host != NULL) { if (c_rows != 0) xb_rt_memcpy2d_async(c_host, c_dev, c_pitch, c_width, c_rows); else xb_rt_memcpy_async(c_host, c_dev, c_bytes); }
  if (staged || xb_rt_blocking()) { xb_rt_sync(); xb_rt_scratch_reset(); }
}

/* ---- strided batch: `count` calls of one packed or BCSC handle in one launch ----------------------------------------------------
 * Call t is kernel(param) with a/b/c.primary advanced by t times their byte strides; everything else in *param (the BCSC pattern
 * and block-column count included) is read once, from call 0. Nothing is staged but a host-readable BCSC pattern, which every call
 * shares: A, B and C must be device-accessible. fsspmdm handles are not batchable: one call already covers every column of B. */
LIBXSMM_API int libxsmm_b200_spgemm_batch_strided(libxsmm_gemmfunction kernel, const libxsmm_gemm_param* param,
                                                  const libxsmm_b200_spgemm_strides* strides, long long count)
{
  const xb_slot* s = xb_slot_of((const void*)kernel);
  xb_sparse_desc d;
  unsigned long long nbc = 0; unsigned int nnzb = 0;
  const void *cp = NULL, *ri = NULL;
  size_t ab, bb, cb, tsa, tsb, tsc;
  int staged = 0, rc;
  if (s == NULL || param == NULL || strides == NULL || count < 0) return -1;
  switch (s->kind) {
    case XB_KIND_SREG: return LIBXSMM_B200_ERROR_NOT_BATCHABLE;
    case XB_KIND_SP_A_CSR: case XB_KIND_SP_B_CSR: case XB_KIND_SP_B_CSC: case XB_KIND_SP_C_CSC:
    case XB_KIND_PK_GEMM: case XB_KIND_PK_AC_RM: case XB_KIND_PK_BC_RM: case XB_KIND_BCSC: break;
    default: return -1;
  }
  d = s->u.sp;
  tsa = libxsmm_typesize((libxsmm_datatype)d.ta); tsb = libxsmm_typesize((libxsmm_datatype)d.tb); tsc = libxsmm_typesize((libxsmm_datatype)d.tc);
  /* a stride must keep every call's operand aligned to its elements */
  if (strides->a < 0 || strides->b < 0 || strides->c < 0) return -1;
  if (strides->a % (long long)tsa != 0 || strides->b % (long long)tsb != 0 || strides->c % (long long)tsc != 0) return -1;
  if (count == 0) return 0;
  if (param->a.primary == NULL || param->b.primary == NULL || param->c.primary == NULL) return -1;
  if (d.kind == XB_KIND_BCSC && (param->b.secondary == NULL || param->b.tertiary == NULL || param->b.quaternary == NULL)) return -1;
  if (xb_rt_ptr_kind(param->a.primary) == 0 || xb_rt_ptr_kind(param->b.primary) == 0 || xb_rt_ptr_kind(param->c.primary) == 0) return -4;
  if (d.kind == XB_KIND_BCSC) {
    if (xb_bcsc_pattern(param, &nbc, &nnzb, &cp, &ri, &staged)) return 0;     /* no block-columns: nothing to run, like a single call */
    if (cp == NULL || ri == NULL) { xb_rt_scratch_reset(); return 2; }
  }
  xb_sparse_extents(&d, nbc, nnzb, &ab, &bb, &cb);
  if (count > 1 && strides->c < (long long)cb) { if (staged) xb_rt_scratch_reset(); return -1; }   /* C of call t reaches into call t + 1 */
  if (d.kind == XB_KIND_BCSC) {
    d.calls.count = count; d.calls.s_a = strides->a; d.calls.s_b = strides->b; d.calls.s_c = strides->c;
    rc = xb_bcsc_launch(&d, param->a.primary, param->b.primary, (const unsigned int*)cp, (const unsigned int*)ri, nbc, nnzb, param->c.primary);
  } else {
    rc = xb_packed_sp_launch(&d, param->a.primary, param->b.primary, param->c.primary, count, strides->a, strides->b, strides->c);
  }
  if (rc == 0 && (staged || xb_rt_blocking())) rc = xb_rt_sync();
  if (staged) xb_rt_scratch_reset();
  return rc;
}

/* ---- fsspmdm ------------------------------------------------------------------------------------------------ */
struct libxsmm_fsspmdm {
  libxsmm_gemmfunction kernel;
  libxsmm_datatype datatype;
  int M, N, K, ldb, ldc;
};

LIBXSMM_API libxsmm_fsspmdm* libxsmm_fsspmdm_create(libxsmm_datatype datatype,
  libxsmm_blasint M, libxsmm_blasint N, libxsmm_blasint K, libxsmm_blasint lda, libxsmm_blasint ldb, libxsmm_blasint ldc,
  const void* alpha, const void* beta, const void* a_dense, int c_is_nt, libxsmm_timer_tickint (*timer_tick)(void))
{
  static int error_once = 0;
  libxsmm_fsspmdm* handle = NULL;
  unsigned int *rowptr = NULL, *colidx = NULL; double* values = NULL;
  libxsmm_bitfield flags = 0;
  int i, j, nnz = 0, vl;
  double fbeta, falpha;
  (void)timer_tick;   /* the reference's timing tournament picks among x86 code variants; one kernel here */
  if (a_dense == NULL || (datatype != LIBXSMM_DATATYPE_F64 && datatype != LIBXSMM_DATATYPE_F32) || M <= 0 || N <= 0 || K <= 0) {
    if (libxsmm_verbosity != 0 && 0 == error_once++) fprintf(stderr, "LIBXSMM ERROR (libxsmm_fsspmdm_create): invalid input!\n");
    return NULL;
  }
  LIBXSMM_INIT
  vl = 64 / (int)libxsmm_typesize(datatype);          /* vector length of the reference's AVX-512 target */
  if (datatype == LIBXSMM_DATATYPE_F64) { fbeta = (beta != NULL) ? *(const double*)beta : 1.0; falpha = (alpha != NULL) ? *(const double*)alpha : 1.0; }
  else { fbeta = (beta != NULL) ? (double)*(const float*)beta : 1.0; falpha = (alpha != NULL) ? (double)*(const float*)alpha : 1.0; }
  if ((N % vl) != 0 || !(fbeta == 1.0 || fbeta == 0.0) || lda < K || ldc < N || ldb < N) {   /* src/libxsmm_fsspmdm.c:80-131 */
    if (libxsmm_verbosity != 0 && 0 == error_once++) fprintf(stderr, "LIBXSMM ERROR (libxsmm_fsspmdm_create): unsupported input!\n");
    return NULL;
  }
  if (fbeta == 0.0) flags |= LIBXSMM_GEMM_FLAG_BETA_0 | (c_is_nt ? LIBXSMM_GEMM_FLAG_ALIGN_C_NTS_HINT : 0);
  rowptr = (unsigned int*)malloc(((size_t)M + 1) * sizeof(unsigned int));
  colidx = (unsigned int*)malloc((size_t)M * K * sizeof(unsigned int));
  values = (double*)malloc((size_t)M * K * sizeof(double));
  if (rowptr == NULL || colidx == NULL || values == NULL) { free(rowptr); free(colidx); free(values); return NULL; }
  for (i = 0; i < M; ++i) {                            /* CSR with alpha folded in; exact zeros dropped (:190-238) */
    rowptr[i] = (unsigned int)nnz;
    for (j = 0; j < K; ++j) {
      double v;
      if (datatype == LIBXSMM_DATATYPE_F64) v = falpha * ((const double*)a_dense)[(size_t)i * lda + j];
      else v = (double)((float)falpha * ((const float*)a_dense)[(size_t)i * lda + j]);
      if (v != 0.0) { values[nnz] = v; colidx[nnz] = (unsigned int)j; ++nnz; }
    }
  }
  rowptr[M] = (unsigned int)nnz;
  if (nnz == 0) {                                      /* empty matrix => NULL (:133-140) */
    if (libxsmm_verbosity != 0 && 0 == error_once++) fprintf(stderr, "LIBXSMM WARNING (libxsmm_fsspmdm_create): discovered an empty matrix!\n");
  } else {
    handle = (libxsmm_fsspmdm*)calloc(1, sizeof(*handle));
    if (handle != NULL) {
      const libxsmm_gemm_shape shape = libxsmm_create_gemm_shape(M, vl, K, 0, ldb, ldc, datatype, datatype, datatype, datatype);
      handle->kernel = libxsmm_create_spgemm_csr_areg(shape, flags, LIBXSMM_GEMM_PREFETCH_NONE, N, rowptr, colidx, values);
      handle->datatype = datatype; handle->M = M; handle->N = N; handle->K = K; handle->ldb = ldb; handle->ldc = ldc;
      if (handle->kernel == NULL) { free(handle); handle = NULL; }
    }
  }
  free(rowptr); free(colidx); free(values);
  return handle;
}

LIBXSMM_API libxsmm_dfsspmdm* libxsmm_dfsspmdm_create(libxsmm_blasint M, libxsmm_blasint N, libxsmm_blasint K,
  libxsmm_blasint lda, libxsmm_blasint ldb, libxsmm_blasint ldc, double alpha, double beta, const double* a_dense,
  int c_is_nt, libxsmm_timer_tickint (*timer_tick)(void))
{
  return libxsmm_fsspmdm_create(LIBXSMM_DATATYPE_F64, M, N, K, lda, ldb, ldc, &alpha, &beta, a_dense, c_is_nt, timer_tick);
}

LIBXSMM_API libxsmm_sfsspmdm* libxsmm_sfsspmdm_create(libxsmm_blasint M, libxsmm_blasint N, libxsmm_blasint K,
  libxsmm_blasint lda, libxsmm_blasint ldb, libxsmm_blasint ldc, float alpha, float beta, const float* a_dense,
  int c_is_nt, libxsmm_timer_tickint (*timer_tick)(void))
{
  return libxsmm_fsspmdm_create(LIBXSMM_DATATYPE_F32, M, N, K, lda, ldb, ldc, &alpha, &beta, a_dense, c_is_nt, timer_tick);
}

LIBXSMM_API void libxsmm_fsspmdm_execute(const libxsmm_fsspmdm* handle, const void* B, void* C) {
  libxsmm_gemm_param p;
  if (handle == NULL || handle->kernel == NULL) return;
  memset(&p, 0, sizeof(p));
  p.b.primary = (void*)(uintptr_t)B; p.c.primary = C;
  handle->kernel(&p);
}
const xb_sparse_desc* xb_fsspmdm_desc(const libxsmm_fsspmdm* handle) {
  const xb_slot* s = (handle != NULL) ? xb_slot_of((const void*)handle->kernel) : NULL;
  return (s != NULL && s->kind == XB_KIND_SREG) ? &s->u.sp : NULL;
}
LIBXSMM_API void libxsmm_dfsspmdm_execute(const libxsmm_dfsspmdm* handle, const double* B, double* C) { libxsmm_fsspmdm_execute(handle, B, C); }
LIBXSMM_API void libxsmm_sfsspmdm_execute(const libxsmm_sfsspmdm* handle, const float* B, float* C) { libxsmm_fsspmdm_execute(handle, B, C); }

LIBXSMM_API void libxsmm_fsspmdm_destroy(libxsmm_fsspmdm* handle) {
  if (handle == NULL) return;
  libxsmm_release_kernel((const void*)handle->kernel);
  free(handle);
}
LIBXSMM_API void libxsmm_dfsspmdm_destroy(libxsmm_dfsspmdm* handle) { libxsmm_fsspmdm_destroy(handle); }
LIBXSMM_API void libxsmm_sfsspmdm_destroy(libxsmm_sfsspmdm* handle) { libxsmm_fsspmdm_destroy(handle); }
