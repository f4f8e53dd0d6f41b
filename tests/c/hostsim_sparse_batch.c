/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * Packed-sparse, packed-dense and BCSC launches for the simulated device of tests/c/hostsim_runtime.c (which refuses them).
 * tests/test_sparse_batch_hostsim.py links the host_*.c objects, that runtime and this file with
 * -Wl,--wrap=xb_packed_sp_launch,--wrap=xb_bcsc_launch,--wrap=xb_rt_ptr_kind: every launch, single call or batch, is answered call
 * by call by the oracle, each call's A, B and C advanced by its strides, and the pattern, the block-column count and the block
 * count each launch was handed are recorded. Address ranges the test marks are "pageable host memory"; every other pointer is
 * what the runtime says. What this checks is the host half of the batch form, not any kernel. */
#include <stdint.h>
#include <string.h>
#include "../../libxsmm_b200/csrc/xb_internal.h"

extern int oracle_packed_sp(int is_csc, int dtype, const int* dims, unsigned int flags, int P,
                            const unsigned int* ptr, const unsigned int* idx, const void* values, void* a, void* b, void* c);
extern int oracle_packed_dense(int kind, int dtype, const int* dims, unsigned int flags, int P, const void* a, const void* b, void* c);
extern int oracle_bcsc(const int* types, const int* geo, unsigned int flags, void* A, void* Bvals, unsigned int* colptr,
                       unsigned int* rowidx, void* C);
extern int __real_xb_rt_ptr_kind(const void* p);

static unsigned long long g_launches = 0, g_calls = 0;
static const void* g_colptr = NULL; static const void* g_rowidx = NULL;
static unsigned long long g_nblocks = 0; static unsigned int g_nnzb = 0;
static struct { uintptr_t lo, hi; } g_pageable[8]; static int g_npageable = 0;

/* launches answered (one per single call or batch) and calls computed */
unsigned long long hostsim_sparse_launches(void) { return g_launches; }
unsigned long long hostsim_sparse_calls(void) { return g_calls; }
/* what the last BCSC launch was handed: colptr, rowidx, block-columns, block count (0: unknown on the host) */
void hostsim_sparse_last_bcsc(const void** colptr, const void** rowidx, unsigned long long* n_blocks, unsigned int* nnzb) {
  *colptr = g_colptr; *rowidx = g_rowidx; *n_blocks = g_nblocks; *nnzb = g_nnzb;
}
void hostsim_sparse_mark_pageable(const void* p, size_t bytes) {
  if (g_npageable < 8) { g_pageable[g_npageable].lo = (uintptr_t)p; g_pageable[g_npageable].hi = (uintptr_t)p + bytes; ++g_npageable; }
}
void hostsim_sparse_clear_pageable(void) { g_npageable = 0; }

int __wrap_xb_rt_ptr_kind(const void* p) {
  int i;
  for (i = 0; i < g_npageable; ++i) if ((uintptr_t)p >= g_pageable[i].lo && (uintptr_t)p < g_pageable[i].hi) return 0;
  return __real_xb_rt_ptr_kind(p);
}

int __wrap_xb_packed_sp_launch(const xb_sparse_desc* d, const void* a, const void* b, void* c, long long count,
                               long long sa, long long sb, long long sc) {
  const int dims[6] = { d->m, d->n, d->k, d->lda, d->ldb, d->ldc };
  const int dense = (d->kind == XB_KIND_PK_GEMM || d->kind == XB_KIND_PK_AC_RM || d->kind == XB_KIND_PK_BC_RM);
  const int is_csc = (d->kind == XB_KIND_SP_B_CSC || d->kind == XB_KIND_SP_C_CSC);
  long long t; int rc = 0;
  if (count <= 0) return 0;
  ++g_launches;
  for (t = 0; t < count && rc == 0; ++t, ++g_calls) {
    const char* at = (const char*)a + t * sa; const char* bt = (const char*)b + t * sb; char* ct = (char*)c + t * sc;
    if (dense) rc = oracle_packed_dense(d->kind - XB_KIND_PK_GEMM, d->ta, dims, d->flags, d->packed_width, at, bt, ct);
    else rc = oracle_packed_sp(is_csc, d->ta, dims, d->flags, d->packed_width, d->d_ptr, d->d_idx, NULL, (void*)(uintptr_t)at, (void*)(uintptr_t)bt, ct);
  }
  return rc;
}

int __wrap_xb_bcsc_launch(xb_sparse_desc* d, const void* a, const void* b_vals, const unsigned int* colptr, const unsigned int* rowidx,
                          unsigned long long n_blocks, unsigned int nnzb, void* c) {
  const int types[4] = { d->ta, d->tb, d->tcomp, d->tc };
  const int geo[6] = { d->m, d->packed_width, d->k, (int)(n_blocks * (unsigned long long)d->bn), d->bk, d->bn };
  const long long count = (d->calls.count > 1) ? d->calls.count : 1;
  long long t; int rc = 0;
  g_colptr = colptr; g_rowidx = rowidx; g_nblocks = n_blocks; g_nnzb = nnzb;
  if (d->m <= 0 || n_blocks == 0) return 0;
  ++g_launches;
  for (t = 0; t < count && rc == 0; ++t, ++g_calls) {
    rc = oracle_bcsc(types, geo, d->flags, (char*)(uintptr_t)a + t * d->calls.s_a, (char*)(uintptr_t)b_vals + t * d->calls.s_b,
                     (unsigned int*)(uintptr_t)colptr, (unsigned int*)(uintptr_t)rowidx, (char*)c + t * d->calls.s_c);
  }
  return rc;
}
