/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * Low-bit weight tiles (I2X4 / I1X8 x I8 / U8 -> I32, MXFP4X2 x I8 -> F32 / BF16) for the simulated device of tests/c/hostsim_runtime.c.
 * tests/test_lowbit_hostsim.py links the host_*.c objects, that runtime and this file with -Wl,--wrap=xb_gemm_simt_launch: a launch of
 * such a descriptor is answered tile by tile by the low-bit oracle (oracle/oracle_lowbit.c) with the operands and block scales the host
 * code resolved (single calls: L->one, strided batches: the per-tile strides, per-tile records: each record); every other launch goes
 * on to the runtime's own launcher. Missing MXFP4 scales are noted like the real launcher does and launch nothing. */
#include <stdio.h>
#include <string.h>
#include "../../libxsmm_b200/csrc/xb_internal.h"

extern int __real_xb_gemm_simt_launch(const xb_gemm_launch* L);
extern int oracle_gemm_lowbit(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                              unsigned long long br, const void* a, const void* b, void* c, const long long* offs_a, const long long* offs_b,
                              const void* scf_a, const void* scf_b);

int __wrap_xb_gemm_simt_launch(const xb_gemm_launch* L) {
  const xb_gemm_desc* d = &L->d;
  const int dims[6] = { d->m, d->n, d->k, d->lda, d->ldb, d->ldc }, types[4] = { d->ta, d->tb, d->tcomp, d->tc };
  const int form = xb_lowbit_form(d), single = (L->recs == NULL && L->a == NULL && L->c == NULL);
  long long t; int rc = 0;
  if (form == XB_LB_NONE) return __real_xb_gemm_simt_launch(L);
  for (t = 0; t < L->count && rc == 0; ++t) {
    xb_gemm_rec r;
    if (L->recs != NULL) r = L->recs[t];
    else if (single) r = L->one;
    else {
      r = L->one;
      r.a = (const char*)L->a + t * L->tile_stride_a; r.b = (const char*)L->b + t * L->tile_stride_b; r.c = (char*)L->c + t * L->tile_stride_c;
      r.br = L->br;
      r.a_s = (L->one.a_s == NULL) ? NULL : (const char*)L->one.a_s + t * L->tile_stride_as;
      r.b_s = (L->one.b_s == NULL) ? NULL : (const char*)L->one.b_s + t * L->tile_stride_bs;
    }
    if (form == XB_LB_MXFP4 && (r.a_s == NULL || r.b_s == NULL)) {
      xb_rt_note_error(1, "MXFP4 x I8: block scales missing (a.tertiary, b.tertiary)");
      return 1;
    }
    xb_rt_count_launch();
    rc = oracle_gemm_lowbit(dims, types, d->flags, d->br_type, d->br_stride_a, d->br_stride_b, d->br_type ? r.br : 1, r.a, r.b, r.c,
                            (const long long*)r.a_aux, (const long long*)r.b_aux, r.a_s, r.b_s);
  }
  if (rc != 0) fprintf(stderr, "hostsim: the low-bit oracle refused a GEMM tile (rc %d)\n", rc);
  return rc;
}
