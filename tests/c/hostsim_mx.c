/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * MX fp8 tiles for the simulated device of tests/c/hostsim_runtime.c. tests/test_mxfp8_hostsim.py links the host_*.c objects, that
 * runtime and this file with -Wl,--wrap=xb_gemm_simt_launch: a launch of an MXBF8 / MXHF8 descriptor is answered tile by tile by
 * the MX oracle (oracle/oracle_mx.c) with the block scales the host code resolved (single calls: L->one, strided batches: the
 * per-tile scale strides); every other launch goes on to the runtime's own launcher. */
#include <stdio.h>
#include <string.h>
#include "../../libxsmm_b200/csrc/xb_internal.h"

extern int __real_xb_gemm_simt_launch(const xb_gemm_launch* L);
extern int oracle_gemm_mx(const int* dims, const int* types, unsigned int flags, int br_type, unsigned long long br,
                          const unsigned char* a, const unsigned char* b, void* c, const unsigned char* a_s, const unsigned char* b_s,
                          unsigned char* c_s);

int __wrap_xb_gemm_simt_launch(const xb_gemm_launch* L) {
  const xb_gemm_desc* d = &L->d;
  const int dims[6] = { d->m, d->n, d->k, d->lda, d->ldb, d->ldc }, types[4] = { d->ta, d->tb, d->tcomp, d->tc };
  const int single = (L->a == NULL && L->c == NULL);
  long long t; int rc = 0;
  if (d->ta != LIBXSMM_DATATYPE_MXBF8 && d->ta != LIBXSMM_DATATYPE_MXHF8) return __real_xb_gemm_simt_launch(L);
  if (L->recs != NULL) return 1;                 /* MX handles never reach the per-tile record forms */
  for (t = 0; t < L->count && rc == 0; ++t) {
    const char* a = single ? (const char*)L->one.a : (const char*)L->a + t * L->tile_stride_a;
    const char* b = single ? (const char*)L->one.b : (const char*)L->b + t * L->tile_stride_b;
    char* c = single ? (char*)L->one.c : (char*)L->c + t * L->tile_stride_c;
    const char* as = (const char*)L->one.a_s + (single ? 0 : t * L->tile_stride_as);
    const char* bs = (const char*)L->one.b_s + (single ? 0 : t * L->tile_stride_bs);
    char* cs = (L->one.c_s == NULL) ? NULL : (char*)L->one.c_s + (single ? 0 : t * L->tile_stride_cs);
    xb_rt_count_launch();
    rc = oracle_gemm_mx(dims, types, d->flags, d->br_type, single ? L->one.br : L->br, (const unsigned char*)a, (const unsigned char*)b, c,
                        (const unsigned char*)as, (const unsigned char*)bs, (unsigned char*)cs);
  }
  if (rc != 0) fprintf(stderr, "hostsim: the MX oracle refused a GEMM tile (rc %d)\n", rc);
  return rc;
}
