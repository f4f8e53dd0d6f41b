/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * MX fp8 tiles for the simulated device of tests/c/hostsim_runtime.c. tests/test_mxfp8_hostsim.py links the host_*.c objects, that
 * runtime and this file with -Wl,--wrap=xb_gemm_simt_launch: a launch of an MXBF8 / MXHF8 descriptor is answered tile by tile by
 * the MX oracle (oracle/oracle_mx.c) with the block scales the host code resolved (xb_gemm_tile); every other launch goes on to the
 * runtime's own launcher. */
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
  long long t; int rc = 0;
  if (d->path != P_MX8) return __real_xb_gemm_simt_launch(L);
  for (t = 0; t < L->count && rc == 0; ++t) {
    const xb_gemm_rec r = xb_gemm_tile(L, t);
    xb_rt_count_launch();
    rc = oracle_gemm_mx(dims, types, d->flags, d->br_type, r.br, (const unsigned char*)r.a, (const unsigned char*)r.b, r.c,
                        (const unsigned char*)r.a_s, (const unsigned char*)r.b_s, (unsigned char*)r.c_s);
  }
  if (rc != 0) fprintf(stderr, "hostsim: the MX oracle refused a GEMM tile (rc %d)\n", rc);
  return rc;
}
