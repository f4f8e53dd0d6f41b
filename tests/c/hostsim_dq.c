/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * Dequantising-A tiles (I8 x BF16, I8 / I4 / U4 / BF8 x F16) for the simulated device of tests/c/hostsim_runtime.c.
 * tests/test_dequant_hostsim.py links the host_*.c objects, that runtime and this file with -Wl,--wrap=xb_gemm_simt_launch: a launch of
 * such a descriptor is answered tile by tile by the dequantising oracle (oracle/oracle_dq.c) with the operands, row scales and zero
 * points the host code resolved (xb_gemm_tile); every other launch goes on to the runtime's own launcher. */
#include <stdio.h>
#include <string.h>
#include "../../libxsmm_b200/csrc/xb_internal.h"

extern int __real_xb_gemm_simt_launch(const xb_gemm_launch* L);
extern int oracle_gemm_dq(const int* dims, const int* types, unsigned int flags, int br_type, long long stride_a, long long stride_b,
                          unsigned long long br, const void* a, const void* b, void* c, const long long* offs_a, const long long* offs_b,
                          const void* scf, const void* zpt);

int __wrap_xb_gemm_simt_launch(const xb_gemm_launch* L) {
  const xb_gemm_desc* d = &L->d;
  const int dims[6] = { d->m, d->n, d->k, d->lda, d->ldb, d->ldc }, types[4] = { d->ta, d->tb, d->tcomp, d->tc };
  long long t; int rc = 0;
  if (d->path != P_DQ) return __real_xb_gemm_simt_launch(L);
  for (t = 0; t < L->count && rc == 0; ++t) {
    const xb_gemm_rec r = xb_gemm_tile(L, t);
    xb_rt_count_launch();
    rc = oracle_gemm_dq(dims, types, d->flags, d->br_type, d->br_stride_a, d->br_stride_b, d->br_type ? r.br : 1, r.a, r.b, r.c,
                        (const long long*)r.a_aux, (const long long*)r.b_aux, r.a_s, r.a_q);
  }
  if (rc != 0) fprintf(stderr, "hostsim: the dequantising oracle refused a GEMM tile (rc %d)\n", rc);
  return rc;
}
