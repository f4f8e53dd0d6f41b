/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * Counts the calls of the exact-order GEMM launcher for the simulated device of tests/c/hostsim_runtime.c, whose launcher answers a
 * launch tile by tile (and counts each tile as a launch). tests/test_gemm_ext_batch_hostsim.py links it with
 * -Wl,--wrap=xb_gemm_simt_launch: every launch is counted once here and then goes on to the runtime's launcher unchanged. */
#include "../../libxsmm_b200/csrc/xb_internal.h"

extern int __real_xb_gemm_simt_launch(const xb_gemm_launch* L);

static unsigned long long g_gemm_launches = 0;
unsigned long long hostsim_gemm_launches(void) { return g_gemm_launches; }

int __wrap_xb_gemm_simt_launch(const xb_gemm_launch* L) {
  ++g_gemm_launches;
  return __real_xb_gemm_simt_launch(L);
}
