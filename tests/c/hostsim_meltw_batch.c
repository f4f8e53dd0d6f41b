/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * Batched matrix-eltwise launches for the simulated device of tests/c/hostsim_runtime.c. tests/test_meltw_batch_hostsim.py links the
 * host_*.c objects, that runtime and this file with -Wl,--wrap=xb_meltw_launch: a launch with a tile axis (count > 1) is answered
 * call by call, each call's operands advanced by its strides, through the runtime's own launcher (the oracle); every other launch
 * goes on to that launcher unchanged. What this checks is the host half of the batch forms, not any kernel. */
#include <string.h>
#include "../../libxsmm_b200/csrc/xb_internal.h"

extern int __real_xb_meltw_launch(const xb_meltw_desc* d, const xb_meltw_args* a);

static unsigned long long g_batch_launches = 0;
/* launches with a tile axis seen by the wrapper: one per batch (per node and chunk for an equation) */
unsigned long long hostsim_batch_launches(void) { return g_batch_launches; }

int __wrap_xb_meltw_launch(const xb_meltw_desc* d, const xb_meltw_args* a) {
  long long t; int rc = 0;
  if (a->count <= 1) return __real_xb_meltw_launch(d, a);
  ++g_batch_launches;
  for (t = 0; t < a->count && rc == 0; ++t) {
    xb_meltw_args c = *a;
    c.count = 0;
    c.in0 = a->in0 ? (const char*)a->in0 + t * a->s_in0 : NULL;
    c.in1 = a->in1 ? (const char*)a->in1 + t * a->s_in1 : NULL;
    c.in2 = a->in2 ? (const char*)a->in2 + t * a->s_in2 : NULL;
    c.in_aux = a->in_aux ? (const char*)a->in_aux + t * a->s_in_aux : NULL;
    c.out = a->out ? (char*)a->out + t * a->s_out : NULL;
    c.out_aux = a->out_aux ? (char*)a->out_aux + t * a->s_out_aux : NULL;
    rc = __real_xb_meltw_launch(d, &c);
  }
  return rc;
}
