/* TEST INFRASTRUCTURE ONLY -- never linked into libxsmm_b200.so.
 *
 * What a matrix-eltwise call stages, for the simulated device of tests/c/hostsim_runtime.c. tests/test_meltw_stage_hostsim.py links
 * the host_*.c objects, that runtime and this file with -Wl,--wrap for xb_rt_upload, xb_rt_memcpy_async and xb_meltw_launch: every
 * upload and every copy back is logged with its host pointer and byte count, and a launch is recorded (its argument struct) and
 * answered with 0 without running anything. What this pins is the host half of a call: which operands travel, how many bytes, and
 * what reaches the launcher. */
#include <string.h>
#include "../../libxsmm_b200/csrc/xb_internal.h"

extern int __real_xb_rt_upload(void* dst_dev, const void* src_host, size_t size);
extern int __real_xb_rt_memcpy_async(void* dst, const void* src, size_t size);

#define XB_STAGE_LOG 64
typedef struct stage_copy { const void* host; unsigned long long bytes; } stage_copy;
static stage_copy g_up[XB_STAGE_LOG], g_down[XB_STAGE_LOG];
static int g_nup = 0, g_ndown = 0, g_nlaunch = 0;
static xb_meltw_args g_args;

void hostsim_stage_reset(void) { g_nup = g_ndown = g_nlaunch = 0; memset(&g_args, 0, sizeof(g_args)); }
/* what the last call did: the uploads and copies back (host pointer, bytes), the number of launches and the last launch's arguments */
int hostsim_stage_uploads(const stage_copy** log) { *log = g_up; return g_nup; }
int hostsim_stage_copies_back(const stage_copy** log) { *log = g_down; return g_ndown; }
int hostsim_stage_launches(void) { return g_nlaunch; }
const xb_meltw_args* hostsim_stage_args(void) { return &g_args; }

int __wrap_xb_rt_upload(void* dst_dev, const void* src_host, size_t size) {
  if (g_nup < XB_STAGE_LOG) { g_up[g_nup].host = src_host; g_up[g_nup].bytes = size; ++g_nup; }
  return __real_xb_rt_upload(dst_dev, src_host, size);
}
int __wrap_xb_rt_memcpy_async(void* dst, const void* src, size_t size) {
  if (g_ndown < XB_STAGE_LOG) { g_down[g_ndown].host = dst; g_down[g_ndown].bytes = size; ++g_ndown; }
  return __real_xb_rt_memcpy_async(dst, src, size);
}
int __wrap_xb_meltw_launch(const xb_meltw_desc* d, const xb_meltw_args* a) {
  (void)d;
  g_args = *a; ++g_nlaunch;
  return 0;
}
