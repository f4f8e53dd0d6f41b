// libxsmm_b200 -- thin CUDA runtime shim used by the plain-C host code: device/stream selection per
// host thread, sticky error reporting (kernels return void, like the reference's handles), memory,
// pointer classification and a per-thread device scratch arena used to stage host-resident operands.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include "xb_internal.h"

namespace {
struct ThreadState {
  cudaStream_t stream = nullptr;
  int blocking = 1;
  char* scratch = nullptr; size_t scratch_cap = 0, scratch_used = 0;
  int scratch_device = -1;                  // the arena belongs to one device: a thread that switches device gets a new one
  // overflow blocks (kept until reset) when a request does not fit the arena
  void* spill[64]; int nspill = 0;
};
thread_local ThreadState tls;
std::atomic<int> g_last_error{0};
std::atomic<unsigned long long> g_launches{0};
std::atomic<unsigned long long> g_launches_by[LIBXSMM_B200_BACKEND_NOOP + 1];   // per kernel family (libxsmm_b200_backend)
char g_error_where[128] = {0};
int g_have_gpu = -1;
}  // namespace

extern "C" {

int xb_rt_have_gpu(void) {
  if (g_have_gpu < 0) {
    int n = 0;
    const cudaError_t e = cudaGetDeviceCount(&n);
    g_have_gpu = (e == cudaSuccess && n > 0) ? 1 : 0;
    if (e != cudaSuccess) (void)cudaGetLastError();
  }
  return g_have_gpu;
}

int xb_rt_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  return n;
}

int xb_rt_set_device(int ordinal) {
  const cudaError_t e = cudaSetDevice(ordinal);
  if (e != cudaSuccess) { xb_rt_note_error((int)e, "set_device"); return (int)e; }
  return 0;
}

void xb_rt_set_stream(void* stream) { tls.stream = (cudaStream_t)stream; }
void* xb_rt_stream(void) { return (void*)tls.stream; }
void xb_rt_set_blocking(int on) { tls.blocking = on ? 1 : 0; }
int xb_rt_blocking(void) { return tls.blocking; }

void xb_rt_note_error(int code, const char* where) {
  int expected = 0;
  bool first = false;
  if (g_last_error.compare_exchange_strong(expected, code)) {
    snprintf(g_error_where, sizeof(g_error_where), "%s", where ? where : "?");
    first = true;
  }
  // handles return void (reference ABI): the first failure is always reported, there is no CPU path to fall back to
  if (first || libxsmm_verbosity != 0) {
    fprintf(stderr, "LIBXSMM-B200 ERROR (%s): %s\n", where ? where : "?", cudaGetErrorString((cudaError_t)code));
  }
}

int xb_rt_sync(void) {
  const cudaError_t e = cudaStreamSynchronize(tls.stream);
  if (e != cudaSuccess) xb_rt_note_error((int)e, "sync");
  return g_last_error.load();
}

int xb_rt_last_error(void) { return g_last_error.load(); }
const char* xb_rt_last_error_string(void) {
  static thread_local char buf[256];
  const int e = g_last_error.load();
  if (e == 0) return "";
  snprintf(buf, sizeof(buf), "%s: %s", g_error_where, cudaGetErrorString((cudaError_t)e));
  return buf;
}

unsigned long long xb_rt_launch_count(void) { return g_launches.load(); }
void xb_rt_count_launch(void) { g_launches.fetch_add(1, std::memory_order_relaxed); }
void xb_rt_count_launch_backend(int backend) {
  xb_rt_count_launch();
  if (backend >= 0 && backend <= LIBXSMM_B200_BACKEND_NOOP) g_launches_by[backend].fetch_add(1, std::memory_order_relaxed);
}
LIBXSMM_API unsigned long long libxsmm_b200_launch_count_backend(int backend) {
  return (backend >= 0 && backend <= LIBXSMM_B200_BACKEND_NOOP) ? g_launches_by[backend].load() : 0ull;
}

void* xb_rt_device_malloc(size_t size) {
  void* p = nullptr;
  const cudaError_t e = cudaMalloc(&p, size ? size : 1);
  if (e != cudaSuccess) { xb_rt_note_error((int)e, "device_malloc"); return nullptr; }
  return p;
}
void xb_rt_device_free(void* p) { if (p) cudaFree(p); }
void* xb_rt_host_malloc(size_t size) {
  void* p = nullptr;
  const cudaError_t e = cudaMallocHost(&p, size ? size : 1);
  if (e != cudaSuccess) { xb_rt_note_error((int)e, "host_malloc"); return nullptr; }
  return p;
}
void xb_rt_host_free(void* p) { if (p) cudaFreeHost(p); }
void* xb_rt_managed_malloc(size_t size) {
  void* p = nullptr;
  const cudaError_t e = cudaMallocManaged(&p, size ? size : 1, cudaMemAttachGlobal);
  if (e != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
  return p;
}
void xb_rt_managed_free(void* p) { if (p) cudaFree(p); }

int xb_rt_memcpy(void* dst, const void* src, size_t size) {
  if (size == 0) return 0;
  cudaError_t e = cudaMemcpyAsync(dst, src, size, cudaMemcpyDefault, tls.stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(tls.stream);
  if (e != cudaSuccess) { xb_rt_note_error((int)e, "memcpy"); return (int)e; }
  return 0;
}
int xb_rt_memcpy_async(void* dst, const void* src, size_t size) {
  if (size == 0) return 0;
  const cudaError_t e = cudaMemcpyAsync(dst, src, size, cudaMemcpyDefault, tls.stream);
  if (e != cudaSuccess) { xb_rt_note_error((int)e, "memcpy_async"); return (int)e; }
  return 0;
}
int xb_rt_upload(void* dst_dev, const void* src_host, size_t size) { return xb_rt_memcpy_async(dst_dev, src_host, size); }
// `rows` pieces of `width` bytes, `pitch` bytes apart on both sides, on the thread's stream: a column block of a wider row-major matrix
int xb_rt_memcpy2d_async(void* dst, const void* src, size_t pitch, size_t width, size_t rows) {
  if (width == 0 || rows == 0) return 0;
  const cudaError_t e = cudaMemcpy2DAsync(dst, pitch, src, pitch, width, rows, cudaMemcpyDefault, tls.stream);
  if (e != cudaSuccess) { xb_rt_note_error((int)e, "memcpy2d_async"); return (int)e; }
  return 0;
}

int xb_rt_ptr_kind(const void* p) {
  if (p == nullptr) return 0;
  cudaPointerAttributes at;
  const cudaError_t e = cudaPointerGetAttributes(&at, p);
  if (e != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  switch (at.type) {
    case cudaMemoryTypeDevice: return 1;
    case cudaMemoryTypeManaged: return 2;
    case cudaMemoryTypeHost: return 3;
    default: return 0;
  }
}

// ---- chunked host <-> device pipeline ------------------------------------------------------------------------------
// Host-resident batches are cut into chunks that flow through three streams (H2D copy, kernel, D2H copy) over two sets
// of staging buffers, so that the copy engines run in both PCIe directions while the kernel of the previous chunk executes.
namespace {
struct Pipe {
  cudaStream_t s_in = nullptr, s_k = nullptr, s_out = nullptr;
  cudaEvent_t in_done[2] = {nullptr, nullptr}, k_done[2] = {nullptr, nullptr}, out_done[2] = {nullptr, nullptr};
  char* buf[2] = {nullptr, nullptr}; size_t cap = 0;
  int device = -1;
};
thread_local Pipe xb_pipe_state;
bool xb_pipe_setup(size_t bytes_per_slot) {
  int dev = 0; cudaGetDevice(&dev);
  if (xb_pipe_state.device != dev) {             // first use on this thread / device change: (re)create streams and events
    xb_pipe_state = Pipe(); xb_pipe_state.device = dev;
    if (cudaStreamCreateWithFlags(&xb_pipe_state.s_in, cudaStreamNonBlocking) != cudaSuccess) return false;
    if (cudaStreamCreateWithFlags(&xb_pipe_state.s_k, cudaStreamNonBlocking) != cudaSuccess) return false;
    if (cudaStreamCreateWithFlags(&xb_pipe_state.s_out, cudaStreamNonBlocking) != cudaSuccess) return false;
    for (int i = 0; i < 2; ++i) {
      if (cudaEventCreateWithFlags(&xb_pipe_state.in_done[i], cudaEventDisableTiming) != cudaSuccess) return false;
      if (cudaEventCreateWithFlags(&xb_pipe_state.k_done[i], cudaEventDisableTiming) != cudaSuccess) return false;
      if (cudaEventCreateWithFlags(&xb_pipe_state.out_done[i], cudaEventDisableTiming) != cudaSuccess) return false;
    }
  }
  if (xb_pipe_state.cap < bytes_per_slot) {
    for (int i = 0; i < 2; ++i) { if (xb_pipe_state.buf[i]) cudaFree(xb_pipe_state.buf[i]); xb_pipe_state.buf[i] = nullptr; }
    xb_pipe_state.cap = 0;
    for (int i = 0; i < 2; ++i) if (cudaMalloc((void**)&xb_pipe_state.buf[i], bytes_per_slot) != cudaSuccess) return false;
    xb_pipe_state.cap = bytes_per_slot;
  }
  return true;
}
}  // namespace

int xb_rt_pipeline(long long nchunks, size_t max_a, size_t max_b, size_t max_c, xb_pipe_describe_fn describe, xb_pipe_launch_fn launch, void* ctx) {
  const size_t oa = 0, ob = (max_a + 255) & ~(size_t)255, oc = ob + ((max_b + 255) & ~(size_t)255);
  const size_t per_slot = oc + ((max_c + 255) & ~(size_t)255);
  if (!xb_pipe_setup(per_slot)) { xb_rt_note_error((int)cudaGetLastError(), "pipeline"); return 2; }
  cudaStream_t user = tls.stream;
  cudaError_t e = cudaStreamSynchronize(user);         // everything the caller queued before this call
  int rc = 0;
  for (long long i = 0; i < nchunks && e == cudaSuccess && rc == 0; ++i) {
    const int s = (int)(i & 1);
    xb_pipe_chunk ch; describe(ctx, i, &ch);
    char* da = xb_pipe_state.buf[s] + oa; char* db = xb_pipe_state.buf[s] + ob; char* dc = xb_pipe_state.buf[s] + oc;
    if (i >= 2) e = cudaStreamWaitEvent(xb_pipe_state.s_in, xb_pipe_state.out_done[s], 0);     // slot free again (its result left the device)
    if (e == cudaSuccess && ch.bytes_a) e = cudaMemcpyAsync(da, ch.host_a, ch.bytes_a, cudaMemcpyHostToDevice, xb_pipe_state.s_in);
    if (e == cudaSuccess && ch.bytes_b) e = cudaMemcpyAsync(db, ch.host_b, ch.bytes_b, cudaMemcpyHostToDevice, xb_pipe_state.s_in);
    if (e == cudaSuccess && ch.copy_c_in && ch.bytes_c) e = cudaMemcpyAsync(dc, ch.host_c, ch.bytes_c, cudaMemcpyHostToDevice, xb_pipe_state.s_in);
    if (e == cudaSuccess) e = cudaEventRecord(xb_pipe_state.in_done[s], xb_pipe_state.s_in);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(xb_pipe_state.s_k, xb_pipe_state.in_done[s], 0);
    if (e != cudaSuccess) break;
    tls.stream = xb_pipe_state.s_k;
    rc = launch(ctx, &ch, da, db, dc);
    tls.stream = user;
    if (rc != 0) break;
    e = cudaEventRecord(xb_pipe_state.k_done[s], xb_pipe_state.s_k);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(xb_pipe_state.s_out, xb_pipe_state.k_done[s], 0);
    if (e == cudaSuccess && ch.bytes_c) e = cudaMemcpyAsync(ch.host_c, dc, ch.bytes_c, cudaMemcpyDeviceToHost, xb_pipe_state.s_out);
    if (e == cudaSuccess) e = cudaEventRecord(xb_pipe_state.out_done[s], xb_pipe_state.s_out);
  }
  cudaError_t e2 = cudaStreamSynchronize(xb_pipe_state.s_in); if (e == cudaSuccess) e = e2;
  e2 = cudaStreamSynchronize(xb_pipe_state.s_k); if (e == cudaSuccess) e = e2;
  e2 = cudaStreamSynchronize(xb_pipe_state.s_out); if (e == cudaSuccess) e = e2;
  if (e != cudaSuccess) { xb_rt_note_error((int)e, "pipeline"); return (int)e; }
  return rc;
}

int xb_rt_current_device(void) { int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); dev = 0; } return dev; }

/* per-(kernel, device) one-time work such as cudaFuncSetAttribute: `mask` holds one bit per device ordinal */
int xb_rt_first_use_on_device(unsigned long long* mask) {
  const int dev = xb_rt_current_device();
  if (dev < 0 || dev >= 64) return 1;
  const unsigned long long bit = 1ull << dev;
  const unsigned long long old = __atomic_fetch_or(mask, bit, __ATOMIC_ACQ_REL);
  return (old & bit) == 0;
}

void* xb_rt_scratch(size_t bytes) {
  bytes = (bytes + 255) & ~(size_t)255;
  {
    const int dev = xb_rt_current_device();
    if (tls.scratch != nullptr && tls.scratch_device != dev && tls.scratch_used == 0) {   // device switched: drop the old arena
      const int cur = dev; cudaSetDevice(tls.scratch_device); cudaFree(tls.scratch); cudaSetDevice(cur);
      tls.scratch = nullptr; tls.scratch_cap = 0;
    }
    tls.scratch_device = dev;
  }
  if (tls.scratch_used + bytes <= tls.scratch_cap) {
    void* p = tls.scratch + tls.scratch_used; tls.scratch_used += bytes; return p;
  }
  if (tls.scratch_used == 0) {               // nothing handed out: grow the arena
    if (tls.scratch) cudaFree(tls.scratch);
    size_t cap = tls.scratch_cap ? tls.scratch_cap : ((size_t)1 << 22);
    while (cap < bytes) cap <<= 1;
    tls.scratch = nullptr; tls.scratch_cap = 0;
    if (cudaMalloc((void**)&tls.scratch, cap) != cudaSuccess) { xb_rt_note_error((int)cudaGetLastError(), "scratch"); return nullptr; }
    tls.scratch_cap = cap; tls.scratch_used = bytes; return tls.scratch;
  }
  if (tls.nspill < 64) {                     // arena in use: one-off block until the next reset
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) { xb_rt_note_error((int)cudaGetLastError(), "scratch"); return nullptr; }
    tls.spill[tls.nspill++] = p; return p;
  }
  return nullptr;
}

void xb_rt_scratch_reset(void) {
  for (int i = 0; i < tls.nspill; ++i) cudaFree(tls.spill[i]);
  tls.nspill = 0; tls.scratch_used = 0;
}

}  // extern "C"
