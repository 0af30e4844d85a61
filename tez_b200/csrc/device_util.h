// device_util.h -- host-side RAII helpers (device selection, device / pinned buffers) for libtezgpu.
#pragma once
#include <cudaTypedefs.h>

#include "../../include/tezgpu.h"
#include "common.cuh"

namespace tezgpu {

// Device bytes a group of DeviceBuffers holds, and the most it held at once.  A buffer allocated while a thread has
// g_device_tally set counts against that tally until it is freed (merge_steps.cuh reports a bounded merge's peak).
struct DeviceTally {
  uint64_t live = 0, peak = 0;
  void add(size_t b) { live += b; if (live > peak) peak = live; }
};
inline thread_local DeviceTally *g_device_tally = nullptr;

struct TallyScope {
  DeviceTally *prev;
  explicit TallyScope(DeviceTally *t) : prev(g_device_tally) { g_device_tally = t; }
  ~TallyScope() { g_device_tally = prev; }
};

// The device a C ABI call runs on: every entry point that touches CUDA opens one scope, on its handle's conf.device or
// its device argument, and everything under it (streams, events, buffers, kernels) uses the current device.  The
// calling thread's CUDA context is current again when the call returns or throws.  A thread that had none is left on
// the call's device: selecting device 0, which it reports, would create a context on a device it never used.
class DeviceScope {
  CUcontext prev = nullptr;
  // cuCtxGetCurrent / cuCtxSetCurrent, looked up through the runtime so that the library does not link libcuda
  struct CtxApi {
    PFN_cuCtxGetCurrent get = nullptr;
    PFN_cuCtxSetCurrent set = nullptr;
    CtxApi() {
      TG_CUDA(cudaGetDriverEntryPoint("cuCtxGetCurrent", (void **)&get, cudaEnableDefault));
      TG_CUDA(cudaGetDriverEntryPoint("cuCtxSetCurrent", (void **)&set, cudaEnableDefault));
      TG_CHECK(get && set, TEZGPU_E_CUDA, "the CUDA driver has no cuCtxGetCurrent / cuCtxSetCurrent");
    }
  };
  static const CtxApi &ctx() {
    static const CtxApi api;
    return api;
  }

 public:
  explicit DeviceScope(int d) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
      cudaGetLastError();
      throw Error(TEZGPU_E_CUDA, "no CUDA device available (libtezgpu has no CPU fallback)");
    }
    TG_CHECK(d >= 0 && d < n, TEZGPU_E_INVALID, "bad device ordinal");
    if (ctx().get(&prev) != CUDA_SUCCESS) prev = nullptr;
    TG_CUDA(cudaSetDevice(d));
  }
  ~DeviceScope() {
    if (prev) ctx().set(prev);
  }
  DeviceScope(const DeviceScope &) = delete;
  DeviceScope &operator=(const DeviceScope &) = delete;
};

struct DeviceBuffer {
  void *p = nullptr;
  size_t cap = 0;
  DeviceTally *tally = nullptr;
  ~DeviceBuffer() { release(); }
  DeviceBuffer() = default;
  DeviceBuffer(const DeviceBuffer &) = delete;
  DeviceBuffer &operator=(const DeviceBuffer &) = delete;
  void release() {
    if (p) cudaFree(p);
    if (tally) tally->live -= cap;
    p = nullptr;
    cap = 0;
    tally = nullptr;
  }
  void counted(size_t bytes) {
    tally = g_device_tally;
    if (tally) tally->add(bytes);
  }
  // grow-only; contents are NOT preserved
  void ensure(size_t bytes) {
    bytes = align_up(bytes ? bytes : 16, 256);
    if (bytes <= cap) return;
    release();
    TG_CUDA(cudaMalloc(&p, bytes));
    cap = bytes;
    counted(bytes);
  }
  // grow preserving the first `keep` bytes
  void grow_preserve(size_t bytes, size_t keep, cudaStream_t st) {
    bytes = align_up(bytes ? bytes : 16, 256);
    if (bytes <= cap) return;
    size_t ncap = cap ? cap : 4096;
    while (ncap < bytes) ncap = ncap + ncap / 2;
    ncap = align_up(ncap, 256);
    void *np = nullptr;
    cudaError_t e = cudaMalloc(&np, ncap);
    if (e != cudaSuccess) {
      cudaGetLastError();
      ncap = bytes;  // retry with the exact size before giving up
      TG_CUDA(cudaMalloc(&np, ncap));
    }
    if (keep) {
      TG_CUDA(cudaMemcpyAsync(np, p, keep, cudaMemcpyDeviceToDevice, st));
      TG_CUDA(cudaStreamSynchronize(st));
    }
    DeviceTally *t = g_device_tally;
    if (t) t->add(ncap);  // old and new are both held until the copy is done
    release();
    p = np;
    cap = ncap;
    tally = t;
  }
  template <typename T>
  T *as() const { return reinterpret_cast<T *>(p); }
};

struct PinnedBuffer {
  void *p = nullptr;
  size_t cap = 0;
  ~PinnedBuffer() { release(); }
  PinnedBuffer() = default;
  PinnedBuffer(const PinnedBuffer &) = delete;
  PinnedBuffer &operator=(const PinnedBuffer &) = delete;
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
  void ensure(size_t bytes) {
    bytes = align_up(bytes ? bytes : 16, 4096);
    if (bytes <= cap) return;
    release();
    TG_CUDA(cudaHostAlloc(&p, bytes, cudaHostAllocDefault));
    cap = bytes;
  }
  template <typename T>
  T *as() const { return reinterpret_cast<T *>(p); }
};

struct EventTimer {
  cudaEvent_t ev[8];
  int n = 0;
  EventTimer() { for (auto &e : ev) cudaEventCreate(&e); }
  ~EventTimer() { for (auto &e : ev) cudaEventDestroy(e); }
  void mark(cudaStream_t st) { if (n < 8) cudaEventRecord(ev[n++], st); }
  float ms(int a, int b) {
    float f = 0;
    if (a < n && b < n) cudaEventElapsedTime(&f, ev[a], ev[b]);
    return f;
  }
  void reset() { n = 0; }
};

}  // namespace tezgpu
