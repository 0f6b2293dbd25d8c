// launch.cuh -- the one place the library issues a kernel, and the per-device state of its launchers.
#pragma once

#include <atomic>
#include <mutex>

#include <cuda_runtime.h>

namespace ovrfsr {

// Work the launchers do once per device ordinal: kernel attributes, the NIS filter banks and the SM count all belong to
// ONE device, so a process that drives several GPUs needs each on each.  The first call on a device runs
// make(dev, value) under a lock; a concurrent call on that device waits for it, so whatever make did (a synchronous
// upload) is done before either caller goes on.  Later calls return the stored `value` without the lock.  A make that
// fails is not recorded, and the next call runs it again.  Ordinals >= kMaxDevices are not cached: make runs each time.
class PerDevice {
 public:
  template <class Make>
  cudaError_t once(Make &&make, int *value = nullptr) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const bool cached = dev >= 0 && dev < kMaxDevices;
    if (!cached || !done_[dev].load(std::memory_order_acquire)) {
      std::lock_guard<std::mutex> lock(mu_);
      if (!cached) {
        int v = 0;
        e = make(dev, v);
        if (value) *value = v;
        return e;
      }
      if (!done_[dev].load(std::memory_order_relaxed)) {
        if ((e = make(dev, value_[dev])) != cudaSuccess) return e;
        done_[dev].store(true, std::memory_order_release);
      }
    }
    if (value) *value = value_[dev];
    return cudaSuccess;
  }

 private:
  static constexpr int kMaxDevices = 64;
  std::mutex mu_;
  std::atomic<bool> done_[kMaxDevices] = {};
  int value_[kMaxDevices] = {};
};

// the multiprocessor count of the current device (132, an H100 SXM's, where it cannot be read)
inline int sm_count() {
  static PerDevice counts;
  int n = 0;
  const cudaError_t e = counts.once([](int dev, int &v) { return cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev); }, &n);
  return e == cudaSuccess && n > 0 ? n : 132;
}

// A kernel's dynamic shared memory above the default 48 KB: `bytes` is what it may ask for (0: no opt-in), and
// `maxCarveout` also asks for the largest shared-memory carve-out of the SM.
struct SmemOptIn {
  int bytes;
  bool maxCarveout;
};
constexpr SmemOptIn kNoOptIn = {0, false};

// bumped by launch() once per kernel it issues (ovrfsr_kernel_launches)
void count_launch();

// Issues Kernel<<<grid, threads, smem, s>>>(args...) and returns the launch's status.  With an opt-in, the kernel's
// attributes are set first, once per device (cudaFuncSetAttribute applies to the current device only); a kernel without
// one makes no other CUDA call here.
template <auto Kernel, class... A>
cudaError_t launch(dim3 grid, int threads, size_t smem, SmemOptIn optIn, cudaStream_t s, const A &...args) {
  if (optIn.bytes) {
    static PerDevice attributes;
    const cudaError_t e = attributes.once([&](int, int &) {
      cudaError_t r = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optIn.bytes);
      if (r == cudaSuccess && optIn.maxCarveout)
        r = cudaFuncSetAttribute(Kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
      return r;
    });
    if (e != cudaSuccess) return e;
  }
  Kernel<<<grid, threads, smem, s>>>(args...);
  count_launch();
  return cudaGetLastError();
}

} // namespace ovrfsr
