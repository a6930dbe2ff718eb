// kuq_buffers.cuh — move-only owners of CUDA resources: device memory, pinned host memory, streams and events.
//
// An owner frees what it holds when it is reset, re-allocated, assigned another owner or goes out of scope, on the
// device that was current when it was allocated (the current device is restored afterwards).  So an error return frees
// every temporary made before it, and a struct of owners needs no list of frees kept in step with its members.  Owners
// convert to the raw pointer or handle, so they pass to kernels, Params and copies as they are.  cudaFree synchronises
// the device: where a temporary must go before further work, reset() it there.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

namespace kuq {

template <typename Kind>
class Owned {
 public:
  using Handle = typename Kind::Handle;
  Owned() = default;
  Owned(const Owned &) = delete;
  Owned &operator=(const Owned &) = delete;
  Owned(Owned &&o) noexcept : h_(std::exchange(o.h_, nullptr)), dev_(o.dev_) {}
  Owned &operator=(Owned &&o) noexcept {
    if (this != &o) { reset(); h_ = std::exchange(o.h_, nullptr); dev_ = o.dev_; }
    return *this;
  }
  ~Owned() { reset(); }

  // frees what the owner held, then makes `n` items of memory, or a stream / event with the flags `n`, on the current
  // device; the owner stays empty when that fails
  cudaError_t alloc(uint64_t n) {
    reset();
    cudaGetDevice(&dev_);
    const cudaError_t e = Kind::make(&h_, n);
    if (e != cudaSuccess) h_ = nullptr;
    return e;
  }
  void reset() {
    if (!h_) return;
    int cur = dev_;
    cudaGetDevice(&cur);
    if (cur != dev_) cudaSetDevice(dev_);
    Kind::destroy(std::exchange(h_, nullptr));
    if (cur != dev_) cudaSetDevice(cur);
  }
  Handle release() { return std::exchange(h_, nullptr); }   // the caller takes over the resource and its free
  Handle get() const { return h_; }
  operator Handle() const { return h_; }

 private:
  Handle h_ = nullptr;
  int dev_ = 0;
};

template <typename T>
struct DeviceMemory {
  using Handle = T *;
  static cudaError_t make(T **p, uint64_t n) { return cudaMalloc((void **)p, n * sizeof(T)); }
  static void destroy(T *p) { cudaFree(p); }
};
template <typename T>
struct PinnedMemory {
  using Handle = T *;
  static cudaError_t make(T **p, uint64_t n) { return cudaMallocHost((void **)p, n * sizeof(T)); }
  static void destroy(T *p) { cudaFreeHost(p); }
};
struct StreamHandle {
  using Handle = cudaStream_t;
  static cudaError_t make(cudaStream_t *s, uint64_t flags) { return cudaStreamCreateWithFlags(s, (unsigned)flags); }
  static void destroy(cudaStream_t s) { cudaStreamDestroy(s); }
};
struct EventHandle {
  using Handle = cudaEvent_t;
  static cudaError_t make(cudaEvent_t *e, uint64_t flags) { return cudaEventCreateWithFlags(e, (unsigned)flags); }
  static void destroy(cudaEvent_t e) { cudaEventDestroy(e); }
};

template <typename T>
using DevBuf = Owned<DeviceMemory<T>>;
template <typename T>
using HostBuf = Owned<PinnedMemory<T>>;
using Stream = Owned<StreamHandle>;
using Event = Owned<EventHandle>;

}  // namespace kuq
