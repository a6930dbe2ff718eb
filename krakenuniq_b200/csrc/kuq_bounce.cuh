// Copies between large host images and device memory through two pinned bounce buffers.  The images are usually
// mmap'ed files: a plain cudaMemcpy from pageable memory goes through the driver's single-threaded staging (~7 GB/s,
// page faults included).  Instead NT threads fault the pages in and copy a piece of at most CH bytes into one pinned
// buffer while the previous piece travels.  If pinned memory is refused the buffers are ordinary heap memory: the
// same copies, at the pageable rate.
#ifndef KUQ_BOUNCE_CUH
#define KUQ_BOUNCE_CUH
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

namespace kuq {

struct PinnedBounce {
  static constexpr uint64_t CH = 64ull << 20;
  static constexpr int NT = 8;
  uint8_t *buf[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  bool pinned = false;
  uint64_t next = 0;

  cudaError_t init() {
    pinned = cudaHostAlloc((void **)&buf[0], CH, cudaHostAllocPortable) == cudaSuccess &&
             cudaHostAlloc((void **)&buf[1], CH, cudaHostAllocPortable) == cudaSuccess;
    if (!pinned) {
      (void)cudaGetLastError();
      for (auto &b : buf) { if (b) cudaFreeHost(b); b = (uint8_t *)malloc(CH); }
      if (!buf[0] || !buf[1]) return cudaErrorMemoryAllocation;
    }
    for (auto &e : ev) {
      cudaError_t rc = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
      if (rc != cudaSuccess) return rc;
    }
    return cudaSuccess;
  }
  ~PinnedBounce() {
    for (int b = 0; b < 2; b++) {
      if (ev[b]) { cudaEventSynchronize(ev[b]); cudaEventDestroy(ev[b]); }
      if (buf[b]) { if (pinned) cudaFreeHost(buf[b]); else free(buf[b]); }
    }
  }
  static void host_copy(void *dst, const void *src, uint64_t n) {
    std::vector<std::thread> th;
    const uint64_t per = (n + NT - 1) / NT;
    for (int t = 0; t < NT; t++) {
      const uint64_t a = std::min(n, per * t), e = std::min(n, per * (t + 1));
      if (e > a) th.emplace_back([=] { memcpy((uint8_t *)dst + a, (const uint8_t *)src + a, e - a); });
    }
    for (auto &x : th) x.join();
  }
  // one piece (n <= CH) h_src → d_dst, queued on st behind the work already there; returns once h_src has been read
  cudaError_t h2d(void *d_dst, const void *h_src, uint64_t n, cudaStream_t st) {
    const int b = (int)(next++ & 1);
    cudaError_t rc = cudaEventSynchronize(ev[b]);                // the buffer's previous piece has left
    if (rc != cudaSuccess) return rc;
    host_copy(buf[b], h_src, n);
    if ((rc = cudaMemcpyAsync(d_dst, buf[b], n, cudaMemcpyHostToDevice, st)) != cudaSuccess) return rc;
    return cudaEventRecord(ev[b], st);
  }
  // one piece (n <= CH) d_src → a bounce buffer, after the work queued on st; *out holds it until the next call but one
  cudaError_t d2h(const uint8_t **out, const void *d_src, uint64_t n, cudaStream_t st) {
    const int b = (int)(next++ & 1);
    cudaError_t rc = cudaEventSynchronize(ev[b]);
    if (rc == cudaSuccess) rc = cudaMemcpyAsync(buf[b], d_src, n, cudaMemcpyDeviceToHost, st);
    if (rc == cudaSuccess) rc = cudaEventRecord(ev[b], st);
    if (rc == cudaSuccess) rc = cudaEventSynchronize(ev[b]);
    *out = buf[b];
    return rc;
  }
  // whole images, piece by piece
  cudaError_t to_device(void *d_dst, const void *h_src, uint64_t bytes, cudaStream_t st) {
    for (uint64_t off = 0; off < bytes; off += CH) {
      cudaError_t rc = h2d((uint8_t *)d_dst + off, (const uint8_t *)h_src + off, std::min(CH, bytes - off), st);
      if (rc != cudaSuccess) return rc;
    }
    return cudaSuccess;
  }
  cudaError_t to_host(void *h_dst, const void *d_src, uint64_t bytes, cudaStream_t st) {
    for (uint64_t off = 0; off < bytes; off += CH) {
      const uint64_t n = std::min(CH, bytes - off);
      const uint8_t *piece = nullptr;
      cudaError_t rc = d2h(&piece, (const uint8_t *)d_src + off, n, st);
      if (rc != cudaSuccess) return rc;
      host_copy((uint8_t *)h_dst + off, piece, n);
    }
    return cudaSuccess;
  }
};

}  // namespace kuq
#endif
