// Scratch of one device-form call: one allocation from the library's stream-ordered pool, made and freed on the call's stream,
// so calls on different streams never share scratch and none synchronises the host.  The pool (one per device, created on first
// use and kept for the life of the process; the device's default pool is left to the rest of the process) keeps what is freed
// instead of unmapping it at each synchronisation, and never hands out memory still pending on another stream, which would add
// a hidden wait on that stream: it grows instead.
#pragma once
#include "common.h"

namespace sivo {
cudaMemPool_t scratch_pool(int device);  // stream_scratch.cu

class StreamScratch {
 public:
  // one allocation of `bytes` on the current device, ordered on `s`; nothing at 0 bytes
  StreamScratch(size_t bytes, cudaStream_t s) : stream_(s) {
    if (!bytes) return;
    int dev;
    SIVO_CUDA(cudaGetDevice(&dev));
    SIVO_CUDA(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&base_), bytes, scratch_pool(dev), s));
    size_ = bytes;
  }
  // frees on the same stream, after the work the call enqueued; never throws
  ~StreamScratch() { if (base_) cudaFreeAsync(base_, stream_); }
  StreamScratch(const StreamScratch&) = delete;
  StreamScratch& operator=(const StreamScratch&) = delete;
  // the room take<T>(count) needs, to size the allocation
  template <class T> static size_t bytes(size_t count) { return (count * sizeof(T) + 255) & ~static_cast<size_t>(255); }
  // the next 256-byte-aligned piece of `count` elements
  template <class T> T* take(size_t count) {
    const size_t off = bytes<uint8_t>(used_);
    used_ = off + count * sizeof(T);
    if (used_ > size_) fail(SIVO_EINVAL, "internal: %zu bytes taken from a scratch of %zu", used_, size_);
    return reinterpret_cast<T*>(base_ + off);
  }
 private:
  uint8_t* base_ = nullptr;
  size_t size_ = 0, used_ = 0;
  cudaStream_t stream_;
};
}  // namespace sivo
