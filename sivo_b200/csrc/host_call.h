// Staging for the host-buffer entry points (stereo / Hamming / information selection / projection searches / pose): per thread and
// device, device memory that only grows and one non-blocking stream.  Each such call uploads and takes its buffers after begin()
// and synchronises before it returns, so the calls of one thread share it.
// (Allocating and freeing half a dozen buffers per call and running on the legacy default stream synchronises the whole device,
// i.e. serialises every per-frame call against the SegNet graph and the extractors' streams.)
#pragma once
#include <algorithm>
#include <vector>

#include "common.h"

namespace sivo {

struct HostCall {
  int device = -1;
  cudaStream_t stream = nullptr;
  // Buffers are taken from the last block.  A take that does not fit opens another block, so pointers taken earlier in the
  // call stay valid; the next begin() merges the blocks into one that holds the same call again without growing.
  std::vector<DevBuf> blocks;
  size_t used = 0;  // of blocks.back()

  void begin(int dev) {
    SIVO_CUDA(cudaSetDevice(dev));
    if (device != dev) {
      if (stream) { cudaSetDevice(device); cudaStreamDestroy(stream); cudaSetDevice(dev); }
      blocks.clear();
      SIVO_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
      device = dev;
    }
    if (blocks.size() > 1) {
      SIVO_CUDA(cudaStreamSynchronize(stream));
      const size_t total = held();
      blocks.clear();
      blocks.emplace_back(total);
    }
    used = 0;
  }
  // 256-byte-aligned device memory for max(count, 1) elements, valid until the next begin() on this thread
  template <class T> T* take(size_t count) {
    const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
    used = (used + 255) & ~static_cast<size_t>(255);
    if (blocks.empty() || used + bytes > blocks.back().bytes) {
      blocks.emplace_back(std::max(bytes, held() / 2));
      used = 0;
    }
    T* p = reinterpret_cast<T*>(blocks.back().as<uint8_t>() + used);
    used += bytes;
    return p;
  }
  // take() + copy on the stream; a null `host` or a zero count copies nothing
  template <class T> T* upload(const T* host, size_t count) {
    T* dev = take<T>(count);
    if (host && count) SIVO_CUDA(cudaMemcpyAsync(dev, host, count * sizeof(T), cudaMemcpyHostToDevice, stream));
    return dev;
  }
  template <class T> void download(T* host, const T* dev, size_t count) {
    if (host && count) SIVO_CUDA(cudaMemcpyAsync(host, dev, count * sizeof(T), cudaMemcpyDeviceToHost, stream));
  }
  void sync() { SIVO_CUDA(cudaStreamSynchronize(stream)); }
  ~HostCall() { if (stream) { cudaSetDevice(device); cudaStreamDestroy(stream); } }
  size_t held() const {
    size_t b = 0;
    for (const DevBuf& blk : blocks) b += blk.bytes;
    return b;
  }
};
HostCall& host_call();  // the calling thread's instance (stereo.cu)

}  // namespace sivo
