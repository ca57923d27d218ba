#include <mutex>

#include "stream_scratch.h"

namespace sivo {
cudaMemPool_t scratch_pool(int device) {
  static std::mutex mu;
  static std::vector<cudaMemPool_t> pools;
  std::lock_guard<std::mutex> lock(mu);
  if (device >= static_cast<int>(pools.size())) pools.resize(device + 1, nullptr);
  if (pools[device]) return pools[device];
  cudaMemPoolProps props{};
  props.allocType = cudaMemAllocationTypePinned;
  props.location = {cudaMemLocationTypeDevice, device};
  uint64_t keep = UINT64_MAX;
  int internal_deps = 0;
  cudaMemPool_t pool;
  SIVO_CUDA(cudaMemPoolCreate(&pool, &props));
  SIVO_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
  SIVO_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolReuseAllowInternalDependencies, &internal_deps));
  return pools[device] = pool;
}
}  // namespace sivo
