// Block-level rules shared by the SLAM kernels: the device count's clamp, ordered compaction, and the fixed reduction tree.
// Only integer ops and IEEE adds: the files that include this header build with and without -fmad=false, and compute the same.
#pragma once
#include <cuda_runtime.h>

namespace sivo {

// A device count clamped to the capacity; a negative count is passed on as -1.
__device__ __forceinline__ int clamp_count(long long n, int cap) {
  return n < 0 ? -1 : static_cast<int>(min(n, static_cast<long long>(cap)));
}

// The rank of this thread's `flag` among the set flags of a kThreads-thread block, in thread order (warp ballots, then the
// per-warp counts), with the block's count in *total; every thread must call it.  warp_count: kThreads / 32 ints of shared
// memory.  Ends after the barrier that publishes warp_count: the caller needs another barrier before warp_count is reused.
template <int kThreads>
__device__ __forceinline__ int block_rank(bool flag, int* warp_count, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ballot = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_count[warp] = __popc(ballot);
  __syncthreads();
  int before = 0, sum = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const int k = warp_count[w];
    before += w < warp ? k : 0;
    sum += k;
  }
  *total = sum;
  return before + __popc(ballot & ((1u << lane) - 1u));
}

// Ordered stream compaction by one block, one chunk of kThreads consecutive items at a time: a kept item `i` goes to
// out[base + its rank in the chunk], so the kept indices come out ascending, as a sequential host loop builds them.  Returns
// `base` plus the chunk's kept count, the running offset for the next chunk.  out may be NULL (count only).
template <int kThreads>
__device__ __forceinline__ int compact_chunk(bool keep, int i, int base, int* warp_kept, int* out) {
  int total;
  const int rank = block_rank<kThreads>(keep, warp_kept, &total);
  if (keep && out) out[base + rank] = i;
  __syncthreads();  // warp_kept is rewritten by the next chunk
  return base + total;
}

// The fixed reduction tree, in double.  A warp's sum: xor shuffles 16, 8, 4, 2, 1 (every lane ends with it).
__device__ __forceinline__ double warp_tree_sum(double v) {
#pragma unroll
  for (int s = 16; s; s >>= 1) v = v + __shfl_xor_sync(0xffffffffu, v, s);
  return v;
}

// Then the kWarps warp totals w[0 .. kWarps), folded in place as w[i] + w[i + s] for s = kWarps / 2, ..., 1; returns w[0].
template <int kWarps>
__device__ __forceinline__ double fold_warp_totals(double* w) {
#pragma unroll
  for (int s = kWarps / 2; s; s >>= 1)
#pragma unroll
    for (int i = 0; i < s; ++i) w[i] = w[i] + w[i + s];
  return w[0];
}

}  // namespace sivo
