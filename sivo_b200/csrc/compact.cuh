// Ordered stream compaction by one block: the kept indices of a list come out ascending, as a sequential host loop builds them.
#pragma once
#include <cuda_runtime.h>

namespace sivo {

// One chunk of kThreads consecutive items, one per thread of a kThreads-thread block; every thread must call it.  A kept
// item `i` goes to out[base + number of kept items before it in the chunk] (warp ballots, then the per-warp totals), and the
// return value is `base` plus the chunk's kept count -- the running offset for the next chunk.  warp_kept: kThreads / 32 ints
// of shared memory.  out may be NULL (count only).  lane / warp: threadIdx.x & 31 / threadIdx.x >> 5.
template <int kThreads>
__device__ __forceinline__ int compact_chunk(bool keep, int i, int base, int lane, int warp, int* warp_kept, int* out) {
  const unsigned ballot = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_kept[warp] = __popc(ballot);
  __syncthreads();
  int before = 0, total = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const int k = warp_kept[w];
    before += w < warp ? k : 0;
    total += k;
  }
  if (keep && out) out[base + before + __popc(ballot & ((1u << lane) - 1u))] = i;
  __syncthreads();  // warp_kept is rewritten by the next chunk
  return base + total;
}

}  // namespace sivo
