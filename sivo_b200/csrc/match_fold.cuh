// The ORBmatcher rules shared by the matching kernels (stereo.cu, track.cu, bow.cu, mapping.cu).
//
// The best / second-best fold of ORBmatcher's candidate loops (SearchByProjection, ORBmatcher.cc:79-113 and :1352-1376), shared
// by k_hamming_best2 (stereo.cu) and the projection searches (track.cu):
//   for idx in candidates (in order): dist = DescriptorDistance(q, train[idx]);
//     if (dist < bestDist) { bestDist2 = bestDist; bestLevel2 = bestLevel; bestDist = dist; bestLevel = level[idx]; bestIdx = idx; }
//     else if (dist < bestDist2) { bestLevel2 = level[idx]; bestDist2 = dist; }
#pragma once
#include <cuda_runtime.h>

namespace sivo {

// ORBmatcher::DescriptorDistance (ORBmatcher.cc:1582-1596): the popcount of the XOR of two 256-bit descriptors (a0 a1, b0 b1)
__device__ __forceinline__ int descriptor_distance(uint4 a0, uint4 a1, uint4 b0, uint4 b1) {
  return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) +
         __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// The angle rule of the rotation histogram's searches: a key or point angle takes part only if it is finite and in [0, 360].
// With both angles in range, rot is in [0, 360] and the rotation bin in 0..12, inside the 30-bin histogram; a NaN or infinite
// angle, or one off by more than 360, would index outside it.
__host__ __device__ __forceinline__ bool angle_ok(float a) { return a >= 0.f && a <= 360.f; }

struct Best2 {
  int dist = 256, level = -1, idx = -1;    // bestDist, bestLevel, bestIdx
  int dist2 = 256, level2 = -1, idx2 = -1;  // bestDist2, bestLevel2 and the candidate that set them last
};

// Folds lane k's candidate (d, idx, lvl) for k = 0 .. n-1 in lane order; every lane of the warp calls it with the same `b` and
// ends with the same `b`.  A lane without a candidate passes d >= 256, which can change neither distance, so it is skipped.
__device__ __forceinline__ void best2_fold_warp(Best2& b, int d, int idx, int lvl, int n) {
  unsigned live = __ballot_sync(0xffffffffu, d < 256);
  if (n < 32) live &= (1u << n) - 1u;
  while (live) {
    const int k = __ffs(live) - 1;
    live &= live - 1u;
    const int dk = __shfl_sync(0xffffffffu, d, k), ik = __shfl_sync(0xffffffffu, idx, k), lk = __shfl_sync(0xffffffffu, lvl, k);
    if (dk < b.dist) {
      b.dist2 = b.dist; b.level2 = b.level; b.idx2 = b.idx;
      b.dist = dk; b.level = lk; b.idx = ik;
    } else if (dk < b.dist2) {
      b.level2 = lk; b.dist2 = dk; b.idx2 = ik;
    }
  }
}

// ORBmatcher::ComputeThreeMaxima (ORBmatcher.cc:1545-1577) over the rotation histogram's bin sizes, shared by the last-frame search
// (track.cu) and SearchByBoW (bow.cu): keep[0..2] = ind1, ind2, ind3 (-1: none).
__device__ __forceinline__ void three_maxima(const int* counts, int n, int* keep) {
  int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
  for (int i = 0; i < n; ++i) {
    const int s = counts[i];
    if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
    else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
    else if (s > max3) { max3 = s; ind3 = i; }
  }
  if (max2 < 0.1f * static_cast<float>(max1)) { ind2 = -1; ind3 = -1; }
  else if (max3 < 0.1f * static_cast<float>(max1)) ind3 = -1;
  keep[0] = ind1; keep[1] = ind2; keep[2] = ind3;
}

}  // namespace sivo
