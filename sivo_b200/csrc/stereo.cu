// Hamming stage of Frame::ComputeStereoMatches (src/orbslam/Frame.cc:452-533) -- SURVEY 8f row 1.
// One warp per left keypoint scans every right keypoint (<= ~2000, descriptors stay in L2): row band
// [floor(vR - 2 s), ceil(vR + 2 s)] must contain int(vL), octave within +-1, uR in [uL - maxD, uL - minD];
// distance = ORBmatcher::DescriptorDistance (ORBmatcher.cc:1582-1596) as 4 x __popcll.  The reference keeps
// the first strictly smaller distance walking candidates in increasing iR, i.e. (min dist, min iR).
#include "frame_ops.h"
#include "host_call.h"
#include "match_fold.cuh"
#include "stream_scratch.h"

namespace sivo {
namespace {
constexpr int kThHigh = 100;  // ORBmatcher::TH_HIGH (ORBmatcher.cc:37)

// The row-band Hamming search of left keypoint L (descriptor a) over right keypoints [0, nr), warp-wide: every lane calls it with
// the same L and gets the warp's packed best (dist << 20 | idx), or (kThHigh << 20 | 0xFFFFF) if no candidate is below kThHigh.
// Right keypoints whose octave is outside [0, nlevels) are skipped.  Where the reference is undefined (a NaN or out-of-range row
// index into vRowIndices) the rule is: a left key with a non-finite x or y, or with (int) y outside [0, rows), has no candidate,
// and a right key with a non-finite x or y is no candidate.  Every test is made in float, before any conversion to int.
__device__ __forceinline__ unsigned stereo_best_right(const sivo_keypoint L, const ulonglong4 a, const sivo_keypoint* __restrict__ kr,
                                                      const uint8_t* __restrict__ dr, int nr, const float* __restrict__ scale, int nlevels,
                                                      int rows, float min_d, float max_d, int lane) {
  const float min_u = __fsub_rn(L.x, max_d), max_u = __fsub_rn(L.x, min_d);
  unsigned best = (static_cast<unsigned>(kThHigh) << 20) | 0xFFFFFu;  // dist:12 | idx:20
  // (int) y in [0, rows) <=> y in (-1, rows) for finite y; NaN fails both compares
  if (isfinite(L.x) && L.y > -1.f && L.y < static_cast<float>(rows) && max_u >= 0.f) {
    const float row = static_cast<float>(static_cast<int>(L.y));
    for (int i = lane; i < nr; i += 32) {
      const sivo_keypoint R = kr[i];
      if (static_cast<unsigned>(R.octave) >= static_cast<unsigned>(nlevels)) continue;
      if (!isfinite(R.x) || !isfinite(R.y)) continue;
      const float band = __fmul_rn(2.0f, scale[R.octave]);
      if (row < floorf(__fsub_rn(R.y, band)) || row > ceilf(__fadd_rn(R.y, band))) continue;
      if (R.octave < L.octave - 1 || R.octave > L.octave + 1) continue;
      if (!(R.x >= min_u && R.x <= max_u)) continue;
      const ulonglong4 b = *reinterpret_cast<const ulonglong4*>(dr + static_cast<size_t>(i) * 32);
      unsigned d = __popcll(a.x ^ b.x) + __popcll(a.y ^ b.y) + __popcll(a.z ^ b.z) + __popcll(a.w ^ b.w);
      if (d < static_cast<unsigned>(kThHigh)) best = min(best, (d << 20) | static_cast<unsigned>(i));
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  return best;
}

__global__ void k_stereo_hamming(const sivo_keypoint* __restrict__ kl, const uint8_t* __restrict__ dl, int nl,
                                 const sivo_keypoint* __restrict__ kr, const uint8_t* __restrict__ dr, int nr,
                                 const float* __restrict__ scale, int nlevels, int rows, float min_d, float max_d,
                                 int* __restrict__ best_idx, int* __restrict__ best_dist) {
  int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= nl) return;
  const ulonglong4 a = *reinterpret_cast<const ulonglong4*>(dl + static_cast<size_t>(wid) * 32);
  const unsigned best = stereo_best_right(kl[wid], a, kr, dr, nr, scale, nlevels, rows, min_d, max_d, lane);
  if (lane == 0) {
    int d = best >> 20;
    best_dist[wid] = d;
    best_idx[wid] = d < kThHigh ? static_cast<int>(best & 0xFFFFFu) : -1;
  }
}

// ---- the whole of Frame::ComputeStereoMatches (Frame.cc:444-629) for one left keypoint per warp: Hamming search as
// above, then the 11x11 SAD slide over +-5 px on the keypoint's pyramid level (windows are centred-intensity
// differences of u8 pixels, so every L1 distance is an exact integer), parabola sub-pixel fit, disparity gate.
// The median-based outlier cut (:617-628) needs all matches: k_stereo_median_cut does it over the SAD distances.
// `round` of the reference is std::round on a float: roundf, half away from zero.
// Where the reference's rowRange / colRange would throw, the rule is: a key stays unmatched (no SAD enters the median) if its
// 11 x 11 window at its octave (rows sv_l +- 5, columns su_l +- 5) or the right slide (rows sv_l +- 5, columns su_r0 - 10 ..
// su_r0 + 10) leaves that level's image.  The reference's own test (iniu < 0 || endu >= cols) stays as written, one column
// stricter on the right than the slide needs.  The tests are made on the rounded floats, before any conversion to int.

// The per-keypoint body; every lane of the warp calls it with the same left keypoint L and descriptor row.
__device__ __forceinline__ void stereo_match_key(const sivo_keypoint L, const uint8_t* __restrict__ dl_key, const sivo_keypoint* __restrict__ kr,
                                                 const uint8_t* __restrict__ dr, int nr, const float* __restrict__ scale,
                                                 const float* __restrict__ inv_scale, const uint8_t* __restrict__ pyr_l, const OrbLevelTable& lt_l,
                                                 const uint8_t* __restrict__ pyr_r, const OrbLevelTable& lt_r, float mb, float mbf, int lane,
                                                 float& out_u, float& out_z, int& out_sad) {
  const float min_d = 0.f, max_d = __fdiv_rn(mbf, mb);
  const unsigned best = stereo_best_right(L, *reinterpret_cast<const ulonglong4*>(dl_key), kr, dr, nr, scale, lt_l.nlevels, lt_l.lv[0].h,
                                          min_d, max_d, lane);
  out_u = -1.f;
  out_z = -1.f;
  out_sad = -1;
  const int hd = best >> 20;
  if (hd < (kThHigh + 50) / 2) {  // thOrbDist = (TH_HIGH + TH_LOW) / 2 (:448)
    const int ir = best & 0xFFFFFu;
    const int oct = L.octave;
    const float sf = inv_scale[oct];
    const float su_l = roundf(__fmul_rn(L.x, sf)), sv_l = roundf(__fmul_rn(L.y, sf)), su_r0 = roundf(__fmul_rn(kr[ir].x, sf));
    const OrbLevel ll = lt_l.lv[oct], lr = lt_r.lv[oct];
    const float iniu = su_r0 + 5.f - 5.f, endu = su_r0 + 5.f + 5.f + 1.f;
    const bool slide_in = su_r0 >= 10.f && sv_l >= 5.f && sv_l <= static_cast<float>(lr.h - 6);
    const bool left_in = su_l >= 5.f && su_l <= static_cast<float>(ll.w - 6) && sv_l >= 5.f && sv_l <= static_cast<float>(ll.h - 6);
    if (!(iniu < 0.f || endu >= static_cast<float>(lr.w)) && slide_in && left_in) {
      const int cx_l = static_cast<int>(su_l), cy = static_cast<int>(sv_l), cx_r = static_cast<int>(su_r0);
      const uint8_t* pl = pyr_l + ll.img_off + static_cast<size_t>(cy + kEdge) * ll.pitch + cx_l + kEdge;
      const uint8_t* pr = pyr_r + lr.img_off + static_cast<size_t>(cy + kEdge) * lr.pitch + cx_r + kEdge;
      const int lc = pl[0];
      int dists[11];
#pragma unroll
      for (int inc = -5; inc <= 5; ++inc) {
        const int rc = pr[inc];
        int s = 0;
        for (int e = lane; e < 121; e += 32) {
          const int dy = e / 11 - 5, dx = e % 11 - 5;
          const int vl = static_cast<int>(pl[dy * ll.pitch + dx]) - lc;
          const int vr = static_cast<int>(pr[dy * lr.pitch + dx + inc]) - rc;
          s += abs(vl - vr);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        dists[inc + 5] = s;
      }
      int bd = 0x7fffffff, binc = 0;
#pragma unroll
      for (int i = 0; i < 11; ++i)
        if (dists[i] < bd) { bd = dists[i]; binc = i - 5; }
      if (binc != -5 && binc != 5) {
        float d1 = 0.f, d2 = 0.f, d3 = 0.f;
#pragma unroll
        for (int i = 1; i < 10; ++i)
          if (i - 5 == binc) { d1 = static_cast<float>(dists[i - 1]); d2 = static_cast<float>(dists[i]); d3 = static_cast<float>(dists[i + 1]); }
        const float delta = __fdiv_rn(__fsub_rn(d1, d3), __fmul_rn(2.0f, __fsub_rn(__fadd_rn(d1, d3), __fmul_rn(2.0f, d2))));
        if (!(delta < -1.f || delta > 1.f)) {
          float best_u = __fmul_rn(scale[oct], __fadd_rn(__fadd_rn(su_r0, static_cast<float>(binc)), delta));
          float disp = __fsub_rn(L.x, best_u);
          if (disp >= min_d && disp < max_d) {
            if (disp <= 0.f) {
              disp = 0.01f;
              best_u = static_cast<float>(static_cast<double>(L.x) - 0.01);
            }
            out_z = __fdiv_rn(mbf, disp);
            out_u = best_u;
            out_sad = bd;
          }
        }
      }
    }
  }
}

// Counts and (optionally) the left keypoint indices live on the device.  Warp j handles left keypoint keep_idx[j] (j when keep_idx
// is NULL) for j < min(*n_left, cap_l); right keypoints [0, min(*n_right, cap_r)).  A left keypoint whose octave or index is out
// of range stays unmatched.
__global__ void k_stereo_match(const sivo_keypoint* __restrict__ kl, const uint8_t* __restrict__ dl, const int* __restrict__ keep_idx,
                               const long long* __restrict__ n_left, int cap_l, const sivo_keypoint* __restrict__ kr,
                               const uint8_t* __restrict__ dr, const long long* __restrict__ n_right, int cap_r,
                               const float* __restrict__ scale, const float* __restrict__ inv_scale, const uint8_t* __restrict__ pyr_l,
                               OrbLevelTable lt_l, const uint8_t* __restrict__ pyr_r, OrbLevelTable lt_r, float mb, float mbf,
                               float* __restrict__ u_right, float* __restrict__ depth, int* __restrict__ sad_dist) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= cap_l || wid >= *n_left) return;
  const long long nr64 = *n_right;
  const int nr = nr64 < 0 ? 0 : static_cast<int>(min(nr64, static_cast<long long>(cap_r)));
  const int k = keep_idx ? keep_idx[wid] : wid;
  float out_u = -1.f, out_z = -1.f;
  int out_sad = -1;
  if (k >= 0 && k < cap_l) {
    const sivo_keypoint L = kl[k];
    if (static_cast<unsigned>(L.octave) < static_cast<unsigned>(lt_l.nlevels))
      stereo_match_key(L, dl + static_cast<size_t>(k) * 32, kr, dr, nr, scale, inv_scale, pyr_l, lt_l, pyr_r, lt_r, mb, mbf, lane,
                       out_u, out_z, out_sad);
  }
  if (lane == 0) {
    u_right[wid] = out_u;
    depth[wid] = out_z;
    sad_dist[wid] = out_sad;
  }
}

// ---- median-based outlier cut (Frame.cc:617-628) on the device, one block.  m = number of matched keys (SAD >= 0); the median
// is the SAD at index m / 2 of the ascending order.  Every SAD is an integer <= 121 * 510 < 2^16, so an exact two-pass radix
// select (high byte, then low byte, 256-bin shared histograms) finds it without sorting.  th = 1.5f * 1.4f * median in float; every
// matched key with (float) sad >= th -- exactly the tail the reference walks down the sorted distances -- is unmatched (-1).
constexpr int kCutThreads = 1024;

// warp 0: the bin holding the element of rank `k` (0-based, ascending) of the 256-bin histogram, and its rank within that bin
__device__ __forceinline__ void hist_select(const int* hist, int k, int lane, int* bin, int* rank_in_bin) {
  int c[8], sum = 0;
#pragma unroll
  for (int b = 0; b < 8; ++b) { c[b] = hist[lane * 8 + b]; sum += c[b]; }
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  int before = incl - sum;
  if (k >= before && k < incl) {
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      if (k < before + c[b]) { *bin = lane * 8 + b; *rank_in_bin = k - before; break; }
      before += c[b];
    }
  }
}

__global__ void __launch_bounds__(kCutThreads) k_stereo_median_cut(const long long* __restrict__ n_left, int cap, const int* __restrict__ sad,
                                                                   float* __restrict__ u_right, float* __restrict__ depth) {
  __shared__ int hist[256];
  __shared__ int s_m, s_bin, s_rank;
  const long long n64 = *n_left;
  const int n = n64 < 0 ? 0 : static_cast<int>(min(n64, static_cast<long long>(cap)));
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid < 256) hist[tid] = 0;
  __syncthreads();
  for (int i = tid; i < n; i += kCutThreads) {
    const int s = sad[i];
    if (s >= 0) atomicAdd(&hist[s >> 8], 1);
  }
  __syncthreads();
  if (tid < 32) {
    int m = 0;
#pragma unroll
    for (int b = 0; b < 8; ++b) m += hist[lane * 8 + b];
#pragma unroll
    for (int o = 16; o; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
    if (lane == 0) s_m = m;
    if (m > 0) hist_select(hist, m / 2, lane, &s_bin, &s_rank);
  }
  __syncthreads();
  if (s_m == 0) return;  // nothing matched: nothing to cut
  const int hi = s_bin;
  if (tid < 256) hist[tid] = 0;
  __syncthreads();
  for (int i = tid; i < n; i += kCutThreads) {
    const int s = sad[i];
    if (s >= 0 && (s >> 8) == hi) atomicAdd(&hist[s & 255], 1);
  }
  __syncthreads();
  if (tid < 32) {
    const int k = s_rank;
    __syncwarp();  // every lane has read the rank before one of them overwrites it
    hist_select(hist, k, lane, &s_bin, &s_rank);
  }
  __syncthreads();
  const float median = static_cast<float>((hi << 8) | s_bin);
  const float th = 1.5f * 1.4f * median;
  for (int i = tid; i < n; i += kCutThreads) {
    const int s = sad[i];
    if (s >= 0 && static_cast<float>(s) >= th) {
      u_right[i] = -1.f;
      depth[i] = -1.f;
    }
  }
}

// Both forms: the match kernel over cap_l outputs, then the median cut over their SAD distances in `sad` (cap_l ints), on `s`.
void launch_stereo(const Orb& left, const Orb& right, const sivo_keypoint* kl, const uint8_t* dl, const int* keep_idx, const long long* n_left,
                   int cap_l, const sivo_keypoint* kr, const uint8_t* dr, const long long* n_right, int cap_r, float mb, float mbf,
                   float* u_right, float* depth, int* sad, cudaStream_t s) {
  k_stereo_match<<<ceil_div(cap_l * 32, 128), 128, 0, s>>>(kl, dl, keep_idx, n_left, cap_l, kr, dr, n_right, cap_r, left.dev_scale(),
                                                           left.dev_inv_scale(), left.dev_pyramid(), left.levels(), right.dev_pyramid(),
                                                           right.levels(), mb, mbf, u_right, depth, sad);
  SIVO_CUDA(cudaGetLastError());
  k_stereo_median_cut<<<1, kCutThreads, 0, s>>>(n_left, cap_l, sad, u_right, depth);
  SIVO_CUDA(cudaGetLastError());
}

// The SAD windows of both images are read at the left key's octave with one set of rounded coordinates: the two extractors' last
// runs must have the same level tables (same image size and scale factor), or the right reads would leave its pyramid.
void check_extractors(const Orb& left, const Orb& right) {
  if (!left.has_run() || !right.has_run()) fail(SIVO_EINVAL, "stereo: run both extractors first");
  if (left.device() != right.device() || left.nlevels() != right.nlevels()) fail(SIVO_EINVAL, "stereo: extractors differ");
  for (int l = 0; l < left.nlevels(); ++l)
    if (left.levels().lv[l].w != right.levels().lv[l].w || left.levels().lv[l].h != right.levels().lv[l].h)
      fail(SIVO_EINVAL, "stereo: level %d is %d x %d on the left and %d x %d on the right", l, left.levels().lv[l].w,
           left.levels().lv[l].h, right.levels().lv[l].w, right.levels().lv[l].h);
}

void check_octaves(const sivo_keypoint* left, int nl, const sivo_keypoint* right, int nr, int nlevels) {
  for (int i = 0; i < nl; ++i) if (left[i].octave < 0 || left[i].octave >= nlevels) fail(SIVO_EINVAL, "stereo: left octave out of range");
  for (int i = 0; i < nr; ++i) if (right[i].octave < 0 || right[i].octave >= nlevels) fail(SIVO_EINVAL, "stereo: right octave out of range");
}

}  // namespace

HostCall& host_call() {
  static thread_local HostCall hc;
  return hc;
}

void stereo_hamming(int device, const sivo_keypoint* left, const uint8_t* dl, int nl, const sivo_keypoint* right,
                    const uint8_t* dr, int nr, const float* scale, int nlevels, int rows, float min_d, float max_d,
                    int* best_idx, int* best_dist) {
  if (nl < 0 || nr < 0 || nr >= (1 << 20)) fail(SIVO_EINVAL, "stereo: bad keypoint counts %d / %d", nl, nr);
  if (nl == 0) return;
  check_octaves(left, nl, right, nr, nlevels);
  HostCall& hc = host_call();
  hc.begin(device);
  const sivo_keypoint* d_kl = hc.upload(left, nl);
  const uint8_t* d_dl = hc.upload(dl, static_cast<size_t>(nl) * 32);
  const sivo_keypoint* d_kr = hc.upload(right, nr);
  const uint8_t* d_dr = hc.upload(dr, static_cast<size_t>(nr) * 32);
  const float* d_sc = hc.upload(scale, nlevels);
  int* d_bi = hc.take<int>(nl);
  int* d_bd = hc.take<int>(nl);
  k_stereo_hamming<<<ceil_div(nl * 32, 128), 128, 0, hc.stream>>>(d_kl, d_dl, nl, d_kr, d_dr, nr, d_sc, nlevels, rows, min_d, max_d, d_bi,
                                                                  d_bd);
  SIVO_CUDA(cudaGetLastError());
  hc.download(best_idx, d_bi, nl);
  hc.download(best_dist, d_bd, nl);
  hc.sync();
}

// ---- best / second-best descriptor match over per-query candidate lists: the inner loop shared by
// ORBmatcher::SearchByProjection (ORBmatcher.cc:79-113 and :1278-), SearchForTriangulation (:631-) and SearchBySim3 --
//   bestDist = bestDist2 = 256, bestLevel = bestLevel2 = -1, bestIdx = -1;
//   for idx in candidates (in order): dist = DescriptorDistance(q, train[idx]);
//     if (dist < bestDist) { bestDist2 = bestDist; bestLevel2 = bestLevel; bestDist = dist; bestLevel = level[idx]; bestIdx = idx; }
//     else if (dist < bestDist2) { bestLevel2 = level[idx]; bestDist2 = dist; }
// One warp per query: the lanes compute 32 distances at a time, the warp folds them in candidate order (best2_fold_warp,
// match_fold.cuh) so that ties fall exactly as in the sequential loop.
namespace {
__global__ void k_hamming_best2(const uint8_t* __restrict__ query, int nq, const uint8_t* __restrict__ train,
                                const int* __restrict__ cand_off, const int* __restrict__ cand_idx, const int* __restrict__ level,
                                int* __restrict__ out) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= nq) return;
  const ulonglong4 a = *reinterpret_cast<const ulonglong4*>(query + static_cast<size_t>(wid) * 32);
  const int b = cand_off[wid], e = cand_off[wid + 1];
  Best2 best;
  for (int base = b; base < e; base += 32) {
    const int i = base + lane;
    int d = 0x7FFFFFFF, idx = -1, lvl = -1;
    if (i < e) {
      idx = cand_idx[i];
      const ulonglong4 t = *reinterpret_cast<const ulonglong4*>(train + static_cast<size_t>(idx) * 32);
      d = __popcll(a.x ^ t.x) + __popcll(a.y ^ t.y) + __popcll(a.z ^ t.z) + __popcll(a.w ^ t.w);
      lvl = level ? level[idx] : 0;
    }
    best2_fold_warp(best, d, idx, lvl, min(32, e - base));  // warp-uniform fold in candidate order
  }
  if (lane == 0) {
    int* o = out + static_cast<size_t>(wid) * 5;
    o[0] = best.idx; o[1] = best.dist; o[2] = best.level; o[3] = best.dist2; o[4] = best.level2;
  }
}
}  // namespace

void hamming_best2(int device, const uint8_t* query, int nq, const uint8_t* train, int nt, const int* cand_off, const int* cand_idx,
                   const int* train_level, int* out5) {
  if (nq < 0 || nt < 0) fail(SIVO_EINVAL, "hamming_best2: negative counts");
  if (nq == 0) return;
  if (cand_off[0] != 0) fail(SIVO_EINVAL, "hamming_best2: candidate offsets must start at 0");
  for (int i = 0; i < nq; ++i) if (cand_off[i + 1] < cand_off[i]) fail(SIVO_EINVAL, "hamming_best2: candidate offsets must not decrease");
  const int nc = cand_off[nq];
  for (int i = 0; i < nc; ++i) if (cand_idx[i] < 0 || cand_idx[i] >= nt) fail(SIVO_ERANGE, "hamming_best2: candidate %d names train descriptor %d of %d", i, cand_idx[i], nt);
  HostCall& hc = host_call();
  hc.begin(device);
  const uint8_t* d_q = hc.upload(query, static_cast<size_t>(nq) * 32);
  const uint8_t* d_t = hc.upload(train, static_cast<size_t>(nt) * 32);
  const int* d_off = hc.upload(cand_off, nq + 1);
  const int* d_idx = hc.upload(cand_idx, nc);
  const int* d_lvl = hc.upload(train_level, nt);
  int* d_out = hc.take<int>(static_cast<size_t>(nq) * 5);
  k_hamming_best2<<<ceil_div(nq * 32, 128), 128, 0, hc.stream>>>(d_q, nq, d_t, d_off, d_idx, train_level ? d_lvl : nullptr, d_out);
  SIVO_CUDA(cudaGetLastError());
  hc.download(out5, d_out, static_cast<size_t>(nq) * 5);
  hc.sync();
}

}  // namespace sivo

namespace sivo {
// ComputeStereoMatches end to end; `left` / `right` are the extractors whose last runs produced the keypoints.
void stereo_match(const Orb& left, const Orb& right, const sivo_keypoint* kl, const uint8_t* dl, int nl, const sivo_keypoint* kr,
                  const uint8_t* dr, int nr, float mb, float mbf, float* u_right, float* depth) {
  check_extractors(left, right);
  if (nl < 0 || nr < 0 || nr >= (1 << 20) || !(mb > 0.f) || !(mbf > 0.f)) fail(SIVO_EINVAL, "stereo: bad arguments");
  for (int i = 0; i < nl; ++i) { u_right[i] = -1.f; depth[i] = -1.f; }
  if (nl == 0 || nr == 0) return;
  check_octaves(kl, nl, kr, nr, left.nlevels());
  HostCall& hc = host_call();
  hc.begin(left.device());
  const sivo_keypoint* d_kl = hc.upload(kl, nl);
  const uint8_t* d_dl = hc.upload(dl, static_cast<size_t>(nl) * 32);
  const sivo_keypoint* d_kr = hc.upload(kr, nr);
  const uint8_t* d_dr = hc.upload(dr, static_cast<size_t>(nr) * 32);
  const long long counts[2] = {nl, nr};
  const long long* d_n = hc.upload(counts, 2);
  float* d_u = hc.take<float>(nl);
  float* d_z = hc.take<float>(nl);
  int* d_s = hc.take<int>(nl);
  // the pyramids were written on the two extractors' own streams; their synchronous run() has returned, so they are complete
  launch_stereo(left, right, d_kl, d_dl, nullptr, d_n, nl, d_kr, d_dr, d_n + 1, nr, mb, mbf, d_u, d_z, d_s, hc.stream);
  hc.download(u_right, d_u, nl);
  hc.download(depth, d_z, nl);
  hc.sync();
}

// ComputeStereoMatches on device-resident keypoints, descriptors and counts, enqueued on `s` (NULL: the left extractor's stream)
// without a host synchronisation.  `s` first waits for everything enqueued so far on both extractors' streams (their pyramids
// are read).  The SAD distances go to the call's own stream-ordered scratch.
void stereo_match_device(Orb& left, Orb& right, const sivo_keypoint* kl, const uint8_t* dl, const int* keep_idx, const long long* n_left,
                         const sivo_keypoint* kr, const uint8_t* dr, const long long* n_right, float mb, float mbf, float* u_right,
                         float* depth, cudaStream_t s) {
  check_extractors(left, right);
  if (!(mb > 0.f) || !(mbf > 0.f)) fail(SIVO_EINVAL, "stereo: bad arguments");
  // the Hamming search packs a right index into 20 bits
  if (right.capacity() >= (1 << 20)) fail(SIVO_EINVAL, "stereo: right extractor capacity %d needs more than 20 index bits", right.capacity());
  s = left.enter(s);
  left.stream_wait(s);
  right.stream_wait(s);
  StreamScratch sc(StreamScratch::bytes<int>(left.capacity()), s);
  launch_stereo(left, right, kl, dl, keep_idx, n_left, left.capacity(), kr, dr, n_right, right.capacity(), mb, mbf, u_right, depth,
                sc.take<int>(left.capacity()), s);
}

// Test hook: k_stereo_median_cut alone over n SAD distances (negative = unmatched), cutting u / z in place.
void stereo_median_cut(int device, const int* sad, int n, float* u, float* z) {
  if (n < 0) fail(SIVO_EINVAL, "stereo_median_cut: n = %d", n);
  if (n == 0) return;
  HostCall& hc = host_call();
  hc.begin(device);
  const long long count = n;
  const long long* d_n = hc.upload(&count, 1);
  const int* d_s = hc.upload(sad, n);
  float* d_u = hc.upload(u, n);
  float* d_z = hc.upload(z, n);
  k_stereo_median_cut<<<1, kCutThreads, 0, hc.stream>>>(d_n, n, d_s, d_u, d_z);
  SIVO_CUDA(cudaGetLastError());
  hc.download(u, d_u, n);
  hc.download(z, d_z, n);
  hc.sync();
}
}  // namespace sivo
