// SIVO's information-based map-point selection (Tracking.cc:470-520 / 953-1000 with sivo_helpers.cpp:64-88, 160-218): per semantic
// key the mutual information between the pose and the stereo measurement, minus the classification entropy, against a threshold.
// The rule is spelled out in include/sivo_b200.h and oracle/info_oracle.py.  This file is compiled with -fmad=false: no
// multiply-add is contracted, so every float / double intermediate is the correctly rounded result of the operation as written
// (the divisions and log2 keep the math library's own sequences).
#include <cmath>

#include "block_ops.cuh"
#include "frame_ops.h"
#include "host_call.h"
#include "info_mi.cuh"
#include "stream_scratch.h"

namespace sivo {

// what the kernels need of the Frame and the extractor, by value (~450 B of kernel parameters)
struct InfoParams {
  double sigma[36];  // mSigmacw, row-major
  double threshold;
  float fx, fy, cx, cy, invfx, invfy, mb;
  float rwc[9], ow[3];
  float sigma2[kOrbMaxLevels];  // GetScaleSigmaSquares
  int nlevels;
};

namespace {
constexpr int kInfoThreads = 128;
constexpr int kInfoShared = 81 * kInfoThreads * static_cast<int>(sizeof(double));  // one 9 x 9 matrix per thread
constexpr int kCompactThreads = 512;

// One thread per semantic key j < min(*count, cap): the decision goes to flags[j] (1 = selected), the optional outputs to
// world[3 j ..], reduction[j] and the three determinants.  The working 9 x 9 matrix lives in dynamic shared memory as
// [element][thread], so that one element of a warp's 32 matrices is 32 consecutive words.
__global__ void __launch_bounds__(kInfoThreads) k_info_select(const InfoParams p, const sivo_keypoint* __restrict__ kps,
                                                              const double* __restrict__ entropy, const int* __restrict__ keep_idx,
                                                              const long long* __restrict__ count, int cap,
                                                              const float* __restrict__ depth, float* __restrict__ world,
                                                              double* __restrict__ reduction, uint8_t* __restrict__ flags,
                                                              double* __restrict__ det_state, double* __restrict__ det_meas,
                                                              double* __restrict__ det_joint) {
  extern __shared__ double ws_all[];
  const long long n64 = *count;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (n64 < 0 || j >= cap || j >= n64) return;
  const int k = keep_idx ? keep_idx[j] : j;
  const float z = depth[j];
  sivo_keypoint kp{};
  bool valid = k >= 0 && k < cap && z > 0.f;
  if (valid) {
    kp = kps[k];
    valid = kp.octave >= 0 && kp.octave < p.nlevels;
  }
  if (!valid) {
    if (world) world[3 * j] = world[3 * j + 1] = world[3 * j + 2] = __int_as_float(0x7fc00000);
    if (reduction) reduction[j] = __longlong_as_double(0x7ff8000000000000ll);
    if (det_state) det_state[j] = det_meas[j] = det_joint[j] = __longlong_as_double(0x7ff8000000000000ll);
    flags[j] = 0;
    return;
  }
  // Frame::UnprojectStereo: x3Dc = ((u - cx) z invfx, (v - cy) z invfy, z); wP = Rwc x3Dc + Ow (cv::gemm, float)
  const float xc[3] = {(kp.x - p.cx) * z * p.invfx, (kp.y - p.cy) * z * p.invfy, z};
  float w[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) w[r] = p.rwc[3 * r] * xc[0] + p.rwc[3 * r + 1] * xc[1] + p.rwc[3 * r + 2] * xc[2] + p.ow[r];
  if (world) { world[3 * j] = w[0]; world[3 * j + 1] = w[1]; world[3 * j + 2] = w[2]; }

  const double s2 = p.sigma2[kp.octave];
  // the working 9 x 9 matrix: element e of this thread's at ws_all[e * kInfoThreads + threadIdx.x]
  const StereoMiTerms t = stereo_mi_terms(p.sigma, p.fx, p.fy, p.mb, w[0], w[1], w[2], s2, ws_all + threadIdx.x, kInfoThreads);
  const double det_s = t.det_state, det_m33 = t.det_meas, det_m = t.det_joint;
  const double mi = 0.5 * log2(det_s * det_m33 / det_m);
  const double red = mi - entropy[k];
  if (reduction) reduction[j] = red;
  if (det_state) { det_state[j] = det_s; det_meas[j] = det_m33; det_joint[j] = det_m; }
  flags[j] = red > p.threshold ? 1 : 0;
}

// selected[0 .. n_selected) = the j with flags[j] set, ascending (one block, chunks of kCompactThreads)
__global__ void __launch_bounds__(kCompactThreads) k_info_compact(const long long* __restrict__ count, int cap,
                                                                 const uint8_t* __restrict__ flags, int* __restrict__ selected,
                                                                 long long* __restrict__ n_selected) {
  __shared__ int warp_kept[kCompactThreads / 32];
  const int n = clamp_count(*count, cap);
  if (n < 0) {
    if (threadIdx.x == 0 && n_selected) *n_selected = -1;
    return;
  }
  int base = 0;
  for (int c0 = 0; c0 < n; c0 += kCompactThreads) {
    const int i = c0 + threadIdx.x;
    base = compact_chunk<kCompactThreads>(i < n && flags[i], i, base, warp_kept, selected);
  }
  if (threadIdx.x == 0 && n_selected) *n_selected = base;
}

InfoParams make_params(const Orb& left, const sivo_info_camera& cam, double threshold) {
  InfoParams p{};
  for (int i = 0; i < 36; ++i) p.sigma[i] = cam.sigma_cw[i];
  p.threshold = threshold;
  p.fx = cam.fx; p.fy = cam.fy; p.cx = cam.cx; p.cy = cam.cy; p.invfx = cam.invfx; p.invfy = cam.invfy; p.mb = cam.mb;
  for (int i = 0; i < 9; ++i) p.rwc[i] = cam.Rwc[i];
  for (int i = 0; i < 3; ++i) p.ow[i] = cam.Ow[i];
  p.nlevels = left.nlevels();
  for (int l = 0; l < p.nlevels; ++l) p.sigma2[l] = left.tables().sigma2[l];
  return p;
}

// Both forms: the per-key kernel over `cap` keys, then the compaction if its outputs are wanted.
void launch_info_select(const InfoParams& p, const sivo_keypoint* kps, const double* entropy, const int* keep_idx, const long long* count,
                        int cap, const float* depth, float* world, double* reduction, uint8_t* flags, int* selected, long long* n_selected,
                        double* det_state, double* det_meas, double* det_joint, cudaStream_t s) {
  SIVO_CUDA(cudaFuncSetAttribute(k_info_select, cudaFuncAttributeMaxDynamicSharedMemorySize, kInfoShared));
  if (cap > 0)
    k_info_select<<<ceil_div(cap, kInfoThreads), kInfoThreads, kInfoShared, s>>>(p, kps, entropy, keep_idx, count, cap, depth, world, reduction,
                                                                                 flags, det_state, det_meas, det_joint);
  SIVO_CUDA(cudaGetLastError());
  if (selected || n_selected) {
    k_info_compact<<<1, kCompactThreads, 0, s>>>(count, cap, flags, selected, n_selected);
    SIVO_CUDA(cudaGetLastError());
  }
}

// The host form and the test hook: upload the gathered keys, run the kernels on the host-call workspace, download.
void info_host(const Orb& left, const sivo_keypoint* kps, const float* depth, const double* entropy, int n, const sivo_info_camera& cam,
               double threshold, float* world, double* reduction, int* selected, int* n_selected, double* det_state, double* det_meas,
               double* det_joint) {
  if (n < 0) fail(SIVO_EINVAL, "info_select: n = %d", n);
  const InfoParams p = make_params(left, cam, threshold);
  const bool dets = det_state || det_meas || det_joint;
  HostCall& hc = host_call();
  hc.begin(left.device());
  const sivo_keypoint* d_kps = hc.upload(kps, n);
  const float* d_depth = hc.upload(depth, n);
  double* d_ent = hc.upload(entropy, n);
  if (!entropy && n) SIVO_CUDA(cudaMemsetAsync(d_ent, 0, n * sizeof(double), hc.stream));
  const long long count = n;
  const long long* d_count = hc.upload(&count, 1);
  float* d_world = world ? hc.take<float>(3 * static_cast<size_t>(n)) : nullptr;
  double* d_red = reduction ? hc.take<double>(n) : nullptr;
  uint8_t* d_flags = hc.take<uint8_t>(n);
  int* d_sel = selected ? hc.take<int>(n) : nullptr;
  long long* d_nsel = selected || n_selected ? hc.take<long long>(1) : nullptr;
  double* d_det[3] = {nullptr, nullptr, nullptr};
  if (dets)
    for (auto& d : d_det) d = hc.take<double>(n);
  launch_info_select(p, d_kps, d_ent, nullptr, d_count, n, d_depth, d_world, d_red, d_flags, d_sel, d_nsel, d_det[0], d_det[1], d_det[2],
                     hc.stream);
  long long nsel = 0;
  hc.download(world, d_world, 3 * static_cast<size_t>(n));
  hc.download(reduction, d_red, n);
  if (d_nsel) hc.download(&nsel, d_nsel, 1);
  hc.sync();  // the selected list's length is known only now
  if (nsel > 0) hc.download(selected, d_sel, nsel);
  double* out_det[3] = {det_state, det_meas, det_joint};
  for (int i = 0; i < 3; ++i) hc.download(out_det[i], d_det[i], n);
  hc.sync();
  if (n_selected) *n_selected = static_cast<int>(nsel);
}
}  // namespace

void info_select(const Orb& left, const sivo_keypoint* kps, const float* depth, const double* entropy, int n, const sivo_info_camera& cam,
                 double threshold, float* world, double* reduction, int* selected, int* n_selected) {
  info_host(left, kps, depth, entropy, n, cam, threshold, world, reduction, selected, n_selected, nullptr, nullptr, nullptr);
}

void info_terms(const Orb& left, const sivo_keypoint* kps, const float* depth, int n, const sivo_info_camera& cam, float* world,
                double* det_state, double* det_meas, double* det_joint) {
  info_host(left, kps, depth, nullptr, n, cam, 0.0, world, nullptr, nullptr, nullptr, det_state, det_meas, det_joint);
}

// Enqueued on `s` (NULL: the left extractor's stream); no waits and no host synchronisation.
void info_select_device(const Orb& left, const sivo_keypoint* kps, const double* kp_entropy, const int* keep_idx, const long long* n_keep,
                        const float* depth, const sivo_info_camera& cam, double threshold, float* world, double* reduction, int* selected,
                        long long* n_selected, cudaStream_t s) {
  s = left.enter(s);
  StreamScratch sc(StreamScratch::bytes<uint8_t>(left.capacity()), s);
  launch_info_select(make_params(left, cam, threshold), kps, kp_entropy, keep_idx, n_keep, left.capacity(), depth, world, reduction,
                     sc.take<uint8_t>(left.capacity()), selected, n_selected, nullptr, nullptr, nullptr, s);
}

}  // namespace sivo
