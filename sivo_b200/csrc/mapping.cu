// A keyframe's new map points: LocalMapping::CreateNewMapPoints (LocalMapping.cc:198-472) with ORBmatcher::SearchForTriangulation
// (ORBmatcher.cc:631-785), CheckDistEpipolarLine (:137-159), ComputeF12 (LocalMapping.cc:639-654) and SIVO's CheckSemantics
// (:474-545).  The rule is spelled out in include/sivo_b200.h and oracle/mapping_oracle.py.  This file is compiled with
// -fmad=false: every float / double intermediate is the correctly rounded result of the operation as written.
//
// The reference never sets vbMatched2 and runs no orientation check, and a neighbour's own map points change only after its
// search, so each current key is one independent walk over the neighbours that stops at its first created point:
//   host             per neighbour: the baseline test, F12 and the epipole (cv::Mat forms, pinned in tests/test_oracle_mapping.py)
//   k_map_create     one warp per current key: per neighbour, lanes scan the neighbour's keys for the key's vocabulary node (in
//                    key order, so a node's candidates come in the order of its FeatureVector entry), fold the best match,
//                    then triangulate, check and run CheckSemantics; stop at the first created point.
//   k_map_list       one block: the created points neighbour-major, key ascending (mlpRecentAddedMapPoints' order).
#include <cmath>

#include "block_ops.cuh"
#include "frame_ops.h"
#include "host_call.h"
#include "info_mi.cuh"
#include "jacobi.cuh"
#include "match_fold.cuh"
#include "stream_scratch.h"

namespace sivo {
namespace {
constexpr int kMaxNeighbours = 32;
constexpr int kThLow = 50;  // ORBmatcher::TH_LOW
constexpr int kMapThreads = 128, kMapWarps = kMapThreads / 32;
constexpr int kListThreads = 1024;
constexpr int kVoid = 255;  // Classes::VOID
enum { kHasPoint = 0, kBaseline, kNoMatch, kParallax, kWZero, kZ1, kZ2, kReproj1, kReproj2, kScale, kSemantic, kCreated };

struct MapKf {  // one keyframe's keys (device) and pose
  const sivo_keypoint* kps;
  const uint4* desc;
  const float* ur;
  const float* depth;
  const uint8_t* cls;
  const double* conf;
  const double* ent;
  const int* node;
  const uint8_t* hp;
  const long long* count;
  float rcw[9], tcw[3], ow[3], rwc[9];
};

struct MapNb {
  MapKf kf;
  float F[9];  // F12, row-major
  float ex, ey;
  int skip;    // below the baseline
};

struct MapParams {
  MapKf kf1;
  MapNb nb[kMaxNeighbours];
  double sigma[36];
  float fx, fy, cx, cy, invfx, invfy, mb, mbf, ratio_factor, th_conf, th_red;
  float scale[kOrbMaxLevels], sigma2[kOrbMaxLevels];
  int n_nb, nlevels, cap, stride, max_class, full;
};

// any keyframe's count negative (every lane of the warp gets the same answer)
__device__ __forceinline__ bool any_negative(const MapParams& p, int lane) {
  const bool neg = (lane < p.n_nb && *p.nb[lane].kf.count < 0) || (lane == 0 && *p.kf1.count < 0);
  return __any_sync(0xffffffffu, neg);
}

// cv::gemm(R, x) for 3 x 3 floats with x a column: ((R0 x0 + R1 x1) + R2 x2) in float, + t when given
__device__ __forceinline__ void gemm3(const float* R, const float* x, const float* t, float* out) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float s = (R[3 * r] * x[0] + R[3 * r + 1] * x[1]) + R[3 * r + 2] * x[2];
    out[r] = t ? s + t[r] : s;
  }
}

// Mat::dot of two 3-float vectors: ((0 + a0 b0) + a1 b1) + a2 b2 in double
__device__ __forceinline__ double dot3(const float* a, const float* b) {
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) s = s + static_cast<double>(a[i]) * static_cast<double>(b[i]);
  return s;
}

// cos(2 * atan2(mb / 2, depth)) with the float overloads, as the correctly rounded float functions (within an ulp of glibc's)
__device__ __forceinline__ float cos_parallax_stereo(float mb, float depth) {
  const float half = mb / 2.f;
  const float a = static_cast<float>(atan2(static_cast<double>(half), static_cast<double>(depth)));
  return static_cast<float>(cos(static_cast<double>(2.f * a)));
}

// The triangulation's right singular vector (the documented rule, jacobi.cuh): the rotated identity's column of least norm.
__device__ void svd_null_vector(double a[4][4], double out[4]) {
  double v[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) v[r][c] = r == c ? 1.0 : 0.0;
  jacobi_sweeps<4, 4>(a, v);
  int best = 0;
  double best_n = 0.0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    double n = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) n = n + a[r][c] * a[r][c];
    if (c == 0 || n < best_n) { best_n = n; best = c; }
  }
#pragma unroll
  for (int c = 0; c < 4; ++c)
    if (c == best)
#pragma unroll
      for (int r = 0; r < 4; ++r) out[r] = v[r][c];
}

// A.row(k) = s * T.row(i) - T.row(j) as addWeighted(T.row(i), s, T.row(j), -1, 0): in double, rounded to float
__device__ __forceinline__ void a_row(float s, const float* R, const float* t, int i, int j, double* out) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float ti = c < 3 ? R[3 * i + c] : t[i], tj = c < 3 ? R[3 * j + c] : t[j];
    const double v = static_cast<double>(ti) * static_cast<double>(s) + static_cast<double>(tj) * -1.0 + 0.0;
    out[c] = static_cast<double>(static_cast<float>(v));
  }
}

// KeyFrame::UnprojectStereo: Rwc x3Dc + Ow
__device__ __forceinline__ void unproject(const MapParams& p, const MapKf& kf, float u, float v, float z, float* w) {
  const float xc[3] = {(u - p.cx) * z * p.invfx, (v - p.cy) * z * p.invfy, z};
  gemm3(kf.rwc, xc, kf.ow, w);
}

// reprojection error test in one keyframe: false = rejected
__device__ __forceinline__ bool reproj_ok(const MapParams& p, const MapKf& kf, const float* x3, float z, sivo_keypoint kp, bool stereo,
                                          float ur) {
  const float s2 = p.sigma2[kp.octave];
  const float x = static_cast<float>(dot3(kf.rcw, x3) + static_cast<double>(kf.tcw[0]));
  const float y = static_cast<float>(dot3(kf.rcw + 3, x3) + static_cast<double>(kf.tcw[1]));
  const float invz = 1.0f / z;
  const float u = p.fx * x * invz + p.cx, v = p.fy * y * invz + p.cy;
  const float ex = u - kp.x, ey = v - kp.y;
  if (!stereo) return !(static_cast<double>(ex * ex + ey * ey) > 5.991 * static_cast<double>(s2));
  const float er = (u - p.mbf * invz) - ur;
  return !(static_cast<double>(ex * ex + ey * ey + er * er) > 7.8 * static_cast<double>(s2));
}

__device__ __forceinline__ float dist_to(const float* x3, const float* o) {
  const float d[3] = {x3[0] - o[0], x3[1] - o[1], x3[2] - o[2]};
  return static_cast<float>(sqrt(dot3(d, d)));
}

// CheckSemantics' MI - H of the current key (out of line: it keeps the walk's registers free)
__device__ __noinline__ double semantic_reduction(const MapParams& p, const float* x3, int octave, double entropy, double* ws) {
  const StereoMiTerms t = stereo_mi_terms(p.sigma, p.fx, p.fy, p.mb, x3[0], x3[1], x3[2], p.sigma2[octave], ws, 1);
  return 0.5 * log2(t.det_state * t.det_meas / t.det_joint) - entropy;
}

// ---- one warp per current key
__global__ void __launch_bounds__(kMapThreads) k_map_create(const __grid_constant__ MapParams p, int* __restrict__ made_nb,
                                                            int* __restrict__ made_idx, float* __restrict__ world,
                                                            int* __restrict__ dbg_match, int* __restrict__ dbg_stage,
                                                            double* __restrict__ dbg_red) {
  __shared__ double ws_all[kMapWarps][81];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * kMapWarps + warp;
  if (any_negative(p, lane)) return;
  const int n1 = clamp_count(*p.kf1.count, p.cap);
  if (j >= n1) return;
  const MapKf& k1 = p.kf1;
  const sivo_keypoint kp1 = k1.kps[j];
  const uint4 q0 = k1.desc[2 * j], q1 = k1.desc[2 * j + 1];
  const float ur1 = k1.ur[j], z1d = k1.depth[j];
  const int node1 = k1.node[j];
  const bool stereo1 = ur1 >= 0.f;
  const int cls1 = k1.cls[j];
  // CheckSemantics' per-key criteria; a key failing them is never created, so the production path does not search it
  const bool key_ok = z1d > 0.f && cls1 <= p.max_class && k1.conf[j] >= static_cast<double>(p.th_conf);
  const bool search = kp1.octave >= 0 && kp1.octave < p.nlevels && node1 >= 0 && (p.full || key_ok);
  bool has = k1.hp[j] != 0;
  const float xn1[3] = {(kp1.x - p.cx) * p.invfx, (kp1.y - p.cy) * p.invfy, 1.0f};
  float ray1[3];
  gemm3(k1.rwc, xn1, nullptr, ray1);
  int out_nb = -1, out_idx = -1;
  float out_w[3] = {__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000)};
  for (int i = 0; i < p.n_nb; ++i) {
    const MapNb& nb = p.nb[i];
    const MapKf& k2 = nb.kf;
    int stage = kNoMatch, m = -1;
    double red = __longlong_as_double(0x7ff8000000000000ll);
    if (nb.skip) stage = kBaseline;
    else if (has) stage = kHasPoint;
    else if (search) {
      // SearchForTriangulation for key j: lanes take the neighbour's keys in order
      const int n2 = clamp_count(*k2.count, p.cap);
      const float la = (kp1.x * nb.F[0] + kp1.y * nb.F[3]) + nb.F[6];  // CheckDistEpipolarLine's line
      const float lb = (kp1.x * nb.F[1] + kp1.y * nb.F[4]) + nb.F[7];
      const float lc = (kp1.x * nb.F[2] + kp1.y * nb.F[5]) + nb.F[8];
      int bd = kThLow, bi = -1;
      for (int base = 0; base < n2; base += 32) {
        const int i2 = base + lane;
        const bool cand = i2 < n2 && k2.node[i2] == node1 && !k2.hp[i2];
        if (!__any_sync(0xffffffffu, cand)) continue;
        if (!cand) continue;
        const sivo_keypoint kp2 = k2.kps[i2];
        if (kp2.octave < 0 || kp2.octave >= p.nlevels) continue;
        const int d = descriptor_distance(q0, q1, k2.desc[2 * i2], k2.desc[2 * i2 + 1]);
        if (d > bd) continue;
        if (!stereo1 && !(k2.ur[i2] >= 0.f)) {
          const float dex = nb.ex - kp2.x, dey = nb.ey - kp2.y;
          if (dex * dex + dey * dey < 100.f * p.scale[kp2.octave]) continue;
        }
        const float num = (la * kp2.x + lb * kp2.y) + lc, den = la * la + lb * lb;
        if (den == 0.f) continue;
        const float dsqr = num * num / den;
        if (!(static_cast<double>(dsqr) < 3.84 * static_cast<double>(p.sigma2[kp2.octave]))) continue;
        bd = d;
        bi = i2;
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const int od = __shfl_xor_sync(0xffffffffu, bd, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (od < bd || (od == bd && oi > bi)) { bd = od; bi = oi; }
      }
      m = bi;
    }
    if (m >= 0) {
      // the triangulation and its checks (every lane computes the same values)
      const sivo_keypoint kp2 = k2.kps[m];
      const float ur2 = k2.ur[m], z2d = k2.depth[m];
      const bool stereo2 = ur2 >= 0.f;
      const float xn2[3] = {(kp2.x - p.cx) * p.invfx, (kp2.y - p.cy) * p.invfy, 1.0f};
      float ray2[3];
      gemm3(k2.rwc, xn2, nullptr, ray2);
      const float cos_rays = static_cast<float>(dot3(ray1, ray2) / (sqrt(dot3(ray1, ray1)) * sqrt(dot3(ray2, ray2))));
      float cs1 = cos_rays + 1.0f, cs2 = cs1;
      if (stereo1) cs1 = cos_parallax_stereo(p.mb, z1d);
      else if (stereo2) cs2 = cos_parallax_stereo(p.mb, z2d);
      const float cs = cs2 < cs1 ? cs2 : cs1;  // std::min
      float x3[3];
      stage = kCreated;
      if (cos_rays < cs && cos_rays > 0.f && (stereo1 || stereo2 || static_cast<double>(cos_rays) < 0.9998)) {
        double A[4][4], v[4];
        a_row(xn1[0], k1.rcw, k1.tcw, 2, 0, A[0]);
        a_row(xn1[1], k1.rcw, k1.tcw, 2, 1, A[1]);
        a_row(xn2[0], k2.rcw, k2.tcw, 2, 0, A[2]);
        a_row(xn2[1], k2.rcw, k2.tcw, 2, 1, A[3]);
        svd_null_vector(A, v);
        const float w3 = static_cast<float>(v[3]);
        if (w3 == 0.f) stage = kWZero;
        else
          for (int r = 0; r < 3; ++r) x3[r] = static_cast<float>(v[r]) / w3;
      } else if (stereo1 && cs1 < cs2 && z1d > 0.f) {
        unproject(p, k1, kp1.x, kp1.y, z1d, x3);
      } else if (stereo2 && cs2 < cs1 && z2d > 0.f) {
        unproject(p, k2, kp2.x, kp2.y, z2d, x3);
      } else {
        stage = kParallax;
      }
      float z1 = 0.f, z2 = 0.f;
      if (stage == kCreated) {
        z1 = static_cast<float>(dot3(k1.rcw + 6, x3) + static_cast<double>(k1.tcw[2]));
        if (z1 <= 0.f) stage = kZ1;
      }
      if (stage == kCreated) {
        z2 = static_cast<float>(dot3(k2.rcw + 6, x3) + static_cast<double>(k2.tcw[2]));
        if (z2 <= 0.f) stage = kZ2;
      }
      if (stage == kCreated && !reproj_ok(p, k1, x3, z1, kp1, stereo1, ur1)) stage = kReproj1;
      if (stage == kCreated && !reproj_ok(p, k2, x3, z2, kp2, stereo2, ur2)) stage = kReproj2;
      if (stage == kCreated) {
        const float dist1 = dist_to(x3, k1.ow), dist2 = dist_to(x3, k2.ow);
        if (dist1 == 0.f || dist2 == 0.f) stage = kScale;
        else {
          const float ratio_dist = dist2 / dist1, ratio_octave = p.scale[kp1.octave] / p.scale[kp2.octave];
          if (ratio_dist * p.ratio_factor < ratio_octave || ratio_dist > ratio_octave * p.ratio_factor) stage = kScale;
        }
      }
      if (stage == kCreated) {
        // CheckSemantics(current, j, wP, true) and CheckSemantics(neighbour, m, wP, false)
        int c1 = kVoid;
        if (key_ok) {
          if (lane == 0) red = semantic_reduction(p, x3, kp1.octave, k1.ent[j], ws_all[warp]);
          red = __shfl_sync(0xffffffffu, red, 0);
          c1 = red < static_cast<double>(p.th_red) ? kVoid : cls1;
        }
        if (!(c1 == static_cast<int>(k2.cls[m]) && c1 != kVoid)) stage = kSemantic;
      }
      if (stage == kCreated) {
        has = true;
        out_nb = i;
        out_idx = m;
        out_w[0] = x3[0]; out_w[1] = x3[1]; out_w[2] = x3[2];
      }
    }
    if (dbg_stage && lane == 0) {
      const size_t e = static_cast<size_t>(i) * p.stride + j;
      dbg_stage[e] = stage;
      dbg_match[e] = m;
      dbg_red[e] = red;
    }
  }
  if (lane == 0) {
    made_nb[j] = out_nb;
    if (made_idx) made_idx[j] = out_idx;
    if (world) { world[3 * j] = out_w[0]; world[3 * j + 1] = out_w[1]; world[3 * j + 2] = out_w[2]; }
  }
}

// ---- the created points in the reference's order: neighbour-major, key ascending
__global__ void __launch_bounds__(kListThreads) k_map_list(const __grid_constant__ MapParams p, const int* __restrict__ made_nb,
                                                           int* __restrict__ keys, int* __restrict__ list, long long* __restrict__ n_created) {
  __shared__ int warp_kept[kListThreads / 32];
  const int tid = threadIdx.x;
  if (any_negative(p, tid & 31)) {
    if (tid == 0 && n_created) *n_created = -1;
    return;
  }
  const int n1 = clamp_count(*p.kf1.count, p.cap);
  int base = 0;
  for (int i = 0; i < p.n_nb; ++i)
    for (int c0 = 0; c0 < n1; c0 += kListThreads) {
      const int j = c0 + tid;
      base = compact_chunk<kListThreads>(j < n1 && made_nb[j] == i, j, base, warp_kept, keys);
    }
  if (list)
    for (int e = tid; e < base; e += kListThreads) {
      const int j = keys[e];
      list[2 * e] = made_nb[j];
      list[2 * e + 1] = j;
    }
  if (tid == 0 && n_created) *n_created = base;
}

// ---- KeyFrame's copy of the Frame's semantic keys
__global__ void k_kf_gather(const sivo_keypoint* __restrict__ kps, const uint4* __restrict__ desc, const int* __restrict__ keep_idx,
                            const long long* __restrict__ n_keep, int cap, const float* __restrict__ ur, const float* __restrict__ depth,
                            const uint8_t* __restrict__ cls, const double* __restrict__ conf, const double* __restrict__ ent,
                            sivo_keypoint* __restrict__ o_kps, uint4* __restrict__ o_desc, float* __restrict__ o_ur,
                            float* __restrict__ o_depth, uint8_t* __restrict__ o_cls, double* __restrict__ o_conf,
                            double* __restrict__ o_ent, long long* __restrict__ o_count) {
  const int n = clamp_count(*n_keep, cap);
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j == 0) *o_count = n;
  if (j >= n) return;
  const int k = keep_idx ? keep_idx[j] : j;
  o_ur[j] = ur[j];
  o_depth[j] = depth[j];
  if (k < 0 || k >= cap) {
    sivo_keypoint bad{};
    bad.octave = -1;
    o_kps[j] = bad;
    o_desc[2 * j] = o_desc[2 * j + 1] = make_uint4(0, 0, 0, 0);
    o_cls[j] = kVoid;
    o_conf[j] = 0.0;
    o_ent[j] = 0.0;
    return;
  }
  o_kps[j] = kps[k];
  o_desc[2 * j] = desc[2 * k];
  o_desc[2 * j + 1] = desc[2 * k + 1];
  o_cls[j] = cls[k];
  o_conf[j] = conf[k];
  o_ent[j] = ent[k];
}

// ---- host: the per-neighbour cv::Mat forms
// R1 R2^T (cv::gemm with GEMM_2_T): each entry the double sum of the three products, rounded to float
void mul_abt(const float* A, const float* B, float* out) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double s = static_cast<double>(A[3 * r]) * B[3 * c];
      s = s + static_cast<double>(A[3 * r + 1]) * B[3 * c + 1];
      s = s + static_cast<double>(A[3 * r + 2]) * B[3 * c + 2];
      out[3 * r + c] = static_cast<float>(s);
    }
}
// A B (cv::gemm, 3 x 3 floats): (A0 B0 + A1 B1) + A2 B2 in float
void mul_ab(const float* A, const float* B, float* out) {
  float t[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) t[3 * r + c] = (A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c]) + A[3 * r + 2] * B[6 + c];
  for (int i = 0; i < 9; ++i) out[i] = t[i];
}
// cv::Mat::inv of a 3 x 3 float matrix (DECOMP_LU's closed form): cofactors times 1 / det in double, rounded to float
void inv3(const float* m, float* out) {
  double a[9];
  for (int i = 0; i < 9; ++i) a[i] = m[i];
#define M(r, c) a[3 * (r) + (c)]
  double d = M(0, 0) * (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) - M(0, 1) * (M(1, 0) * M(2, 2) - M(1, 2) * M(2, 0)) +
             M(0, 2) * (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0));
  d = 1.0 / d;
  const double b[9] = {(M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) * d, (M(0, 2) * M(2, 1) - M(0, 1) * M(2, 2)) * d,
                       (M(0, 1) * M(1, 2) - M(0, 2) * M(1, 1)) * d, (M(1, 2) * M(2, 0) - M(1, 0) * M(2, 2)) * d,
                       (M(0, 0) * M(2, 2) - M(0, 2) * M(2, 0)) * d, (M(0, 2) * M(1, 0) - M(0, 0) * M(1, 2)) * d,
                       (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0)) * d, (M(0, 1) * M(2, 0) - M(0, 0) * M(2, 1)) * d,
                       (M(0, 0) * M(1, 1) - M(0, 1) * M(1, 0)) * d};
#undef M
  for (int i = 0; i < 9; ++i) out[i] = static_cast<float>(b[i]);
}
float norm3f(const float* a) {
  double s = 0.0;
  for (int i = 0; i < 3; ++i) s = s + static_cast<double>(a[i]) * a[i];
  return static_cast<float>(std::sqrt(s));
}

MapKf make_kf(const sivo_keyframe_keys& k) {
  MapKf m{};
  m.kps = k.kps;
  m.desc = reinterpret_cast<const uint4*>(k.desc);
  m.ur = k.u_right; m.depth = k.depth; m.cls = k.kp_class; m.conf = k.kp_conf; m.ent = k.kp_entropy;
  m.node = k.node; m.hp = k.has_point; m.count = k.count;
  for (int i = 0; i < 9; ++i) m.rcw[i] = k.Rcw[i];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) m.rwc[3 * r + c] = k.Rcw[3 * c + r];
  for (int i = 0; i < 3; ++i) { m.tcw[i] = k.tcw[i]; m.ow[i] = k.Ow[i]; }
  return m;
}

// The baseline test, ComputeF12 and SearchForTriangulation's epipole of neighbour nb against the current keyframe kf1.
void neighbour_terms(const MapParams& p, const sivo_keyframe_keys& kf1, const sivo_keyframe_keys& kf2, MapNb& nb) {
  const float vb[3] = {kf2.Ow[0] - kf1.Ow[0], kf2.Ow[1] - kf1.Ow[1], kf2.Ow[2] - kf1.Ow[2]};
  nb.skip = norm3f(vb) < p.mb;
  // R12 = R1w R2w^T; t12 = -R1w R2w^T t2w + t1w; F12 = K1^-T [t12]x R12 K2^-1
  float R12[9], t12[3], K[9] = {p.fx, 0.f, p.cx, 0.f, p.fy, p.cy, 0.f, 0.f, 1.f}, Kt[9], Kti[9], Ki[9], tx[9], F[9];
  mul_abt(kf1.Rcw, kf2.Rcw, R12);
  for (int r = 0; r < 3; ++r)
    t12[r] = ((-R12[3 * r] * kf2.tcw[0] + -R12[3 * r + 1] * kf2.tcw[1]) + -R12[3 * r + 2] * kf2.tcw[2]) + kf1.tcw[r];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Kt[3 * r + c] = K[3 * c + r];
  inv3(Kt, Kti);
  inv3(K, Ki);
  const float skew[9] = {0.f, -t12[2], t12[1], t12[2], 0.f, -t12[0], -t12[1], t12[0], 0.f};
  for (int i = 0; i < 9; ++i) tx[i] = skew[i];
  mul_ab(Kti, tx, F);
  mul_ab(F, R12, F);
  mul_ab(F, Ki, F);
  for (int i = 0; i < 9; ++i) nb.F[i] = F[i];
  // C2 = R2w Cw + t2w (the current keyframe's centre in the neighbour's frame)
  float C2[3];
  for (int r = 0; r < 3; ++r)
    C2[r] = ((kf2.Rcw[3 * r] * kf1.Ow[0] + kf2.Rcw[3 * r + 1] * kf1.Ow[1]) + kf2.Rcw[3 * r + 2] * kf1.Ow[2]) + kf2.tcw[r];
  const float invz = 1.0f / C2[2];
  nb.ex = p.fx * C2[0] * invz + p.cx;
  nb.ey = p.fy * C2[1] * invz + p.cy;
}

MapParams make_params(const Orb& left, const sivo_keyframe_keys& kf1, const sivo_keyframe_keys* nbs, int n_nb, const sivo_mapping_params& prm,
                      int cap, int stride, bool full) {
  if (n_nb < 0 || n_nb > kMaxNeighbours) fail(SIVO_EINVAL, "create_map_points: %d neighbours (at most %d)", n_nb, kMaxNeighbours);
  MapParams p{};
  p.fx = prm.fx; p.fy = prm.fy; p.cx = prm.cx; p.cy = prm.cy; p.invfx = prm.invfx; p.invfy = prm.invfy; p.mb = prm.mb; p.mbf = prm.mbf;
  for (int i = 0; i < 36; ++i) p.sigma[i] = prm.sigma_cw[i];
  p.max_class = prm.max_static_class;
  p.th_conf = prm.th_confidence;
  p.th_red = prm.th_entropy_reduction;
  p.ratio_factor = 1.5f * left.scale_factor();
  p.nlevels = left.nlevels();
  for (int l = 0; l < p.nlevels; ++l) { p.scale[l] = left.tables().scale[l]; p.sigma2[l] = left.tables().sigma2[l]; }
  p.cap = cap;
  p.stride = stride;
  p.full = full;
  p.n_nb = n_nb;
  p.kf1 = make_kf(kf1);
  for (int i = 0; i < n_nb; ++i) {
    p.nb[i].kf = make_kf(nbs[i]);
    neighbour_terms(p, kf1, nbs[i], p.nb[i]);
  }
  return p;
}

void launch_create(const MapParams& p, int* made_nb, int* made_idx, float* world, int* keys, int* list, long long* n_created, int* dbg_match,
                   int* dbg_stage, double* dbg_red, cudaStream_t s) {
  if (p.cap > 0) {
    k_map_create<<<ceil_div(p.cap, kMapWarps), kMapThreads, 0, s>>>(p, made_nb, made_idx, world, dbg_match, dbg_stage, dbg_red);
    SIVO_CUDA(cudaGetLastError());
  }
  k_map_list<<<1, kListThreads, 0, s>>>(p, made_nb, keys, list, n_created);
  SIVO_CUDA(cudaGetLastError());
}

void check_keys(const sivo_keyframe_keys& k, bool need_arrays) {
  if (!k.count || (need_arrays && (!k.kps || !k.desc || !k.u_right || !k.depth || !k.kp_class || !k.kp_conf || !k.kp_entropy || !k.node ||
                                   !k.has_point)))
    fail(SIVO_EINVAL, "create_map_points: null keyframe array");
}
}  // namespace

void create_map_points_device(const Orb& left, const sivo_keyframe_keys& kf1, const sivo_keyframe_keys* nbs, int n_nb,
                              const sivo_mapping_params& prm, int* created_nb, int* created_idx, float* world, int* created_list,
                              long long* n_created, cudaStream_t s) {
  if (n_nb < 0 || n_nb > kMaxNeighbours) fail(SIVO_EINVAL, "create_map_points: %d neighbours (at most %d)", n_nb, kMaxNeighbours);
  if (n_nb > 0 && !nbs) fail(SIVO_EINVAL, "create_map_points: null neighbours");
  check_keys(kf1, true);
  for (int i = 0; i < n_nb; ++i) check_keys(nbs[i], true);
  const int cap = left.capacity();
  const MapParams p = make_params(left, kf1, nbs, n_nb, prm, cap, cap, false);
  s = left.enter(s);
  const size_t c = std::max(cap, 1);
  StreamScratch sc(2 * StreamScratch::bytes<int>(c), s);
  int* made = sc.take<int>(c);
  launch_create(p, created_nb ? created_nb : made, created_idx, world, sc.take<int>(c), created_list, n_created, nullptr, nullptr, nullptr, s);
}

// The host form and the test hook: stage every keyframe's keys, run the kernels, download.
void create_map_points_host(const Orb& left, const sivo_keyframe_keys& kf1, const sivo_keyframe_keys* nbs, int n_nb,
                            const sivo_mapping_params& prm, int* dbg_match, int* dbg_stage, double* dbg_red, int* created_nb,
                            int* created_idx, float* world, int* created_list, long long* n_created) {
  if (n_nb < 0 || n_nb > kMaxNeighbours) fail(SIVO_EINVAL, "create_map_points: %d neighbours (at most %d)", n_nb, kMaxNeighbours);
  if (n_nb > 0 && !nbs) fail(SIVO_EINVAL, "create_map_points: null neighbours");
  const bool dbg = dbg_match || dbg_stage || dbg_red;
  HostCall& hc = host_call();
  hc.begin(left.device());
  auto stage_kf = [&](const sivo_keyframe_keys& k) {
    check_keys(k, false);
    const long long n = std::max(*k.count, 0ll);
    if (n && (!k.kps || !k.desc || !k.u_right || !k.depth || !k.kp_class || !k.kp_conf || !k.kp_entropy || !k.node || !k.has_point))
      fail(SIVO_EINVAL, "create_map_points: null keyframe array");
    sivo_keyframe_keys d = k;
    d.kps = hc.upload(k.kps, n);
    d.desc = hc.upload(k.desc, 32 * n);
    d.u_right = hc.upload(k.u_right, n);
    d.depth = hc.upload(k.depth, n);
    d.kp_class = hc.upload(k.kp_class, n);
    d.kp_conf = hc.upload(k.kp_conf, n);
    d.kp_entropy = hc.upload(k.kp_entropy, n);
    d.node = hc.upload(k.node, n);
    d.has_point = hc.upload(k.has_point, n);
    d.count = hc.upload(k.count, 1);
    return d;
  };
  const sivo_keyframe_keys d1 = stage_kf(kf1);
  sivo_keyframe_keys dn[kMaxNeighbours];
  int cap = static_cast<int>(std::max(*kf1.count, 0ll));
  for (int i = 0; i < n_nb; ++i) {
    dn[i] = stage_kf(nbs[i]);
    cap = std::max(cap, static_cast<int>(std::max(*nbs[i].count, 0ll)));
  }
  const int n1 = static_cast<int>(std::max(*kf1.count, 0ll));
  const MapParams p = make_params(left, d1, dn, n_nb, prm, cap, n1, dbg);
  const size_t np = static_cast<size_t>(n_nb) * n1;
  int* d_made = hc.take<int>(n1);
  int* d_idx = hc.take<int>(n1);
  float* d_world = hc.take<float>(3 * static_cast<size_t>(n1));
  int* d_keys = hc.take<int>(n1);
  int* d_list = hc.take<int>(2 * static_cast<size_t>(n1));
  long long* d_n = hc.take<long long>(1);
  int* d_m = dbg ? hc.take<int>(np) : nullptr;
  int* d_st = dbg ? hc.take<int>(np) : nullptr;
  double* d_red = dbg ? hc.take<double>(np) : nullptr;
  launch_create(p, d_made, d_idx, d_world, d_keys, d_list, d_n, d_m, d_st, d_red, hc.stream);
  long long nc = 0;
  hc.download(&nc, d_n, 1);
  hc.sync();
  if (n_created) *n_created = nc;
  if (nc < 0) return;
  hc.download(created_nb, d_made, n1);
  hc.download(created_idx, d_idx, n1);
  hc.download(world, d_world, 3 * static_cast<size_t>(n1));
  hc.download(created_list, d_list, 2 * static_cast<size_t>(nc));
  hc.download(dbg_match, d_m, np);
  hc.download(dbg_stage, d_st, np);
  hc.download(dbg_red, d_red, np);
  hc.sync();
}

void keyframe_gather_device(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                            const float* u_right, const float* depth, const uint8_t* cls, const double* conf, const double* ent,
                            sivo_keypoint* o_kps, uint8_t* o_desc, float* o_ur, float* o_depth, uint8_t* o_cls, double* o_conf,
                            double* o_ent, long long* o_count, cudaStream_t s) {
  s = left.enter(s);
  const int cap = left.capacity();
  k_kf_gather<<<ceil_div(std::max(cap, 1), 256), 256, 0, s>>>(kps, reinterpret_cast<const uint4*>(desc), keep_idx, n_keep, cap, u_right, depth,
                                                              cls, conf, ent, o_kps, reinterpret_cast<uint4*>(o_desc), o_ur, o_depth, o_cls,
                                                              o_conf, o_ent, o_count);
  SIVO_CUDA(cudaGetLastError());
}

}  // namespace sivo
