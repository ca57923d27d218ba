// Map points matched to a frame's semantic keys by projection: the Frame's grid (AssignFeaturesToGrid / PosInGrid /
// GetFeaturesInArea, Frame.cc:205-223, 326-404), Frame::isInFrustum + MapPoint::PredictScale (Frame.cc:267-324, MapPoint.cc:439-453)
// and the two per-frame forms of ORBmatcher::SearchByProjection (ORBmatcher.cc:44-127, 1278-1418).  The rules are spelled out in
// include/sivo_b200.h and oracle/track_oracle.py.  This file is compiled with -fmad=false: every float / double intermediate is the
// correctly rounded result of the operation as written.
//
// Three launches per search, all on the caller's stream:
//   k_track_grid       one block: gathers the semantic keys (position, level, mvRight, descriptor, angle) and builds the 64 x 48
//                      cell CSR (cell index ix * 48 + iy, so the cells of one column of a window are contiguous) by a counting
//                      sort, each cell's short list then sorted by key index.
//   k_track_project    one warp per point: projection and window, then the fold over the window's candidates in
//                      GetFeaturesInArea order with only the entry mask applied (best and second-best recorded).
//   k_track_ordered    one warp walks the points in order with the per-key blocked / owner state in shared memory.  A fold's
//                      result depends on a removed candidate only if that candidate was its best or its second-best, so only
//                      the points whose recorded best (local: or second) key an earlier point took are searched again.  The
//                      last-frame search then runs the rotation histogram and ComputeThreeMaxima.
//
// LocalMapping::SearchInNeighbors' ORBmatcher::Fuse(pKF, vpMapPoints, th) (ORBmatcher.cc:787-930) shares the grid builder, the
// area walk, to_camera and predict_scale: k_fuse_grid builds one grid per target keyframe (one block each), k_fuse_decide runs one
// warp per (target, point).  Fuse claims no key, so it needs no ordered pass.
#include <climits>
#include <cmath>
#include <vector>

#include "block_ops.cuh"
#include "frame_ops.h"
#include "host_call.h"
#include "match_fold.cuh"
#include "stream_scratch.h"

namespace sivo {
namespace {
constexpr int kCols = 64, kRows = 48, kCells = kCols * kRows;  // FRAME_GRID_COLS / _ROWS
constexpr int kThHigh = 100;                                   // ORBmatcher::TH_HIGH
constexpr int kHisto = 30;                                     // ORBmatcher::HISTO_LENGTH
constexpr int kGridThreads = 1024;
constexpr int kProjectThreads = 128;

struct TrackParams {
  float fx, fy, cx, cy, mbf;
  float min_x, max_x, min_y, max_y, w_inv, h_inv;
  float rcw[9], tcw[3], ow[3];
  float scale[kOrbMaxLevels];
  float log_scale;  // Frame::mfLogScaleFactor
  float th, nnratio;
  int nlevels;
  int last_frame;  // 0: local-map search, 1: last-frame search
  int forward, backward;
};

struct TrackKey {  // one semantic key as the area walk reads it
  float x, y, ur;
  int octave;
};

struct TrackWin {  // one point's projection and window
  float u, v, rad, xr;
  int lmin, lmax, in_view, pad;
};

struct TrackBufs {  // scratch of one call, taken in order by carve()
  int* cell_start;  // kCells + 1
  int* cell_keys;   // cap
  int* cell_of;     // cap
  TrackKey* keys;   // cap
  uint4* desc;      // 2 cap
  float* angle;     // cap
  TrackWin* win;    // n_points
  Best2* fold;      // n_points
  int* hist;        // n_points
};

// `grids` grids of cap keys each (the Fuse keeps one per target, grid_at) and the per-point arrays of np points
size_t scratch_bytes(int cap, int np, int grids = 1) {
  const size_t c = static_cast<size_t>(std::max(cap, 1)) * grids, p = std::max(np, 1);
  return StreamScratch::bytes<int>(static_cast<size_t>(kCells + 1) * grids) + 2 * StreamScratch::bytes<int>(c) +
         StreamScratch::bytes<TrackKey>(c) + StreamScratch::bytes<uint4>(2 * c) + StreamScratch::bytes<float>(c) +
         StreamScratch::bytes<TrackWin>(p) + StreamScratch::bytes<Best2>(p) + StreamScratch::bytes<int>(p);
}

// takes the buffers, in order, from a HostCall or a StreamScratch of scratch_bytes(cap, np, grids)
template <class Scratch> TrackBufs carve(Scratch& a, int cap, int np, int grids = 1) {
  const size_t c = static_cast<size_t>(std::max(cap, 1)) * grids, p = std::max(np, 1);
  return {a.template take<int>(static_cast<size_t>(kCells + 1) * grids), a.template take<int>(c),
          a.template take<int>(c),                                      a.template take<TrackKey>(c),
          a.template take<uint4>(2 * c),                                a.template take<float>(c),
          a.template take<TrackWin>(p),                                 a.template take<Best2>(p),
          a.template take<int>(p)};
}

// grid g of a carve(.., cap, .., grids)
__device__ __forceinline__ TrackBufs grid_at(TrackBufs b, int g, int cap) {
  const size_t c = static_cast<size_t>(max(cap, 1)) * g;
  b.cell_start += static_cast<size_t>(kCells + 1) * g;
  b.cell_keys += c;
  b.cell_of += c;
  b.keys += c;
  b.desc += 2 * c;
  b.angle += c;
  return b;
}

// ---- grid: one block of kGridThreads builds the grid of keys j < n (n >= 0, already clamped to cap)
__device__ __forceinline__ void build_grid(const TrackParams& p, const sivo_keypoint* __restrict__ kps, const uint8_t* __restrict__ desc,
                                           const int* __restrict__ keep_idx, int n, int cap, const float* __restrict__ u_right,
                                           const TrackBufs& b) {
  __shared__ int cnt[kCells];
  __shared__ int warp_sum[kGridThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int c = tid; c < kCells; c += kGridThreads) cnt[c] = 0;
  __syncthreads();
  for (int j = tid; j < n; j += kGridThreads) {
    const int k = keep_idx ? keep_idx[j] : j;
    int cell = -1;
    TrackKey key{__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), -1.f, -1};
    float ang = 0.f;
    uint4 d0 = make_uint4(0, 0, 0, 0), d1 = d0;
    if (k >= 0 && k < cap) {
      const sivo_keypoint kp = kps[k];
      key = TrackKey{kp.x, kp.y, u_right[j], kp.octave};
      ang = kp.angle;
      d0 = reinterpret_cast<const uint4*>(desc + static_cast<size_t>(k) * 32)[0];
      d1 = reinterpret_cast<const uint4*>(desc + static_cast<size_t>(k) * 32)[1];
      // PosInGrid: round half away from zero; the comparisons in float keep a NaN or huge coordinate out of the int conversion.
      // A key whose angle breaks the angle rule goes in no cell.
      const float gx = roundf((kp.x - p.min_x) * p.w_inv), gy = roundf((kp.y - p.min_y) * p.h_inv);
      if (angle_ok(kp.angle) && gx >= 0.f && gx < static_cast<float>(kCols) && gy >= 0.f && gy < static_cast<float>(kRows)) {
        cell = static_cast<int>(gx) * kRows + static_cast<int>(gy);
        atomicAdd(&cnt[cell], 1);
      }
    }
    b.keys[j] = key;
    b.desc[2 * j] = d0;
    b.desc[2 * j + 1] = d1;
    b.angle[j] = ang;
    b.cell_of[j] = cell;
  }
  __syncthreads();
  // exclusive scan of the 3072 counts: three consecutive cells per thread
  constexpr int kPer = kCells / kGridThreads;
  int local[kPer], sum = 0;
#pragma unroll
  for (int q = 0; q < kPer; ++q) { local[q] = cnt[tid * kPer + q]; sum += local[q]; }
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_sum[warp] = incl;
  __syncthreads();
  int before = 0;
  for (int w = 0; w < warp; ++w) before += warp_sum[w];
  int run = before + incl - sum;
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const int c = tid * kPer + q;
    b.cell_start[c] = run;
    cnt[c] = run;  // becomes the scatter cursor
    run += local[q];
  }
  if (tid == kGridThreads - 1) b.cell_start[kCells] = run;
  __syncthreads();
  for (int j = tid; j < n; j += kGridThreads) {
    const int c = b.cell_of[j];
    if (c >= 0) b.cell_keys[atomicAdd(&cnt[c], 1)] = j;
  }
  __syncthreads();
  // each cell's list in ascending key order (the lists are a few keys long)
  for (int c = tid; c < kCells; c += kGridThreads) {
    const int s = b.cell_start[c], e = b.cell_start[c + 1];
    for (int i = s + 1; i < e; ++i) {
      const int v = b.cell_keys[i];
      int q = i - 1;
      while (q >= s && b.cell_keys[q] > v) { b.cell_keys[q + 1] = b.cell_keys[q]; --q; }
      b.cell_keys[q + 1] = v;
    }
  }
}

__global__ void __launch_bounds__(kGridThreads, 1) k_track_grid(const TrackParams p, const sivo_keypoint* __restrict__ kps,
                                                                const uint8_t* __restrict__ desc, const int* __restrict__ keep_idx,
                                                                const long long* __restrict__ n_keep, int cap,
                                                                const float* __restrict__ u_right, TrackBufs b) {
  const int n = clamp_count(*n_keep, cap);
  if (n < 0) return;
  build_grid(p, kps, desc, keep_idx, n, cap, u_right, b);
}

// ---- GetFeaturesInArea: visits the window's candidates 32 at a time in the reference's order.  visit(ok, j, n_in_chunk) is
// called by every lane of the warp for every chunk; lane i holds the chunk's i-th key (ok: it passes the level and position
// filters).  Returns without visiting when an early return of Frame.cc:334-358 applies.
template <class Visit>
__device__ __forceinline__ void walk_area(const TrackParams& p, const TrackBufs& b, float x, float y, float r, int min_level,
                                          int max_level, int lane, Visit&& visit) {
  const int min_cx = max(0, static_cast<int>(floorf(((x - p.min_x) - r) * p.w_inv)));
  if (min_cx >= kCols) return;
  const int max_cx = min(kCols - 1, static_cast<int>(ceilf(((x - p.min_x) + r) * p.w_inv)));
  if (max_cx < 0) return;
  const int min_cy = max(0, static_cast<int>(floorf(((y - p.min_y) - r) * p.h_inv)));
  if (min_cy >= kRows) return;
  const int max_cy = min(kRows - 1, static_cast<int>(ceilf(((y - p.min_y) + r) * p.h_inv)));
  if (max_cy < 0) return;
  const bool check_levels = min_level > 0 || max_level >= 0;
  for (int ix = min_cx; ix <= max_cx; ++ix) {
    const int s = b.cell_start[ix * kRows + min_cy], e = b.cell_start[ix * kRows + max_cy + 1];
    for (int base = s; base < e; base += 32) {
      const int i = base + lane;
      int j = -1;
      bool ok = false;
      if (i < e) {
        j = b.cell_keys[i];
        const TrackKey k = b.keys[j];
        ok = !(check_levels && (k.octave < min_level || (max_level >= 0 && k.octave > max_level))) && fabsf(k.x - x) < r &&
             fabsf(k.y - y) < r;
      }
      visit(ok, j, min(32, e - base));
    }
  }
}

// The candidate loop of both searches over the window `w` with the key mask `blocked` (NULL: none): the stereo gate, the
// distance and the fold in candidate order.
__device__ __forceinline__ Best2 search_window(const TrackParams& p, const TrackBufs& b, const TrackWin& w, const uint4 q0, const uint4 q1,
                                               const uint8_t* blocked, int lane) {
  Best2 best;
  walk_area(p, b, w.u, w.v, w.rad, w.lmin, w.lmax, lane, [&](bool ok, int j, int n) {
    int d = 0x7FFFFFFF, lvl = -1;
    if (ok && !(blocked && blocked[j])) {
      const TrackKey k = b.keys[j];
      if (!(k.ur > 0.f && fabsf(w.xr - k.ur) > w.rad)) {
        const uint4 t0 = b.desc[2 * j], t1 = b.desc[2 * j + 1];
        d = descriptor_distance(q0, q1, t0, t1);
        lvl = k.octave;
      }
    }
    best2_fold_warp(best, d, j, lvl, n);
  });
  return best;
}

// Pc = Rcw P + tcw as cv::gemm computes it for 3 x 3 floats
__device__ __forceinline__ void to_camera(const float* rcw, const float* tcw, const float* P, float* pc) {
#pragma unroll
  for (int r = 0; r < 3; ++r) pc[r] = ((rcw[3 * r] * P[0] + rcw[3 * r + 1] * P[1]) + rcw[3 * r + 2] * P[2]) + tcw[r];
}

// MapPoint::PredictScale(dist, F / pKF): ceil(logf(max_distance / dist) / logf(scale_factor)) clamped to [0, nlevels); -1 for a
// NaN quotient (the reference converts it to int)
__device__ __forceinline__ int predict_scale(const TrackParams& p, float max_distance, float dist) {
  const float ratio = max_distance / dist;
  const float lq = static_cast<float>(log(static_cast<double>(ratio))) / p.log_scale;
  if (isnan(lq)) return -1;
  const float c = ceilf(lq);
  return c < 0.f ? 0 : (c >= static_cast<float>(p.nlevels) ? p.nlevels - 1 : static_cast<int>(c));
}

// The projection and window of one point; in_view = 0 when it is not searched.
__device__ TrackWin project(const TrackParams& p, const sivo_map_point& mp) {
  TrackWin w{0.f, 0.f, 0.f, 0.f, 0, 0, 0, 0};
  float pc[3];
  to_camera(p.rcw, p.tcw, mp.pos, pc);
  if (!p.last_frame) {
    // Frame::isInFrustum(pMP, 0.5)
    if (pc[2] < 0.0f) return w;
    const float invz = 1.0f / pc[2];
    const float u = p.fx * pc[0] * invz + p.cx, v = p.fy * pc[1] * invz + p.cy;
    if (isnan(u) || isnan(v)) return w;
    if (u < p.min_x || u > p.max_x || v < p.min_y || v > p.max_y) return w;
    const float max_d = 1.2f * mp.max_distance, min_d = 0.8f * mp.min_distance;
    const float a0 = mp.pos[0] - p.ow[0], a1 = mp.pos[1] - p.ow[1], a2 = mp.pos[2] - p.ow[2];
    double ss = 0.0;
    ss = ss + static_cast<double>(a0) * a0;
    ss = ss + static_cast<double>(a1) * a1;
    ss = ss + static_cast<double>(a2) * a2;
    const float dist = static_cast<float>(sqrt(ss));
    if (dist < min_d || dist > max_d) return w;
    double dot = 0.0;
    dot = dot + static_cast<double>(a0) * mp.normal[0];
    dot = dot + static_cast<double>(a1) * mp.normal[1];
    dot = dot + static_cast<double>(a2) * mp.normal[2];
    const float view_cos = static_cast<float>(dot / static_cast<double>(dist));
    if (isnan(view_cos) || view_cos < 0.5f) return w;
    const int level = predict_scale(p, mp.max_distance, dist);
    if (level < 0) return w;
    // ORBmatcher::SearchByProjection(F, vpMapPoints, th)
    float r = static_cast<double>(view_cos) > 0.998 ? 2.5f : 4.0f;
    if (p.th != 1.0f) r *= p.th;
    w = TrackWin{u, v, r * p.scale[level], u - p.mbf * invz, level - 1, level, 1, 0};
    return w;
  }
  // SearchByProjection(CurrentFrame, LastFrame, th)
  const float invzc = static_cast<float>(1.0 / static_cast<double>(pc[2]));
  if (invzc < 0) return w;
  const float u = p.fx * pc[0] * invzc + p.cx, v = p.fy * pc[1] * invzc + p.cy;
  if (isnan(u) || isnan(v)) return w;
  if (u < p.min_x || u > p.max_x || v < p.min_y || v > p.max_y) return w;
  const int o = mp.octave;
  if (o < 0 || o >= p.nlevels || !angle_ok(mp.angle)) return w;
  const float radius = p.th * p.scale[o];
  int lmin = o - 1, lmax = o + 1;
  if (p.forward) { lmin = o; lmax = -1; }
  else if (p.backward) { lmin = 0; lmax = o; }
  w = TrackWin{u, v, radius, u - p.mbf * invzc, lmin, lmax, 1, 0};
  return w;
}

__device__ __forceinline__ void load_desc(const sivo_map_point* mp, uint4& q0, uint4& q1) {
  q0 = reinterpret_cast<const uint4*>(mp->desc)[0];
  q1 = reinterpret_cast<const uint4*>(mp->desc)[1];
}

// ---- the unconstrained pass: one warp per point
__global__ void __launch_bounds__(kProjectThreads) k_track_project(const TrackParams p, const long long* __restrict__ n_keep,
                                                                   const sivo_map_point* __restrict__ pts, int n_points,
                                                                   const uint8_t* __restrict__ blocked, TrackBufs b,
                                                                   uint8_t* __restrict__ in_view) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n_points || *n_keep < 0) return;
  const TrackWin w = project(p, pts[i]);
  Best2 best;
  if (w.in_view) {
    uint4 q0, q1;
    load_desc(pts + i, q0, q1);
    best = search_window(p, b, w, q0, q1, blocked, lane);
  }
  if (lane == 0) {
    b.win[i] = w;
    b.fold[i] = best;
    if (in_view) in_view[i] = static_cast<uint8_t>(w.in_view);
  }
}

// ---- the ordered pass: one warp, the key state in dynamic shared memory (owner: cap ints, blocked: cap bytes)
__global__ void __launch_bounds__(32) k_track_ordered(const TrackParams p, const long long* __restrict__ n_keep, int cap,
                                                      const sivo_map_point* __restrict__ pts, int n_points,
                                                      const uint8_t* __restrict__ blocked_in, TrackBufs b, int* __restrict__ match,
                                                      long long* __restrict__ n_matches) {
  extern __shared__ int owner[];
  __shared__ int hist_count[kHisto];
  uint8_t* blocked = reinterpret_cast<uint8_t*>(owner + cap);
  const int lane = threadIdx.x;
  const int n = clamp_count(*n_keep, cap);
  if (n < 0) {
    if (lane == 0 && n_matches) *n_matches = -1;
    return;
  }
  for (int j = lane; j < n; j += 32) {
    owner[j] = -1;
    blocked[j] = blocked_in ? blocked_in[j] : 0;
  }
  if (lane < kHisto) hist_count[lane] = 0;
  __syncwarp();
  int count = 0, n_hist = 0;
  for (int base = 0; base < n_points; base += 32) {
    const int mine = base + lane;
    Best2 f;
    int view = 0;
    if (mine < n_points) {
      f = b.fold[mine];
      view = b.win[mine].in_view;
    }
    const int m = min(32, n_points - base);
    for (int k = 0; k < m; ++k) {
      if (!__shfl_sync(0xffffffffu, view, k)) continue;
      const int i = base + k;
      Best2 r;
      r.idx = __shfl_sync(0xffffffffu, f.idx, k);
      if (r.idx < 0) continue;  // no candidate at all; taking keys only removes candidates
      r.idx2 = __shfl_sync(0xffffffffu, f.idx2, k);
      if (blocked[r.idx] || (!p.last_frame && r.idx2 >= 0 && blocked[r.idx2])) {
        uint4 q0, q1;
        load_desc(pts + i, q0, q1);
        r = search_window(p, b, b.win[i], q0, q1, blocked, lane);
        if (r.idx < 0) continue;
      } else {
        r.dist = __shfl_sync(0xffffffffu, f.dist, k);
        r.level = __shfl_sync(0xffffffffu, f.level, k);
        r.dist2 = __shfl_sync(0xffffffffu, f.dist2, k);
        r.level2 = __shfl_sync(0xffffffffu, f.level2, k);
      }
      if (r.dist > kThHigh) continue;
      if (!p.last_frame && r.level == r.level2 && static_cast<float>(r.dist) > p.nnratio * static_cast<float>(r.dist2)) continue;
      ++count;
      const sivo_map_point& mp = pts[i];
      if (lane == 0) {
        owner[r.idx] = i;
        if (mp.observed > 0) blocked[r.idx] = 1;
      }
      if (p.last_frame) {
        float rot = mp.angle - b.angle[r.idx];
        if (rot < 0.0f) rot += 360.0f;
        int bin = static_cast<int>(roundf(rot * (1.0f / kHisto)));
        if (bin == kHisto) bin = 0;
        if (lane == 0) {
          b.hist[n_hist] = r.idx | (bin << 24);
          ++hist_count[bin];
        }
        ++n_hist;
      }
      __syncwarp();
    }
  }
  if (p.last_frame) {
    __syncwarp();
    __shared__ int keep_bin[3];
    if (lane == 0) three_maxima(hist_count, kHisto, keep_bin);
    __syncwarp();
    int culled = 0;
    for (int e = lane; e < n_hist; e += 32) {
      const int v = b.hist[e], bin = v >> 24;
      if (bin != keep_bin[0] && bin != keep_bin[1] && bin != keep_bin[2]) {
        owner[v & 0xFFFFFF] = -1;
        ++culled;
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) culled += __shfl_xor_sync(0xffffffffu, culled, o);
    count -= culled;
    __syncwarp();
  }
  if (match)
    for (int j = lane; j < n; j += 32) match[j] = owner[j];
  if (lane == 0 && n_matches) *n_matches = count;
}

// test hook kernels: per-query list lengths, then the lists
__global__ void k_area_lists(const TrackParams p, TrackBufs b, const float* __restrict__ xyr, const int* __restrict__ levels, int nq,
                             const int* __restrict__ offsets, int* __restrict__ out) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (q >= nq) return;
  int pos = offsets ? offsets[q] : 0;
  walk_area(p, b, xyr[3 * q], xyr[3 * q + 1], xyr[3 * q + 2], levels[2 * q], levels[2 * q + 1], lane, [&](bool ok, int j, int) {
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (ok && offsets) out[pos + __popc(m & ((1u << lane) - 1u))] = j;
    pos += __popc(m);
  });
  if (!offsets && lane == 0) out[q] = pos;
}

TrackParams make_params(const Orb& left, const sivo_track_frame& f) {
  if (!(f.max_x > f.min_x) || !(f.max_y > f.min_y)) fail(SIVO_EINVAL, "track: image bounds need max > min");
  TrackParams p{};
  p.fx = f.fx; p.fy = f.fy; p.cx = f.cx; p.cy = f.cy; p.mbf = f.mbf;
  p.min_x = f.min_x; p.max_x = f.max_x; p.min_y = f.min_y; p.max_y = f.max_y;
  p.w_inv = static_cast<float>(kCols) / (f.max_x - f.min_x);
  p.h_inv = static_cast<float>(kRows) / (f.max_y - f.min_y);
  for (int i = 0; i < 9; ++i) p.rcw[i] = f.Rcw[i];
  for (int i = 0; i < 3; ++i) { p.tcw[i] = f.tcw[i]; p.ow[i] = f.Ow[i]; }
  p.nlevels = left.nlevels();
  for (int l = 0; l < p.nlevels; ++l) p.scale[l] = left.tables().scale[l];
  p.log_scale = static_cast<float>(std::log(static_cast<double>(left.tables().scale.size() > 1 ? left.tables().scale[1] : 1.0f)));
  return p;
}

// the forward / backward decision of the last-frame search (ORBmatcher.cc:1290-1301)
void last_frame_direction(TrackParams& p, const sivo_track_frame& f, const float* Rlw, const float* tlw) {
  float twc[3], tlc[3];
  for (int r = 0; r < 3; ++r) {
    double s = 0.0;
    s = s + static_cast<double>(f.Rcw[r]) * f.tcw[0];
    s = s + static_cast<double>(f.Rcw[3 + r]) * f.tcw[1];
    s = s + static_cast<double>(f.Rcw[6 + r]) * f.tcw[2];
    twc[r] = -static_cast<float>(s);
  }
  for (int r = 0; r < 3; ++r) tlc[r] = ((Rlw[3 * r] * twc[0] + Rlw[3 * r + 1] * twc[1]) + Rlw[3 * r + 2] * twc[2]) + tlw[r];
  p.forward = tlc[2] > f.mb;
  p.backward = -tlc[2] > f.mb;
}

size_t ordered_smem(int cap) { return static_cast<size_t>(std::max(cap, 1)) * (sizeof(int) + 1); }

void launch_search(const TrackParams& p, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                   int cap, const float* u_right, const uint8_t* blocked, const sivo_map_point* pts, int n_points, const TrackBufs& b,
                   uint8_t* in_view, int* match, long long* n_matches, cudaStream_t s) {
  const size_t smem = ordered_smem(cap);
  if (smem > 200 * 1024) fail(SIVO_EINVAL, "track: capacity %d exceeds the ordered pass's shared memory", cap);
  SIVO_CUDA(cudaFuncSetAttribute(k_track_ordered, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  k_track_grid<<<1, kGridThreads, 0, s>>>(p, kps, desc, keep_idx, n_keep, cap, u_right, b);
  SIVO_CUDA(cudaGetLastError());
  if (n_points > 0) {
    k_track_project<<<ceil_div(n_points, kProjectThreads / 32), kProjectThreads, 0, s>>>(p, n_keep, pts, n_points, blocked, b, in_view);
    SIVO_CUDA(cudaGetLastError());
  }
  k_track_ordered<<<1, 32, smem, s>>>(p, n_keep, cap, pts, n_points, blocked, b, match, n_matches);
  SIVO_CUDA(cudaGetLastError());
}

void check_args(int n_points, float th, float nnratio) {
  if (n_points < 0 || !(th > 0.f) || !std::isfinite(th) || !std::isfinite(nnratio)) fail(SIVO_EINVAL, "track: bad arguments");
}

// The host forms: stage the gathered keys and the points on the host-call workspace, run the device forms' kernels, download.
void search_host(const Orb& left, bool last, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right, const uint8_t* blocked,
                 int n, const sivo_map_point* pts, int n_points, const sivo_track_frame& f, const float* Rlw, const float* tlw, float th,
                 float nnratio, uint8_t* in_view, int* match, int* n_matches) {
  if (n < 0) fail(SIVO_EINVAL, "track: n = %d", n);
  check_args(n_points, th, nnratio);
  TrackParams p = make_params(left, f);
  p.th = th;
  p.nnratio = nnratio;
  p.last_frame = last;
  for (int j = 0; j < n; ++j)
    if (!angle_ok(kps[j].angle)) fail(SIVO_ERANGE, "track: key %d has angle %g outside [0, 360]", j, kps[j].angle);
  if (last) {
    last_frame_direction(p, f, Rlw, tlw);
    for (int i = 0; i < n_points; ++i) {
      if (pts[i].octave < 0 || pts[i].octave >= p.nlevels) fail(SIVO_ERANGE, "track: point %d has octave %d", i, pts[i].octave);
      if (!angle_ok(pts[i].angle)) fail(SIVO_ERANGE, "track: point %d has angle %g outside [0, 360]", i, pts[i].angle);
    }
  }
  HostCall& hc = host_call();
  hc.begin(left.device());
  const sivo_keypoint* d_kps = hc.upload(kps, n);
  const uint8_t* d_desc = hc.upload(desc, static_cast<size_t>(n) * 32);
  const float* d_ur = hc.upload(u_right, n);
  const uint8_t* d_blocked = blocked ? hc.upload(blocked, n) : nullptr;
  const sivo_map_point* d_pts = hc.upload(pts, n_points);
  const long long count = n;
  const long long* d_count = hc.upload(&count, 1);
  uint8_t* d_view = hc.take<uint8_t>(n_points);
  int* d_match = hc.take<int>(n);
  long long* d_nm = hc.take<long long>(1);
  const TrackBufs b = carve(hc, n, n_points);
  launch_search(p, d_kps, d_desc, nullptr, d_count, n, d_ur, d_blocked, d_pts, n_points, b, d_view, d_match, d_nm, hc.stream);
  long long nm = 0;
  hc.download(in_view, d_view, n_points);
  hc.download(match, d_match, n);
  hc.download(&nm, d_nm, 1);
  hc.sync();
  if (n_matches) *n_matches = static_cast<int>(nm);
}

void search_device(const Orb& left, bool last, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                   const float* u_right, const uint8_t* blocked, const sivo_map_point* pts, int n_points, const sivo_track_frame& f,
                   const float* Rlw, const float* tlw, float th, float nnratio, uint8_t* in_view, int* match, long long* n_matches,
                   cudaStream_t s) {
  check_args(n_points, th, nnratio);
  TrackParams p = make_params(left, f);
  p.th = th;
  p.nnratio = nnratio;
  p.last_frame = last;
  if (last) last_frame_direction(p, f, Rlw, tlw);
  s = left.enter(s);
  const int cap = left.capacity();
  StreamScratch sc(scratch_bytes(cap, n_points), s);
  const TrackBufs b = carve(sc, cap, n_points);
  launch_search(p, kps, desc, keep_idx, n_keep, cap, u_right, blocked, pts, n_points, b, in_view, match, n_matches, s);
}

// ---- ORBmatcher::Fuse(pKF, vpMapPoints, th) over a chunk of targets: every target's grid in one launch (block k builds target
// k's), then one warp per (target, point) pair.  The pair's decision depends only on the point and the target, so the pairs run
// independently; the caller's map bookkeeping replays them in the reference's order (include/sivo_b200.h).
constexpr int kFuseChunk = 64;  // targets per launch: their records ride in the kernel parameters
constexpr int kFuseThreads = 128;
constexpr int kThLow = 50;      // ORBmatcher::TH_LOW
enum { kFuseNegative = -1, kFuseDepth = 0, kFuseImage, kFuseDistance, kFuseAngle, kFuseNoCandidate, kFuseAboveThLow, kFuseMatched };

struct FuseTarget {
  const sivo_keypoint* kps;
  const uint8_t* desc;
  const float* ur;
  const long long* count;
  float rcw[9], tcw[3], ow[3];
};

struct FuseParams {
  TrackParams geo;  // the shared camera, bounds and scale tables (its pose is unused)
  float inv_sigma2[kOrbMaxLevels];
  int cap, n_targets, base, n_points;  // base: the chunk's first target
  FuseTarget t[kFuseChunk];
};

__global__ void __launch_bounds__(kGridThreads, 1) k_fuse_grid(const __grid_constant__ FuseParams p, TrackBufs g) {
  const FuseTarget& t = p.t[blockIdx.x];
  const int n = clamp_count(*t.count, p.cap);
  if (n < 0) return;
  build_grid(p.geo, t.kps, t.desc, nullptr, n, p.cap, t.ur, grid_at(g, blockIdx.x, p.cap));
}

// One warp per pair: (blockIdx.y = target in the chunk, point).  Writes match / dist / stage at (base + k) n_points + i.
__global__ void __launch_bounds__(kFuseThreads) k_fuse_decide(const __grid_constant__ FuseParams p, TrackBufs g,
                                                              const sivo_map_point* __restrict__ pts, float th, int* __restrict__ match,
                                                              int* __restrict__ dist, int* __restrict__ stage_out) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31, k = blockIdx.y;
  if (i >= p.n_points) return;
  const FuseTarget& t = p.t[k];
  const TrackParams& c = p.geo;
  const sivo_map_point& mp = pts[i];
  int stage = kFuseNegative, bd = 256, bi = -1;
  if (*t.count >= 0) {
    float pc[3];
    to_camera(t.rcw, t.tcw, mp.pos, pc);
    stage = kFuseDepth;
    if (!(pc[2] < 0.0f)) {
      const float invz = 1 / pc[2];
      const float x = pc[0] * invz, y = pc[1] * invz;
      const float u = c.fx * x + c.cx, v = c.fy * y + c.cy;
      stage = kFuseImage;
      // KeyFrame::IsInImage: strict upper bounds; a NaN is out
      if (u >= c.min_x && u < c.max_x && v >= c.min_y && v < c.max_y) {
        const float ur = u - c.mbf * invz;
        const float max_d = 1.2f * mp.max_distance, min_d = 0.8f * mp.min_distance;
        const float a[3] = {mp.pos[0] - t.ow[0], mp.pos[1] - t.ow[1], mp.pos[2] - t.ow[2]};
        double ss = 0.0, dot = 0.0;
#pragma unroll
        for (int r = 0; r < 3; ++r) ss = ss + static_cast<double>(a[r]) * a[r];
        const float dist3 = static_cast<float>(sqrt(ss));
#pragma unroll
        for (int r = 0; r < 3; ++r) dot = dot + static_cast<double>(a[r]) * mp.normal[r];
        stage = kFuseDistance;
        if (!(dist3 < min_d || dist3 > max_d)) {
          stage = kFuseAngle;
          if (!(dot < 0.5 * static_cast<double>(dist3))) {
            const int level = predict_scale(c, mp.max_distance, dist3);
            stage = kFuseNoCandidate;  // also a NaN level quotient: nothing is searched
            if (level >= 0) {
              const float radius = th * c.scale[level];
              const uint4 q0 = reinterpret_cast<const uint4*>(mp.desc)[0], q1 = reinterpret_cast<const uint4*>(mp.desc)[1];
              const TrackBufs b = grid_at(g, k, p.cap);
              bool any = false;
              walk_area(c, b, u, v, radius, -1, -1, lane, [&](bool ok, int j, int) {
                any |= __any_sync(0xffffffffu, ok);
                unsigned key = 256u << 5 | 31u;
                if (ok) {
                  const TrackKey kp = b.keys[j];
                  const int o = kp.octave;
                  if (o >= level - 1 && o <= level && o >= 0 && o < c.nlevels) {
                    const float ex = u - kp.x, ey = v - kp.y;
                    bool pass;
                    if (kp.ur >= 0.f) {
                      const float er = ur - kp.ur;
                      const float e2 = (ex * ex + ey * ey) + er * er;
                      pass = !(static_cast<double>(e2 * p.inv_sigma2[o]) > 7.8);
                    } else {
                      const float e2 = ex * ex + ey * ey;
                      pass = !(static_cast<double>(e2 * p.inv_sigma2[o]) > 5.99);
                    }
                    if (pass) key = static_cast<unsigned>(descriptor_distance(q0, q1, b.desc[2 * j], b.desc[2 * j + 1])) << 5 | lane;
                  }
                }
                // the chunk's smallest distance, first in walk order on ties; a later chunk takes over only when strictly smaller
                const unsigned m = __reduce_min_sync(0xffffffffu, key);
                const int jm = __shfl_sync(0xffffffffu, j, m & 31u);
                if (static_cast<int>(m >> 5) < bd) { bd = static_cast<int>(m >> 5); bi = jm; }
              });
              if (any) stage = bd <= kThLow ? kFuseMatched : kFuseAboveThLow;
            }
          }
        }
      }
    }
  }
  if (lane == 0) {
    const size_t e = static_cast<size_t>(p.base + k) * p.n_points + i;
    match[e] = stage == kFuseMatched ? bi : -1;
    if (dist) dist[e] = bd;
    if (stage_out) stage_out[e] = stage;
  }
}

FuseParams fuse_params(const Orb& left, const sivo_fuse_camera& cam, int cap, int n_points) {
  sivo_track_frame f{};
  f.fx = cam.fx; f.fy = cam.fy; f.cx = cam.cx; f.cy = cam.cy; f.mbf = cam.mbf;
  f.min_x = cam.min_x; f.max_x = cam.max_x; f.min_y = cam.min_y; f.max_y = cam.max_y;
  FuseParams p{};
  p.geo = make_params(left, f);
  for (int l = 0; l < p.geo.nlevels; ++l) p.inv_sigma2[l] = left.tables().inv_sigma2[l];
  p.cap = cap;
  p.n_points = n_points;
  return p;
}

void check_fuse_args(const sivo_keyframe_keys* targets, int n_targets, int n_points, float th) {
  if (n_targets < 0 || n_points < 0) fail(SIVO_EINVAL, "fuse: n_targets %d, n_points %d", n_targets, n_points);
  if (static_cast<long long>(n_targets) * n_points > INT_MAX) fail(SIVO_EINVAL, "fuse: %d x %d pairs exceed INT_MAX", n_targets, n_points);
  if (!(th > 0.f) || !std::isfinite(th)) fail(SIVO_EINVAL, "fuse: th %g", th);
  if (n_targets > 0 && !targets) fail(SIVO_EINVAL, "fuse: null targets");
  for (int k = 0; k < n_targets; ++k)
    if (!targets[k].count) fail(SIVO_EINVAL, "fuse: target %d has no count", k);
}

// Runs every chunk of targets (t: device pointers) with the grids g (min(n_targets, kFuseChunk) of them).
void launch_fuse(FuseParams& p, const FuseTarget* t, int n_targets, const TrackBufs& g, const sivo_map_point* pts, float th, int* match,
                 int* dist, int* stage, cudaStream_t s) {
  if (p.n_points == 0) return;
  for (int base = 0; base < n_targets; base += kFuseChunk) {
    p.base = base;
    p.n_targets = std::min(kFuseChunk, n_targets - base);
    for (int k = 0; k < p.n_targets; ++k) p.t[k] = t[base + k];
    k_fuse_grid<<<p.n_targets, kGridThreads, 0, s>>>(p, g);
    SIVO_CUDA(cudaGetLastError());
    k_fuse_decide<<<dim3(ceil_div(p.n_points, kFuseThreads / 32), p.n_targets), kFuseThreads, 0, s>>>(p, g, pts, th, match, dist, stage);
    SIVO_CUDA(cudaGetLastError());
  }
}

FuseTarget fuse_target(const sivo_keyframe_keys& k, const sivo_keypoint* kps, const uint8_t* desc, const float* ur, const long long* count) {
  FuseTarget t{kps, desc, ur, count, {}, {}, {}};
  for (int i = 0; i < 9; ++i) t.rcw[i] = k.Rcw[i];
  for (int i = 0; i < 3; ++i) { t.tcw[i] = k.tcw[i]; t.ow[i] = k.Ow[i]; }
  return t;
}
}  // namespace

void search_local_points(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right, const uint8_t* blocked, int n,
                         const sivo_map_point* pts, int n_points, const sivo_track_frame& f, float th, float nnratio, uint8_t* in_view,
                         int* match, int* n_matches) {
  search_host(left, false, kps, desc, u_right, blocked, n, pts, n_points, f, nullptr, nullptr, th, nnratio, in_view, match, n_matches);
}

void search_last_frame(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const float* u_right, int n, const sivo_map_point* pts,
                       int n_points, const sivo_track_frame& f, const float* Rlw, const float* tlw, float th, int* match, int* n_matches) {
  search_host(left, true, kps, desc, u_right, nullptr, n, pts, n_points, f, Rlw, tlw, th, 0.f, nullptr, match, n_matches);
}

void search_local_points_device(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                                const float* u_right, const uint8_t* blocked, const sivo_map_point* pts, int n_points,
                                const sivo_track_frame& f, float th, float nnratio, uint8_t* in_view, int* match, long long* n_matches,
                                cudaStream_t s) {
  search_device(left, false, kps, desc, keep_idx, n_keep, u_right, blocked, pts, n_points, f, nullptr, nullptr, th, nnratio, in_view, match,
                n_matches, s);
}

void search_last_frame_device(const Orb& left, const sivo_keypoint* kps, const uint8_t* desc, const int* keep_idx, const long long* n_keep,
                              const float* u_right, const sivo_map_point* pts, int n_points, const sivo_track_frame& f, const float* Rlw,
                              const float* tlw, float th, int* match, long long* n_matches, cudaStream_t s) {
  search_device(left, true, kps, desc, keep_idx, n_keep, u_right, nullptr, pts, n_points, f, Rlw, tlw, th, 0.f, nullptr, match, n_matches, s);
}

// GetFeaturesInArea on the device grid of n host keys: lengths, host scan, lists
void features_in_area(const Orb& left, const sivo_keypoint* kps, int n, const sivo_track_frame& f, const float* xyr, const int* levels, int nq,
                      int* offsets, int* idx, int idx_cap) {
  if (n < 0 || nq < 0) fail(SIVO_EINVAL, "features_in_area: negative counts");
  const TrackParams p = make_params(left, f);
  HostCall& hc = host_call();
  hc.begin(left.device());
  cudaStream_t st = hc.stream;
  const sivo_keypoint* d_kps = hc.upload(kps, n);
  uint8_t* d_desc = hc.take<uint8_t>(static_cast<size_t>(n) * 32);
  float* d_ur = hc.take<float>(n);
  if (n) {
    SIVO_CUDA(cudaMemsetAsync(d_desc, 0, static_cast<size_t>(n) * 32, st));
    SIVO_CUDA(cudaMemsetAsync(d_ur, 0, n * sizeof(float), st));
  }
  const long long count = n;
  const long long* d_count = hc.upload(&count, 1);
  const float* d_xyr = hc.upload(xyr, 3 * static_cast<size_t>(nq));
  const int* d_lv = hc.upload(levels, 2 * static_cast<size_t>(nq));
  int* d_off = hc.take<int>(nq + 1);
  int* d_idx = hc.take<int>(std::max(idx_cap, 0));
  const TrackBufs b = carve(hc, n, 0);
  k_track_grid<<<1, kGridThreads, 0, st>>>(p, d_kps, d_desc, nullptr, d_count, n, d_ur, b);
  SIVO_CUDA(cudaGetLastError());
  std::vector<int> len(std::max(nq, 1));
  if (nq) {
    k_area_lists<<<ceil_div(nq * 32, 128), 128, 0, st>>>(p, b, d_xyr, d_lv, nq, nullptr, d_off);
    SIVO_CUDA(cudaGetLastError());
    hc.download(len.data(), d_off, nq);
  }
  hc.sync();
  offsets[0] = 0;
  for (int q = 0; q < nq; ++q) offsets[q + 1] = offsets[q] + len[q];
  if (offsets[nq] > idx_cap) fail(SIVO_ERANGE, "features_in_area: %d candidates, room for %d", offsets[nq], idx_cap);
  if (!offsets[nq]) return;
  SIVO_CUDA(cudaMemcpyAsync(d_off, offsets, (nq + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
  k_area_lists<<<ceil_div(nq * 32, 128), 128, 0, st>>>(p, b, d_xyr, d_lv, nq, d_off, d_idx);
  SIVO_CUDA(cudaGetLastError());
  hc.download(idx, d_idx, offsets[nq]);
  hc.sync();
}

void fuse_device(const Orb& left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera& cam, const sivo_map_point* pts,
                 int n_points, float th, int* match, int* dist, cudaStream_t s) {
  check_fuse_args(targets, n_targets, n_points, th);
  const int cap = left.capacity();
  FuseParams p = fuse_params(left, cam, cap, n_points);
  std::vector<FuseTarget> t(n_targets);
  for (int k = 0; k < n_targets; ++k) {
    const sivo_keyframe_keys& tk = targets[k];
    if (!tk.kps || !tk.desc || !tk.u_right) fail(SIVO_EINVAL, "fuse: null array in target %d", k);
    t[k] = fuse_target(tk, tk.kps, tk.desc, tk.u_right, tk.count);
  }
  if (!n_targets || !n_points) return;
  s = left.enter(s);
  const int grids = std::min(n_targets, kFuseChunk);
  StreamScratch sc(scratch_bytes(cap, 0, grids), s);
  const TrackBufs g = carve(sc, cap, 0, grids);
  launch_fuse(p, t.data(), n_targets, g, pts, th, match, dist, nullptr, s);
}

// The host form and the test hook: stage every target's keys and the points, run the device form's kernels, download.
void fuse_host(const Orb& left, const sivo_keyframe_keys* targets, int n_targets, const sivo_fuse_camera& cam, const sivo_map_point* pts,
               int n_points, float th, int* match, int* dist, int* stage) {
  check_fuse_args(targets, n_targets, n_points, th);
  int cap = 0;
  for (int k = 0; k < n_targets; ++k) {
    const sivo_keyframe_keys& tk = targets[k];
    const long long n = *tk.count;
    if (n > INT_MAX) fail(SIVO_EINVAL, "fuse: target %d has %lld keys", k, n);
    if (n > 0 && (!tk.kps || !tk.desc || !tk.u_right)) fail(SIVO_EINVAL, "fuse: null array in target %d", k);
    for (long long j = 0; j < n; ++j)
      if (!angle_ok(tk.kps[j].angle)) fail(SIVO_ERANGE, "fuse: target %d key %lld has angle %g outside [0, 360]", k, j, tk.kps[j].angle);
    cap = std::max(cap, static_cast<int>(std::max(n, 0ll)));
  }
  FuseParams p = fuse_params(left, cam, cap, n_points);
  if (!n_targets || !n_points) return;
  HostCall& hc = host_call();
  hc.begin(left.device());
  std::vector<FuseTarget> t(n_targets);
  for (int k = 0; k < n_targets; ++k) {
    const sivo_keyframe_keys& tk = targets[k];
    const size_t n = static_cast<size_t>(std::max(*tk.count, 0ll));
    t[k] = fuse_target(tk, hc.upload(tk.kps, n), hc.upload(tk.desc, 32 * n), hc.upload(tk.u_right, n), hc.upload(tk.count, 1));
  }
  const sivo_map_point* d_pts = hc.upload(pts, n_points);
  const size_t np = static_cast<size_t>(n_targets) * n_points;
  int* d_match = hc.take<int>(np);
  int* d_dist = hc.take<int>(np);
  int* d_stage = stage ? hc.take<int>(np) : nullptr;
  const TrackBufs g = carve(hc, cap, 0, std::min(n_targets, kFuseChunk));
  launch_fuse(p, t.data(), n_targets, g, d_pts, th, d_match, d_dist, d_stage, hc.stream);
  hc.download(match, d_match, np);
  hc.download(dist, d_dist, np);
  hc.download(stage, d_stage, np);
  hc.sync();
}

}  // namespace sivo
