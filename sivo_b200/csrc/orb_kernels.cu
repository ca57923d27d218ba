// ORB extractor kernels.  All integer / byte work, bit-exact against oracle/orb_oracle.py (which is pinned
// to cv2): pyramid (cv::resize INTER_LINEAR fixed point + REFLECT_101 border), FAST-9/16 score map,
// per-cell threshold / 3x3 NMS / ordered compaction, 7x7 sigma-2 fixed-point blur, IC angle, rBRIEF.
// Everything here is latency/launch bound on the GPU (~8 MB touched per image), so the design goal is few
// launches over all 8 levels at once rather than bandwidth tricks.
#include "orb.h"

namespace sivo {
namespace {

__constant__ int8_t c_pattern[256 * 4];

const int8_t h_pattern[256 * 4] = {
#include "orb_pattern.inc"
};

__device__ __forceinline__ int reflect101(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

// ---- level 0: copyMakeBorder(image, 19, BORDER_REFLECT_101) (ORBextractor.cc:1112-1119)
__global__ void k_level0(const uint8_t* __restrict__ gray, size_t gpitch, uint8_t* __restrict__ dst, OrbLevel lv) {
  ORB_PDL_PROLOGUE();
  int bx = blockIdx.x * blockDim.x + threadIdx.x, by = blockIdx.y;
  if (bx >= lv.w + 2 * kEdge) return;
  int x = reflect101(bx - kEdge, lv.w), y = reflect101(by - kEdge, lv.h);
  dst[lv.img_off + static_cast<size_t>(by) * lv.pitch + bx] = gray[static_cast<size_t>(y) * gpitch + x];
}

// ---- level k from level k-1: cv::resize(INTER_LINEAR) 8-bit fixed point, then the REFLECT_101 border
// (ORBextractor.cc:1097-1110).  Coefficient rule as pinned in oracle/orb_oracle.py::resize_linear_u8.
struct Coef { int s0, s1, a0, a1; };
__device__ __forceinline__ Coef lin_coef(int d, int dn, int sn) {
  double scale = static_cast<double>(sn) / static_cast<double>(dn);
  float f = static_cast<float>((d + 0.5) * scale - 0.5);
  int s0 = static_cast<int>(floorf(f));
  float fr = __fsub_rn(f, static_cast<float>(s0));
  if (s0 < 0) { fr = 0.f; s0 = 0; }
  if (s0 >= sn - 1) { fr = 0.f; s0 = sn - 1; }
  Coef c;
  c.s0 = s0;
  c.s1 = min(s0 + 1, sn - 1);
  c.a1 = __float2int_rn(__fmul_rn(fr, 2048.f));
  c.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fr), 2048.f));
  return c;
}

__global__ void k_resize(uint8_t* __restrict__ pyr, OrbLevel src, OrbLevel dst) {
  ORB_PDL_PROLOGUE();
  int bx = blockIdx.x * blockDim.x + threadIdx.x, by = blockIdx.y;
  if (bx >= dst.w + 2 * kEdge) return;
  int dx = reflect101(bx - kEdge, dst.w), dy = reflect101(by - kEdge, dst.h);
  Coef cx = lin_coef(dx, dst.w, src.w), cy = lin_coef(dy, dst.h, src.h);
  const uint8_t* s = pyr + src.img_off + static_cast<size_t>(kEdge) * src.pitch + kEdge;
  const uint8_t* r0 = s + static_cast<size_t>(cy.s0) * src.pitch;
  const uint8_t* r1 = s + static_cast<size_t>(cy.s1) * src.pitch;
  int S0 = r0[cx.s0] * cx.a0 + r0[cx.s1] * cx.a1;
  int S1 = r1[cx.s0] * cx.a0 + r1[cx.s1] * cx.a1;
  int v = (((cy.a0 * (S0 >> 4)) >> 16) + ((cy.a1 * (S1 >> 4)) >> 16) + 2) >> 2;
  pyr[dst.img_off + static_cast<size_t>(by) * dst.pitch + bx] = static_cast<uint8_t>(v);
}

// ---- FAST-9/16 corner score (cv::FAST's cornerScore<16>): S = max over the 16 contiguous 9-arcs of
// min(+-(ring - p)) - 1; p is a corner at threshold t iff S >= t.  One thread per pixel, all levels in
// one launch (grid.y = level).  Only [19, w-19) x [19, h-19) can ever be a keypoint (cell interiors).
// `t_min` = the smallest threshold any consumer applies (min(iniThFAST, minThFAST)): a 9-arc covers at least two of the four
// compass points, so a pixel with fewer than two compass points brighter than p + t_min and fewer than two darker than
// p - t_min has S < t_min, is zeroed by every threshold, and gets 0 without the full score (most pixels).
__device__ __forceinline__ int fast_score_at(const uint8_t* __restrict__ pyr, const OrbLevel& lv, int x, int y, int t_min) {
  if (!(x >= kEdge && x < lv.w - kEdge && y >= kEdge && y < lv.h - kEdge)) return 0;
  const uint8_t* c = pyr + lv.img_off + static_cast<size_t>(y + kEdge) * lv.pitch + x + kEdge;
  const int P = lv.pitch;
  const int off[16] = {3 * P,      3 * P + 1,  2 * P + 2,  P + 3,  3,  -P + 3,  -2 * P + 2, -3 * P + 1,
                       -3 * P,     -3 * P - 1, -2 * P - 2, -P - 3, -3, P - 3,   2 * P - 2,  3 * P - 1};
  const int v = c[0];
  {
    const int q[4] = {static_cast<int>(c[3 * P]) - v, static_cast<int>(c[3]) - v, static_cast<int>(c[-3 * P]) - v, static_cast<int>(c[-3]) - v};
    int nb = 0, nd = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) { nb += q[k] > t_min; nd += q[k] < -t_min; }
    if (nb < 2 && nd < 2) return 0;
  }
  int d[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) d[k] = static_cast<int>(c[off[k]]) - v;
  int best = -255;
#pragma unroll
  for (int sgn = 0; sgn < 2; ++sgn) {
    int m2[16], m4[16], m8[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) m2[k] = min(d[k], d[(k + 1) & 15]);
#pragma unroll
    for (int k = 0; k < 16; ++k) m4[k] = min(m2[k], m2[(k + 2) & 15]);
#pragma unroll
    for (int k = 0; k < 16; ++k) m8[k] = min(m4[k], m4[(k + 4) & 15]);
#pragma unroll
    for (int k = 0; k < 16; ++k) best = max(best, min(m8[k], d[(k + 8) & 15]));
#pragma unroll
    for (int k = 0; k < 16; ++k) d[k] = -d[k];
  }
  return max(best - 1, 0);
}

__global__ void k_fast_score(const uint8_t* __restrict__ pyr, uint8_t* __restrict__ score, OrbLevelTable t, int t_min) {
  const OrbLevel lv = t.lv[blockIdx.y];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= lv.w * lv.h) return;
  score[lv.flat_off + i] = static_cast<uint8_t>(fast_score_at(pyr, lv, i % lv.w, i / lv.w, t_min));
}

// ---- one block per 30-px cell: cv::FAST(cell, iniThFAST, NMS) with the minThFAST retry when the cell
// comes back empty (ORBextractor.cc:793-807), emitted in sub-image row-major order.
constexpr int kCellThreads = 256;
constexpr int kCellMaxDim = 62;  // interior side bound: wCell = ceil(width / floor(width/30)) <= 59

__device__ int block_exclusive_scan(int flag, int* s_warp, int& total) {
  unsigned b = __ballot_sync(0xffffffffu, flag);
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int within = __popc(b & ((1u << lane) - 1));
  if (lane == 0) s_warp[wid] = __popc(b);
  __syncthreads();
  int base = 0, tot = 0;
  for (int w = 0; w < kCellThreads / 32; ++w) {
    int c = s_warp[w];
    if (w < wid) base += c;
    tot += c;
  }
  __syncthreads();
  total = tot;
  return base + within;
}

// score == nullptr: the cell computes its own FAST scores from the pyramid (cell interiors tile the level without overlap, so
// this is the same work as the score-map kernel minus one launch and the 1.1 MB map written and read back)
__global__ void __launch_bounds__(kCellThreads) k_cells(const uint8_t* __restrict__ score, const uint8_t* __restrict__ pyr, OrbLevelTable t,
                                                        const OrbCell* __restrict__ cells, int ini_th, int min_th,
                                                        int* __restrict__ cell_count, uint32_t* __restrict__ cell_items) {
  ORB_PDL_PROLOGUE();
  __shared__ uint8_t s[(kCellMaxDim + 2) * (kCellMaxDim + 2)];
  __shared__ int s_warp[kCellThreads / 32];
  __shared__ int s_any;
  const OrbCell cell = cells[blockIdx.x];
  const OrbLevel lv = t.lv[cell.level];
  const int ix0 = cell.x0 + 3, iy0 = cell.y0 + 3;
  const int iw = cell.x1 - 3 - ix0, ih = cell.y1 - 3 - iy0;  // interior size
  if (iw <= 0 || ih <= 0) {
    if (threadIdx.x == 0) cell_count[blockIdx.x] = 0;
    return;
  }
  const int sw = iw + 2;
  const uint8_t* sc = score + lv.flat_off;
  for (int e = threadIdx.x; e < (ih + 2) * sw; e += kCellThreads) {
    int x = e % sw - 1, y = e / sw - 1;
    uint8_t v = 0;
    if (x >= 0 && x < iw && y >= 0 && y < ih)
      v = score ? sc[static_cast<size_t>(iy0 + y) * lv.w + ix0 + x]
                : static_cast<uint8_t>(fast_score_at(pyr, lv, ix0 + x, iy0 + y, min(ini_th, min_th)));
    s[e] = v;  // outside the sub-image's 3-px apron the score is 0 by construction of cv::FAST
  }
  if (threadIdx.x == 0) s_any = 0;
  __syncthreads();
  int th = ini_th;
  for (int pass = 0; pass < 2; ++pass) {
    // does any pixel survive threshold + NMS at this threshold?
    int any = 0;
    for (int e = threadIdx.x; e < iw * ih; e += kCellThreads) {
      int x = e % iw, y = e / iw;
      const uint8_t* p = s + (y + 1) * sw + x + 1;
      int v = p[0];
      if (v < th) continue;
      auto nb = [&](int o) { int q = p[o]; return q >= th ? q : 0; };
      if (v > nb(-sw - 1) && v > nb(-sw) && v > nb(-sw + 1) && v > nb(-1) && v > nb(1) && v > nb(sw - 1) && v > nb(sw) &&
          v > nb(sw + 1))
        any = 1;
    }
    if (any) s_any = 1;
    __syncthreads();
    if (s_any) break;
    th = min_th;
    __syncthreads();
  }
  if (!s_any) {
    if (threadIdx.x == 0) cell_count[blockIdx.x] = 0;
    return;
  }
  // ordered compaction, row-major
  int written = 0;
  uint32_t* out = cell_items + static_cast<size_t>(blockIdx.x) * kCellCap;
  const int relx = ix0 - (kEdge - 3), rely = iy0 - (kEdge - 3);  // relative to (minBorderX, minBorderY)
  for (int base = 0; base < iw * ih; base += kCellThreads) {
    int e = base + threadIdx.x;
    int flag = 0, v = 0, x = 0, y = 0;
    if (e < iw * ih) {
      x = e % iw;
      y = e / iw;
      const uint8_t* p = s + (y + 1) * sw + x + 1;
      v = p[0];
      if (v >= th) {
        auto nb = [&](int o) { int q = p[o]; return q >= th ? q : 0; };
        flag = v > nb(-sw - 1) && v > nb(-sw) && v > nb(-sw + 1) && v > nb(-1) && v > nb(1) && v > nb(sw - 1) &&
               v > nb(sw) && v > nb(sw + 1);
      }
    }
    int total;
    int pos = written + block_exclusive_scan(flag, s_warp, total);
    if (flag && pos < kCellCap)
      out[pos] = static_cast<uint32_t>(relx + x) | (static_cast<uint32_t>(rely + y) << 12) | (static_cast<uint32_t>(v) << 24);
    written += total;
  }
  if (threadIdx.x == 0) cell_count[blockIdx.x] = min(written, kCellCap);
}

// ---- cell lists -> one candidate array in the reference's vToDistributeKeys order (level, cell row, cell col)
__global__ void k_scan_cells(OrbLevelTable t, int ncells, const int* __restrict__ cell_count, int* __restrict__ cell_offset,
                             int* __restrict__ level_offsets) {
  // single block of 256 threads, ncells < 2048: eight consecutive cells per thread, warp + block scan of the partial sums
  __shared__ int s[2049];
  __shared__ int wsum[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int v[8], sum = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = tid * 8 + k;
    v[k] = i < ncells ? cell_count[i] : 0;
    sum += v[k];
  }
  int inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int x = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += x;
  }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  int base = 0;
  for (int w = 0; w < warp; ++w) base += wsum[w];
  int run = base + inc - sum;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int i = tid * 8 + k;
    if (i <= 2048) s[i] = run;
    run += v[k];
  }
  if (tid == 255) s[2048] = run;
  __syncthreads();
  for (int i = tid; i <= ncells; i += blockDim.x) cell_offset[i] = s[i];
  if (tid <= t.nlevels) {
    const int l = tid;
    level_offsets[l] = l < t.nlevels ? s[t.lv[l].cell_begin] : s[ncells];
  }
}

__global__ void k_gather_cells(const int* __restrict__ cell_count, const int* __restrict__ cell_offset,
                               const uint32_t* __restrict__ cell_items, uint32_t* __restrict__ cand, int cand_cap) {
  int n = cell_count[blockIdx.x], off = cell_offset[blockIdx.x];
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (off + i < cand_cap) cand[off + i] = cell_items[static_cast<size_t>(blockIdx.x) * kCellCap + i];
}

// ---- cv::GaussianBlur(7x7, sigma 2, REFLECT_101) on 8-bit: 8.8 fixed-point kernel [18 34 48 56 48 34 18],
// exact integer accumulation over both passes, one final rounding (v + 2^15) >> 16.  The 19-px reflected
// border of the pyramid buffer supplies the 3-px halo.  Output is the borderless w*h plane the reference
// blurs (`mvImagePyramid[level].clone()`, ORBextractor.cc:1060-1062).
// One thread = four horizontally adjacent pixels: 10 bytes per source row serve four 7-tap row sums.
__global__ void k_blur(const uint8_t* __restrict__ pyr, uint8_t* __restrict__ blur, OrbLevelTable t) {
  ORB_PDL_PROLOGUE();
  const OrbLevel lv = t.lv[blockIdx.y];
  const int wq = (lv.w + 3) >> 2;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= wq * lv.h) return;
  const int x = (i % wq) * 4, y = i / wq;
  const int g[7] = {18, 34, 48, 56, 48, 34, 18};
  // columns x-3 .. x+6 exist in the bordered buffer for every x < w (19-px border), also for the ragged last quad
  const uint8_t* c = pyr + lv.img_off + static_cast<size_t>(y + kEdge - 3) * lv.pitch + x + kEdge - 3;
  unsigned acc[4] = {0, 0, 0, 0};
#pragma unroll
  for (int ky = 0; ky < 7; ++ky) {
    unsigned v[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) v[k] = c[k];
#pragma unroll
    for (int o = 0; o < 4; ++o) {
      unsigned r = 0;
#pragma unroll
      for (int kx = 0; kx < 7; ++kx) r += g[kx] * v[o + kx];
      acc[o] += g[ky] * r;
    }
    c += lv.pitch;
  }
  uint8_t* d = blur + lv.flat_off + static_cast<size_t>(y) * lv.w + x;
#pragma unroll
  for (int o = 0; o < 4; ++o)
    if (x + o < lv.w) d[o] = static_cast<uint8_t>((acc[o] + 32768u) >> 16);
}

// ---- cv::fastAtan2 (degrees): 7th-order odd polynomial in float32 without FMA contraction.
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {
  const float scale = static_cast<float>(180.0 / 3.141592653589793238462643383279502884);
  const float p1 = __fmul_rn(0.9997878412794807f, scale), p3 = __fmul_rn(-0.3258083974640975f, scale),
              p5 = __fmul_rn(0.1555786518463281f, scale), p7 = __fmul_rn(-0.04432655554792128f, scale);
  const float eps = 2.220446049250313e-16f;
  float ax = fabsf(x), ay = fabsf(y), a, c, c2;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, eps));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, eps));
    c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0.f) a = __fsub_rn(180.f, a);
  if (y < 0.f) a = __fsub_rn(360.f, a);
  return a;
}

// ---- one warp per keypoint: IC_Angle (ORBextractor.cc:75-100) then computeOrbDescriptor (:104-150).
// Device-tree form (sel_packed != nullptr): the per-level selections of k_distribute are concatenated level-major on the fly --
// every warp derives the level offsets from the eight counts -- and the finished keypoint record is written here
// (ComputeKeyPointsOctTree :824-835, operator() :1071-1078), so no separate pass builds the OrbSelected list.
__global__ void k_describe(const uint8_t* __restrict__ pyr, const uint8_t* __restrict__ blur, OrbLevelTable t,
                           const OrbSelected* __restrict__ sel, int n, const int* __restrict__ umax,
                           float* __restrict__ angles, uint8_t* __restrict__ desc, const uint32_t* __restrict__ sel_packed,
                           const int* __restrict__ level_count, OrbTreeParams prm, sivo_keypoint* __restrict__ kps,
                           int* __restrict__ n_out, long long* __restrict__ n_out_i64, int* __restrict__ out_error) {
  ORB_PDL_PROLOGUE();
  int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  OrbSelected kp;
  uint32_t packed = 0;
  if (sel_packed) {
    int off = 0, lvl = -1, idx = 0;
    for (int l = 0; l < t.nlevels; ++l) {
      const int c = level_count[l];
      if (lvl < 0 && wid < off + c) { lvl = l; idx = wid - off; }
      off += c;
    }
    const bool too_many = off > n;  // n = capacity of the output buffers
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      if (too_many) atomicOr(out_error, 1 << 30);
      *n_out = too_many ? 0 : off;
      if (n_out_i64) *n_out_i64 = too_many ? 0 : off;
    }
    if (too_many || lvl < 0) return;
    packed = sel_packed[lvl * kTreeSelCap + idx];
    kp.x = static_cast<short>(static_cast<int>(packed & 0xFFF) + prm.min_b);
    kp.y = static_cast<short>(static_cast<int>((packed >> 12) & 0xFFF) + prm.min_b);
    kp.level = static_cast<short>(lvl);
    kp.pad = 0;
  } else {
    if (wid >= n) return;
    kp = sel[wid];
  }
  const OrbLevel lv = t.lv[kp.level];
  // intensity centroid over the radius-15 disc: lane = row v + 15
  int m10 = 0, m01 = 0;
  if (lane < 2 * kHalfPatch + 1) {
    int v = lane - kHalfPatch;
    int d = umax[abs(v)];
    const uint8_t* row = pyr + lv.img_off + static_cast<size_t>(kp.y + v + kEdge) * lv.pitch + kp.x + kEdge;
    int sum = 0;
    for (int u = -d; u <= d; ++u) {
      int val = row[u];
      m10 += u * val;
      sum += val;
    }
    m01 = v * sum;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    m10 += __shfl_xor_sync(0xffffffffu, m10, o);
    m01 += __shfl_xor_sync(0xffffffffu, m01, o);
  }
  const float angle = fast_atan2_deg(static_cast<float>(m01), static_cast<float>(m10));
  if (lane == 0) {
    if (sel_packed) {
      sivo_keypoint o;
      o.x = static_cast<float>(kp.x);
      o.y = static_cast<float>(kp.y);
      if (kp.level != 0) { o.x = __fmul_rn(o.x, prm.scale[kp.level]); o.y = __fmul_rn(o.y, prm.scale[kp.level]); }
      o.size = prm.size[kp.level];
      o.angle = angle;
      o.response = static_cast<float>(packed >> 24);
      o.octave = kp.level;
      o.class_id = -1;
      kps[wid] = o;
    } else {
      angles[wid] = angle;
    }
  }
  // rotated BRIEF: lane = descriptor byte
  const float factor_pi = static_cast<float>(3.141592653589793238462643383279502884 / 180.f);
  const float ang = __fmul_rn(angle, factor_pi);
  const float a = static_cast<float>(cos(static_cast<double>(ang)));
  const float b = static_cast<float>(sin(static_cast<double>(ang)));
  const uint8_t* img = blur + lv.flat_off;
  const int npx = lv.w * lv.h;
  int val = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int8_t* pt = c_pattern + (lane * 8 + k) * 4;
    int tv[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      float px = static_cast<float>(pt[2 * q]), py = static_cast<float>(pt[2 * q + 1]);
      int ry = __float2int_rn(__fadd_rn(__fmul_rn(px, b), __fmul_rn(py, a)));
      int rx = __float2int_rn(__fsub_rn(__fmul_rn(px, a), __fmul_rn(py, b)));
      int idx = (kp.y + ry) * lv.w + kp.x + rx;  // flat index into the continuous clone, as the reference computes it
      tv[q] = (idx >= 0 && idx < npx) ? img[idx] : 0;
    }
    val |= (tv[0] < tv[1]) << k;
  }
  desc[static_cast<size_t>(wid) * 32 + lane] = static_cast<uint8_t>(val);
}

}  // namespace

void orb_upload_pattern() { SIVO_CUDA(cudaMemcpyToSymbol(c_pattern, h_pattern, sizeof(h_pattern))); }

void orb_launch_pyramid(const uint8_t* gray, int rows, int cols, size_t gray_pitch, uint8_t* pyr, const OrbLevelTable& t,
                        cudaStream_t s) {
  (void)rows; (void)cols;
  for (int l = 0; l < t.nlevels; ++l) {
    const OrbLevel& lv = t.lv[l];
    dim3 grid(ceil_div(lv.w + 2 * kEdge, 128), lv.h + 2 * kEdge);
    if (l == 0) orb_launch_pdl(k_level0, grid, dim3(128), 0, s, gray, gray_pitch, pyr, lv);
    else orb_launch_pdl(k_resize, grid, dim3(128), 0, s, pyr, t.lv[l - 1], lv);
  }
  SIVO_CUDA(cudaGetLastError());
}

void orb_launch_score(const uint8_t* pyr, uint8_t* score, const OrbLevelTable& t, int t_min, cudaStream_t s) {
  dim3 grid(ceil_div(t.lv[0].w * t.lv[0].h, 128), t.nlevels);
  k_fast_score<<<grid, 128, 0, s>>>(pyr, score, t, t_min);
  SIVO_CUDA(cudaGetLastError());
}

void orb_launch_cells(const uint8_t* score, const uint8_t* pyr, const OrbLevelTable& t, const OrbCell* cells, int ncells, int ini_th,
                      int min_th, int* cell_count, uint32_t* cell_items, cudaStream_t s) {
  if (ncells == 0) return;
  orb_launch_pdl(k_cells, dim3(ncells), dim3(kCellThreads), 0, s, score, pyr, t, cells, ini_th, min_th, cell_count, cell_items);
  SIVO_CUDA(cudaGetLastError());
}

void orb_launch_compact(const OrbLevelTable& t, const OrbCell* cells, int ncells, const int* cell_count,
                        const uint32_t* cell_items, int* cell_offset, int* level_offsets, uint32_t* cand, int cand_cap,
                        cudaStream_t s) {
  (void)cells;
  if (ncells >= 2047) fail(SIVO_EINVAL, "image too large: %d FAST cells", ncells);
  k_scan_cells<<<1, 256, 0, s>>>(t, ncells, cell_count, cell_offset, level_offsets);
  if (ncells) k_gather_cells<<<ncells, 128, 0, s>>>(cell_count, cell_offset, cell_items, cand, cand_cap);
  SIVO_CUDA(cudaGetLastError());
}

void orb_launch_blur(const uint8_t* pyr, uint8_t* blur, const OrbLevelTable& t, cudaStream_t s) {
  dim3 grid(ceil_div(((t.lv[0].w + 3) / 4) * t.lv[0].h, 128), t.nlevels);
  orb_launch_pdl(k_blur, grid, dim3(128), 0, s, pyr, blur, t);
  SIVO_CUDA(cudaGetLastError());
}

void orb_launch_describe(const uint8_t* pyr, const uint8_t* blur, const OrbLevelTable& t, const OrbSelected* sel, int n,
                         const int* umax, float* angles, uint8_t* desc, cudaStream_t s) {
  if (n == 0) return;
  k_describe<<<ceil_div(n * 32, 128), 128, 0, s>>>(pyr, blur, t, sel, n, umax, angles, desc, nullptr, nullptr, OrbTreeParams{}, nullptr, nullptr, nullptr, nullptr);
  SIVO_CUDA(cudaGetLastError());
}

void orb_launch_describe_dev(const uint8_t* pyr, const uint8_t* blur, const OrbLevelTable& t, const uint32_t* sel_packed,
                             const int* level_count, const OrbTreeParams& prm, int cap, const int* umax, sivo_keypoint* kps,
                             uint8_t* desc, int* n_out, long long* n_out_i64, int* error, cudaStream_t s) {
  if (cap == 0) return;
  orb_launch_pdl(k_describe, dim3(ceil_div(cap * 32, 128)), dim3(128), 0, s, pyr, blur, t, static_cast<const OrbSelected*>(nullptr), cap, umax,
                 static_cast<float*>(nullptr), desc, sel_packed, level_count, prm, kps, n_out, n_out_i64, error);
  SIVO_CUDA(cudaGetLastError());
}

}  // namespace sivo
