// Optimizer::PoseOptimization (Optimizer.cc:273-491) with the g2o Levenberg-Marquardt it runs, and its marginal covariance
// (computeMarginals -> MarginalCovarianceCholesky).  The rules and the reference facts kept are spelled out in
// include/sivo_b200.h and oracle/pose_oracle.py.  This file is compiled with -fmad=false: every float / double intermediate is
// the correctly rounded result of the operation as written.
//
//   k_pose_optimize  one CTA per problem (grid 1 for Tracking's calls), resident for the whole call: 4 rounds x <= 10 iterations
//                    x <= 10 trials.  Threads own edges (edge e on thread e % 256) and compute the error, chi2 and Huber weights,
//                    plus the Jacobian and the 21 + 6 partial sums of H and b on linearisation passes; the block reduces them in
//                    a fixed tree (pose_reduce), in double.  Thread 0 factors the damped 6 x 6 system (LL^T), applies the exp
//                    update, keeps the lambda / rho bookkeeping and hands the pose to the block through shared memory.
//   k_pose_system    the same setup and one linearisation pass (test hook).
//   k_pose_gather    xw[j] = points[match[j]].pos for the semantic keys with a match.
#include <cfloat>
#include <cmath>

#include "block_ops.cuh"
#include "frame_ops.h"
#include "host_call.h"
#include "stream_scratch.h"

namespace sivo {
namespace {
constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int kTerms = 28;  // 21 upper entries of H (row by row), 6 of g (b = -g), the robust chi2
constexpr int kRounds = 4, kIterations = 10, kMaxTrials = 10;

struct PoseParams {
  double fx, fy, cx, cy, bf;
  float inv_sigma2[kOrbMaxLevels];
  int nlevels;
};

struct PoseEdge {  // one edge, in semantic-key order (80 bytes)
  double X[3], obs[3], info, chi2;
  int key, stereo, outlier, pad;
};

struct DPose { double q[4], t[3]; };  // SE3Quat: q = (x, y, z, w)

size_t edges_bytes(int cap) { return static_cast<size_t>(std::max(cap, 1)) * sizeof(PoseEdge); }

// ---- SE3Quat and Eigen 3's quaternion formulas
__device__ void normalize_rotation(double* q) {
  if (q[3] < 0) for (int i = 0; i < 4; ++i) q[i] = -q[i];
  const double n2 = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3];
  if (n2 > 0) {
    const double n = sqrt(n2);
    for (int i = 0; i < 4; ++i) q[i] = q[i] / n;
  }
}

__device__ void quat_from_matrix(const double (&m)[3][3], double* q) {
  double t = (m[0][0] + m[1][1]) + m[2][2];
  if (t > 0) {
    t = sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[2][1] - m[1][2]) * t;
    q[1] = (m[0][2] - m[2][0]) * t;
    q[2] = (m[1][0] - m[0][1]) * t;
  } else {
    int i = 0;
    if (m[1][1] > m[0][0]) i = 1;
    if (m[2][2] > m[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(((m[i][i] - m[j][j]) - m[k][k]) + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m[k][j] - m[j][k]) * t;
    q[j] = (m[j][i] + m[i][j]) * t;
    q[k] = (m[k][i] + m[i][k]) * t;
  }
}

__device__ __forceinline__ void cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

// Eigen's q * v: uv = q.vec x v; uv += uv; v + w uv + q.vec x uv
__device__ __forceinline__ void transform(const double* q, const double* v, double* out) {
  double uv[3], c[3];
  cross(q, v, uv);
  for (int i = 0; i < 3; ++i) uv[i] = uv[i] + uv[i];
  cross(q, uv, c);
  for (int i = 0; i < 3; ++i) out[i] = (v[i] + q[3] * uv[i]) + c[i];
}

__device__ void rotation_matrix(const double* q, double (&r)[3][3]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  r[0][0] = 1.0 - (tyy + tzz); r[0][1] = txy - twz; r[0][2] = txz + twy;
  r[1][0] = txy + twz; r[1][1] = 1.0 - (txx + tzz); r[1][2] = tyz - twx;
  r[2][0] = txz - twy; r[2][1] = tyz + twx; r[2][2] = 1.0 - (txx + tyy);
}

// Converter::toSE3Quat of the float 3 x 4 pose
__device__ void to_se3quat(const float* T, DPose& P) {
  double m[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) m[r][c] = T[4 * r + c];
  quat_from_matrix(m, P.q);
  normalize_rotation(P.q);
  for (int r = 0; r < 3; ++r) P.t[r] = T[4 * r + 3];
}

__device__ __forceinline__ void mat3(const double (&a)[3][3], const double (&b)[3][3], double (&c)[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c[i][j] = (a[i][0] * b[0][j] + a[i][1] * b[1][j]) + a[i][2] * b[2][j];
}

// VertexSE3Expmap::oplusImpl: SE3Quat::exp(d) * T.  kTrace: tv = (theta, sin theta, cos theta, pow(theta, 3)), the last three
// written only when the theta >= 1e-5 branch calls them.
template <bool kTrace = false>
__device__ void oplus(const double* d, const DPose& T, DPose& out, double* tv = nullptr) {
  const double theta = sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
  const double O[3][3] = {{0.0, -d[2], d[1]}, {d[2], 0.0, -d[0]}, {-d[1], d[0], 0.0}};
  double O2[3][3], R[3][3], V[3][3];
  mat3(O, O, O2);
  if (theta < 0.00001) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) R[i][j] = V[i][j] = ((i == j ? 1.0 : 0.0) + O[i][j]) + O2[i][j];
  } else {
    const double s = sin(theta), c = cos(theta);
    const double a = s / theta, b = (1 - c) / (theta * theta), e = (theta - s) / pow(theta, 3.0);
    if constexpr (kTrace) { tv[1] = s; tv[2] = c; tv[3] = pow(theta, 3.0); }  // pow is a pure function: the value e used
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const double id = i == j ? 1.0 : 0.0;
        R[i][j] = (id + a * O[i][j]) + b * O2[i][j];
        V[i][j] = (id + b * O[i][j]) + e * O2[i][j];
      }
  }
  if constexpr (kTrace) tv[0] = theta;
  double eq[4], et[3];
  quat_from_matrix(R, eq);
  normalize_rotation(eq);
  for (int i = 0; i < 3; ++i) et[i] = (V[i][0] * d[3] + V[i][1] * d[4]) + V[i][2] * d[5];
  // SE3Quat::operator*: t = exp.t + exp.q * T.t, q = exp.q * T.q (quat_product), normalised
  double tt[3];
  transform(eq, T.t, tt);
  for (int i = 0; i < 3; ++i) out.t[i] = et[i] + tt[i];
  const double *a = eq, *b = T.q;
  out.q[0] = ((a[3] * b[0] + a[0] * b[3]) + a[1] * b[2]) - a[2] * b[1];
  out.q[1] = ((a[3] * b[1] + a[1] * b[3]) + a[2] * b[0]) - a[0] * b[2];
  out.q[2] = ((a[3] * b[2] + a[2] * b[3]) + a[0] * b[1]) - a[1] * b[0];
  out.q[3] = ((a[3] * b[3] - a[0] * b[0]) - a[1] * b[1]) - a[2] * b[2];
  normalize_rotation(out.q);
}

// ---- one edge at a pose: computeError, chi2, RobustKernelHuber, linearizeOplus
struct EdgeEval {
  double e[3], chi2, rho0, rho1;
  bool valid;
};

template <bool kJacobian>
__device__ __forceinline__ EdgeEval eval_edge(const PoseEdge& E, const DPose& T, const PoseParams& p, bool robust, double (&J)[3][6]) {
  EdgeEval o;
  double P[3];
  transform(T.q, E.X, P);
  const double x = P[0] + T.t[0], y = P[1] + T.t[1], z = P[2] + T.t[2];
  if (E.stereo) {
    const double invz_f = static_cast<float>(1.0 / z);  // `const float invz = 1.0f / trans_xyz[2]`
    const double u = (x * invz_f) * p.fx + p.cx, v = (y * invz_f) * p.fy + p.cy;
    o.e[0] = E.obs[0] - u;
    o.e[1] = E.obs[1] - v;
    o.e[2] = E.obs[2] - (u - p.bf * invz_f);
  } else {
    o.e[0] = E.obs[0] - ((x / z) * p.fx + p.cx);
    o.e[1] = E.obs[1] - ((y / z) * p.fy + p.cy);
    o.e[2] = 0.0;
  }
  const double info = E.info;
  double chi2 = o.e[0] * (info * o.e[0]) + o.e[1] * (info * o.e[1]);
  if (E.stereo) chi2 = chi2 + o.e[2] * (info * o.e[2]);
  const double invz = 1.0 / z, invz_2 = invz * invz;
  o.valid = isfinite(chi2) && isfinite(invz_2);  // the NaN rule
  o.chi2 = o.valid ? chi2 : __longlong_as_double(0x7ff8000000000000ll);
  o.rho0 = o.chi2;
  o.rho1 = 1.0;
  if (robust) {
    const double delta = E.stereo ? static_cast<double>(sqrtf(7.815f)) : static_cast<double>(sqrtf(5.991f));
    const double dsqr = delta * delta;
    if (!(o.chi2 <= dsqr)) {
      const double sqrte = sqrt(o.chi2);
      o.rho0 = (2 * sqrte) * delta - dsqr;
      o.rho1 = delta / sqrte;
    }
  }
  if (kJacobian) {
    const double fx = p.fx, fy = p.fy, bf = p.bf;
    J[0][0] = ((x * y) * invz_2) * fx;
    J[0][1] = (-(1 + ((x * x) * invz_2))) * fx;
    J[0][2] = (y * invz) * fx;
    J[0][3] = (-invz) * fx;
    J[0][4] = 0.0;
    J[0][5] = (x * invz_2) * fx;
    J[1][0] = (1 + ((y * y) * invz_2)) * fy;
    J[1][1] = (((-x) * y) * invz_2) * fy;
    J[1][2] = ((-x) * invz) * fy;
    J[1][3] = 0.0;
    J[1][4] = (-invz) * fy;
    J[1][5] = (y * invz_2) * fy;
    if (E.stereo) {
      J[2][0] = J[0][0] - ((bf * y) * invz_2);
      J[2][1] = J[0][1] + ((bf * x) * invz_2);
      J[2][2] = J[0][2];
      J[2][3] = J[0][3];
      J[2][4] = 0.0;
      J[2][5] = J[0][5] - (bf * invz_2);
    } else {
      for (int k = 0; k < 6; ++k) J[2][k] = 0.0;
    }
  }
  return o;
}

// constructQuadraticForm's terms: h[k][l] = sum_i (A[i][k] w) A[i][l] (w = rho1 info), g[k] = sum_i ((rho1 A[i][k]) info) e[i]
__device__ __forceinline__ void add_terms(const PoseEdge& E, const EdgeEval& o, const double (&J)[3][6], double (&acc)[kTerms]) {
  const double w = o.rho1 * E.info;
  int q = 0;
#pragma unroll
  for (int k = 0; k < 6; ++k)
#pragma unroll
    for (int l = k; l < 6; ++l, ++q) {
      double s = (J[0][k] * w) * J[0][l] + (J[1][k] * w) * J[1][l];
      if (E.stereo) s = s + (J[2][k] * w) * J[2][l];
      acc[q] = acc[q] + s;
    }
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    double s = ((o.rho1 * J[0][k]) * E.info) * o.e[0] + ((o.rho1 * J[1][k]) * E.info) * o.e[1];
    if (E.stereo) s = s + ((o.rho1 * J[2][k]) * E.info) * o.e[2];
    acc[21 + k] = acc[21 + k] + s;
  }
  acc[27] = acc[27] + o.rho0;
}

// The fixed reduction tree (block_ops.cuh) over the per-thread sums (above).  out[q] is valid after the call (it ends with
// __syncthreads).
template <int M>
__device__ void pose_reduce(double (&v)[M], double (*sh)[kTerms], double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < M; ++q) v[q] = warp_tree_sum(v[q]);
  if (lane == 0)
#pragma unroll
    for (int q = 0; q < M; ++q) sh[warp][q] = v[q];
  __syncthreads();
  if (threadIdx.x < M) {
    double w[kWarps];
    for (int i = 0; i < kWarps; ++i) w[i] = sh[i][threadIdx.x];
    out[threadIdx.x] = fold_warp_totals<kWarps>(w);
  }
  __syncthreads();
}

// ---- dense 6 x 6: LL^T in natural order (false when a pivot is not > 0), the two triangular solves, the marginal recursion
__device__ bool cholesky6(const double (&A)[6][6], double (&L)[6][6]) {
  for (int j = 0; j < 6; ++j) {
    double d = A[j][j];
    for (int k = 0; k < j; ++k) d = d - L[j][k] * L[j][k];
    if (!(d > 0)) return false;
    L[j][j] = sqrt(d);
    for (int i = j + 1; i < 6; ++i) {
      double s = A[i][j];
      for (int k = 0; k < j; ++k) s = s - L[i][k] * L[j][k];
      L[i][j] = s / L[j][j];
    }
  }
  return true;
}

__device__ void cholesky6_solve(const double (&L)[6][6], const double* b, double* x) {
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s = s - L[i][k] * y[k];
    y[i] = s / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double s = y[i];
    for (int k = i + 1; k < 6; ++k) s = s - L[k][i] * x[k];
    x[i] = s / L[i][i];
  }
}

// MarginalCovarianceCholesky::computeEntry for every (r <= c), by decreasing c then decreasing r (its sort order)
__device__ void marginal6(const double (&L)[6][6], double* sigma) {
  double C[6][6], diag[6];
  for (int r = 0; r < 6; ++r) diag[r] = 1.0 / L[r][r];
  for (int c = 5; c >= 0; --c)
    for (int r = c; r >= 0; --r) {
      double s = 0.;
      for (int rr = r + 1; rr < 6; ++rr) s += (rr < c ? C[rr][c] : C[c][rr]) * L[rr][r];
      C[r][c] = r == c ? diag[r] * (diag[r] - s) : -s * diag[r];
    }
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) sigma[6 * r + c] = r <= c ? C[r][c] : C[c][r];
}

// ---- setup shared by both kernels: the edges of the semantic keys with a map point, compacted in key order
__device__ int build_edges(const PoseParams& p, const sivo_keypoint* __restrict__ kps, const int* __restrict__ keep_idx, int n, int cap,
                           const float* __restrict__ u_right, const float* __restrict__ xw, const uint8_t* __restrict__ level1,
                           PoseEdge* __restrict__ edges, int* warp_count) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int total = 0;
  for (int base = 0; base < n; base += kThreads) {
    const int j = base + threadIdx.x;
    PoseEdge E;
    bool ok = false;
    if (j < n) {
      const int k = keep_idx ? keep_idx[j] : j;
      if (k >= 0 && k < cap) {
        const sivo_keypoint kp = kps[k];
        const float X0 = xw[3 * j];
        if (!isnan(X0) && kp.octave >= 0 && kp.octave < p.nlevels) {
          ok = true;
          const float ur = u_right[j];
          E.stereo = !(ur < 0.f);
          E.X[0] = X0; E.X[1] = xw[3 * j + 1]; E.X[2] = xw[3 * j + 2];
          E.obs[0] = kp.x; E.obs[1] = kp.y; E.obs[2] = E.stereo ? static_cast<double>(ur) : 0.0;
          E.info = p.inv_sigma2[kp.octave];
          E.chi2 = __longlong_as_double(0x7ff8000000000000ll);
          E.key = j;
          E.outlier = level1 ? (level1[j] != 0) : 0;
          E.pad = 0;
        }
      }
    }
    // block_rank (block_ops.cuh) written out with `warp` computed once, outside the loop: on block_rank, which computes it per
    // chunk, k_pose_optimize needs two more registers
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) warp_count[warp] = __popc(m);
    __syncthreads();
    int before = total;
    for (int w = 0; w < warp; ++w) before += warp_count[w];
    if (ok) edges[before + __popc(m & ((1u << lane) - 1u))] = E;
    for (int w = 0; w < kWarps; ++w) total += warp_count[w];
    __syncthreads();
  }
  return total;
}

struct PoseShared {
  double red[kWarps][kTerms];
  double sum[kTerms];
  double H[6][6], b[6], x[6];
  DPose in, cur, trial;
  double lam, ni, current, rho;
  int ok2, go, n_active, n_bad, warp_count[kWarps];
};

// A linearisation pass (computeActiveErrors + activeRobustChi2 + buildSystem) over the active edges at s.cur, into s.H / s.b /
// s.current; each active edge keeps its chi2.
__device__ void linearise(const PoseParams& p, PoseEdge* edges, int ne, bool robust_stereo, PoseShared& s) {
  double acc[kTerms];
#pragma unroll
  for (int q = 0; q < kTerms; ++q) acc[q] = 0.0;
  const DPose T = s.cur;
  for (int e = threadIdx.x; e < ne; e += kThreads) {
    PoseEdge E = edges[e];
    if (E.outlier) continue;
    double J[3][6];
    const EdgeEval o = eval_edge<true>(E, T, p, !E.stereo || robust_stereo, J);
    edges[e].chi2 = o.chi2;
    if (o.valid) add_terms(E, o, J, acc);
  }
  pose_reduce(acc, s.red, s.sum);
  if (threadIdx.x == 0) {
    int q = 0;
    for (int k = 0; k < 6; ++k)
      for (int l = k; l < 6; ++l, ++q) s.H[k][l] = s.H[l][k] = s.sum[q];
    for (int k = 0; k < 6; ++k) s.b[k] = -s.sum[21 + k];
    s.current = s.sum[27];
  }
  __syncthreads();
}

// An error pass (computeActiveErrors + activeRobustChi2) at s.trial; returns the robust chi2 on every thread.
__device__ double error_pass(const PoseParams& p, PoseEdge* edges, int ne, bool robust_stereo, PoseShared& s) {
  double acc[1] = {0.0};
  const DPose T = s.trial;
  double J[3][6];
  for (int e = threadIdx.x; e < ne; e += kThreads) {
    const PoseEdge& E = edges[e];
    if (E.outlier) continue;
    const EdgeEval o = eval_edge<false>(E, T, p, !E.stereo || robust_stereo, J);
    edges[e].chi2 = o.chi2;
    if (o.valid) acc[0] = acc[0] + o.rho0;
  }
  pose_reduce(acc, s.red, s.sum);
  return s.sum[0];
}

__device__ void write_pose(const float* T, const DPose& P, sivo_pose_result* r) {
  for (int i = 0; i < 12; ++i) r->Tcw[i] = T[i];
  for (int i = 0; i < 4; ++i) r->q[i] = P.q[i];
  for (int i = 0; i < 3; ++i) r->t[i] = P.t[i];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) {
      r->Rcw[3 * i + j] = T[4 * i + j];
      r->Rwc[3 * j + i] = T[4 * i + j];
    }
    r->tcw[i] = T[4 * i + 3];
  }
  // Frame::UpdatePoseMatrices: mOw = -mRcw^T mtcw (cv::gemm: the three products summed in double, rounded to float)
  for (int c = 0; c < 3; ++c) {
    double a = static_cast<double>(T[c]) * T[3];
    a = a + static_cast<double>(T[4 + c]) * T[7];
    a = a + static_cast<double>(T[8 + c]) * T[11];
    r->Ow[c] = -static_cast<float>(a);
  }
}

// Converter::toCvMat of the estimate: toRotationMatrix and t rounded to float, then write_pose
__device__ void write_estimate(const DPose& P, sivo_pose_result* r) {
  double R[3][3];
  rotation_matrix(P.q, R);
  float T[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[4 * i + j] = static_cast<float>(R[i][j]);
    T[4 * i + 3] = static_cast<float>(P.t[i]);
  }
  write_pose(T, P, r);
}

// Thread 0's record stream of the traced kernel (sivo_dbg_pose_trace): records past the caller's capacity are counted, not written.
struct Tracer {
  sivo_pose_trace_rec* rec;
  int cap, n;
  __device__ sivo_pose_trace_rec* add(int kind, int round, int it, int trial) {
    sivo_pose_trace_rec* r = n < cap ? rec + n : nullptr;
    ++n;
    if (r) {
      *r = sivo_pose_trace_rec{};
      r->kind = kind; r->round = round; r->iteration = it; r->trial = trial;
    }
    return r;
  }
  __device__ void call(int kind, int round, int it, int trial, double arg, double value) {
    if (sivo_pose_trace_rec* r = add(kind, round, it, trial)) { r->arg = arg; r->value = value; }
  }
};

// kTrace (sivo_dbg_pose_trace): thread 0 also appends its records to trace (trace_cap of them) and writes their count to
// *trace_count; the production instantiation ignores the three.
template <bool kTrace>
__global__ void __launch_bounds__(kThreads, 1)
    k_pose_optimize(const PoseParams p, const sivo_keypoint* __restrict__ kps, const int* __restrict__ keep_idx,
                    const long long* __restrict__ n_keep, int cap, const float* __restrict__ u_right, const float* __restrict__ xw,
                    const float* Tcw_in, PoseEdge* __restrict__ edges_all, sivo_pose_result* results,
                    uint8_t* __restrict__ outlier_all, sivo_pose_trace_rec* trace, int trace_cap, int* trace_count) {
  __shared__ PoseShared s;
  Tracer tr{trace, trace_cap, 0};
  double lam0 = 0.0, ni0 = 0.0, cur0 = 0.0;
  // Tcw_in may be the Tcw of *results (an in-place update): it is read into shared memory before anything is written to results.
  // problem blockIdx.x: its keys, points and outputs at stride cap (a batch of problems is a grid size away)
  const int prob = blockIdx.x;
  if (keep_idx) keep_idx += static_cast<size_t>(prob) * cap;
  u_right += static_cast<size_t>(prob) * cap;
  xw += static_cast<size_t>(prob) * cap * 3;
  Tcw_in += 12 * prob;
  PoseEdge* edges = edges_all + static_cast<size_t>(prob) * cap;
  uint8_t* outlier = outlier_all ? outlier_all + static_cast<size_t>(prob) * cap : nullptr;
  sivo_pose_result* res = results + prob;
  const int tid = threadIdx.x;
  const int n = clamp_count(n_keep[prob], cap);
  if (n < 0) {
    if (tid == 0) res->n_good = -1;
    return;
  }
  if (outlier)
    for (int j = tid; j < n; j += kThreads) outlier[j] = 0;
  const int ne = build_edges(p, kps, keep_idx, n, cap, u_right, xw, nullptr, edges, s.warp_count);
  __shared__ float tin[12];
  if (tid < 12) tin[tid] = Tcw_in[tid];
  __syncthreads();
  if (tid == 0) {
    to_se3quat(tin, s.in);
    for (int i = 0; i < 6; ++i) s.x[i] = 0.0;
  }
  __syncthreads();
  if (ne < 3) {  // nInitialCorrespondences < 3: return 0, the pose untouched
    if (tid == 0) {
      write_pose(tin, s.in, res);
      for (int i = 0; i < 36; ++i) res->sigma_cw[i] = 0.0;
      res->sigma_valid = 0; res->n_initial = ne; res->n_bad = 0; res->n_good = 0; res->rounds_run = 0; res->reserved = 0;
    }
    return;
  }
  bool robust_stereo = true, have_h = false;
  int rounds = 0, n_bad = 0;
  for (int round = 0; round < kRounds; ++round) {
    if (tid == 0) { s.cur = s.in; s.n_active = 0; s.n_bad = 0; }
    __syncthreads();
    int mine = 0;
    for (int e = tid; e < ne; e += kThreads) mine += !edges[e].outlier;
    if (mine) atomicAdd(&s.n_active, mine);
    __syncthreads();
    have_h = s.n_active > 0;  // no level-0 edge: optimize() returns -1, the estimate stays the input pose
    for (int it = 0; have_h && it < kIterations; ++it) {
      linearise(p, edges, ne, robust_stereo, s);
      if (tid == 0) {
        if (it == 0) {  // computeLambdaInit
          double m = 0.0;
          for (int j = 0; j < 6; ++j) { const double a = fabs(s.H[j][j]); m = a < m ? m : a; }
          s.lam = 1e-5 * m;
          s.ni = 2.0;
        }
        s.rho = 0.0;
      }
      int qmax = 0;
      while (true) {
        if (tid == 0) {
          double A[6][6], L[6][6];
          for (int i = 0; i < 6; ++i)
            for (int j = 0; j < 6; ++j) A[i][j] = s.H[i][j];
          for (int j = 0; j < 6; ++j) A[j][j] = A[j][j] + s.lam;
          s.ok2 = cholesky6(A, L);
          if (s.ok2) cholesky6_solve(L, s.b, s.x);  // a failed factorisation leaves x as it was
          if constexpr (kTrace) {
            double tv[4];
            oplus<true>(s.x, s.cur, s.trial, tv);
            if (!(tv[0] < 0.00001)) {
              tr.call(SIVO_POSE_TRACE_SIN, round, it, qmax, tv[0], tv[1]);
              tr.call(SIVO_POSE_TRACE_COS, round, it, qmax, tv[0], tv[2]);
              tr.call(SIVO_POSE_TRACE_POW_THETA, round, it, qmax, tv[0], tv[3]);
            }
            lam0 = s.lam;
            ni0 = s.ni;
          } else {
            oplus(s.x, s.cur, s.trial);
          }
        }
        __syncthreads();
        const double temp_computed = error_pass(p, edges, ne, robust_stereo, s);
        if (tid == 0) {
          const double temp = s.ok2 ? temp_computed : DBL_MAX;
          double rho = s.current - temp, scale = 0.;
          for (int j = 0; j < 6; ++j) scale += s.x[j] * (s.lam * s.x[j] + s.b[j]);
          scale += 1e-3;
          rho /= scale;
          s.go = 1;
          if constexpr (kTrace) cur0 = s.current;
          if (rho > 0 && isfinite(temp)) {
            double alpha = 1. - pow((2 * rho - 1), 3.0);
            if constexpr (kTrace) tr.call(SIVO_POSE_TRACE_POW_RHO, round, it, qmax, 2 * rho - 1, pow((2 * rho - 1), 3.0));
            alpha = (2. / 3.) < alpha ? (2. / 3.) : alpha;
            s.lam *= (1. / 3.) < alpha ? alpha : (1. / 3.);
            s.ni = 2;
            s.current = temp;
            s.cur = s.trial;
          } else {
            s.lam *= s.ni;
            s.ni *= 2;
            if (!isfinite(s.lam)) s.go = 0;
          }
          s.rho = rho;
          if constexpr (kTrace) {
            if (sivo_pose_trace_rec* r = tr.add(SIVO_POSE_TRACE_TRIAL, round, it, qmax)) {
              r->ok2 = s.ok2; r->accepted = rho > 0 && isfinite(temp);
              r->current = cur0; r->temp = temp; r->rho = rho;
              r->lam_before = lam0; r->ni_before = ni0; r->lam_after = s.lam; r->ni_after = s.ni;
              for (int j = 0; j < 6; ++j) r->x[j] = s.x[j];
              for (int j = 0; j < 4; ++j) r->q[j] = s.trial.q[j];
              for (int j = 0; j < 3; ++j) r->t[j] = s.trial.t[j];
            }
          }
        }
        __syncthreads();
        if (!s.go) break;
        ++qmax;
        if (!(s.rho < 0 && qmax < kMaxTrials)) break;
      }
      const bool terminate = qmax == kMaxTrials || s.rho == 0 || !isfinite(s.lam);
      __syncthreads();
      if (terminate) break;
    }
    // classify the stereo edges: an outlier recomputes its error at the final estimate, an inlier keeps its last chi2
    {
      const DPose T = s.cur;
      double J[3][6];
      int bad = 0;
      for (int e = tid; e < ne; e += kThreads) {
        PoseEdge& E = edges[e];
        if (!E.stereo) continue;
        double chi2 = E.chi2;
        if (E.outlier) {
          chi2 = eval_edge<false>(E, T, p, robust_stereo, J).chi2;
          E.chi2 = chi2;
        }
        E.outlier = !(static_cast<float>(chi2) <= 7.815f);
        bad += E.outlier;
      }
      if (bad) atomicAdd(&s.n_bad, bad);
      __syncthreads();
      if (tid == 0) n_bad = s.n_bad;  // only thread 0 reads it: it alone resets it for the next round
    }
    if constexpr (kTrace)
      if (tid == 0)
        if (sivo_pose_trace_rec* r = tr.add(SIVO_POSE_TRACE_ROUND, round, -1, -1)) {
          r->n_active = s.n_active; r->n_bad = n_bad; r->robust_stereo = robust_stereo;
        }
    if (round == 2) robust_stereo = false;
    rounds = round + 1;
    if (ne < 10) break;
  }
  if (tid == 0) {
    double L[6][6];
    const bool valid = have_h && cholesky6(s.H, L);
    if (valid) marginal6(L, res->sigma_cw);
    else for (int i = 0; i < 36; ++i) res->sigma_cw[i] = 0.0;
    write_estimate(s.cur, res);
    res->sigma_valid = valid; res->n_initial = ne; res->n_bad = n_bad; res->n_good = ne - n_bad; res->rounds_run = rounds;
    res->reserved = 0;
    if constexpr (kTrace) *trace_count = tr.n;
  }
  if (outlier)
    for (int e = tid; e < ne; e += kThreads) outlier[edges[e].key] = static_cast<uint8_t>(edges[e].outlier);
}

// test hook: the setup and one linearisation pass at a given pose; per-key outputs (NaN for a key without an edge)
__global__ void __launch_bounds__(kThreads, 1)
    k_pose_system(const PoseParams p, const sivo_keypoint* __restrict__ kps, int n, const float* __restrict__ u_right,
                  const float* __restrict__ xw, const uint8_t* __restrict__ level1, const double* __restrict__ pose7, int robust_stereo,
                  PoseEdge* __restrict__ edges, double* __restrict__ err, double* __restrict__ chi2, double* __restrict__ rho,
                  double* __restrict__ jac, double* __restrict__ Hb) {
  __shared__ PoseShared s;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int j = threadIdx.x; j < n; j += kThreads) {
    for (int i = 0; i < 3; ++i) err[3 * j + i] = nan;
    chi2[j] = nan;
    rho[2 * j] = rho[2 * j + 1] = nan;
    for (int i = 0; i < 18; ++i) jac[18 * j + i] = nan;
  }
  const int ne = build_edges(p, kps, nullptr, n, n, u_right, xw, level1, edges, s.warp_count);
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) s.cur.q[i] = pose7[i];
    for (int i = 0; i < 3; ++i) s.cur.t[i] = pose7[4 + i];
  }
  __syncthreads();
  const DPose T = s.cur;
  for (int e = threadIdx.x; e < ne; e += kThreads) {
    const PoseEdge E = edges[e];
    double J[3][6];
    const EdgeEval o = eval_edge<true>(E, T, p, !E.stereo || robust_stereo, J);
    const int j = E.key;
    for (int i = 0; i < 3; ++i) err[3 * j + i] = o.e[i];
    chi2[j] = o.chi2;
    rho[2 * j] = o.rho0;
    rho[2 * j + 1] = o.rho1;
    for (int i = 0; i < 18; ++i) jac[18 * j + i] = J[i / 6][i % 6];
  }
  __syncthreads();
  linearise(p, edges, ne, robust_stereo, s);
  if (threadIdx.x == 0) {
    for (int i = 0; i < 36; ++i) Hb[i] = s.H[i / 6][i % 6];
    for (int i = 0; i < 6; ++i) Hb[36 + i] = s.b[i];
    Hb[42] = s.current;
  }
}

// test hook: per entry i, P = to_se3quat(T[i]), then oplus(d[i], P) as the trial step computes it, and its write_estimate
__global__ void k_pose_se3(int n, const float* __restrict__ T, const double* __restrict__ d, double* __restrict__ se3, double* __restrict__ up,
                           double* __restrict__ tv, sivo_pose_result* __restrict__ res) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float Ti[12];
  for (int k = 0; k < 12; ++k) Ti[k] = T[12 * i + k];
  double di[6];
  for (int k = 0; k < 6; ++k) di[k] = d[6 * i + k];
  DPose P, U;
  to_se3quat(Ti, P);
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  double t[4] = {nan, nan, nan, nan};
  oplus<true>(di, P, U, t);
  for (int k = 0; k < 4; ++k) { se3[7 * i + k] = P.q[k]; up[7 * i + k] = U.q[k]; tv[4 * i + k] = t[k]; }
  for (int k = 0; k < 3; ++k) { se3[7 * i + 4 + k] = P.t[k]; up[7 * i + 4 + k] = U.t[k]; }
  write_estimate(U, res + i);
}

__global__ void k_pose_gather(const int* __restrict__ match, const long long* __restrict__ n_keep, int cap,
                              const sivo_map_point* __restrict__ pts, int n_points, float* __restrict__ xw) {
  const int n = clamp_count(*n_keep, cap);
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int m = match[j];
  if (m < 0 || m >= n_points) return;
  for (int i = 0; i < 3; ++i) xw[3 * j + i] = pts[m].pos[i];
}

PoseParams make_params(const Orb& left, float fx, float fy, float cx, float cy, float mbf) {
  if (!(std::isfinite(fx) && fx > 0.f) || !(std::isfinite(fy) && fy > 0.f) || !(std::isfinite(mbf) && mbf > 0.f) || !std::isfinite(cx) ||
      !std::isfinite(cy))
    fail(SIVO_EINVAL, "pose: fx, fy and mbf must be finite and positive, cx and cy finite");
  PoseParams p{};
  p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy; p.bf = mbf;
  p.nlevels = left.nlevels();
  for (int l = 0; l < p.nlevels; ++l) p.inv_sigma2[l] = left.tables().inv_sigma2[l];
  return p;
}

void launch_optimize(const PoseParams& p, const sivo_keypoint* kps, const int* keep_idx, const long long* n_keep, int cap,
                     const float* u_right, const float* xw, const float* Tcw_in, PoseEdge* edges, sivo_pose_result* result,
                     uint8_t* outlier, cudaStream_t s) {
  k_pose_optimize<false><<<1, kThreads, 0, s>>>(p, kps, keep_idx, n_keep, cap, u_right, xw, Tcw_in, edges, result, outlier, nullptr, 0,
                                                nullptr);
  SIVO_CUDA(cudaGetLastError());
}

// the host forms refuse a key that has a point (xw not NaN) and an octave outside the extractor's levels
void check_octaves(const char* who, const sivo_keypoint* kps, const float* xw, int n, int nlevels) {
  for (int j = 0; j < n; ++j)
    if (!std::isnan(xw[3 * j]) && (kps[j].octave < 0 || kps[j].octave >= nlevels))
      fail(SIVO_ERANGE, "%s: key %d has octave %d", who, j, kps[j].octave);
}
}  // namespace

void pose_optimize_device(const Orb& left, const sivo_keypoint* kps, const int* keep_idx, const long long* n_keep, const float* u_right,
                          const float* xw, float fx, float fy, float cx, float cy, float mbf, const float* Tcw_in,
                          sivo_pose_result* result, uint8_t* outlier, cudaStream_t s) {
  const PoseParams p = make_params(left, fx, fy, cx, cy, mbf);
  s = left.enter(s);
  const int cap = left.capacity();
  StreamScratch sc(edges_bytes(cap), s);
  launch_optimize(p, kps, keep_idx, n_keep, cap, u_right, xw, Tcw_in, sc.take<PoseEdge>(std::max(cap, 1)), result, outlier, s);
}

void pose_gather_device(const Orb& left, const int* match, const long long* n_keep, const sivo_map_point* pts, int n_points, float* xw,
                        cudaStream_t s) {
  if (n_points < 0) fail(SIVO_EINVAL, "pose_gather: n_points = %d", n_points);
  s = left.enter(s);
  const int cap = left.capacity();
  k_pose_gather<<<ceil_div(std::max(cap, 1), kThreads), kThreads, 0, s>>>(match, n_keep, cap, pts, n_points, xw);
  SIVO_CUDA(cudaGetLastError());
}

// The host form: stage the gathered keys on the host-call workspace, run the device form's kernel, download.
void pose_optimize(const Orb& left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx, float fy, float cx,
                   float cy, float mbf, const float* Tcw_in, sivo_pose_result* result, uint8_t* outlier) {
  if (n < 0) fail(SIVO_EINVAL, "pose: n = %d", n);
  const PoseParams p = make_params(left, fx, fy, cx, cy, mbf);
  check_octaves("pose", kps, xw, n, p.nlevels);
  HostCall& hc = host_call();
  hc.begin(left.device());
  const sivo_keypoint* d_kps = hc.upload(kps, n);
  const float* d_ur = hc.upload(u_right, n);
  const float* d_xw = hc.upload(xw, 3 * static_cast<size_t>(n));
  const float* d_T = hc.upload(Tcw_in, 12);
  const long long count = n;
  const long long* d_count = hc.upload(&count, 1);
  sivo_pose_result* d_res = hc.take<sivo_pose_result>(1);
  uint8_t* d_out = hc.take<uint8_t>(n);
  PoseEdge* d_edges = reinterpret_cast<PoseEdge*>(hc.take<uint8_t>(edges_bytes(n)));
  launch_optimize(p, d_kps, nullptr, d_count, n, d_ur, d_xw, d_T, d_edges, d_res, d_out, hc.stream);
  hc.download(result, d_res, 1);
  hc.download(outlier, d_out, n);
  hc.sync();
}

int pose_trace(const Orb& left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx, float fy, float cx,
               float cy, float mbf, const float* Tcw_in, sivo_pose_result* result, uint8_t* outlier, sivo_pose_trace_rec* trace,
               int trace_cap) {
  if (n < 0 || trace_cap < 0 || (trace_cap && !trace)) fail(SIVO_EINVAL, "pose_trace: n = %d, trace_cap = %d", n, trace_cap);
  const PoseParams p = make_params(left, fx, fy, cx, cy, mbf);
  check_octaves("pose_trace", kps, xw, n, p.nlevels);
  HostCall& hc = host_call();
  hc.begin(left.device());
  const sivo_keypoint* d_kps = hc.upload(kps, n);
  const float* d_ur = hc.upload(u_right, n);
  const float* d_xw = hc.upload(xw, 3 * static_cast<size_t>(n));
  const float* d_T = hc.upload(Tcw_in, 12);
  const long long count = n;
  const long long* d_count = hc.upload(&count, 1);
  const int zero = 0;
  int* d_nrec = hc.upload(&zero, 1);
  sivo_pose_result* d_res = hc.take<sivo_pose_result>(1);
  uint8_t* d_out = hc.take<uint8_t>(n);
  sivo_pose_trace_rec* d_tr = hc.take<sivo_pose_trace_rec>(std::max(trace_cap, 1));
  PoseEdge* d_edges = reinterpret_cast<PoseEdge*>(hc.take<uint8_t>(edges_bytes(n)));
  k_pose_optimize<true><<<1, kThreads, 0, hc.stream>>>(p, d_kps, nullptr, d_count, n, d_ur, d_xw, d_T, d_edges, d_res, d_out, d_tr,
                                                       trace_cap, d_nrec);
  SIVO_CUDA(cudaGetLastError());
  int n_rec = 0;
  hc.download(result, d_res, 1);
  if (outlier) hc.download(outlier, d_out, n);
  hc.download(&n_rec, d_nrec, 1);
  hc.sync();
  if (trace_cap) {
    hc.download(trace, d_tr, std::min(n_rec, trace_cap));
    hc.sync();
  }
  return n_rec;
}

void pose_se3(int device, int n, const float* T, const double* d, double* se3, double* up, double* tv, sivo_pose_result* res) {
  if (n < 1 || !T || !d || !se3 || !up || !tv || !res) fail(SIVO_EINVAL, "pose_se3: null argument or n < 1");
  HostCall& hc = host_call();
  hc.begin(device);
  const float* d_T = hc.upload(T, 12 * static_cast<size_t>(n));
  const double* d_d = hc.upload(d, 6 * static_cast<size_t>(n));
  double* d_out = hc.take<double>(18 * static_cast<size_t>(n));
  sivo_pose_result* d_res = hc.take<sivo_pose_result>(n);
  k_pose_se3<<<ceil_div(n, kThreads), kThreads, 0, hc.stream>>>(n, d_T, d_d, d_out, d_out + 7 * static_cast<size_t>(n),
                                                               d_out + 14 * static_cast<size_t>(n), d_res);
  SIVO_CUDA(cudaGetLastError());
  hc.download(se3, d_out, 7 * static_cast<size_t>(n));
  hc.download(up, d_out + 7 * static_cast<size_t>(n), 7 * static_cast<size_t>(n));
  hc.download(tv, d_out + 14 * static_cast<size_t>(n), 4 * static_cast<size_t>(n));
  hc.download(res, d_res, n);
  hc.sync();
}

void pose_system(const Orb& left, const sivo_keypoint* kps, const float* u_right, const float* xw, int n, float fx, float fy, float cx,
                 float cy, float mbf, const double* pose7, int robust_stereo, const uint8_t* level1, double* err, double* chi2, double* rho,
                 double* jac, double* H, double* b, double* chi) {
  if (n < 0) fail(SIVO_EINVAL, "pose_system: n = %d", n);
  const PoseParams p = make_params(left, fx, fy, cx, cy, mbf);
  check_octaves("pose_system", kps, xw, n, p.nlevels);
  HostCall& hc = host_call();
  hc.begin(left.device());
  const sivo_keypoint* d_kps = hc.upload(kps, n);
  const float* d_ur = hc.upload(u_right, n);
  const float* d_xw = hc.upload(xw, 3 * static_cast<size_t>(n));
  const uint8_t* d_l1 = hc.upload(level1, n);
  const double* d_pose = hc.upload(pose7, 7);
  double* d_per = hc.take<double>(24 * static_cast<size_t>(n));
  double* d_Hb = hc.take<double>(43);
  PoseEdge* d_edges = reinterpret_cast<PoseEdge*>(hc.take<uint8_t>(edges_bytes(n)));
  double *d_err = d_per, *d_chi2 = d_per + 3 * static_cast<size_t>(n), *d_rho = d_per + 4 * static_cast<size_t>(n),
         *d_jac = d_per + 6 * static_cast<size_t>(n);
  k_pose_system<<<1, kThreads, 0, hc.stream>>>(p, d_kps, n, d_ur, d_xw, level1 ? d_l1 : nullptr, d_pose, robust_stereo, d_edges, d_err,
                                               d_chi2, d_rho, d_jac, d_Hb);
  SIVO_CUDA(cudaGetLastError());
  double Hb[43];
  hc.download(err, d_err, 3 * static_cast<size_t>(n));
  hc.download(chi2, d_chi2, n);
  hc.download(rho, d_rho, 2 * static_cast<size_t>(n));
  hc.download(jac, d_jac, 18 * static_cast<size_t>(n));
  hc.download(Hb, d_Hb, 43);
  hc.sync();
  if (H) for (int i = 0; i < 36; ++i) H[i] = Hb[i];
  if (b) for (int i = 0; i < 6; ++i) b[i] = Hb[36 + i];
  if (chi) *chi = Hb[42];
}

}  // namespace sivo
