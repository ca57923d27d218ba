// Relocalization's pose hypotheses: PnPsolver (PnPsolver.cc) with SetRansacParameters(0.99, 10, 300, 4, 0.5, 5.991), batched over
// the candidate keyframes.  The rule is spelled out in include/sivo_b200.h and oracle/pnp_oracle.py.  This file is compiled with
// -fmad=false: every float / double intermediate is the correctly rounded result of the operation as written.
//
// A hypothesis depends only on (candidate, hypothesis index) (counter-based draws), so one launch runs every hypothesis a call
// may need, and a second walks them in the reference's order:
//   k_pnp_setup   one block per candidate: the correspondences in key order, N, minInliers, epsilon, maxIts; resets the state.
//   k_pnp_hyp     one warp per (active candidate, hypothesis): lane 0 draws and runs EPnP on the minimal set, the lanes run
//                 CheckInliers into a bit mask.
//   k_pnp_decide  one block per active candidate: the iterate() loop over the hypotheses' counts, Refine on the best set so far
//                 (alphas across threads, MtM in the documented tree of mtm_tree), the call's outputs.  EPnP's decompositions,
//                 Gauss-Newton and pose recovery run in one thread (lane 0 / thread 0); their 12 x 12 and 6 x K working arrays do
//                 not fit in registers, so k_pnp_hyp and k_pnp_decide use 255 registers with a few hundred bytes of spills.
#include <cmath>

#include "block_ops.cuh"
#include "frame_ops.h"
#include "host_call.h"
#include "jacobi.cuh"
#include "philox.cuh"
#include "stream_scratch.h"

namespace sivo {
namespace {
constexpr int kMinSet = 4, kMinInliers = 10, kMaxIterations = 300;
constexpr int kItsBound = 35;  // maxIts never exceeds 35: epsilon >= 0.5 gives ceil(log(0.01) / log(1 - 0.125)) = 35
constexpr int kHypWarps = 4, kHypThreads = 32 * kHypWarps;
constexpr int kDecideThreads = 256, kDecideWarps = kDecideThreads / 32;
constexpr float kTh2 = 5.991f;

struct Cam { double fu, fv, uc, vc; };

// ---------------------------------------------------------------------------------------------------- decompositions
// cvSolve(A, b, CV_SVD) for 6 x K: x_i = sum over kept j (descending) of V[i][j] ((B_j . b) / n2_j), j kept iff sigma_j > 2^-51
// times the sum of the sigmas (OpenCV's SVBkSb threshold)
template <int M, int K>
__device__ void solve_svd(double (&a)[M][K], const double* b, double* x) {
  double v[K][K], n2[K];
  int ord[K];
#pragma unroll
  for (int r = 0; r < K; ++r)
#pragma unroll
    for (int c = 0; c < K; ++c) v[r][c] = r == c ? 1.0 : 0.0;
  jacobi_sweeps<M, K>(a, v);
  jacobi_order<M, K>(a, n2, ord);
  double thr = 0.0;
  for (int j = 0; j < K; ++j) thr = thr + sqrt(n2[ord[j]]);
  thr = thr * 0x1p-51;
  for (int i = 0; i < K; ++i) x[i] = 0.0;
  for (int jj = 0; jj < K; ++jj) {
    const int j = ord[jj];
    if (!(sqrt(n2[j]) > thr)) continue;
    double s = 0.0;
    for (int r = 0; r < M; ++r) s = s + a[r][j] * b[r];
    const double w = s / n2[j];
    for (int i = 0; i < K; ++i) x[i] = x[i] + v[i][j] * w;
  }
}

__device__ __forceinline__ double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
__device__ __forceinline__ double dist2(const double* a, const double* b) {
  return (a[0] - b[0]) * (a[0] - b[0]) + (a[1] - b[1]) * (a[1] - b[1]) + (a[2] - b[2]) * (a[2] - b[2]);
}

// ---------------------------------------------------------------------------------------------------- EPnP pieces
// choose_control_points and compute_barycentric_coordinates' inverse (one thread)
__device__ void epnp_control(const double* pws, int n, double cws[4][3], double ci[9]) {
  double c0[3] = {0.0, 0.0, 0.0};
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) c0[j] = c0[j] + pws[3 * i + j];
  for (int j = 0; j < 3; ++j) c0[j] = c0[j] / n;
  double ptp[3][3];
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      double s = 0.0;
      for (int i = 0; i < n; ++i) s = s + (pws[3 * i + a] - c0[a]) * (pws[3 * i + b] - c0[b]);
      ptp[a][b] = s;
    }
  double v[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}}, n2[3];
  int ord[3];
  jacobi_sweeps<3, 3>(ptp, v);
  jacobi_order<3, 3>(ptp, n2, ord);
  for (int j = 0; j < 3; ++j) cws[0][j] = c0[j];
  for (int i = 1; i < 4; ++i) {
    const double k = sqrt(sqrt(n2[ord[i - 1]]) / n);
    for (int j = 0; j < 3; ++j) cws[i][j] = c0[j] + k * v[j][ord[i - 1]];
  }
  // cvInvert(CC, CV_SVD): column k of the inverse solves CC x = e_k
  double cc[3][3];
  for (int k = 0; k < 3; ++k) {
    for (int i = 0; i < 3; ++i)
      for (int j = 1; j < 4; ++j) cc[i][j - 1] = cws[j][i] - cws[0][i];
    const double e[3] = {k == 0 ? 1.0 : 0.0, k == 1 ? 1.0 : 0.0, k == 2 ? 1.0 : 0.0};
    double x[3];
    solve_svd<3, 3>(cc, e, x);
    for (int i = 0; i < 3; ++i) ci[3 * i + k] = x[i];
  }
}

__device__ __forceinline__ void epnp_alpha(const double cws[4][3], const double* ci, const double* p, double* a) {
  for (int j = 0; j < 3; ++j)
    a[1 + j] = ci[3 * j] * (p[0] - cws[0][0]) + ci[3 * j + 1] * (p[1] - cws[0][1]) + ci[3 * j + 2] * (p[2] - cws[0][2]);
  a[0] = 1.0 - a[1] - a[2] - a[3];
}

// fill_M's entry (row 2i + h, column c) for correspondence i
__device__ __forceinline__ double m_entry(const double* a, double u, double v, const Cam& k, int h, int c) {
  const int i = c / 3, comp = c % 3;
  if (h == 0) return comp == 0 ? a[i] * k.fu : comp == 1 ? 0.0 : a[i] * (k.uc - u);
  return comp == 0 ? 0.0 : comp == 1 ? a[i] * k.fv : a[i] * (k.vc - v);
}

// cvMulTransposed(M, MtM, 1)'s entry (r, c): the rows summed in order
__device__ double mtm_entry(const double* alphas, const double* us, int n, const Cam& k, int r, int c) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) {
    const double* a = alphas + 4 * i;
    const double u = us[2 * i], v = us[2 * i + 1];
    s = s + m_entry(a, u, v, k, 0, r) * m_entry(a, u, v, k, 0, c);
    s = s + m_entry(a, u, v, k, 1, r) * m_entry(a, u, v, k, 1, c);
  }
  return s;
}

__device__ void gauss_newton(const double (&L)[6][10], const double* rho, double* betas) {
  double x[4] = {0.0, 0.0, 0.0, 0.0};
  for (int it = 0; it < 5; ++it) {
    double A[6][4], b[6];
    for (int i = 0; i < 6; ++i) {
      const double* r = L[i];
      A[i][0] = 2 * r[0] * betas[0] + r[1] * betas[1] + r[3] * betas[2] + r[6] * betas[3];
      A[i][1] = r[1] * betas[0] + 2 * r[2] * betas[1] + r[4] * betas[2] + r[7] * betas[3];
      A[i][2] = r[3] * betas[0] + r[4] * betas[1] + 2 * r[5] * betas[2] + r[8] * betas[3];
      A[i][3] = r[6] * betas[0] + r[7] * betas[1] + r[8] * betas[2] + 2 * r[9] * betas[3];
      b[i] = rho[i] - (r[0] * betas[0] * betas[0] + r[1] * betas[0] * betas[1] + r[2] * betas[1] * betas[1] + r[3] * betas[0] * betas[2] +
                       r[4] * betas[1] * betas[2] + r[5] * betas[2] * betas[2] + r[6] * betas[0] * betas[3] + r[7] * betas[1] * betas[3] +
                       r[8] * betas[2] * betas[3] + r[9] * betas[3] * betas[3]);
    }
    // qr_solve (PnPsolver.cc:865-955); its early return on a zero column leaves x as it was
    double A1[4], A2[4];
    bool singular = false;
    for (int k = 0; k < 4 && !singular; ++k) {
      double eta = fabs(A[k][k]);
      for (int i = k + 1; i < 6; ++i) {
        const double elt = fabs(A[i][k]);
        if (eta < elt) eta = elt;
      }
      if (eta == 0) { singular = true; break; }
      double s = 0.0;
      const double inv_eta = 1. / eta;
      for (int i = k; i < 6; ++i) {
        A[i][k] = A[i][k] * inv_eta;
        s = s + A[i][k] * A[i][k];
      }
      double sigma = sqrt(s);
      if (A[k][k] < 0) sigma = -sigma;
      A[k][k] = A[k][k] + sigma;
      A1[k] = sigma * A[k][k];
      A2[k] = -eta * sigma;
      for (int j = k + 1; j < 4; ++j) {
        double s2 = 0;
        for (int i = k; i < 6; ++i) s2 = s2 + A[i][k] * A[i][j];
        const double tau = s2 / A1[k];
        for (int i = k; i < 6; ++i) A[i][j] = A[i][j] - tau * A[i][k];
      }
    }
    if (!singular) {
      for (int j = 0; j < 4; ++j) {
        double tau = 0;
        for (int i = j; i < 6; ++i) tau = tau + A[i][j] * b[i];
        tau = tau / A1[j];
        for (int i = j; i < 6; ++i) b[i] = b[i] - tau * A[i][j];
      }
      x[3] = b[3] / A2[3];
      for (int i = 2; i >= 0; --i) {
        double s = 0;
        for (int j = i + 1; j < 4; ++j) s = s + A[i][j] * x[j];
        x[i] = (b[i] - s) / A2[i];
      }
    }
    for (int i = 0; i < 4; ++i) betas[i] = betas[i] + x[i];
  }
}

// compute_ccs, compute_pcs, solve_for_sign, estimate_R_and_t, reprojection_error (pcs: n x 3 scratch)
__device__ double compute_R_and_t(const double (*v)[12], const int* ord, const double* betas, const double* alphas, const double* pws,
                                  const double* us, double* pcs, int n, const Cam& k, double R[3][3], double t[3]) {
  double ccs[4][3];
  for (int i = 0; i < 4; ++i) ccs[i][0] = ccs[i][1] = ccs[i][2] = 0.0;
  for (int i = 0; i < 4; ++i) {
    const int col = ord[11 - i];
    for (int j = 0; j < 4; ++j)
      for (int c = 0; c < 3; ++c) ccs[j][c] = ccs[j][c] + betas[i] * v[3 * j + c][col];
  }
  for (int i = 0; i < n; ++i) {
    const double* a = alphas + 4 * i;
    for (int j = 0; j < 3; ++j) pcs[3 * i + j] = a[0] * ccs[0][j] + a[1] * ccs[1][j] + a[2] * ccs[2][j] + a[3] * ccs[3][j];
  }
  if (pcs[2] < 0.0)
    for (int i = 0; i < 3 * n; ++i) pcs[i] = -pcs[i];
  double pc0[3] = {0.0, 0.0, 0.0}, pw0[3] = {0.0, 0.0, 0.0};
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) {
      pc0[j] = pc0[j] + pcs[3 * i + j];
      pw0[j] = pw0[j] + pws[3 * i + j];
    }
  for (int j = 0; j < 3; ++j) {
    pc0[j] = pc0[j] / n;
    pw0[j] = pw0[j] / n;
  }
  double abt[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j)
      for (int c = 0; c < 3; ++c) abt[j][c] = abt[j][c] + (pcs[3 * i + j] - pc0[j]) * (pws[3 * i + c] - pw0[c]);
  double vv[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}}, n2[3];
  int o[3];
  jacobi_sweeps<3, 3>(abt, vv);
  jacobi_order<3, 3>(abt, n2, o);
  double U[3][3], V[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      U[r][c] = abt[r][o[c]] / sqrt(n2[o[c]]);
      V[r][c] = vv[r][o[c]];
    }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i][j] = dot3(U[i], V[j]);
  const double det = R[0][0] * R[1][1] * R[2][2] + R[0][1] * R[1][2] * R[2][0] + R[0][2] * R[1][0] * R[2][1] -
                     R[0][2] * R[1][1] * R[2][0] - R[0][1] * R[1][0] * R[2][2] - R[0][0] * R[1][2] * R[2][1];
  if (det < 0) {
    R[2][0] = -R[2][0];
    R[2][1] = -R[2][1];
    R[2][2] = -R[2][2];
  }
  for (int i = 0; i < 3; ++i) t[i] = pc0[i] - dot3(R[i], pw0);
  double sum2 = 0.0;
  for (int i = 0; i < n; ++i) {
    const double* pw = pws + 3 * i;
    const double Xc = dot3(R[0], pw) + t[0], Yc = dot3(R[1], pw) + t[1];
    const double inv_Zc = 1.0 / (dot3(R[2], pw) + t[2]);
    const double ue = k.uc + k.fu * Xc * inv_Zc, ve = k.vc + k.fv * Yc * inv_Zc;
    const double u = us[2 * i], vv2 = us[2 * i + 1];
    sum2 = sum2 + sqrt((u - ue) * (u - ue) + (vv2 - ve) * (vv2 - ve));
  }
  return sum2 / n;
}

// the rest of compute_pose after MtM (one thread): its SVD, L_6x10, rho, the three beta approximations with Gauss-Newton, and
// the pose of least reprojection error.  mtm is destroyed; v receives V.
__device__ void epnp_finish(double (*mtm)[12], double (*v)[12], const double cws[4][3], const double* pws, const double* us,
                            const double* alphas, double* pcs, int n, const Cam& k, double R[3][3], double t[3],
                            sivo_pnp_pose_debug* dbg) {
  for (int r = 0; r < 12; ++r)
    for (int c = 0; c < 12; ++c) v[r][c] = r == c ? 1.0 : 0.0;
  jacobi_sweeps<12, 12>(mtm, v);
  double n2[12];
  int ord[12];
  jacobi_order<12, 12>(mtm, n2, ord);
  // compute_L_6x10: v_i = ut row 11 - i = V's column for the (11 - i)-th singular value
  double dv[4][6][3];
  for (int i = 0; i < 4; ++i) {
    const int col = ord[11 - i];
    int a = 0, b = 1;
    for (int j = 0; j < 6; ++j) {
      for (int c = 0; c < 3; ++c) dv[i][j][c] = v[3 * a + c][col] - v[3 * b + c][col];
      ++b;
      if (b > 3) { ++a; b = a + 1; }
    }
  }
  double L[6][10], rho[6];
  for (int i = 0; i < 6; ++i) {
    L[i][0] = dot3(dv[0][i], dv[0][i]);
    L[i][1] = 2.0 * dot3(dv[0][i], dv[1][i]);
    L[i][2] = dot3(dv[1][i], dv[1][i]);
    L[i][3] = 2.0 * dot3(dv[0][i], dv[2][i]);
    L[i][4] = 2.0 * dot3(dv[1][i], dv[2][i]);
    L[i][5] = dot3(dv[2][i], dv[2][i]);
    L[i][6] = 2.0 * dot3(dv[0][i], dv[3][i]);
    L[i][7] = 2.0 * dot3(dv[1][i], dv[3][i]);
    L[i][8] = 2.0 * dot3(dv[2][i], dv[3][i]);
    L[i][9] = dot3(dv[3][i], dv[3][i]);
  }
  rho[0] = dist2(cws[0], cws[1]);
  rho[1] = dist2(cws[0], cws[2]);
  rho[2] = dist2(cws[0], cws[3]);
  rho[3] = dist2(cws[1], cws[2]);
  rho[4] = dist2(cws[1], cws[3]);
  rho[5] = dist2(cws[2], cws[3]);
  double betas[4][4] = {}, rep[4] = {}, Rs[4][3][3], ts[4][3];
  {  // find_betas_approx_1
    double a[6][4], x[4];
    for (int i = 0; i < 6; ++i) { a[i][0] = L[i][0]; a[i][1] = L[i][1]; a[i][2] = L[i][3]; a[i][3] = L[i][6]; }
    solve_svd<6, 4>(a, rho, x);
    double* B = betas[1];
    if (x[0] < 0) {
      B[0] = sqrt(-x[0]);
      B[1] = -x[1] / B[0]; B[2] = -x[2] / B[0]; B[3] = -x[3] / B[0];
    } else {
      B[0] = sqrt(x[0]);
      B[1] = x[1] / B[0]; B[2] = x[2] / B[0]; B[3] = x[3] / B[0];
    }
  }
  {  // find_betas_approx_2
    double a[6][3], x[3];
    for (int i = 0; i < 6; ++i) { a[i][0] = L[i][0]; a[i][1] = L[i][1]; a[i][2] = L[i][2]; }
    solve_svd<6, 3>(a, rho, x);
    double* B = betas[2];
    if (x[0] < 0) {
      B[0] = sqrt(-x[0]);
      B[1] = (x[2] < 0) ? sqrt(-x[2]) : 0.0;
    } else {
      B[0] = sqrt(x[0]);
      B[1] = (x[2] > 0) ? sqrt(x[2]) : 0.0;
    }
    if (x[1] < 0) B[0] = -B[0];
    B[2] = 0.0;
    B[3] = 0.0;
  }
  {  // find_betas_approx_3
    double a[6][5], x[5];
    for (int i = 0; i < 6; ++i)
      for (int c = 0; c < 5; ++c) a[i][c] = L[i][c];
    solve_svd<6, 5>(a, rho, x);
    double* B = betas[3];
    if (x[0] < 0) {
      B[0] = sqrt(-x[0]);
      B[1] = (x[2] < 0) ? sqrt(-x[2]) : 0.0;
    } else {
      B[0] = sqrt(x[0]);
      B[1] = (x[2] > 0) ? sqrt(x[2]) : 0.0;
    }
    if (x[1] < 0) B[0] = -B[0];
    B[2] = x[3] / B[0];
    B[3] = 0.0;
  }
  for (int b = 1; b < 4; ++b) {
    gauss_newton(L, rho, betas[b]);
    rep[b] = compute_R_and_t(v, ord, betas[b], alphas, pws, us, pcs, n, k, Rs[b], ts[b]);
  }
  int N = 1;
  if (rep[2] < rep[1]) N = 2;
  if (rep[3] < rep[N]) N = 3;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) R[i][j] = Rs[N][i][j];
    t[i] = ts[N][i];
  }
  if (dbg) {
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 3; ++j) dbg->cws[3 * i + j] = cws[i][j];
    for (int r = 0; r < 12; ++r) {
      dbg->d[r] = sqrt(n2[ord[r]]);
      for (int c = 0; c < 12; ++c) dbg->ut[12 * r + c] = v[c][ord[r]];
    }
    for (int i = 0; i < 6; ++i) {
      dbg->rho[i] = rho[i];
      for (int c = 0; c < 10; ++c) dbg->l_6x10[10 * i + c] = L[i][c];
    }
    for (int b = 0; b < 3; ++b) {
      dbg->rep_errors[b] = rep[b + 1];
      for (int i = 0; i < 4; ++i) dbg->betas[4 * b + i] = betas[b + 1][i];
      for (int i = 0; i < 3; ++i) {
        dbg->ts[3 * b + i] = ts[b + 1][i];
        for (int j = 0; j < 3; ++j) dbg->Rs[9 * b + 3 * i + j] = Rs[b + 1][i][j];
      }
    }
    for (int i = 0; i < 3; ++i) {
      dbg->t[i] = t[i];
      for (int j = 0; j < 3; ++j) dbg->R[3 * i + j] = R[i][j];
    }
    dbg->best = N;
  }
}

// CheckInliers (PnPsolver.cc:318-347) for one correspondence
__device__ __forceinline__ bool inlier(const double (*R)[3], const double* t, const float* p3, float2 p2, float max_err, const Cam& k) {
  const double x = p3[0], y = p3[1], z = p3[2];
  const float Xc = static_cast<float>(R[0][0] * x + R[0][1] * y + R[0][2] * z + t[0]);
  const float Yc = static_cast<float>(R[1][0] * x + R[1][1] * y + R[1][2] * z + t[1]);
  const float invZc = static_cast<float>(1 / (R[2][0] * x + R[2][1] * y + R[2][2] * z + t[2]));
  const double ue = k.uc + k.fu * Xc * invZc, ve = k.vc + k.fv * Yc * invZc;
  const float dx = static_cast<float>(p2.x - ue), dy = static_cast<float>(p2.y - ve);
  const float e2 = dx * dx + dy * dy;
  return e2 < max_err;
}

__device__ __forceinline__ void tcw_of(const double (*R)[3], const double* t, float* T) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T[4 * i + j] = static_cast<float>(R[i][j]);
    T[4 * i + 3] = static_cast<float>(t[i]);
  }
}

// the draws of hypothesis g among N correspondences: Philox words, then the reference's swap-remove
__device__ __forceinline__ void draw4(uint64_t seed, uint32_t kf_id, uint64_t frame_id, uint32_t g, int N, int* idx) {
  uint32_t w[4];
  philox4x32_10(g, kf_id, static_cast<uint32_t>(frame_id), static_cast<uint32_t>(frame_id >> 32), static_cast<uint32_t>(seed),
                static_cast<uint32_t>(seed >> 32), w);
  int pos[kMinSet], val[kMinSet], m = 0;  // positions of vAvailableIndices that no longer hold their own index
  for (int i = 0; i < kMinSet; ++i) {
    const int avail = N - i;
    const int r = static_cast<int>(static_cast<double>(w[i]) / 4294967296.0 * static_cast<double>(avail));
    int at_r = r, at_back = avail - 1;
    for (int e = 0; e < m; ++e) {
      if (pos[e] == r) at_r = val[e];
      if (pos[e] == avail - 1) at_back = val[e];
    }
    idx[i] = at_r;
    bool found = false;
    for (int e = 0; e < m; ++e)
      if (pos[e] == r) { val[e] = at_back; found = true; }
    if (!found) { pos[m] = r; val[m] = at_back; ++m; }
  }
}

// SetRansacParameters(0.99, 10, 300, 4, 0.5, 5.991) for N correspondences
__device__ void ransac_parameters(int N, int* min_inl, float* eps_out, int* max_its) {
  int nmin = static_cast<int>(static_cast<float>(N) * 0.5f);
  if (nmin < kMinInliers) nmin = kMinInliers;
  if (nmin < kMinSet) nmin = kMinSet;
  float eps = 0.5f;
  if (eps < static_cast<float>(nmin) / N) eps = static_cast<float>(nmin) / N;
  int n_it;
  if (nmin == N) {
    n_it = 1;
  } else {
    const double e = eps;
    const double x = log(1 - 0.99) / log(1 - e * e * e);
    n_it = (x != x || isinf(x)) ? INT_MIN : static_cast<int>(ceil(x));
  }
  *min_inl = nmin;
  *eps_out = eps;
  *max_its = max(1, min(n_it, kMaxIterations));
}

struct PnpState {  // one candidate's PnPsolver members (device)
  int N, min_inl, max_its, iters, best, refine_failed, dead;
  uint32_t kf_id;
  float eps;
  float best_tcw[12];
};

struct PnpArrays {
  PnpState* st;
  float2* p2d;
  float* p3d;
  float* max_err;
  int* key;    // the correspondence's semantic key
  int* point;  // its map point (the match row's entry)
  uint32_t* best_mask;
  int cap, words;
};

struct SetupParams {
  PnpArrays a;
  const sivo_keypoint* kps;
  const int* keep_idx;
  const long long* n_keep;
  const int* match;
  const long long* n_matches;
  const sivo_map_point* points;
  int n_points, nlevels, n_kf;
  float sigma2[kOrbMaxLevels];
  uint32_t kf_id[kPnpMaxCandidates];
};

__global__ void __launch_bounds__(256) k_pnp_setup(const __grid_constant__ SetupParams p) {
  __shared__ int warp_tot[8];
  const int kf = blockIdx.x, cap = p.a.cap;
  const long long nk = *p.n_keep, nm = p.n_matches[kf];
  const bool dead = nk < 0 || nm < 0;
  const int n = dead ? 0 : static_cast<int>(min(nk, static_cast<long long>(cap)));
  const size_t base = static_cast<size_t>(kf) * cap;
  int count = 0;
  for (int j0 = 0; j0 < n; j0 += blockDim.x) {
    const int j = j0 + threadIdx.x;
    bool valid = false;
    int pt = -1, oct = 0, kidx = 0;
    if (j < n) {
      pt = p.match[base + j];
      kidx = p.keep_idx ? p.keep_idx[j] : j;
      valid = pt >= 0 && pt < p.n_points && kidx >= 0 && kidx < cap;
      if (valid) {
        oct = p.kps[kidx].octave;
        valid = oct >= 0 && oct < p.nlevels;
      }
    }
    int tot;
    __syncthreads();  // the previous chunk has read warp_tot
    const int pos = block_rank<256>(valid, warp_tot, &tot);
    if (valid) {
      const size_t o = base + count + pos;
      const sivo_keypoint kp = p.kps[kidx];
      p.a.p2d[o] = make_float2(kp.x, kp.y);
      for (int c = 0; c < 3; ++c) p.a.p3d[3 * o + c] = p.points[pt].pos[c];
      p.a.max_err[o] = p.sigma2[oct] * kTh2;
      p.a.key[o] = j;
      p.a.point[o] = pt;
    }
    count += tot;
  }
  if (threadIdx.x == 0) {
    PnpState s{};
    s.N = count;
    s.dead = dead ? 1 : 0;
    s.kf_id = p.kf_id[kf];
    ransac_parameters(count, &s.min_inl, &s.eps, &s.max_its);
    p.a.st[kf] = s;
  }
}

struct IterParams {
  PnpArrays a;
  Cam k;
  uint64_t seed, frame_id;
  int n_iterations, H, n_act;
  // outputs
  float* Tcw;
  int* has_pose;
  int* no_more;
  int* inlier_match;
  int* n_inliers;
  // per-call scratch: per (slot, hypothesis) count, pose and mask; per slot Refine's doubles and mask
  int* h_cnt;
  float* h_tcw;
  uint32_t* h_mask;
  double* r_work;   // slot * cap * 12: pws 3, us 2, alphas 4, pcs 3
  uint32_t* r_mask;
  // test hook (sivo_dbg_pnp_hypotheses): hypotheses dbg_first .. dbg_first + n_iterations - 1 and their draws and poses; -1 = a call
  int dbg_first;
  int* dbg_draw;
  double* dbg_rt;
  int act[kPnpMaxCandidates];
};

// the number of hypotheses a call runs unless it returns: while (mnIterations < maxIts || nCurrent < n)
__device__ __forceinline__ int call_length(const PnpState& s, int n_iterations) { return max(max(s.max_its - s.iters, n_iterations), 0); }

struct HypShared {
  double mtm[12][12], v[12][12];
  double pws[12], us[8], alphas[16], pcs[12], R[3][3], t[3];
};

__global__ void __launch_bounds__(kHypThreads) k_pnp_hyp(const __grid_constant__ IterParams p) {
  __shared__ HypShared sh[kHypWarps];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, slot = blockIdx.y, kf = p.act[slot];
  const int h = blockIdx.x * kHypWarps + w;
  const PnpState s = p.a.st[kf];
  const int len = p.dbg_first >= 0 ? p.n_iterations : call_length(s, p.n_iterations);
  if (s.dead || s.N < s.min_inl || h >= len) return;
  const int g = (p.dbg_first >= 0 ? p.dbg_first : s.iters) + h;
  HypShared& e = sh[w];
  const size_t base = static_cast<size_t>(kf) * p.a.cap;
  if (lane == 0) {
    int idx[kMinSet];
    draw4(p.seed, s.kf_id, p.frame_id, static_cast<uint32_t>(g), s.N, idx);
    for (int i = 0; i < kMinSet; ++i) {
      const size_t o = base + idx[i];
      for (int c = 0; c < 3; ++c) e.pws[3 * i + c] = p.a.p3d[3 * o + c];
      e.us[2 * i] = p.a.p2d[o].x;
      e.us[2 * i + 1] = p.a.p2d[o].y;
    }
    double cws[4][3], ci[9];
    epnp_control(e.pws, kMinSet, cws, ci);
    for (int i = 0; i < kMinSet; ++i) epnp_alpha(cws, ci, e.pws + 3 * i, e.alphas + 4 * i);
    for (int r = 0; r < 12; ++r)
      for (int c = r; c < 12; ++c) e.mtm[r][c] = e.mtm[c][r] = mtm_entry(e.alphas, e.us, kMinSet, p.k, r, c);
    epnp_finish(e.mtm, e.v, cws, e.pws, e.us, e.alphas, e.pcs, kMinSet, p.k, e.R, e.t, nullptr);
    if (p.dbg_draw) {
      for (int i = 0; i < kMinSet; ++i) p.dbg_draw[4 * h + i] = idx[i];
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) p.dbg_rt[12 * h + 3 * i + j] = e.R[i][j];
        p.dbg_rt[12 * h + 9 + i] = e.t[i];
      }
    }
  }
  __syncwarp();
  const size_t hs = static_cast<size_t>(slot) * p.H + h;
  uint32_t* mask = p.h_mask + hs * p.a.words;
  int cnt = 0;
  for (int i0 = 0; i0 < s.N; i0 += 32) {
    const int i = i0 + lane;
    const bool in = i < s.N && inlier(e.R, e.t, p.a.p3d + 3 * (base + i), p.a.p2d[base + i], p.a.max_err[base + i], p.k);
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (lane == 0) mask[i0 >> 5] = b;
    cnt += __popc(b);
  }
  if (lane == 0) {
    p.h_cnt[hs] = cnt;
    tcw_of(e.R, e.t, p.h_tcw + 12 * hs);
  }
}

struct RefineShared {
  double mtm[12][12], v[12][12];
  double cws[4][3], ci[9], R[3][3], t[3];
  double part[kDecideWarps][78];
  int warp_tot[kDecideWarps];
  int cnt;
};

// MtM over n correspondences in the documented tree: thread t sums correspondences t, t + 256, ... in order (row 2i, then row
// 2i + 1), xor shuffles 16 .. 1 in each warp, then the 8 warp totals folded by halves, ((w0 + w4) + (w2 + w6)) + ((w1 + w5) + (w3 +
// w7)).  Upper triangle row by row (78 entries), mirrored.
__device__ void mtm_tree(const double* alphas, const double* us, int n, const Cam& k, RefineShared& sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int e = 0;
  for (int r = 0; r < 12; ++r)
    for (int c = r; c < 12; ++c, ++e) {
      double s = 0.0;
      for (int i = threadIdx.x; i < n; i += kDecideThreads) {
        const double* a = alphas + 4 * i;
        const double u = us[2 * i], v = us[2 * i + 1];
        s = s + m_entry(a, u, v, k, 0, r) * m_entry(a, u, v, k, 0, c);
        s = s + m_entry(a, u, v, k, 1, r) * m_entry(a, u, v, k, 1, c);
      }
      s = warp_tree_sum(s);
      if (lane == 0) sh.part[w][e] = s;
    }
  __syncthreads();
  if (threadIdx.x < 78) {
    const int t = threadIdx.x;
    int r = 0, c = t;
    while (c >= 12 - r) { c -= 12 - r; ++r; }
    c += r;
    double q[kDecideWarps];
    for (int i = 0; i < kDecideWarps; ++i) q[i] = sh.part[i][t];
    const double v = fold_warp_totals<kDecideWarps>(q);
    sh.mtm[r][c] = v;
    sh.mtm[c][r] = v;
  }
}

// compute_pose over the correspondences set in `sel` (n of them, in order) and CheckInliers over all N into `out_mask`;
// returns the inlier count (block-wide)
__device__ int block_pose(const PnpArrays& a, size_t base, int N, const uint32_t* sel, int n, double* work, uint32_t* out_mask,
                          const Cam& k, RefineShared& sh, float* tcw, sivo_pnp_pose_debug* dbg) {
  double* pws = work;
  double* us = pws + 3 * static_cast<size_t>(a.cap);
  double* alphas = us + 2 * static_cast<size_t>(a.cap);
  double* pcs = alphas + 4 * static_cast<size_t>(a.cap);
  int count = 0;
  for (int i0 = 0; i0 < N; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const bool in = i < N && ((sel[i >> 5] >> (i & 31)) & 1u);
    int tot;
    __syncthreads();  // the previous chunk has read sh.warp_tot
    const int pos = block_rank<kDecideThreads>(in, sh.warp_tot, &tot);
    if (in) {
      const size_t o = base + i;
      const int d = count + pos;
      for (int c = 0; c < 3; ++c) pws[3 * d + c] = a.p3d[3 * o + c];
      us[2 * d] = a.p2d[o].x;
      us[2 * d + 1] = a.p2d[o].y;
    }
    count += tot;
  }
  __syncthreads();
  if (threadIdx.x == 0) epnp_control(pws, n, sh.cws, sh.ci);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) epnp_alpha(sh.cws, sh.ci, pws + 3 * i, alphas + 4 * i);
  __syncthreads();
  mtm_tree(alphas, us, n, k, sh);
  __syncthreads();
  if (threadIdx.x == 0) {
    epnp_finish(sh.mtm, sh.v, sh.cws, pws, us, alphas, pcs, n, k, sh.R, sh.t, dbg);
    sh.cnt = 0;
    if (tcw) tcw_of(sh.R, sh.t, tcw);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  int cnt = 0;
  for (int i0 = (threadIdx.x >> 5) * 32; i0 < N; i0 += blockDim.x) {
    const int i = i0 + lane;
    const bool in = i < N && inlier(sh.R, sh.t, a.p3d + 3 * (base + i), a.p2d[base + i], a.max_err[base + i], k);
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (lane == 0) out_mask[i0 >> 5] = b;
    cnt += __popc(b);
  }
  if (lane == 0) atomicAdd(&sh.cnt, cnt);
  __syncthreads();
  return sh.cnt;
}

__global__ void __launch_bounds__(kDecideThreads) k_pnp_decide(const __grid_constant__ IterParams p) {
  __shared__ RefineShared sh;
  const int slot = blockIdx.x, kf = p.act[slot], cap = p.a.cap, words = p.a.words;
  const size_t base = static_cast<size_t>(kf) * cap;
  PnpState s = p.a.st[kf];
  int* row = p.inlier_match + base;
  for (int j = threadIdx.x; j < cap; j += blockDim.x) row[j] = -1;
  __syncthreads();
  uint32_t* best_mask = p.a.best_mask + static_cast<size_t>(kf) * words;
  uint32_t* r_mask = p.r_mask + static_cast<size_t>(slot) * words;
  const uint32_t* out_mask = nullptr;
  int has_pose = 0, no_more = 0, n_inl = 0;
  if (s.dead || s.N < s.min_inl) {
    no_more = 1;
  } else {
    const int H = call_length(s, p.n_iterations);
    bool done = false;
    for (int h = 0; h < H && !done; ++h) {
      const size_t hs = static_cast<size_t>(slot) * p.H + h;
      const int c = p.h_cnt[hs];
      ++s.iters;
      if (c < s.min_inl) continue;
      if (c > s.best) {
        s.best = c;
        s.refine_failed = 0;
        for (int i = threadIdx.x; i < words; i += blockDim.x) best_mask[i] = p.h_mask[hs * words + i];
        for (int i = 0; i < 12; ++i) s.best_tcw[i] = p.h_tcw[12 * hs + i];
        __syncthreads();
      }
      if (s.refine_failed) continue;  // Refine of the same best set fails again
      const int rc = block_pose(p.a, base, s.N, best_mask, s.best, p.r_work + static_cast<size_t>(slot) * cap * 12, r_mask, p.k, sh,
                                nullptr, nullptr);
      if (rc > s.min_inl) {
        done = true;
        has_pose = 1;
        n_inl = rc;
        out_mask = r_mask;
        if (threadIdx.x == 0) tcw_of(sh.R, sh.t, p.Tcw + 12 * static_cast<size_t>(kf));
      } else {
        s.refine_failed = 1;
      }
    }
    if (!done && s.iters >= s.max_its) {
      no_more = 1;
      if (s.best >= s.min_inl) {
        has_pose = 1;
        n_inl = s.best;
        out_mask = best_mask;
        if (threadIdx.x < 12) p.Tcw[12 * static_cast<size_t>(kf) + threadIdx.x] = s.best_tcw[threadIdx.x];
      }
    }
  }
  __syncthreads();
  if (out_mask)
    for (int i = threadIdx.x; i < s.N; i += blockDim.x)
      if ((out_mask[i >> 5] >> (i & 31)) & 1u) row[p.a.key[base + i]] = p.a.point[base + i];
  if (threadIdx.x == 0) {
    p.a.st[kf] = s;
    p.has_pose[kf] = has_pose;
    p.no_more[kf] = no_more;
    p.n_inliers[kf] = n_inl;
  }
}

// Refine's block path (block_pose) on n host-given correspondences, all selected (test hook)
__global__ void __launch_bounds__(kDecideThreads) k_pnp_pose_debug(PnpArrays a, Cam k, const uint32_t* sel, double* work,
                                                                  uint32_t* mask, int* n_inliers, sivo_pnp_pose_debug* dbg) {
  __shared__ RefineShared sh;
  const int cnt = block_pose(a, 0, a.cap, sel, a.cap, work, mask, k, sh, nullptr, dbg);
  if (threadIdx.x == 0) *n_inliers = cnt;
}

__global__ void k_pnp_draws(uint64_t seed, uint32_t kf_id, uint64_t frame_id, int first, int n_hyp, int N, int* out) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h < n_hyp) draw4(seed, kf_id, frame_id, static_cast<uint32_t>(first + h), N, out + 4 * h);
}

__global__ void k_pnp_state(const PnpState* st, int n, int* out, float* eps) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const PnpState s = st[k];
  int* o = out + 7 * k;
  o[0] = s.N; o[1] = s.min_inl; o[2] = s.max_its; o[3] = s.iters; o[4] = s.best; o[5] = s.refine_failed; o[6] = s.dead;
  if (eps) eps[k] = s.eps;
}
}  // namespace

// ---------------------------------------------------------------------------------------------------- host side
struct Pnp {
  const Orb* left;
  int device, cap, words, max_cand, n_kf = 0;
  uint64_t seed, frame_id = 0;
  Cam cam{};
  DevBuf st, p2d, p3d, max_err, key, point, best_mask;
  PnpArrays arrays() const {
    return PnpArrays{st.as<PnpState>(), p2d.as<float2>(), p3d.as<float>(), max_err.as<float>(), key.as<int>(), point.as<int>(),
                     best_mask.as<uint32_t>(), cap, words};
  }
};

Pnp* pnp_create(const Orb& left, int max_candidates, uint64_t seed) {
  if (max_candidates < 1 || max_candidates > kPnpMaxCandidates)
    fail(SIVO_EINVAL, "pnp_create: max_candidates %d outside [1, %d]", max_candidates, kPnpMaxCandidates);
  SIVO_CUDA(cudaSetDevice(left.device()));
  auto* h = new Pnp;
  h->left = &left;
  h->device = left.device();
  h->cap = left.capacity();
  h->words = (h->cap + 31) / 32;
  h->max_cand = max_candidates;
  h->seed = seed;
  const size_t cells = static_cast<size_t>(max_candidates) * std::max(h->cap, 1);
  h->st.alloc(sizeof(PnpState) * max_candidates);
  h->p2d.alloc(sizeof(float2) * cells);
  h->p3d.alloc(3 * sizeof(float) * cells);
  h->max_err.alloc(sizeof(float) * cells);
  h->key.alloc(sizeof(int) * cells);
  h->point.alloc(sizeof(int) * cells);
  h->best_mask.alloc(sizeof(uint32_t) * max_candidates * std::max(h->words, 1));
  return h;
}

void pnp_destroy(Pnp* h) { delete h; }

void pnp_setup_device(Pnp& h, const sivo_keypoint* kps, const int* keep_idx, const long long* n_keep, const int* match,
                      const long long* n_matches, const sivo_map_point* points, int n_points, const uint32_t* kf_id, int n_kf,
                      uint64_t frame_id, float fx, float fy, float cx, float cy, cudaStream_t s) {
  if (n_kf < 0 || n_kf > h.max_cand) fail(SIVO_EINVAL, "pnp_setup: n_kf %d outside [0, %d]", n_kf, h.max_cand);
  if (n_points < 0) fail(SIVO_EINVAL, "pnp_setup: n_points %d < 0", n_points);
  if (n_kf > 0 && !kf_id) fail(SIVO_EINVAL, "pnp_setup: null kf_id");
  if (!(std::isfinite(fx) && std::isfinite(fy) && std::isfinite(cx) && std::isfinite(cy)))
    fail(SIVO_EINVAL, "pnp_setup: camera parameters not finite");
  s = h.left->enter(s);
  h.n_kf = n_kf;
  h.frame_id = frame_id;
  h.cam = Cam{fx, fy, cx, cy};
  if (n_kf == 0) return;
  SetupParams p{};
  p.a = h.arrays();
  p.kps = kps;
  p.keep_idx = keep_idx;
  p.n_keep = n_keep;
  p.match = match;
  p.n_matches = n_matches;
  p.points = points;
  p.n_points = n_points;
  p.n_kf = n_kf;
  const OrbTables& t = h.left->tables();
  p.nlevels = h.left->nlevels();
  for (int l = 0; l < p.nlevels; ++l) p.sigma2[l] = t.sigma2[l];
  for (int k = 0; k < n_kf; ++k) p.kf_id[k] = kf_id[k];
  k_pnp_setup<<<n_kf, 256, 0, s>>>(p);
  SIVO_CUDA(cudaGetLastError());
}

void pnp_iterate_device(Pnp& h, int n_iterations, const uint8_t* active, float* Tcw, int* has_pose, int* no_more, int* inlier_match,
                        int* n_inliers, cudaStream_t s) {
  if (h.n_kf > 0 && !active) fail(SIVO_EINVAL, "pnp_iterate: null active");
  s = h.left->enter(s);
  IterParams p{};
  for (int k = 0; k < h.n_kf; ++k)
    if (active[k]) p.act[p.n_act++] = k;
  if (p.n_act == 0) return;
  p.a = h.arrays();
  p.k = h.cam;
  p.seed = h.seed;
  p.frame_id = h.frame_id;
  p.n_iterations = n_iterations;
  p.H = std::max(kItsBound, n_iterations);
  p.dbg_first = -1;
  p.Tcw = Tcw;
  p.has_pose = has_pose;
  p.no_more = no_more;
  p.inlier_match = inlier_match;
  p.n_inliers = n_inliers;
  const size_t cap = std::max(h.cap, 1), words = std::max(h.words, 1), hyps = static_cast<size_t>(p.n_act) * p.H;
  const size_t n_cnt = hyps, n_tcw = hyps * 12, n_mask = hyps * words, n_work = p.n_act * cap * 12, n_rmask = p.n_act * words;
  StreamScratch sc(StreamScratch::bytes<int>(n_cnt) + StreamScratch::bytes<float>(n_tcw) + StreamScratch::bytes<uint32_t>(n_mask) +
                   StreamScratch::bytes<double>(n_work) + StreamScratch::bytes<uint32_t>(n_rmask), s);
  p.h_cnt = sc.take<int>(n_cnt);
  p.h_tcw = sc.take<float>(n_tcw);
  p.h_mask = sc.take<uint32_t>(n_mask);
  p.r_work = sc.take<double>(n_work);
  p.r_mask = sc.take<uint32_t>(n_rmask);
  k_pnp_hyp<<<dim3((p.H + kHypWarps - 1) / kHypWarps, p.n_act), kHypThreads, 0, s>>>(p);
  SIVO_CUDA(cudaGetLastError());
  k_pnp_decide<<<p.n_act, kDecideThreads, 0, s>>>(p);
  SIVO_CUDA(cudaGetLastError());
}

void pnp_state(const Pnp& h, int* out, float* eps) {
  HostCall& hc = host_call();
  hc.begin(h.device);
  const int n = h.n_kf;
  int* d_out = hc.take<int>(7 * static_cast<size_t>(n));
  float* d_eps = hc.take<float>(n);
  SIVO_CUDA(cudaDeviceSynchronize());  // the state was last written on the caller's stream
  if (n) k_pnp_state<<<(n + 127) / 128, 128, 0, hc.stream>>>(h.st.as<PnpState>(), n, d_out, d_eps);
  SIVO_CUDA(cudaGetLastError());
  hc.download(out, d_out, 7 * static_cast<size_t>(n));
  hc.download(eps, d_eps, n);
  hc.sync();
}

void pnp_compute_pose_debug(int device, const float* p3d, const float* p2d, const float* max_err, int n, float fx, float fy, float cx,
                            float cy, double* alphas, uint32_t* mask, int* n_inliers, sivo_pnp_pose_debug* dbg) {
  if (n < 1 || !p3d || !p2d || !max_err || !dbg) fail(SIVO_EINVAL, "pnp_compute_pose: null argument or n < 1");
  HostCall& hc = host_call();
  hc.begin(device);
  const int words = (n + 31) / 32;
  std::vector<uint32_t> all(words, 0xffffffffu);
  PnpArrays a{};
  a.p3d = hc.upload(p3d, 3 * static_cast<size_t>(n));
  a.p2d = reinterpret_cast<float2*>(hc.upload(p2d, 2 * static_cast<size_t>(n)));
  a.max_err = hc.upload(max_err, n);
  a.cap = n;
  a.words = words;
  const uint32_t* d_sel = hc.upload(all.data(), words);
  double* d_work = hc.take<double>(12 * static_cast<size_t>(n));
  uint32_t* d_mask = hc.take<uint32_t>(words);
  int* d_cnt = hc.take<int>(1);
  sivo_pnp_pose_debug* d_dbg = hc.take<sivo_pnp_pose_debug>(1);
  k_pnp_pose_debug<<<1, kDecideThreads, 0, hc.stream>>>(a, Cam{fx, fy, cx, cy}, d_sel, d_work, d_mask, d_cnt, d_dbg);
  SIVO_CUDA(cudaGetLastError());
  hc.download(alphas, d_work + 5 * static_cast<size_t>(n), 4 * static_cast<size_t>(n));
  hc.download(mask, d_mask, words);
  hc.download(n_inliers, d_cnt, 1);
  hc.download(dbg, d_dbg, 1);
  hc.sync();
}

void pnp_hypotheses(Pnp& h, int k, int first, int n_hyp, int* draws, double* Rt, int* counts, uint32_t* masks) {
  if (k < 0 || k >= h.n_kf || first < 0 || n_hyp < 1) fail(SIVO_EINVAL, "pnp_hypotheses: candidate %d of %d, first %d, n_hyp %d", k, h.n_kf, first, n_hyp);
  HostCall& hc = host_call();
  hc.begin(h.device);
  SIVO_CUDA(cudaDeviceSynchronize());  // the state was last written on the caller's stream
  IterParams p{};
  p.a = h.arrays();
  p.k = h.cam;
  p.seed = h.seed;
  p.frame_id = h.frame_id;
  p.n_iterations = n_hyp;
  p.H = n_hyp;
  p.n_act = 1;
  p.act[0] = k;
  p.dbg_first = first;
  const size_t words = std::max(h.words, 1);
  p.h_cnt = hc.take<int>(n_hyp);
  p.h_tcw = hc.take<float>(12 * static_cast<size_t>(n_hyp));
  p.h_mask = hc.take<uint32_t>(words * n_hyp);
  p.dbg_draw = hc.take<int>(4 * static_cast<size_t>(n_hyp));
  p.dbg_rt = hc.take<double>(12 * static_cast<size_t>(n_hyp));
  SIVO_CUDA(cudaMemsetAsync(p.h_cnt, 0xff, sizeof(int) * n_hyp, hc.stream));
  k_pnp_hyp<<<dim3((n_hyp + kHypWarps - 1) / kHypWarps, 1), kHypThreads, 0, hc.stream>>>(p);
  SIVO_CUDA(cudaGetLastError());
  hc.download(draws, p.dbg_draw, 4 * static_cast<size_t>(n_hyp));
  hc.download(Rt, p.dbg_rt, 12 * static_cast<size_t>(n_hyp));
  hc.download(counts, p.h_cnt, n_hyp);
  hc.download(masks, p.h_mask, words * n_hyp);
  hc.sync();
}

void pnp_draws(int device, uint64_t seed, uint32_t kf_id, uint64_t frame_id, int first, int n_hyp, int N, int* out) {
  if (n_hyp < 0 || first < 0 || N < kMinSet || (n_hyp && !out)) fail(SIVO_EINVAL, "pnp_draws: n_hyp, first < 0, N < 4 or null output");
  if (n_hyp == 0) return;
  HostCall& hc = host_call();
  hc.begin(device);
  int* d_out = hc.take<int>(4 * static_cast<size_t>(n_hyp));
  k_pnp_draws<<<(n_hyp + 127) / 128, 128, 0, hc.stream>>>(seed, kf_id, frame_id, first, n_hyp, N, d_out);
  SIVO_CUDA(cudaGetLastError());
  hc.download(out, d_out, 4 * static_cast<size_t>(n_hyp));
  hc.sync();
}

}  // namespace sivo
