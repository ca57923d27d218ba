// SIVO's mutual information between the pose and one stereo measurement (sivo_helpers.cpp:64-88, 160-218), shared by the
// information selection (info.cu) and the semantic check of map-point creation (mapping.cu).  Both files are compiled with
// -fmad=false, so every double intermediate is the correctly rounded result of the operation as written; the rule is spelled out
// in oracle/info_oracle.py.
#pragma once
#include <cuda_runtime.h>

namespace sivo {

// det by LU with partial pivoting of the n x n row-major matrix a[(r * n + c) * stride] (overwritten).  The pivot is the first
// row with the largest |a| in the column (a NaN never displaces it); a zero pivot column is skipped.  The result is the product
// of the diagonal in order, times the permutation sign.
__device__ inline double det_lu(double* a, int n, int stride) {
#define A(r, c) a[((r) * n + (c)) * stride]
  bool neg = false;
  for (int c = 0; c < n; ++c) {
    int p = c;
    double best = fabs(A(c, c));
    for (int r = c + 1; r < n; ++r) {
      const double v = fabs(A(r, c));
      if (v > best) { best = v; p = r; }
    }
    if (best == 0.0) continue;
    if (p != c) {
      for (int j = c; j < n; ++j) { const double t = A(c, j); A(c, j) = A(p, j); A(p, j) = t; }
      neg = !neg;
    }
    const double piv = A(c, c);
    for (int r = c + 1; r < n; ++r) {
      const double l = A(r, c) / piv;
      for (int j = c + 1; j < n; ++j) A(r, j) = A(r, j) - l * A(c, j);
    }
  }
  double d = A(0, 0);
  for (int i = 1; i < n; ++i) d = d * A(i, i);
  return neg ? d * -1.0 : d;
#undef A
}

// computeStereoJacobianPose (sivo_helpers.cpp:64-88), each expression left to right as written; zero when Z == 0
__device__ __forceinline__ void stereo_jacobian_pose(double fx, double fy, double bl, double X, double Y, double Z, double J[3][6]) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 6; ++c) J[r][c] = 0.0;
  if (Z == 0.0) return;
  const double ZZ = Z * Z, Xb = X - bl;
  J[0][0] = fx / Z;
  J[0][2] = -fx * X / ZZ;
  J[0][3] = -fx * X * Y / ZZ;
  J[0][4] = fx * (1.0 + X * X / ZZ);
  J[0][5] = -fx * Y / Z;
  J[1][1] = fy / Z;
  J[1][2] = -fy * Y / ZZ;
  J[1][3] = -fy * (1.0 + Y * Y / ZZ);
  J[1][4] = fy * X * Y / ZZ;
  J[1][5] = fy * X / Z;
  J[2][0] = fx / Z;
  J[2][2] = -fx * Xb / ZZ;
  J[2][3] = -fx * Xb * Y / ZZ;
  J[2][4] = fx * (1.0 + X * Xb / ZZ);
  J[2][5] = -fx * Y / Z;
}

struct StereoMiTerms {
  double det_state, det_meas, det_joint;  // det S, det M33, det M
};

// The three determinants of computeStereoMutualInformation for the world point (X, Y, Z) (the reference passes the world point
// where the Jacobian expects camera coordinates), with S = sigma (6 x 6 row-major) and R = s2 I.  ws: a 9 x 9 working matrix,
// element e at ws[e * stride].  MI = 0.5 log2(det_state * det_meas / det_joint).
__device__ __forceinline__ StereoMiTerms stereo_mi_terms(const double* sigma, double fx, double fy, double bl, double X, double Y,
                                                         double Z, double s2, double* ws, int stride) {
  double J[3][6];
  stereo_jacobian_pose(fx, fy, bl, X, Y, Z, J);
  StereoMiTerms t;
  // det S, by the same LU as det M
  for (int e = 0; e < 36; ++e) ws[e * stride] = sigma[e];
  t.det_state = det_lu(ws, 6, stride);
  // M = [[S, S J^T], [J S, (J S) J^T + R]]
#define M(r, c) ws[((r) * 9 + (c)) * stride]
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int c = 0; c < 6; ++c) M(r, c) = sigma[r * 6 + c];
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      double s = sigma[i * 6] * J[r][0];
#pragma unroll
      for (int q = 1; q < 6; ++q) s = s + sigma[i * 6 + q] * J[r][q];
      M(i, 6 + r) = s;
    }
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      double s = J[r][0] * sigma[c];
#pragma unroll
      for (int q = 1; q < 6; ++q) s = s + J[r][q] * sigma[q * 6 + c];
      M(6 + r, c) = s;
    }
  double m33[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double s = M(6 + r, 0) * J[c][0];
#pragma unroll
      for (int q = 1; q < 6; ++q) s = s + M(6 + r, q) * J[c][q];
      m33[r][c] = s + (r == c ? s2 : 0.0);
      M(6 + r, 6 + c) = m33[r][c];
    }
#undef M
  t.det_meas = m33[0][0] * (m33[1][1] * m33[2][2] - m33[1][2] * m33[2][1]) -
               m33[0][1] * (m33[1][0] * m33[2][2] - m33[1][2] * m33[2][0]) +
               m33[0][2] * (m33[1][0] * m33[2][1] - m33[1][1] * m33[2][0]);
  t.det_joint = det_lu(ws, 9, stride);
  return t;
}

}  // namespace sivo
