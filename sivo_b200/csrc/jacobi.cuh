// The documented decomposition rule shared by the triangulation (mapping.cu) and EPnP (pnp.cu), restated in
// oracle/pnp_oracle.py (jacobi): one-sided Jacobi on the columns of an M x N matrix (M >= N) in double.  Pairs (p, q), p < q, in
// row-major order per sweep; a pair is rotated only while |gamma| > 2^-52 sqrt(alpha beta); at most 30 sweeps, stopping after a
// sweep without a rotation.  Afterwards a = A V (its column norms are the singular values) and v holds V.  Compiled with
// -fmad=false by every includer, so each operation is the correctly rounded one as written.
#pragma once

namespace sivo {

constexpr int kJacobiSweeps = 30;

// a: M rows of N doubles (any a[r][c] indexable), v: N x N, the identity on entry
template <int M, int N, class A, class V>
__device__ __forceinline__ void jacobi_sweeps(A& a, V& v) {
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    bool rotated = false;
#pragma unroll(N <= 4 ? N : 1)
    for (int p = 0; p < N - 1; ++p)
#pragma unroll(N <= 4 ? N : 1)
      for (int q = p + 1; q < N; ++q) {
        double alpha = 0.0, beta = 0.0, gamma = 0.0;
#pragma unroll
        for (int r = 0; r < M; ++r) {
          alpha = alpha + a[r][p] * a[r][p];
          beta = beta + a[r][q] * a[r][q];
          gamma = gamma + a[r][p] * a[r][q];
        }
        if (!(fabs(gamma) > 0x1p-52 * sqrt(alpha * beta))) continue;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
        for (int r = 0; r < M; ++r) {
          const double ap = a[r][p], aq = a[r][q];
          a[r][p] = c * ap - s * aq;
          a[r][q] = s * ap + c * aq;
        }
#pragma unroll
        for (int r = 0; r < N; ++r) {
          const double vp = v[r][p], vq = v[r][q];
          v[r][p] = c * vp - s * vq;
          v[r][q] = s * vp + c * vq;
        }
        rotated = true;
      }
    if (!rotated) break;
  }
}

// n2[c] = the squared norm of a's column c (rows summed in order); order = the columns by descending n2, ties in column order
// (an insertion sort with strict `<`, so a NaN norm stays where it is)
template <int M, int N, class A>
__device__ __forceinline__ void jacobi_order(const A& a, double* n2, int* order) {
  for (int c = 0; c < N; ++c) {
    double s = 0.0;
#pragma unroll
    for (int r = 0; r < M; ++r) s = s + a[r][c] * a[r][c];
    n2[c] = s;
    int pos = c;
    while (pos > 0 && n2[order[pos - 1]] < s) {
      order[pos] = order[pos - 1];
      --pos;
    }
    order[pos] = c;
  }
}

}  // namespace sivo
