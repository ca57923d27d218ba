"""Scalar restatement of PnPsolver (PnPsolver.cc) as Tracking::Relocalization runs it: SetRansacParameters(0.99, 10, 300, 4, 0.5,
5.991), iterate(5) rounds, Refine and CheckInliers, with EPnP's compute_pose (:482-531).

Reference facts kept:
- SetRansacParameters: nMinInliers = (int)(N * 0.5f), raised to 10 and to minSet 4; epsilon raised to (float) minInliers / N;
  nIterations = 1 when minInliers == N, else ceil(log(1 - 0.99) / log(1 - pow(epsilon, 3))) in double (pow(float, int) promotes
  to double); maxIts = max(1, min(nIterations, 300)).  A NaN nIterations (N < 10: epsilon > 1) converts to INT_MIN as on x86,
  so maxIts = 1 there (iterate never reads it: N < minInliers returns bNoMore at once).  maxError[i] = sigma2[octave] * 5.991f in
  float.
- iterate(n): bNoMore and no pose at once when N < minInliers.  The loop runs while mnIterations < maxIts || nCurrent < n, so a
  call runs max(maxIts - mnIterations, n) hypotheses unless it returns.  A hypothesis with count >= minInliers replaces the best
  only with a strictly greater count, then Refine runs on the BEST set so far and returns its pose iff its count > minInliers.
  After the loop, mnIterations >= maxIts gives bNoMore and, when best >= minInliers, the best pose.
- CheckInliers (:318-347): Xc, Yc and invZc = 1 / (...) are double expressions rounded to float; ue = uc + fu * Xc * invZc in
  double; distX, distY rounded to float; error2 = distX^2 + distY^2 in float; inlier iff error2 < maxError[i].
- Poses are Rcw / tcw rounded to float (convertTo(CV_32F)).
- EPnP as written, in double; `1.0f`, `2.0f` and `0.0f` literals are doubles there.

Documented rules where the reference cannot be restated:
- Random draws: DUtils::Random::RandomInt on the global rand() stream is replaced by one Philox4x32-10 call per hypothesis:
  ctr = (hypothesis index g, keyframe id, frame id lo, frame id hi), key = (seed lo, seed hi); draw i (0..3) =
  int((double) word_i / 2^32 * (N - i)), followed by the reference's swap-remove of vAvailableIndices.
- Decompositions (cv::SVD / cvSVD / cvSolve(CV_SVD) / cvInvert(CV_SVD) are not restated): `jacobi` below, one-sided Jacobi on the
  columns in double, the pair order, rotation test and sweep cap of mapping_oracle.svd_null_vector, generalised to m x n (m >= n);
  the columns are then ordered by descending squared norm, ties keeping column order (an insertion sort with strict `<`).
  Singular values are the square roots of those norms, V the rotated identity, U's column j = B's column j / sigma_j.
- Pseudo-inverse solves (cvSolve, cvInvert with CV_SVD): x_i = sum over kept j (descending) of V[i][j] * ((sum_r B[r][j] b[r]) /
  n2_j), j kept iff sigma_j > 2^-51 * (sum of sigma_j in descending order), OpenCV's SVBkSb threshold (2 DBL_EPSILON times the
  sum of the singular values).
- Departures from cv::SVD: vector signs are Jacobi's, not LAPACK's (EPnP is invariant to them up to rounding, except that a sign
  flip in V changes betas' signs, which solve_for_sign / the det < 0 flip undo); U's column for a zero singular value is 0 / 0 =
  NaN where cv::SVD completes an orthonormal basis, so a rank-deficient ABt (coplanar or collinear minimal sets) gives a NaN pose
  that no correspondence accepts.
- gauss_newton's x starts at zero; qr_solve's early return on a zero column leaves the previous iteration's x (the reference
  reads an uninitialised x on the first iteration).
- Sums over correspondences run in correspondence order, as the reference's loops, except Refine's MtM, which the device sums
  in a fixed tree (mtm_tree); the hypotheses' 4-point MtM is in row order.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from oracle.philox import philox4x32_10
from oracle.pose_oracle import tree_sum

F32 = np.float32
MAX_SWEEPS = 30
PROB, MIN_INLIERS, MAX_ITS, MIN_SET, EPSILON, TH2 = 0.99, 10, 300, 4, F32(0.5), F32(5.991)
INT_MIN = -(1 << 31)


# ---------------------------------------------------------------------------------------------------------- decompositions
def jacobi(A):
    """One-sided Jacobi on the columns of A (m x n, m >= n, float64) -> (B = A V, V, n2 = squared column norms of B, order =
    columns by descending n2, ties in column order)."""
    m, n = len(A), len(A[0])
    a = [[float(A[r][c]) for c in range(n)] for r in range(m)]
    v = [[1.0 if r == c else 0.0 for c in range(n)] for r in range(n)]
    for _ in range(MAX_SWEEPS):
        rotated = False
        for p in range(n - 1):
            for q in range(p + 1, n):
                alpha = beta = gamma = 0.0
                for r in range(m):
                    alpha = alpha + a[r][p] * a[r][p]
                    beta = beta + a[r][q] * a[r][q]
                    gamma = gamma + a[r][p] * a[r][q]
                if not abs(gamma) > 2.0 ** -52 * math.sqrt(alpha * beta):
                    continue
                zeta = (beta - alpha) / (2.0 * gamma)
                t = (1.0 if zeta >= 0.0 else -1.0) / (abs(zeta) + math.sqrt(1.0 + zeta * zeta))
                c = 1.0 / math.sqrt(1.0 + t * t)
                s = c * t
                for r in range(m):
                    ap, aq = a[r][p], a[r][q]
                    a[r][p] = c * ap - s * aq
                    a[r][q] = s * ap + c * aq
                for r in range(n):
                    vp, vq = v[r][p], v[r][q]
                    v[r][p] = c * vp - s * vq
                    v[r][q] = s * vp + c * vq
                rotated = True
        if not rotated:
            break
    n2 = []
    for c in range(n):
        s = 0.0
        for r in range(m):
            s = s + a[r][c] * a[r][c]
        n2.append(s)
    order = []
    for c in range(n):
        pos = len(order)
        while pos > 0 and n2[order[pos - 1]] < n2[c]:
            pos -= 1
        order.insert(pos, c)
    return a, v, n2, order


def svd(A):
    """-> (sigma descending, V with the matching columns (n x n), U (m x n))."""
    B, V, n2, order = jacobi(A)
    m, n = len(B), len(B[0])
    sig = [math.sqrt(n2[j]) for j in order]
    Vs = [[V[r][j] for j in order] for r in range(n)]
    U = [[_div(B[r][j], math.sqrt(n2[j])) for j in order] for r in range(m)]
    return sig, Vs, U


def _div(a, b):
    if b == 0.0:
        return math.nan if a == 0.0 or a != a else math.copysign(math.inf, a)
    return a / b


def null_vector4(A):
    """mapping_oracle.svd_null_vector's rule through `jacobi`: V's column of least squared norm, the first on ties."""
    _, v, n2, _ = jacobi(A)
    best = 0
    for c in range(4):
        if c == 0 or n2[c] < n2[best]:
            best = c
    return [v[r][best] for r in range(4)]


def solve_svd(A, b):
    """cvSolve(A, b, x, CV_SVD) for m x n A, m >= n: the documented pseudo-inverse rule."""
    B, V, n2, order = jacobi(A)
    m, n = len(B), len(B[0])
    thr = 0.0
    for j in order:
        thr = thr + math.sqrt(n2[j])
    thr = thr * 2.0 ** -51
    x = [0.0] * n
    for j in order:
        if not math.sqrt(n2[j]) > thr:
            continue
        s = 0.0
        for r in range(m):
            s = s + B[r][j] * b[r]
        w = s / n2[j]
        for i in range(n):
            x[i] = x[i] + V[i][j] * w
    return x


def invert_svd(A):
    """cvInvert(A, Ainv, CV_SVD) for a square A: solve_svd against each unit column."""
    n = len(A)
    cols = [solve_svd(A, [1.0 if r == k else 0.0 for r in range(n)]) for k in range(n)]
    return [[cols[k][i] for k in range(n)] for i in range(n)]


# ---------------------------------------------------------------------------------------------------------- EPnP
@dataclass
class PoseDebug:
    cws: list = None
    alphas: list = None
    ut: list = None          # 144, row r = V's column for the r-th singular value (descending)
    d: list = None           # 12 singular values of MtM
    l_6x10: list = None
    rho: list = None
    betas: list = field(default_factory=lambda: [[0.0] * 4 for _ in range(4)])
    rep_errors: list = field(default_factory=lambda: [0.0] * 4)
    Rs: list = field(default_factory=lambda: [None] * 4)
    ts: list = field(default_factory=lambda: [None] * 4)
    best: int = 1
    R: list = None
    t: list = None
    # which branches the run took (for the scene tests; no value depends on them): per approximation 1..3 the sign of x[0]
    # (and of x[1] for 2, 3), solve_for_sign's pcs flip and the det < 0 flip; qr_solve's early returns over all Gauss-Newton runs
    signs: dict = field(default_factory=dict)
    pcs_flip: list = field(default_factory=lambda: [False] * 4)
    det_flip: list = field(default_factory=lambda: [False] * 4)
    qr_early: int = 0


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _dist2(a, b):
    return (a[0] - b[0]) * (a[0] - b[0]) + (a[1] - b[1]) * (a[1] - b[1]) + (a[2] - b[2]) * (a[2] - b[2])


def qr_solve(A, b):
    """PnPsolver::qr_solve on A (nr x nc, modified in place) and b; None on its early return (X untouched)."""
    nr, nc = len(A), len(A[0])
    A1, A2 = [0.0] * nc, [0.0] * nc
    for k in range(nc):
        eta = abs(A[k][k])
        for i in range(k + 1, nr):
            elt = abs(A[i][k])
            if eta < elt:
                eta = elt
        if eta == 0:
            return None
        s, inv_eta = 0.0, 1.0 / eta
        for i in range(k, nr):
            A[i][k] = A[i][k] * inv_eta
            s = s + A[i][k] * A[i][k]
        sigma = math.sqrt(s)
        if A[k][k] < 0:
            sigma = -sigma
        A[k][k] = A[k][k] + sigma
        A1[k] = sigma * A[k][k]
        A2[k] = -eta * sigma
        for j in range(k + 1, nc):
            s = 0.0
            for i in range(k, nr):
                s = s + A[i][k] * A[i][j]
            tau = s / A1[k]
            for i in range(k, nr):
                A[i][j] = A[i][j] - tau * A[i][k]
    for j in range(nc):
        tau = 0.0
        for i in range(j, nr):
            tau = tau + A[i][j] * b[i]
        tau = tau / A1[j]
        for i in range(j, nr):
            b[i] = b[i] - tau * A[i][j]
    X = [0.0] * nc
    X[nc - 1] = b[nc - 1] / A2[nc - 1]
    for i in range(nc - 2, -1, -1):
        s = 0.0
        for j in range(i + 1, nc):
            s = s + A[i][j] * X[j]
        X[i] = (b[i] - s) / A2[i]
    return X


def _gauss_newton(L, rho, betas, dbg=None):
    x = [0.0] * 4
    for _ in range(5):
        A, b = [], []
        for i in range(6):
            r = L[i]
            A.append([2 * r[0] * betas[0] + r[1] * betas[1] + r[3] * betas[2] + r[6] * betas[3],
                      r[1] * betas[0] + 2 * r[2] * betas[1] + r[4] * betas[2] + r[7] * betas[3],
                      r[3] * betas[0] + r[4] * betas[1] + 2 * r[5] * betas[2] + r[8] * betas[3],
                      r[6] * betas[0] + r[7] * betas[1] + r[8] * betas[2] + 2 * r[9] * betas[3]])
            b.append(rho[i] - (r[0] * betas[0] * betas[0] + r[1] * betas[0] * betas[1] + r[2] * betas[1] * betas[1]
                               + r[3] * betas[0] * betas[2] + r[4] * betas[1] * betas[2] + r[5] * betas[2] * betas[2]
                               + r[6] * betas[0] * betas[3] + r[7] * betas[1] * betas[3] + r[8] * betas[2] * betas[3]
                               + r[9] * betas[3] * betas[3]))
        X = qr_solve(A, b)
        if X is not None:
            x = X
        elif dbg is not None:
            dbg.qr_early += 1
        for i in range(4):
            betas[i] = betas[i] + x[i]


def _sqrt(x):
    return math.sqrt(x) if x >= 0 else math.nan


def mtm_tree(M, a, b):
    """MtM[a][b] in Refine's device order: thread t of 256 sums correspondences t, t + 256, ... (rows 2i then 2i + 1), xor
    shuffles 16 .. 1 within each warp of 32, then the 8 warp totals folded by halves (pose_oracle.tree_sum)."""
    M = np.asarray(M, np.float64)
    n = len(M) // 2
    P1, P2 = M[0::2, a] * M[0::2, b], M[1::2, a] * M[1::2, b]
    s = np.zeros(256)
    t = np.arange(256)
    for j in range((n + 255) // 256):
        i = t + 256 * j
        ok = i < n
        s[ok] = s[ok] + P1[i[ok]]
        s[ok] = s[ok] + P2[i[ok]]
    return float(tree_sum(s))


def compute_pose(pws, us, fu, fv, uc, vc, la=None, tree=False) -> PoseDebug:
    """PnPsolver::compute_pose on n correspondences (pws n x 3, us n x 2, float64; camera as doubles).  `la` supplies svd3 /
    svd12 / solve / invert (default: this module's rules; tests pass cv2-backed ones).  tree: MtM in Refine's device order
    (mtm_tree) instead of row order."""
    la = la or RULE
    n = len(pws)
    dbg = PoseDebug()
    # choose_control_points
    c0 = [0.0, 0.0, 0.0]
    for i in range(n):
        for j in range(3):
            c0[j] = c0[j] + pws[i][j]
    c0 = [c0[j] / n for j in range(3)]
    pw0 = [[pws[i][j] - c0[j] for j in range(3)] for i in range(n)]
    ptp = [[0.0] * 3 for _ in range(3)]
    for a in range(3):
        for b in range(3):
            s = 0.0
            for i in range(n):
                s = s + pw0[i][a] * pw0[i][b]
            ptp[a][b] = s
    dc, uct = la.svd_sym(ptp)
    cws = [c0]
    for i in range(1, 4):
        k = _sqrt(dc[i - 1] / n)
        cws.append([c0[j] + k * uct[3 * (i - 1) + j] for j in range(3)])
    dbg.cws = [x for c in cws for x in c]
    # compute_barycentric_coordinates
    cc = [[cws[j][i] - cws[0][i] for j in range(1, 4)] for i in range(3)]
    ci = la.invert(cc)
    ci = [x for row in ci for x in row]
    alphas = []
    for i in range(n):
        p = pws[i]
        a = [0.0] * 4
        for j in range(3):
            a[1 + j] = ci[3 * j] * (p[0] - cws[0][0]) + ci[3 * j + 1] * (p[1] - cws[0][1]) + ci[3 * j + 2] * (p[2] - cws[0][2])
        a[0] = 1.0 - a[1] - a[2] - a[3]
        alphas.append(a)
    dbg.alphas = alphas
    # fill_M, MtM
    M = []
    for i in range(n):
        a, u, v = alphas[i], us[i][0], us[i][1]
        m1, m2 = [0.0] * 12, [0.0] * 12
        for k in range(4):
            m1[3 * k], m1[3 * k + 1], m1[3 * k + 2] = a[k] * fu, 0.0, a[k] * (uc - u)
            m2[3 * k], m2[3 * k + 1], m2[3 * k + 2] = 0.0, a[k] * fv, a[k] * (vc - v)
        M += [m1, m2]
    mtm = [[0.0] * 12 for _ in range(12)]
    for a in range(12):
        for b in range(a, 12):
            if tree:
                s = mtm_tree(M, a, b)
            else:
                s = 0.0
                for r in range(2 * n):
                    s = s + M[r][a] * M[r][b]
            mtm[a][b] = mtm[b][a] = s
    d, ut = la.svd_sym12(mtm)
    dbg.d, dbg.ut = d, ut
    # compute_L_6x10, compute_rho
    vv = [ut[12 * (11 - i):12 * (12 - i)] for i in range(4)]
    dv = [[None] * 6 for _ in range(4)]
    for i in range(4):
        a, b = 0, 1
        for j in range(6):
            dv[i][j] = [vv[i][3 * a + k] - vv[i][3 * b + k] for k in range(3)]
            b += 1
            if b > 3:
                a += 1
                b = a + 1
    L = []
    for i in range(6):
        L.append([_dot(dv[0][i], dv[0][i]), 2.0 * _dot(dv[0][i], dv[1][i]), _dot(dv[1][i], dv[1][i]),
                  2.0 * _dot(dv[0][i], dv[2][i]), 2.0 * _dot(dv[1][i], dv[2][i]), _dot(dv[2][i], dv[2][i]),
                  2.0 * _dot(dv[0][i], dv[3][i]), 2.0 * _dot(dv[1][i], dv[3][i]), 2.0 * _dot(dv[2][i], dv[3][i]),
                  _dot(dv[3][i], dv[3][i])])
    rho = [_dist2(cws[0], cws[1]), _dist2(cws[0], cws[2]), _dist2(cws[0], cws[3]), _dist2(cws[1], cws[2]),
           _dist2(cws[1], cws[3]), _dist2(cws[2], cws[3])]
    dbg.l_6x10, dbg.rho = [x for r in L for x in r], rho
    # betas
    b4 = la.solve([[r[0], r[1], r[3], r[6]] for r in L], rho)
    B = [0.0] * 4
    if b4[0] < 0:
        B[0] = _sqrt(-b4[0])
        B[1], B[2], B[3] = _div(-b4[1], B[0]), _div(-b4[2], B[0]), _div(-b4[3], B[0])
    else:
        B[0] = _sqrt(b4[0])
        B[1], B[2], B[3] = _div(b4[1], B[0]), _div(b4[2], B[0]), _div(b4[3], B[0])
    dbg.betas[1] = B
    dbg.signs[1] = (b4[0] < 0,)
    b3 = la.solve([[r[0], r[1], r[2]] for r in L], rho)
    B = [0.0] * 4
    if b3[0] < 0:
        B[0] = _sqrt(-b3[0])
        B[1] = _sqrt(-b3[2]) if b3[2] < 0 else 0.0
    else:
        B[0] = _sqrt(b3[0])
        B[1] = _sqrt(b3[2]) if b3[2] > 0 else 0.0
    if b3[1] < 0:
        B[0] = -B[0]
    dbg.betas[2] = B
    dbg.signs[2] = (b3[0] < 0, b3[1] < 0)
    b5 = la.solve([[r[0], r[1], r[2], r[3], r[4]] for r in L], rho)
    B = [0.0] * 4
    if b5[0] < 0:
        B[0] = _sqrt(-b5[0])
        B[1] = _sqrt(-b5[2]) if b5[2] < 0 else 0.0
    else:
        B[0] = _sqrt(b5[0])
        B[1] = _sqrt(b5[2]) if b5[2] > 0 else 0.0
    if b5[1] < 0:
        B[0] = -B[0]
    B[2] = _div(b5[3], B[0])
    dbg.betas[3] = B
    dbg.signs[3] = (b5[0] < 0, b5[1] < 0)
    for k in (1, 2, 3):
        _gauss_newton(L, rho, dbg.betas[k], dbg)
        flips = []
        dbg.Rs[k], dbg.ts[k], dbg.rep_errors[k] = _compute_R_and_t(ut, dbg.betas[k], alphas, pws, us, n, fu, fv, uc, vc, la, flips)
        dbg.pcs_flip[k], dbg.det_flip[k] = flips
    N = 1
    if dbg.rep_errors[2] < dbg.rep_errors[1]:
        N = 2
    if dbg.rep_errors[3] < dbg.rep_errors[N]:
        N = 3
    dbg.best, dbg.R, dbg.t = N, dbg.Rs[N], dbg.ts[N]
    return dbg


def _compute_R_and_t(ut, betas, alphas, pws, us, n, fu, fv, uc, vc, la, flips=None):
    ccs = [[0.0] * 3 for _ in range(4)]
    for i in range(4):
        v = ut[12 * (11 - i):12 * (12 - i)]
        for j in range(4):
            for k in range(3):
                ccs[j][k] = ccs[j][k] + betas[i] * v[3 * j + k]
    pcs = []
    for i in range(n):
        a = alphas[i]
        pcs.append([a[0] * ccs[0][j] + a[1] * ccs[1][j] + a[2] * ccs[2][j] + a[3] * ccs[3][j] for j in range(3)])
    pcs_flip = pcs[0][2] < 0.0
    if pcs_flip:
        pcs = [[-x for x in p] for p in pcs]
    # estimate_R_and_t
    pc0, pw0 = [0.0] * 3, [0.0] * 3
    for i in range(n):
        for j in range(3):
            pc0[j] = pc0[j] + pcs[i][j]
            pw0[j] = pw0[j] + pws[i][j]
    pc0 = [x / n for x in pc0]
    pw0 = [x / n for x in pw0]
    abt = [[0.0] * 3 for _ in range(3)]
    for i in range(n):
        pc, pw = pcs[i], pws[i]
        for j in range(3):
            for k in range(3):
                abt[j][k] = abt[j][k] + (pc[j] - pc0[j]) * (pw[k] - pw0[k])
    U, V = la.svd_uv(abt)
    R = [[_dot(U[i], V[j]) for j in range(3)] for i in range(3)]
    det = (R[0][0] * R[1][1] * R[2][2] + R[0][1] * R[1][2] * R[2][0] + R[0][2] * R[1][0] * R[2][1]
           - R[0][2] * R[1][1] * R[2][0] - R[0][1] * R[1][0] * R[2][2] - R[0][0] * R[1][2] * R[2][1])
    if det < 0:
        R[2] = [-x for x in R[2]]
    if flips is not None:
        flips += [pcs_flip, det < 0]
    t = [pc0[i] - _dot(R[i], pw0) for i in range(3)]
    # reprojection_error
    s2 = 0.0
    for i in range(n):
        pw = pws[i]
        Xc = _dot(R[0], pw) + t[0]
        Yc = _dot(R[1], pw) + t[1]
        inv_Zc = _div(1.0, _dot(R[2], pw) + t[2])
        ue = uc + fu * Xc * inv_Zc
        ve = vc + fv * Yc * inv_Zc
        u, v = us[i]
        s2 = s2 + _sqrt((u - ue) * (u - ue) + (v - ve) * (v - ve))
    return R, t, s2 / n


class _Rule:
    """The documented decompositions."""

    @staticmethod
    def svd_sym(A):  # cvSVD(A, D, Ut, 0, MODIFY_A | U_T) of a symmetric PSD 3 x 3: D, Ut rows = V's columns
        sig, V, _ = svd(A)
        return sig, [V[j][i] for i in range(3) for j in range(3)]

    @staticmethod
    def svd_sym12(A):
        sig, V, _ = svd(A)
        return sig, [V[j][i] for i in range(12) for j in range(12)]

    @staticmethod
    def svd_uv(A):  # cvSVD(A, D, U, V, MODIFY_A): U, V as row-major 3 x 3
        _, V, U = svd(A)
        return U, V

    solve = staticmethod(solve_svd)
    invert = staticmethod(invert_svd)


RULE = _Rule()


# ---------------------------------------------------------------------------------------------------------- RANSAC
def _log(x):
    return math.log(x) if x > 0 else (-math.inf if x == 0 else math.nan)


def ransac_parameters(N: int):
    """SetRansacParameters(0.99, 10, 300, 4, 0.5, 5.991) -> (minInliers, epsilon (float32), maxIts).  pow(epsilon, 3) is the
    correctly rounded cube, (e * e) * e in double (e * e is exact)."""
    min_inl = int(F32(N) * EPSILON)
    if min_inl < MIN_INLIERS:
        min_inl = MIN_INLIERS
    if min_inl < MIN_SET:
        min_inl = MIN_SET
    eps = EPSILON
    with np.errstate(divide="ignore", invalid="ignore"):
        q = F32(F32(min_inl) / F32(N))
    if eps < q:
        eps = q
    if min_inl == N:
        n_it = 1
    else:
        e = float(eps)
        den = _log(1 - e * e * e)
        x = math.nan if den == 0 or den != den else _log(1 - PROB) / den
        n_it = INT_MIN if (x != x or abs(x) == math.inf) else math.ceil(x)
    return min_inl, eps, max(1, min(n_it, MAX_ITS))


def draws(seed: int, kf_id: int, frame_id: int, g: int, N: int):
    """The 4 correspondence indices of hypothesis g (the documented Philox rule, then the reference's swap-remove)."""
    w = philox4x32_10(np.uint32(g), np.uint32(kf_id), np.uint32(frame_id & 0xFFFFFFFF), np.uint32(frame_id >> 32),
                      seed & 0xFFFFFFFF, seed >> 32)
    avail = list(range(N))
    out = []
    for i in range(MIN_SET):
        r = int(float(int(w[i])) / 4294967296.0 * float(len(avail)))
        out.append(avail[r])
        avail[r] = avail[-1]
        avail.pop()
    return out


def check_inliers(R, t, p3d, p2d, fu, fv, uc, vc, max_err):
    """-> (bool mask (N), count).  Elementwise numpy float64 / float32 operations are the IEEE ones, left to right as written."""
    p3 = np.asarray(p3d, F32).astype(np.float64)
    x, y, z = p3[:, 0], p3[:, 1], p3[:, 2]
    with np.errstate(all="ignore"):
        Xc = (R[0][0] * x + R[0][1] * y + R[0][2] * z + t[0]).astype(F32)
        Yc = (R[1][0] * x + R[1][1] * y + R[1][2] * z + t[1]).astype(F32)
        invZc = (1.0 / (R[2][0] * x + R[2][1] * y + R[2][2] * z + t[2])).astype(F32)
        ue = uc + fu * Xc.astype(np.float64) * invZc.astype(np.float64)
        ve = vc + fv * Yc.astype(np.float64) * invZc.astype(np.float64)
        p2 = np.asarray(p2d, F32)
        dx = (p2[:, 0].astype(np.float64) - ue).astype(F32)
        dy = (p2[:, 1].astype(np.float64) - ve).astype(F32)
        e2 = dx * dx + dy * dy
    mask = e2 < np.asarray(max_err, F32)
    return mask, int(mask.sum())


def tcw_of(R, t) -> np.ndarray:
    """3 x 4 float32 [Rcw | tcw] (convertTo(CV_32F))."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.array([[R[i][0], R[i][1], R[i][2], t[i]] for i in range(3)], np.float64).astype(F32)


@dataclass
class IterResult:
    Tcw: np.ndarray | None
    no_more: bool
    inliers: np.ndarray      # bool per correspondence
    n_inliers: int
    hypotheses: int          # run by this call


class Solver:
    """PnPsolver for one candidate: correspondences p2d (N x 2 float32), p3d (N x 3 float32), sigma2 (N float32)."""

    def __init__(self, p2d, p3d, sigma2, fx, fy, cx, cy, seed, kf_id, frame_id, dead=False, log=False):
        self.p2d = np.asarray(p2d, F32).reshape(-1, 2)
        self.p3d = np.asarray(p3d, F32).reshape(-1, 3)
        self.N = len(self.p2d)
        self.max_err = np.asarray(sigma2, F32) * TH2
        self.fu, self.fv, self.uc, self.vc = float(F32(fx)), float(F32(fy)), float(F32(cx)), float(F32(cy))
        self.seed, self.kf_id, self.frame_id, self.dead = seed, kf_id, frame_id, dead
        self.min_inl, self.eps, self.max_its = ransac_parameters(self.N)
        self.iterations, self.best, self.best_mask, self.best_tcw = 0, 0, np.zeros(self.N, bool), None
        self.cache = {}
        # the device's refine_failed: Refine of the current best set has failed, so it fails again (Refine is a function of the
        # set); the device skips it until a hypothesis improves the best count
        self.refine_failed = False
        # log=True: one entry per hypothesis (call, g, count, kind = below / improve / tie / worse, refine = ok / failed / skipped /
        # None, refine_count) and one per call (kind "call"); read by oracle/pnp_scene.paths_reached
        self.log = [] if log else None
        self.calls = 0

    def hypothesis(self, g):
        """-> (draw indices, PoseDebug, mask, count) of hypothesis g, memoised."""
        if g not in self.cache:
            idx = draws(self.seed, self.kf_id, self.frame_id, g, self.N)
            pws = [[float(c) for c in self.p3d[i]] for i in idx]
            us = [[float(c) for c in self.p2d[i]] for i in idx]
            dbg = compute_pose(pws, us, self.fu, self.fv, self.uc, self.vc)
            mask, cnt = check_inliers(dbg.R, dbg.t, self.p3d, self.p2d, self.fu, self.fv, self.uc, self.vc, self.max_err)
            self.cache[g] = (idx, dbg, mask, cnt)
        return self.cache[g]

    def refine(self):
        sel = np.nonzero(self.best_mask)[0]
        pws = [[float(c) for c in self.p3d[i]] for i in sel]
        us = [[float(c) for c in self.p2d[i]] for i in sel]
        dbg = compute_pose(pws, us, self.fu, self.fv, self.uc, self.vc, tree=True)
        mask, cnt = check_inliers(dbg.R, dbg.t, self.p3d, self.p2d, self.fu, self.fv, self.uc, self.vc, self.max_err)
        return cnt > self.min_inl, tcw_of(dbg.R, dbg.t), mask, cnt

    def iterate(self, n_iterations: int) -> IterResult:
        res = self._iterate(n_iterations)
        if self.log is not None:
            self.log.append(dict(kind="call", call=self.calls, n=n_iterations, ran=res.hypotheses, pose=res.Tcw is not None,
                                 no_more=res.no_more, n_inliers=res.n_inliers, end=self.iterations))
        self.calls += 1
        return res

    def _note(self, **e):
        if self.log is not None:
            self.log.append(dict(call=self.calls, **e))

    def _iterate(self, n_iterations: int) -> IterResult:
        empty = np.zeros(self.N, bool)
        if self.dead or self.N < self.min_inl:
            return IterResult(None, True, empty, 0, 0)
        cur = 0
        while self.iterations < self.max_its or cur < n_iterations:
            g = self.iterations
            cur += 1
            self.iterations += 1
            _, dbg, mask, cnt = self.hypothesis(g)
            if cnt < self.min_inl:
                self._note(kind="below", g=g, count=cnt, refine=None, last=False)
                continue
            kind = "improve" if cnt > self.best else "tie" if cnt == self.best else "worse"
            if cnt > self.best:
                self.best, self.best_mask, self.best_tcw = cnt, mask, tcw_of(dbg.R, dbg.t)
                self.refine_failed = False
            elif kind == "tie" and np.array_equal(mask, self.best_mask):
                kind = "tie_same"
            skipped = self.refine_failed  # the reference runs Refine again on the same set; the device skips it
            ok, T, rmask, rcnt = self.refine()
            self._note(kind=kind, g=g, count=cnt, refine="skipped" if skipped else "ok" if ok else "failed", refine_count=rcnt,
                       refine_n=self.best, last=False)
            if ok:
                self._mark_last(cur, n_iterations)
                return IterResult(T, False, rmask, rcnt, cur)
            self.refine_failed = True
        if self.iterations >= self.max_its:
            if self.best >= self.min_inl:
                return IterResult(self.best_tcw, True, self.best_mask, self.best, cur)
            return IterResult(None, True, empty, 0, cur)
        return IterResult(None, False, empty, 0, cur)

    def _mark_last(self, cur, n_iterations):
        """The entry just logged returned a pose on the last hypothesis the call would have run."""
        if self.log is not None:
            self.log[-1]["last"] = cur == max(self.max_its - (self.iterations - cur), n_iterations, 0)


def correspondences(kps, match_row, n_keep, points_pos, sigma2_table, keep_idx=None, cap=None):
    """The PnPsolver constructor over one SearchByBoW row: keys j < n_keep in order with 0 <= match_row[j] < len(points_pos)
    (extractor key keep_idx[j], octave within the table) -> (p2d, p3d, sigma2, key index)."""
    p2d, p3d, s2, key = [], [], [], []
    for j in range(n_keep):
        p = int(match_row[j])
        if p < 0 or p >= len(points_pos):
            continue
        k = j if keep_idx is None else int(keep_idx[j])
        if k < 0 or (cap is not None and k >= cap):
            continue
        oc = int(kps[k]["octave"])
        if oc < 0 or oc >= len(sigma2_table):
            continue
        p2d.append((kps[k]["x"], kps[k]["y"]))
        p3d.append(points_pos[p])
        s2.append(sigma2_table[oc])
        key.append(j)
    return (np.array(p2d, F32).reshape(-1, 2), np.array(p3d, F32).reshape(-1, 3), np.array(s2, F32), np.array(key, np.int64))
