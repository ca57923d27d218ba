"""Accuracy of the documented one-sided Jacobi rule where EPnP depends on it, against a 50-digit reference (mpmath).

The oracle restates the rule bit for bit, so bit equality with the device says nothing about whether the rule is accurate.  These
helpers measure it, each as a ratio to its first-order bound, so that one constant c (C below) bounds every case:

  eigen     MtM's singular values d (descending) against the exact eigenvalues lambda of the stored matrix:
            |d_i - |lambda|_i| <= c eps d_0.
  span      the span of ut rows 8-11 (the four control-point null vectors) against the exact eigenvectors of the four smallest
            |lambda|: sin Theta <= c eps d_0 / (d_7 - d_8), d from the reference (Davis-Kahan with a backward error of c eps d_0).
  solve     a 6 x K pseudo-inverse solve (cvSolve with CV_SVD) against the exact least-squares solution x*:
            |x - x*| <= c eps (cond |x*| + cond^2 |r| / sigma_max) with r = b - A x* (Wedin's first-order bound; the second term
            vanishes for a consistent system).  Solves that drop a singular value (the SVBkSb threshold) are not least-squares
            solutions and are skipped.

eps = 2^-53 (the unit roundoff of double)."""
from __future__ import annotations

import mpmath as mp
import numpy as np

from oracle import pnp_oracle as P

EPS = 2.0 ** -53
C = 50.0  # measured maxima: eigen 21.2, span 1.1, solve 2.3 (generated matrices); eigen 13.7 on EPnP scenes
DPS = 50


def _mp(A):
    return mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.asarray(A, np.float64)])


def mtm_exact(alphas, us, cam):
    """MtM of fill_M's rows in 50 digits from double alphas (n x 4) and float observations (n x 2)."""
    with mp.workdps(DPS):
        fu, fv, uc, vc = (mp.mpf(float(np.float32(c))) for c in cam)
        A = mp.zeros(12, 12)
        for a, (u, v) in zip(np.asarray(alphas, np.float64), np.asarray(us, np.float64)):
            r1, r2 = [mp.mpf(0)] * 12, [mp.mpf(0)] * 12
            for k in range(4):
                ak = mp.mpf(float(a[k]))
                r1[3 * k], r1[3 * k + 2] = ak * fu, ak * (uc - mp.mpf(float(u)))
                r2[3 * k + 1], r2[3 * k + 2] = ak * fv, ak * (vc - mp.mpf(float(v)))
            for i in range(12):
                for j in range(12):
                    A[i, j] += r1[i] * r1[j] + r2[i] * r2[j]
        return A


def eigen_ratios(d, ut, A):
    """(eigen ratio, span ratio, exact eigenvalues descending by magnitude) for singular values d (12, descending), ut (144,
    row r = the vector of d[r]) and the reference matrix A (mpmath or array)."""
    with mp.workdps(DPS):
        A = A if isinstance(A, mp.matrix) else _mp(A)
        E, Q = mp.eigsy(A)
        order = sorted(range(12), key=lambda i: -abs(E[i]))
        lam = [abs(E[i]) for i in order]
        d0 = lam[0]
        if d0 == 0:
            return 0.0, 0.0, [float(x) for x in lam]
        eig = max(abs(mp.mpf(float(d[i])) - lam[i]) for i in range(12)) / (EPS * d0)
        W = mp.matrix(12, 4)
        U = mp.matrix(12, 4)
        for c, i in enumerate(order[8:]):
            for r in range(12):
                W[r, c] = Q[r, i]
                U[r, c] = mp.mpf(float(ut[12 * (8 + c) + r]))
        Pm = U - W * (W.T * U)
        s2 = max(abs(x) for x in mp.eigsy(Pm.T * Pm)[0])
        gap = lam[7] - lam[8]
        span = mp.sqrt(s2) / (EPS * d0 / gap) if gap > 0 else mp.mpf(0)
        return float(eig), float(span), [float(x) for x in lam]


def solve_ratio(A, b):
    """The documented solve of A x = b (6 x K) against the 50-digit least-squares solution -> ratio to the bound, or None when
    the rule drops a singular value."""
    A = np.asarray(A, np.float64)
    _, _, n2, order = P.jacobi(A.tolist())
    thr = 0.0
    for j in order:
        thr = thr + float(np.sqrt(n2[j]))
    if any(not np.sqrt(n2[j]) > thr * 2.0 ** -51 for j in order):
        return None
    x = np.array(P.solve_svd(A.tolist(), list(b)))
    with mp.workdps(DPS):
        Am, bm = _mp(A), mp.matrix([mp.mpf(float(v)) for v in b])
        xs = mp.lu_solve(Am.T * Am, Am.T * bm)
        r = bm - Am * xs
        sv = mp.svd_r(Am, compute_uv=False)
        smax, smin = max(sv), min(sv)
        if smin == 0:
            return None
        cond = smax / smin
        nx = mp.norm(xs)
        bound = EPS * (cond * nx + cond ** 2 * mp.norm(r) / smax)
        err = mp.norm(mp.matrix([mp.mpf(float(v)) for v in x]) - xs)
        return float(err / bound) if bound > 0 else (0.0 if err == 0 else float("inf"))


def beta_systems(l_6x10, rho):
    """The three 6 x K systems of find_betas_approx_1 / 2 / 3."""
    L = np.asarray(l_6x10, np.float64).reshape(6, 10)
    return [(L[:, [0, 1, 3, 6]], rho), (L[:, [0, 1, 2]], rho), (L[:, :5], rho)]


def spectrum_matrix(rng, kind):
    """A 12 x 12 symmetric test matrix: "spread" (eigenvalues log-uniform over 1e-6 .. 1), "cluster" (four eigenvalues within
    1e-3 of each other near 1e-10, the rest spread), "null4" (rank 8: B^T B with B 8 x 12), "equal" (repeated eigenvalues at the
    top and a cluster of four at the bottom), "mtm" (fill_M's MtM of a noise-free scene: one eigenvalue at rounding level)."""
    Q, _ = np.linalg.qr(rng.normal(size=(12, 12)))
    if kind == "spread":
        lam = 10.0 ** rng.uniform(-6, 0, 12)
    elif kind == "cluster":
        lam = np.r_[10.0 ** rng.uniform(-4, 0, 8), 1e-10 * (1 + 1e-3 * rng.random(4))]
    elif kind == "equal":
        lam = np.r_[[1.0] * 4, 10.0 ** rng.uniform(-3, -1, 4), [1e-9] * 4]
    elif kind == "null4":
        B = rng.normal(size=(8, 12)) * 10.0 ** rng.uniform(-2, 2)
        return B.T @ B
    else:
        n = int(rng.integers(6, 60))
        X = np.c_[rng.uniform(-5, 5, n), rng.uniform(-2, 2, n), rng.uniform(5, 40, n)]
        cam = (718.856, 718.856, 607.1928, 185.2157)
        us = np.c_[cam[0] * X[:, 0] / X[:, 2] + cam[2], cam[1] * X[:, 1] / X[:, 2] + cam[3]]
        dbg = P.compute_pose(X.tolist(), us.tolist(), *cam)
        M = []
        for al, (u, v) in zip(dbg.alphas, us):
            M.append([x for k in range(4) for x in (al[k] * cam[0], 0.0, al[k] * (cam[2] - u))])
            M.append([x for k in range(4) for x in (0.0, al[k] * cam[1], al[k] * (cam[3] - v))])
        M = np.array(M)
        return M.T @ M
    return (Q * lam) @ Q.T


CONDITIONING = [(D, s, h) for D in (5.0, 50.0, 300.0) for s in (1.0, 0.1, 0.01) for h in (1.0, 0.01, 0.001)]


def conditioned_scene(D, s, h, n=50, seed=0):
    """n noise-free correspondences at depth D with lateral spread s and depth thickness h (metres), seen by the true pose
    [R | t] -> (p3d float32, p2d float32, R, t)."""
    rng = np.random.default_rng(seed)
    Pc = np.c_[rng.uniform(-s, s, n), rng.uniform(-s, s, n), D + rng.uniform(-h / 2, h / 2, n)]
    a = rng.normal(size=3)
    ang = rng.uniform(0, np.pi)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * (K @ K)
    t = rng.uniform(-3, 3, 3)
    X = ((Pc - t) @ R).astype(np.float32)
    Xc = X.astype(np.float64) @ R.T + t
    cam = (718.856, 718.856, 607.1928, 185.2157)
    us = np.c_[cam[0] * Xc[:, 0] / Xc[:, 2] + cam[2], cam[1] * Xc[:, 1] / Xc[:, 2] + cam[3]].astype(np.float32)
    return X, us, R, t


def pose_error(Rg, tg, R, t):
    """(max |R - R_true|, |t - t_true| / |t_true|)."""
    Rg, tg = np.asarray(Rg, np.float64).reshape(3, 3), np.asarray(tg, np.float64)
    return float(np.abs(Rg - R).max()), float(np.linalg.norm(tg - t) / np.linalg.norm(t))


def check_pose_debug(alphas, us, dbg, cam):
    """The three ratios (eigen, span, worst solve or 0) of one compute_pose's intermediates (PoseDebug or sivo_pnp_pose_debug):
    MtM rebuilt in 50 digits from its alphas and the float observations; the solves on its L_6x10 and rho."""
    A = mtm_exact(alphas, us, cam)
    e, sp, _ = eigen_ratios(list(dbg.d), list(dbg.ut), A)
    sol = [solve_ratio(M, b) for M, b in beta_systems(list(dbg.l_6x10), list(dbg.rho))]
    return e, sp, max([r for r in sol if r is not None] + [0.0])
