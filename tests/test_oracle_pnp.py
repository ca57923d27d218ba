"""CPU: oracle/pnp_oracle.py's rules -- the Jacobi decompositions against numpy and cv2, compute_pose against cv2's EPnP and the
true pose, the RANSAC schedule against a literal transcription, and the draw rule against a literal swap-remove loop."""
import math

import cv2
import numpy as np
import pytest

from oracle import mapping_oracle as MO
from oracle import pnp_oracle as P

F = (718.856, 718.856, 607.1928, 185.2157)


def scene(n, seed, planar=False):
    r = np.random.default_rng(seed)
    Xw = r.uniform(-5, 5, (n, 3))
    if planar:
        Xw[:, 2] = 0.0
    R, _ = cv2.Rodrigues(r.normal(size=3) * 0.3)
    t = np.array([0.1, -0.2, 12.0])
    Xc = Xw @ R.T + t
    fx, fy, cx, cy = F
    u = np.c_[fx * Xc[:, 0] / Xc[:, 2] + cx, fy * Xc[:, 1] / Xc[:, 2] + cy]
    return Xw, u, R, t


def test_null_vector_through_the_shared_jacobi_equals_the_triangulation_rule():
    r = np.random.default_rng(1)
    for _ in range(300):
        A = r.normal(size=(4, 4)) * 10.0 ** r.integers(-3, 4)
        assert P.null_vector4(A) == MO.svd_null_vector(A)


@pytest.mark.parametrize("shape", [(3, 3), (6, 3), (6, 4), (6, 5), (12, 12)])
def test_singular_values_against_numpy(shape):
    r = np.random.default_rng(shape[0] * 7 + shape[1])
    for _ in range(20):
        A = r.normal(size=shape)
        sig, V, U = P.svd(A.tolist())
        ref = np.linalg.svd(A, compute_uv=False)
        assert np.all(np.abs(np.array(sig) - ref) <= 1e-12 * ref[0])


def test_vectors_against_cv2_up_to_sign():
    r = np.random.default_rng(3)
    for n in (3, 12):
        Q, _ = np.linalg.qr(r.normal(size=(n, n)))
        A = Q @ np.diag(np.linspace(10, 1, n)) @ Q.T  # symmetric, separated spectrum
        sig, V, _ = P.svd(A.tolist())
        w, u, vt = cv2.SVDecomp(A)
        V = np.array(V)
        for j in range(n):
            s = np.sign(V[:, j] @ vt[j])
            assert np.abs(V[:, j] * s - vt[j]).max() < 1e-12


def test_solves_and_inverse_against_cv2_including_the_threshold():
    r = np.random.default_rng(4)
    for k in (3, 4, 5):
        A = r.normal(size=(6, k))
        b = r.normal(size=6)
        x = np.array(P.solve_svd(A.tolist(), b.tolist()))
        ref = cv2.solve(A, b, flags=cv2.DECOMP_SVD)[1].ravel()
        assert np.abs(x - ref).max() < 1e-12 * max(1.0, np.abs(ref).max())
    M = r.normal(size=(3, 3))
    assert np.abs(np.array(P.invert_svd(M.tolist())) - cv2.invert(M, flags=cv2.DECOMP_SVD)[1]).max() < 1e-11
    # rank-deficient: a singular value far below 2^-51 * sum(sigma) is dropped by both, one far above is kept by both
    U, _ = np.linalg.qr(r.normal(size=(3, 3)))
    V, _ = np.linalg.qr(r.normal(size=(3, 3)))
    for small, kept in ((1e-18, False), (1e-12, True)):
        A = U @ np.diag([2.0, 1.0, small]) @ V.T
        x = np.array(P.invert_svd(A.tolist()))
        ref = cv2.invert(A, flags=cv2.DECOMP_SVD)[1]
        big = np.abs(x).max() > 1e6
        assert big == kept
        assert np.abs(x - ref).max() <= 1e-4 * np.abs(ref).max()  # cond(A) = 2e12 when kept


@pytest.mark.parametrize("n", [6, 50, 500])
def test_compute_pose_recovers_the_true_pose_and_matches_cv2_epnp(n):
    Xw, u, R, t = scene(n, n)
    d = P.compute_pose(Xw.tolist(), u.tolist(), *F)
    assert np.abs(np.array(d.R) - R).max() <= 1e-9 and np.abs(np.array(d.t) - t).max() <= 1e-9
    K = np.array([[F[0], 0, F[2]], [0, F[1], F[3]], [0, 0, 1.0]])
    ok, rv, tv = cv2.solvePnP(Xw, u, K, None, flags=cv2.SOLVEPNP_EPNP)
    assert ok and np.abs(cv2.Rodrigues(rv)[0] - np.array(d.R)).max() <= 1e-9


def test_four_points_do_not_determine_epnp_and_cv2_agrees():
    """EPnP on a minimal set is not exact: neither the rule nor cv2's own EPnP recovers a 4-point pose in general."""
    Xw, u, R, _ = scene(4, 0)
    d = P.compute_pose(Xw.tolist(), u.tolist(), *F)
    K = np.array([[F[0], 0, F[2]], [0, F[1], F[3]], [0, 0, 1.0]])
    _, rv, _ = cv2.solvePnP(Xw, u, K, None, flags=cv2.SOLVEPNP_EPNP)
    assert np.abs(np.array(d.R) - R).max() > 1e-6 and np.abs(cv2.Rodrigues(rv)[0] - R).max() > 1e-6


def test_gauss_newton_step_against_float64_least_squares():
    r = np.random.default_rng(5)
    A = r.normal(size=(6, 4))
    b = r.normal(size=6)
    x = P.qr_solve([list(row) for row in A], list(b))
    ref = np.linalg.lstsq(A, b, rcond=None)[0]
    assert np.abs(np.array(x) - ref).max() < 1e-12


def test_coplanar_minimal_set_gives_a_nan_pose_and_no_inliers():
    """Coplanar world points make ABt's third column exactly zero: U's column is 0 / 0, so R is NaN and nothing is an inlier."""
    Xw, u, _, _ = scene(4, 2, planar=True)
    d = P.compute_pose(Xw.tolist(), u.tolist(), *F)
    assert np.isnan(np.array(d.R)).any()
    mask, cnt = P.check_inliers(d.R, d.t, Xw.astype(np.float32), u.astype(np.float32), *F, np.full(4, 5.991, np.float32))
    assert cnt == 0 and not mask.any()


class CV2:
    """cv2-backed decompositions for the transcription: cvSVD (U_T / full), cvSolve and cvInvert with DECOMP_SVD."""

    @staticmethod
    def svd_sym(A):
        w, u, vt = cv2.SVDecomp(np.array(A))
        return list(w.ravel()), list(u.T.ravel())

    svd_sym12 = svd_sym

    @staticmethod
    def svd_uv(A):
        w, u, vt = cv2.SVDecomp(np.array(A))
        return u.tolist(), vt.T.tolist()

    @staticmethod
    def solve(A, b):
        return list(cv2.solve(np.array(A), np.array(b), flags=cv2.DECOMP_SVD)[1].ravel())

    @staticmethod
    def invert(A):
        return cv2.invert(np.array(A), flags=cv2.DECOMP_SVD)[1].tolist()


@pytest.mark.parametrize("n", [6, 50, 500])
def test_compute_pose_against_the_transcription_on_cv2_svd(n):
    Xw, u, R, t = scene(n, 100 + n)  # noise-free: with noise the two SVDs' signs can select different beta approximations
    a = P.compute_pose(Xw.tolist(), u.tolist(), *F)
    b = P.compute_pose(Xw.tolist(), u.tolist(), *F, la=CV2)
    assert np.abs(np.array(a.R) - np.array(b.R)).max() <= 1e-9 and np.abs(np.array(a.t) - np.array(b.t)).max() <= 1e-8
    assert abs(a.rep_errors[a.best] - b.rep_errors[b.best]) <= 1e-9


@pytest.mark.parametrize("n", [4, 300, 2000])
def test_refine_tree_sum_against_the_sequential_sum(n):
    Xw, u, _, _ = scene(n, n)
    a = P.compute_pose(Xw.tolist(), u.tolist(), *F)
    b = P.compute_pose(Xw.tolist(), u.tolist(), *F, tree=True)
    M = []
    for i in range(n):
        al = a.alphas[i]
        M.append([x for k in range(4) for x in (al[k] * F[0], 0.0, al[k] * (F[2] - u[i][0]))])
        M.append([x for k in range(4) for x in (0.0, al[k] * F[1], al[k] * (F[3] - u[i][1]))])
    M = np.array(M)
    for r in range(12):
        for c in range(r, 12):
            seq = 0.0
            for x in M[:, r] * M[:, c]:
                seq = seq + x
            tree = P.mtm_tree(M, r, c)
            assert abs(tree - seq) <= 1e-12 * np.abs(M[:, r] * M[:, c]).sum()
    if n > 4:  # a 4-point EPnP is ill-determined: rounding-level changes in MtM move its pose
        assert np.abs(np.array(a.R) - np.array(b.R)).max() <= 1e-9


def literal_parameters(N):
    """SetRansacParameters(0.99, 10, 300, 4, 0.5, 5.991) line by line (float32 where the reference has float)."""
    eps, min_inl, max_its = np.float32(0.5), 10, 300
    nmin = int(np.float32(N) * eps)
    nmin = max(nmin, min_inl)
    nmin = max(nmin, 4)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.float32(nmin) / np.float32(N)
    if eps < q:
        eps = q
    if nmin == N:
        nit = 1
    else:
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.float64(eps)
            x = np.log(1 - 0.99) / np.log(1 - e * e * e)
        nit = -(1 << 31) if not np.isfinite(x) else int(np.ceil(x))
    return nmin, eps, max(1, min(nit, max_its))


def test_parameter_formulas_at_every_N():
    for N in range(0, 4097):
        assert P.ransac_parameters(N) == literal_parameters(N), N
    its = [P.ransac_parameters(N)[2] for N in range(15, 4097)]
    assert min(its) == 14 and max(its) == 35
    small = [P.ransac_parameters(N)[2] for N in range(10, 15)]
    assert small[0] == 1 and small[-1] == 11 and small == sorted(small)
    assert all(P.ransac_parameters(N)[2] == 1 for N in range(0, 10))


def test_draws_against_a_literal_swap_remove_loop():
    for N in (4, 5, 15, 200, 2000):
        for g in range(50):
            w = P.philox4x32_10(np.uint32(g), np.uint32(7), np.uint32(9), np.uint32(0), 1234, 0)
            avail = list(range(N))
            out = []
            for i in range(4):
                r = int(int(w[i]) / 2 ** 32 * (N - i))
                out.append(avail[r])
                avail[r] = avail[len(avail) - 1]
                avail.pop()
            assert P.draws(1234, 7, 9, g, N) == out
            assert len(set(out)) == 4


def synthetic_solver(N, outliers, seed, **kw):
    r = np.random.default_rng(seed)
    Xw, u, _, _ = scene(N, seed)
    bad = r.random(N) < outliers
    u = u + bad[:, None] * r.uniform(-80, 80, (N, 2))
    return P.Solver(u.astype(np.float32), Xw.astype(np.float32), np.ones(N, np.float32), *F, seed=seed, kf_id=3, frame_id=11, **kw)


def test_call_lengths_follow_the_or_condition():
    s = synthetic_solver(40, 0.9, 0)
    s.min_inl = 39  # unreachable: every call runs to its end
    first = s.iterate(5)
    assert first.hypotheses == s.max_its == 35 and first.no_more and first.Tcw is None
    second = s.iterate(5)
    assert second.hypotheses == 5 and s.iterations == 40


def test_refine_runs_on_the_best_set_after_a_non_improving_hypothesis():
    s = synthetic_solver(60, 0.3, 1)
    calls = []
    orig = s.refine

    def spy():
        calls.append((s.iterations, s.best, s.best_mask.copy()))
        ok, T, m, c = orig()
        return False, T, m, c  # force failures so that later hypotheses reach Refine
    s.refine = spy
    s.iterate(50)
    counts = [s.hypothesis(g)[3] for g in range(s.iterations)]
    non_improving = [i for i, (it, best, _) in enumerate(calls) if counts[it - 1] < best]
    assert non_improving, "the scene must contain a hypothesis that reaches minInliers without improving"
    it, best, mask = calls[non_improving[0]]
    assert int(mask.sum()) == best and not np.array_equal(mask, s.hypothesis(it - 1)[2])


def test_no_more_with_and_without_a_best_pose():
    s = synthetic_solver(40, 0.0, 2)
    s.refine = lambda: (False, None, None, 0)
    r = s.iterate(5)
    assert r.no_more and r.Tcw is not None and r.n_inliers == s.best >= s.min_inl
    s = synthetic_solver(40, 1.0, 3)
    r = s.iterate(5)
    assert r.no_more and r.Tcw is None
    s = synthetic_solver(9, 0.0, 4)
    r = s.iterate(5)
    assert r.no_more and r.Tcw is None and r.hypotheses == 0


# ---------------------------------------------------------------------------------------------------------- constructed scenes
def test_constructed_scenes_reach_their_paths_and_together_every_path():
    """oracle/pnp_scene.py: each scene reaches the paths it names, its embedding gives the setup exactly its correspondences,
    and together the scenes reach every path of PATHS except those UNREACHED lists."""
    from oracle import pnp_scene as S
    cap = S.capacity()
    reached = set()
    for sc in S.constructed_scenes():
        s, res, _ = S.run(sc)
        got = S.paths_reached(sc, s, cap=cap)
        assert sc.paths <= got, (sc.name, sc.paths - got)
        reached |= got
        for nlevels in (8, 4):
            if nlevels == 4 and sc.N > 600:
                continue
            fr = S.embed(sc, cap, nlevels, np.random.default_rng(0))
            p2, p3, s2, key = S.frame_correspondences(fr, cap, S.SIGMA2)
            if nlevels == 8:
                assert np.array_equal(p2, sc.p2d) and np.array_equal(p3, sc.p3d) and np.array_equal(s2, S.SIGMA2[sc.octave])
            reached |= fr.paths
    missing = set(S.PATHS) - reached
    assert missing == set(S.UNREACHED), missing
    print(f"{len(reached & set(S.PATHS))} of {len(S.PATHS)} paths reached")


def test_searched_scenes_are_the_first_that_reach_their_paths():
    """SEARCHED records, per family, the first kf_id whose run takes the named paths."""
    from oracle import pnp_scene as S
    for name, kf in S.SEARCHED.items():
        assert S.find_searched(name, 1, kf) == kf, name


def test_the_log_is_additive():
    """The per-hypothesis log changes no result: a logged and an unlogged solver agree call by call."""
    for seed in range(4):
        a, b = synthetic_solver(40, 0.4, seed), synthetic_solver(40, 0.4, seed, log=True)
        for n in (5, 1, 0, 36, 5):
            ra, rb = a.iterate(n), b.iterate(n)
            assert (ra.no_more, ra.n_inliers, ra.hypotheses) == (rb.no_more, rb.n_inliers, rb.hypotheses)
            assert np.array_equal(ra.inliers, rb.inliers) and ((ra.Tcw is None and rb.Tcw is None) or np.array_equal(ra.Tcw, rb.Tcw))
        assert len(b.log) >= 5


# ---------------------------------------------------------------------------------------------------------- 50-digit bounds
def test_jacobi_rule_within_its_bounds_against_50_digits():
    """oracle/pnp_bounds.py on generated matrices: 600 12 x 12 spectra (spread, a clustered near-null four, rank 8, repeated
    eigenvalues, noise-free MtM) and 2400 6 x K solves (K = 3, 4, 5, column scales over 1e-3 .. 1e3, consistent and with a
    residual).  Each error, as a ratio to its first-order bound, stays below C."""
    from oracle import pnp_bounds as B
    rng = np.random.default_rng(2024)
    worst = {"eigen": 0.0, "span": 0.0, "solve": 0.0}
    for i in range(600):
        A = B.spectrum_matrix(rng, ("spread", "cluster", "null4", "equal", "mtm")[i % 5])
        sig, V, _ = P.svd(A.tolist())
        e, sp, _ = B.eigen_ratios(sig, [V[j][r] for r in range(12) for j in range(12)], A)
        worst["eigen"], worst["span"] = max(worst["eigen"], e), max(worst["span"], sp)
    skipped = 0
    for i in range(2400):
        K = 3 + i % 3
        A = rng.normal(size=(6, K)) * 10.0 ** rng.uniform(-3, 3, K)
        if i % 7 == 0:
            A[:, -1] = A[:, 0] + 10.0 ** rng.uniform(-12, -6) * np.abs(A).max() * rng.normal(size=6)  # nearly dependent
        b = A @ rng.normal(size=K) + (rng.normal(size=6) * 10.0 ** rng.uniform(-6, 0) if i % 2 else 0.0)
        r = B.solve_ratio(A, b)
        if r is None:
            skipped += 1
            continue
        worst["solve"] = max(worst["solve"], r)
    print("largest ratio to the bound:", {k: round(v, 2) for k, v in worst.items()}, f"({skipped} solves below the threshold)")
    assert max(worst.values()) <= B.C and skipped < 2400 // 14


def test_compute_pose_within_its_bounds_across_conditioning():
    """The oracle's compute_pose (the device's, bit for bit) on noise-free scenes from 5 m to 300 m depth, spread 1 m to 1 cm,
    thickness 1 m to 1 mm: every decomposition within its bound; the pose error against the true pose is printed."""
    from oracle import pnp_bounds as B
    worst = [0.0, 0.0, 0.0]
    for D, s, h in B.CONDITIONING:
        X, us, R, t = B.conditioned_scene(D, s, h, n=20)
        d = P.compute_pose(X.astype(np.float64).tolist(), us.astype(np.float64).tolist(), *(float(np.float32(c)) for c in F), tree=True)
        r = B.check_pose_debug(d.alphas, us, d, F)
        worst = [max(a, b) for a, b in zip(worst, r)]
        print(f"depth {D:5.0f} m spread {s:5.2f} m thickness {h:6.3f} m: pose error R {B.pose_error(d.R, d.t, R, t)[0]:.1e} "
              f"t {B.pose_error(d.R, d.t, R, t)[1]:.1e}; ratios {[round(x, 2) for x in r]}")
    assert max(worst) <= B.C, worst
