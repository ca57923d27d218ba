"""CPU: oracle/pose_oracle.py, the restatement of Optimizer::PoseOptimization and the g2o code it runs, pinned against closed
forms (scipy's expm, numpy's inverse, central differences) and against its own round and Levenberg-Marquardt rules."""
import math

import numpy as np
import pytest
from scipy.linalg import expm

from oracle import pose_oracle as P
from oracle.pose_scene import CAM, INV_SIGMA2, exact_scene, pose34, rotation, scene

F32 = np.float32


def rot_err(q, R):
    return float(np.abs(P.rotation_matrix(q) - R).max())


# ---------------------------------------------------------------------------------------------------------- SE3Quat::exp
@pytest.mark.parametrize("theta", [0.0, 1e-7, 1e-6, np.nextafter(1e-5, 0), 1e-5, np.nextafter(1e-5, 1), 1e-3, 0.3, 2.0])
def test_exp_against_expm_of_the_twist(theta):
    rng = np.random.default_rng(int(theta * 1e9) % 1000)
    a = rng.standard_normal(3)
    w = theta * a / np.linalg.norm(a)
    ups = rng.standard_normal(3)
    T = P.se3_exp(np.r_[w, ups])
    M = np.zeros((4, 4))
    M[:3, :3] = P.skew(w)
    M[:3, 3] = ups
    E = expm(M)
    assert rot_err(T.q, E[:3, :3]) <= 1e-12
    if math.sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]) < 1e-5:
        # the small branch's V = I + Omega + Omega^2 (g2o's own "TODO: CHECK"), kept as the reference has it: it differs from
        # the exponential's V = I + Omega / 2 + ... by about theta |upsilon| / 2
        O = P.skew(w)
        V = (np.eye(3) + O) + P._mat3(O, O)
        assert np.array_equal(T.t, np.array([(V[i, 0] * ups[0] + V[i, 1] * ups[1]) + V[i, 2] * ups[2] for i in range(3)]))
        assert np.abs(T.t - E[:3, 3]).max() <= theta * np.linalg.norm(ups) + 1e-12
    else:
        assert np.abs(T.t - E[:3, 3]).max() <= 1e-12 * max(1.0, np.abs(E[:3, 3]).max())


def test_oplus_composes_on_the_left():
    rng = np.random.default_rng(3)
    T = P.to_se3quat(pose34(rotation(0.3, -0.2, 0.1), (1.0, -2.0, 0.5)))
    d = np.r_[rng.uniform(-0.1, 0.1, 3), rng.uniform(-0.3, 0.3, 3)]
    U = P.oplus(d, T)
    M = np.eye(4)
    M[:3, :3] = P.rotation_matrix(T.q)
    M[:3, 3] = T.t
    tw = np.zeros((4, 4))
    tw[:3, :3] = P.skew(d[:3])
    tw[:3, 3] = d[3:]
    E = expm(tw) @ M
    assert rot_err(U.q, E[:3, :3]) <= 1e-12 and np.abs(U.t - E[:3, 3]).max() <= 1e-12
    assert U.q[3] >= 0 and abs(np.linalg.norm(U.q) - 1) <= 1e-15


# ---------------------------------------------------------------------------------------------------------- Jacobians, Huber
@pytest.mark.parametrize("stereo", [False, True])
def test_jacobians_against_central_differences(stereo):
    kps, ur, X, Tin, _ = scene(5, n=40, mode="stereo" if stereo else "mono")
    E = P.make_edges(kps, ur, X, INV_SIGMA2)
    T = P.to_se3quat(Tin)
    ev = P.evaluate(E, T, CAM, np.ones(len(E), bool), jacobian=True)
    # the stereo error divides by a float invz, which is piecewise constant at 1e-7 relative: a wider step there
    h, rtol = (1e-3, 2e-4) if stereo else (1e-6, 1e-6)
    for d in range(6):
        step = np.zeros(6)
        step[d] = h
        ep = P.evaluate(E, P.oplus(step, T), CAM, np.ones(len(E), bool)).err
        em = P.evaluate(E, P.oplus(-step, T), CAM, np.ones(len(E), bool)).err
        num = (ep - em) / (2 * h)
        rows = 3 if stereo else 2
        scale = np.abs(ev.J[:, :rows]).max()
        assert np.abs(num[:, :rows] - ev.J[:, :rows, d]).max() <= rtol * scale, d


def test_huber_at_below_and_above_delta_squared():
    for delta in (P.DELTA_MONO, P.DELTA_STEREO):
        d2 = delta * delta
        assert d2 != (5.991 if delta == P.DELTA_MONO else 7.815)
        for e in (np.nextafter(d2, 0), d2):
            r0, r1 = P.huber(e, delta)
            assert r0 == e and r1 == 1.0
        e = np.nextafter(d2, np.inf)
        r0, r1 = P.huber(e, delta)
        assert r0 == (2 * math.sqrt(e)) * delta - d2 and r1 == delta / math.sqrt(e)
        r0, r1 = P.huber(100.0, delta)
        assert r0 == (2 * 10.0) * delta - d2 and r1 == delta / 10.0


# ---------------------------------------------------------------------------------------------------------- marginals
@pytest.mark.parametrize("seed", range(5))
def test_marginal_covariance_is_the_inverse(seed):
    a = np.random.default_rng(seed).standard_normal((6, 6))
    H = a @ a.T + 0.5 * np.eye(6) * (seed + 1)
    S = P.marginal_covariance(P.cholesky(H))
    Ref = np.linalg.inv(H)
    assert np.abs(S - Ref).max() <= 1e-12 * np.abs(Ref).max()
    assert np.array_equal(S, S.T)


def test_cholesky_refuses_a_singular_matrix():
    J = np.random.default_rng(1).standard_normal((3, 6))
    H = J.T @ J
    H[2, :] = H[:, 2] = 0.0
    assert P.cholesky(H) is None


# ---------------------------------------------------------------------------------------------------------- whole optimisation
@pytest.mark.parametrize("mode", ["mono", "stereo", "mixed"])
def test_noise_free_scenes_converge_to_the_true_pose(mode):
    cam, kps, ur, X = exact_scene(mode)
    Tin = pose34(rotation(0.01, -0.02, 0.015), (0.05, -0.03, 0.08))
    r = P.pose_optimization(kps, ur, X, Tin, INV_SIGMA2, cam)
    assert r.rounds_run == 4 and r.n_bad == 0 and r.n_good == len(kps)
    assert rot_err(r.q, np.eye(3)) <= 1e-9 and np.abs(r.t).max() <= 1e-9
    assert r.sigma_valid and np.all(np.linalg.eigvalsh(r.sigma) > 0)


def test_a_rejected_trial_leaves_its_errors_behind():
    """Run to convergence: the trial loop then fails until lambda has grown ten times or a step changes nothing (rho == 0), and
    optimize() ends on a rejected trial.  Every active edge's chi2 is then the one at that trial's estimate, not at the
    restored pose, and the trial's bookkeeping is g2o's."""
    kps, ur, X, Tin, _ = scene(0, n=60, mode="mixed", noise=0.5, outliers=0.3)
    E = P.make_edges(kps, ur, X, INV_SIGMA2)
    robust = np.ones(len(E), bool)
    o = P.optimize(E, P.to_se3quat(Tin), CAM, robust, robust, "sequential", P.LMState(), iterations=200)
    it, trial_no, accepted, current, temp, lam, trial = o.log[-1]
    assert not accepted and it < 199 and (trial_no == P.MAX_TRIALS - 1 or temp == current)
    assert not (np.array_equal(trial.q, o.pose.q) and np.array_equal(trial.t, o.pose.t))
    at_trial = P.evaluate(E, trial, CAM, robust).chi2
    at_pose = P.evaluate(E, o.pose, CAM, robust).chi2
    assert np.array_equal(o.chi2, at_trial) and not np.array_equal(at_trial, at_pose)
    # a rejected trial multiplies lambda by ni = 2, 4, 8, ... and keeps the estimate
    rejected = [e for e in o.log if e[0] == o.log[-1][0]]
    for a, b in zip(rejected, rejected[1:]):
        assert b[5] == a[5] * 2 ** (b[1] + 1)


def test_round_rules():
    # mono edges are never flagged, whatever their error; stereo gross outliers are
    kps, ur, X, Tin, _ = scene(2, n=200, mode="mixed", outliers=0.3)
    r = P.pose_optimization(kps, ur, X, Tin, INV_SIGMA2, CAM)
    mono = ur < 0
    assert not r.outlier[mono].any() and r.outlier[~mono].sum() == r.n_bad > 10
    assert r.n_good == r.n_initial - r.n_bad and r.rounds_run == 4
    # kernels: on for every edge in rounds 0-2, off for stereo edges in round 3; round 0 starts with every edge active and later
    # rounds without some stereo edges; each round starts from the input pose: the currentChi of its first trial is the robust
    # chi2 at the input pose over that round's active edges and kernels
    T_in = P.to_se3quat(Tin)
    for k, log in enumerate(r.logs):
        assert np.array_equal(log["robust"], np.ones(len(r.edges), bool) if k < 3 else ~r.edges.stereo)
        assert log["active"][~r.edges.stereo].all() and (log["active"].all() if k == 0 else not log["active"].all())
        chi_in, _ = P.robust_chi(r.edges, T_in, CAM, log["robust"], log["active"], "sequential")
        assert log["lm"][0][3] == chi_in
    # < 10 edges: one round; < 3: nothing at all, the pose's bits untouched
    keep = np.flatnonzero(~np.isnan(X[:, 0]))[:9]
    X9 = np.full_like(X, np.nan)
    X9[keep] = X[keep]
    assert P.pose_optimization(kps, ur, X9, Tin, INV_SIGMA2, CAM).rounds_run == 1
    X2 = np.full_like(X, np.nan)
    X2[keep[:2]] = X[keep[:2]]
    r2 = P.pose_optimization(kps, ur, X2, Tin, INV_SIGMA2, CAM)
    assert (r2.n_initial, r2.n_good, r2.rounds_run, r2.sigma_valid) == (2, 0, 0, False)
    assert np.array_equal(r2.Tcw, Tin) and not r2.outlier.any()


def test_nan_rule():
    kps, ur, X, Tin, Ttrue = scene(4, n=40, mode="stereo", noise=0.3)
    X = X.copy()
    R, t = Ttrue[:, :3].astype(float), Ttrue[:, 3].astype(float)
    X[0] = ((np.array([0.0, 0.0, 0.0]) - t) @ R).astype(F32)  # on the camera centre at the true pose: z near 0
    X[1] = ((np.array([1.0, 0.5, -10.0]) - t) @ R).astype(F32)  # behind the camera
    E = P.make_edges(kps, ur, X, INV_SIGMA2)
    T = P.to_se3quat(Ttrue)
    Tz = P.Pose(T.q, T.t - T.map(E.X[:1])[0] * np.array([0, 0, 1.0]))  # moves edge 0 onto z = 0 exactly
    ev = P.evaluate(E, Tz, CAM, np.ones(len(E), bool))
    assert P.Pose(Tz.q, Tz.t).map(E.X[:1])[0, 2] == 0 and not ev.valid[0] and np.isnan(ev.chi2[0])
    S = P.system(E, Tz, CAM, np.ones(len(E), bool), np.ones(len(E), bool), "sequential")
    keep = np.ones(len(E), bool)
    keep[0] = False
    S2 = P.system(E, Tz, CAM, np.ones(len(E), bool), keep, "sequential")
    assert np.array_equal(S.H, S2.H) and np.array_equal(S.b, S2.b) and S.chi == S2.chi
    r = P.pose_optimization(kps, ur, X, Ttrue, INV_SIGMA2, CAM)
    assert r.outlier[1]


def test_the_two_reduction_orders_agree():
    for seed, n in ((1, 37), (2, 700), (3, 2000)):
        kps, ur, X, Tin, _ = scene(seed, n=n, outliers=0.1)
        E = P.make_edges(kps, ur, X, INV_SIGMA2)
        T = P.to_se3quat(Tin)
        act = np.random.default_rng(seed).uniform(size=len(E)) > 0.1
        a = P.system(E, T, CAM, np.ones(len(E), bool), act, "sequential")
        b = P.system(E, T, CAM, np.ones(len(E), bool), act, "device")
        assert np.abs(a.H - b.H).max() <= 1e-12 * np.abs(a.H).max()
        assert np.abs(a.b - b.b).max() <= 1e-12 * np.abs(a.b).max() and abs(a.chi - b.chi) <= 1e-12 * a.chi
        assert np.array_equal(a.ev.chi2, b.ev.chi2, equal_nan=True)


# ---------------------------------------------------------------------------------------------------------- constructed scenes
from oracle import pose_scene as PS  # noqa: E402
from scipy.spatial.transform import Rotation  # noqa: E402

_SCENES = {s.name: s for s in PS.constructed_scenes()}


def _run(s):
    return P.pose_optimization(s.kps, s.ur, s.X, s.Tin, PS.INV_SIGMA2, s.camera(), order="device", log=True)


@pytest.mark.parametrize("name", [n for n, s in _SCENES.items() if s.paths])
def test_constructed_scene_reaches_its_paths(name):
    s = _SCENES[name]
    r, log = _run(s)
    assert s.paths <= PS.paths_reached(s, r, log)


def test_constructed_scenes_cover_every_path():
    """Together the scenes reach every path of PATHS.  Not in PATHS because no float input reaches it through a mirrored pair
    or a robust edge: (float) chi2 at the double halfway above 7.815f, chi2 one ulp below delta^2 (see pose_scene.chi2_targets)
    and a lambda that turns non-finite (see pose_scene.overflow_scenes)."""
    got = set()
    for s in _SCENES.values():
        r, log = _run(s)
        got |= PS.paths_reached(s, r, log)
    assert set(PS.PATHS) <= got, set(PS.PATHS) - got


def test_fixed_points_keep_the_input_bits():
    for name in ("fixed_mono", "fixed_stereo", "fixed_mixed", "pair_chi2_7815f"):
        s = _SCENES[name]
        r, log = _run(s)
        assert np.array_equal(r.Tcw, s.Tin) and np.array_equal(r.q, [0, 0, 0, 1]) and np.array_equal(r.t, [0, 0, 0])
        trials = [e for e in log if e["kind"] == "trial"]
        assert len(trials) == 4 and all(e["rho"] == 0 and not e["accepted"] and (e["x"] == 0).all() for e in trials)


def test_pairs_hit_their_chi2_bits():
    for name, target in PS.chi2_targets().items():
        where, stereo, e = PS.pair_errors(name)
        assert PS.chi2_of(e, 1.0, stereo) == target, name
        s = _SCENES["pair_" + name]
        E = P.make_edges(s.kps, s.ur, s.X, PS.INV_SIGMA2)
        c = P.evaluate(E, P.to_se3quat(s.Tin), s.camera(), np.ones(len(E), bool)).chi2
        assert c[-1] == target and c[-2] == target and (c[:-2] == 0).all(), name
    t = float(P.CHI2_STEREO)
    assert int(np.float32(t).view(np.int32)) & 1  # odd mantissa: the halfway double rounds up to the next float
    assert np.float32((t + PS.f32_next(t)) / 2) == np.float32(PS.f32_next(t))


def _sweep_matrices():
    out = []
    for ax in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1), (0.3, -1, 0.2)):
        for ang in np.linspace(0, np.pi, 61):
            out.append(PS.axis_rotation(ax, ang).astype(np.float32).astype(np.float64))
    return out + [m for m in PS._rot_special().values()]


def test_quat_from_matrix_against_scipy():
    for m in _sweep_matrices():
        q = P.normalize_rotation(P.quat_from_matrix(m))
        ref = Rotation.from_matrix(m).as_quat()  # (x, y, z, w), scalar last
        assert min(np.abs(q - ref).max(), np.abs(q + ref).max()) <= 1e-6


def test_to_se3quat_reproduces_the_float_matrix():
    """The float matrix is a rotation to about 1e-7 per entry, so the quaternion's matrix reproduces it to 4e-7."""
    for m in _sweep_matrices():
        T = np.concatenate([m, np.ones((3, 1))], 1).astype(np.float32)
        R = P.rotation_matrix(P.to_se3quat(T).q)
        assert np.abs(R - m).max() <= 4e-7
