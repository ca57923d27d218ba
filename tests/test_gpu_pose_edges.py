"""-m gpu: the frame pose on constructed worst cases (oracle/pose_scene.py), large rotations, KITTI-scale poses and seeded fuzz,
bit for bit against the replay oracle: the host form, the device form and sivo_dbg_pose_trace's per-trial, per-round and
transcendental records, with no tolerance and no exemption.  The device's sin / cos / pow values, which the oracle replays, are
held separately to CUDA's documented ulp bounds."""
import math

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from frame_support import extractor, i64, same_bits, sentinel, upload
from oracle import pose_oracle as P
from oracle import pose_scene as PS
from oracle.keymap import keymap, scatter
from sivo_b200 import pose_optimize, pose_optimize_device
from sivo_b200.pose import (TRACE_COS, TRACE_POW_RHO, TRACE_POW_THETA, TRACE_ROUND, TRACE_SIN, TRACE_TRIAL, pose_se3, pose_trace,
                            result_from_bytes)

pytestmark = pytest.mark.gpu

KIND = {TRACE_TRIAL: "trial", TRACE_ROUND: "round", TRACE_SIN: "sin", TRACE_COS: "cos", TRACE_POW_THETA: "pow_theta",
        TRACE_POW_RHO: "pow_rho"}
FIELDS = {"trial": ("round", "iteration", "trial", "ok2", "accepted", "current", "temp", "lam_before", "ni_before", "lam_after",
                    "ni_after", "rho", "x", "q", "t"),
          "round": ("round", "n_active", "n_bad", "robust_stereo"),
          "call": ("round", "iteration", "trial", "arg", "value")}
# CUDA C++ Programming Guide, "Mathematical Functions" (double precision): sin, cos and pow are within 2 ulp (round to nearest)
ULP_BOUND = {"sin": 2, "cos": 2, "pow_theta": 2, "pow_rho": 2}
CALLS = []  # every device transcendental value the tests saw: (kind, arg, value)


@pytest.fixture(scope="module")
def ext():
    return extractor()


def records(rec):
    out = []
    for r in rec:
        k = KIND[int(r["kind"])]
        out.append({"kind": k, **{f: r[f] for f in FIELDS["call" if k not in ("trial", "round") else k]}})
    return out


def check_log(dev, ref):
    assert [d["kind"] for d in dev] == [r["kind"] for r in ref]
    for i, (d, r) in enumerate(zip(dev, ref)):
        for f in FIELDS["call" if d["kind"] not in ("trial", "round") else d["kind"]]:
            assert same_bits(d[f], r[f]), (i, d["kind"], f, d[f], r[f])


def check_exact(res, outl, ref: P.Result):
    assert np.array_equal(res.pose(), ref.Tcw) and same_bits(res.q, ref.q) and same_bits(res.t, ref.t)
    assert np.array_equal(np.array(res.Rcw, np.float32), ref.Rcw.reshape(-1))
    assert np.array_equal(np.array(res.tcw, np.float32), ref.tcw) and np.array_equal(np.array(res.Rwc, np.float32), ref.Rwc.reshape(-1))
    assert np.array_equal(np.array(res.Ow, np.float32), ref.Ow)
    assert same_bits(res.sigma(), ref.sigma) and bool(res.sigma_valid) == ref.sigma_valid
    assert (res.n_initial, res.n_bad, res.n_good, res.rounds_run) == (ref.n_initial, ref.n_bad, ref.n_good, ref.rounds_run)
    assert np.array_equal(outl, ref.outlier)


def run_all(ext, kps, ur, X, Tin, cam, keep_device=True):
    """The trace hook against the replay oracle, then the host form and the device form (permuted keep_idx with -1 and
    out-of-capacity entries) against the traced result's bytes."""
    intr = (cam.fx, cam.fy, cam.cx, cam.cy, cam.mbf)
    res, outl, rec = pose_trace(ext, kps, ur, X, Tin, *intr)
    dev = records(rec)
    CALLS.extend((d["kind"], float(d["arg"]), float(d["value"])) for d in dev if d["kind"] not in ("trial", "round"))
    ref, log = P.pose_optimization(kps, ur, X, Tin, ext.GetInverseScaleSigmaSquares(), cam, order="device", replay=dev)
    check_log(dev, log)
    check_exact(res, outl, ref)
    h, ho = pose_optimize(ext, kps, ur, X, Tin, *intr)
    assert bytes(h) == bytes(res) and np.array_equal(ho, outl)
    if keep_device:
        device_form(ext, kps, ur, X, Tin, intr, ref)
    return ref, log


def device_form(ext, kps, ur, X, Tin, intr, ref):
    """Keys scattered over the extractor's slots by an oracle/keymap.py map, whose rejected entries have a point but no key slot:
    they have no edge, so the result is the oracle's over the real keys."""
    cap = ext.capacity()
    n = len(kps)
    if n + 2 > cap:
        return
    km = keymap(n, cap, np.random.default_rng(n))
    _, U, W = PS.embed(km, kps, ur, X)
    kb, kk, nn = upload(scatter(kps, km.slots, cap, np.zeros(1, kps.dtype))), upload(km.keep), i64(km.n_keep)
    ub, xb, tb = upload(U), upload(W), upload(np.asarray(Tin, np.float32).reshape(-1)[:12])
    rb, ob = sentinel(512, 0, torch.uint8), sentinel(cap, 7, torch.uint8)
    pose_optimize_device(ext, kb.data_ptr(), kk.data_ptr(), nn.data_ptr(), ub.data_ptr(), xb.data_ptr(), *intr, tb.data_ptr(),
                         rb.data_ptr(), ob.data_ptr())
    torch.cuda.synchronize()
    r = result_from_bytes(rb.cpu().numpy())
    o = ob.cpu().numpy()
    check_exact(r, o[km.real].astype(bool), ref)
    assert not o[:km.n_keep][km.src < 0].any() and (o[km.n_keep:] == 7).all()


# ---------------------------------------------------------------------------------------------------------- constructed scenes
SCENES = {s.name: s for s in PS.constructed_scenes()}


@pytest.mark.parametrize("name", list(SCENES))
def test_constructed_scene(ext, name):
    s = SCENES[name]
    ref, log = run_all(ext, s.kps, s.ur, s.X, s.Tin, s.camera())
    assert s.paths <= PS.paths_reached(s, ref, log)


# ---------------------------------------------------------------------------------------------------------- re-posed SCENES
REPOSED = [(seed, n, mode, out, ang, dist) for seed, (n, mode) in enumerate([(120, "mono"), (400, "stereo"), (800, "mixed"),
                                                                            (2000, "mixed")])
           for out in (0.0, 0.3) for ang, dist in ((2.5, 3.0), (math.pi - 0.01, 350.0))]


@pytest.mark.parametrize("seed,n,mode,out,ang,dist", REPOSED)
def test_scenes_at_large_rotations_and_kitti_scale(ext, seed, n, mode, out, ang, dist):
    rng = np.random.default_rng(seed)
    R = PS.axis_rotation(rng.standard_normal(3), ang)
    C = rng.standard_normal(3)
    C = C / np.linalg.norm(C) * dist
    kps, ur, X, Tin = PS.posed_scene(seed, R, C, n=n, mode=mode, outliers=out)
    run_all(ext, kps, ur, X, Tin, P.Camera(*PS.KITTI))


# ---------------------------------------------------------------------------------------------------------- fuzz
@pytest.mark.parametrize("seed", range(200))
def test_fuzz(ext, seed):
    rng = np.random.default_rng(10_000 + seed)
    n = int(rng.choice([0, 1, 2, 3, 5, 9, 10, 11, 40, 255, 256, 257, 700, ext.capacity()])) if seed % 4 == 0 else int(rng.integers(0, 600))
    R = PS.axis_rotation(rng.standard_normal(3), rng.uniform(0, math.pi))
    C = rng.standard_normal(3) * 10.0 ** rng.uniform(-1, 2.8)
    mode = ("mono", "stereo", "mixed")[seed % 3]
    kps, ur, X, Tin = PS.posed_scene(seed, R, C, n=max(n, 1), mode=mode, outliers=float(rng.uniform(0, 0.5)),
                                     noise=float(rng.uniform(0, 2)), motion=(float(rng.uniform(0, 0.1)), float(rng.uniform(0, 0.5))))
    kps, ur, X = kps[:n], ur[:n], X[:n]
    X[rng.uniform(size=n) < 0.1] = np.nan  # keys without a point
    run_all(ext, kps, ur, X, Tin, P.Camera(*PS.KITTI), keep_device=seed % 5 == 0)


# ---------------------------------------------------------------------------------------------------------- SE3Quat hook
def se3_cases():
    """(T (n, 12) float, d (n, 6)): the rotation sweep and the special matrices, random rotations (every quat_from_matrix branch,
    both signs of w) with steps of every size, and theta at 0, -0, 1e-5 and 1e-5 +- 1 ulp."""
    rng = np.random.default_rng(1)
    Ts, ds = [], []
    mats = [PS.axis_rotation(ax, a) for ax in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)) for a in np.linspace(0, np.pi, 101)]
    mats += list(PS._rot_special().values())
    n_rand = 100_000
    q = rng.standard_normal((n_rand, 4))
    mats_r = Rotation.from_quat(q).as_matrix()
    for m in list(mats) + list(mats_r):
        Ts.append(np.concatenate([m, rng.uniform(-600, 600, (3, 1))], 1).astype(np.float32).reshape(-1))
    k = len(Ts)
    w = rng.standard_normal((k, 3))
    w = w / np.linalg.norm(w, axis=1, keepdims=True) * (10.0 ** rng.uniform(-8, 0.5, (k, 1)))
    d = np.concatenate([w, rng.standard_normal((k, 3))], 1)
    specials = [0.0, -0.0, 1e-5, np.nextafter(1e-5, 0), np.nextafter(1e-5, 1), 3.0, np.pi]
    for i, th in enumerate(specials):
        d[i, :3] = [th, 0.0, 0.0]
        d[len(specials) + i, :3] = [0.0, 0.0, th]
    return np.array(Ts), d


def test_se3_functions_bit_for_bit():
    T, d = se3_cases()
    se3, up, tv, res = pose_se3(T, d)
    branches, flips_in, flips_up = set(), 0, 0
    for i in range(len(T)):
        m = T[i].reshape(3, 4).astype(np.float64)
        P0 = P.to_se3quat(T[i])
        assert same_bits(se3[i], np.r_[P0.q, P0.t]), i
        branches.add(PS.quat_branch(m[:, :3]).split("+")[0])
        flips_in += P.quat_from_matrix(m[:, :3])[3] < 0
        theta = tv[i, 0]
        small = theta < 1e-5
        assert np.isnan(tv[i, 1:]).all() == small
        replay = [] if small else [{"kind": k, "arg": theta, "value": v} for k, v in zip(("sin", "cos", "pow_theta"), tv[i, 1:])]
        tx = P.Transcendentals(replay)
        U = P.oplus(d[i], P0, tx)
        assert tx.used == len(replay)
        assert same_bits(up[i], np.r_[U.q, U.t]), i
        E = P.se3_exp(d[i], P.Transcendentals(replay))
        flips_up += P.quat_mul(E.q, P0.q)[3] < 0
        R = P.rotation_matrix(U.q)
        Tout = np.concatenate([R, U.t[:, None]], 1).astype(np.float32)
        assert np.array_equal(np.array(res[i].Tcw, np.float32), Tout.reshape(-1)), i
        assert np.array_equal(np.array(res[i].Ow, np.float32), P.camera_centre(Tout[:, :3], Tout[:, 3])), i
        if not small:
            CALLS.extend((k, theta, v) for k, v in zip(("sin", "cos", "pow_theta"), tv[i, 1:]))
    assert branches == {"trace_pos", "i0", "i1", "i2"} and flips_in > 0 and flips_up > 0


# ---------------------------------------------------------------------------------------------------------- transcendentals
def test_device_transcendentals_within_cudas_ulp_bounds():
    """Every sin / cos / pow value collected above, against a high-precision reference.  Runs after the tests that collect."""
    if not CALLS:
        pytest.skip("no transcendental values collected (run with the rest of the file)")
    try:
        import mpmath
        mpmath.mp.prec = 160
        exact = {"sin": mpmath.sin, "cos": mpmath.cos, "pow_theta": lambda a: a ** 3, "pow_rho": lambda a: a ** 3}
        big = mpmath.mpf
    except ImportError:  # numpy's extended precision (64-bit mantissa on x86)
        exact = {"sin": np.sin, "cos": np.cos, "pow_theta": lambda a: a ** 3, "pow_rho": lambda a: a ** 3}
        big = np.longdouble
    worst = {k: 0.0 for k in ULP_BOUND}
    for kind, arg, val in set(CALLS):
        if not math.isfinite(arg):
            assert math.isnan(val)
            continue
        ref = exact[kind](big(arg))
        err = float(abs(big(val) - ref)) / float(np.spacing(abs(float(ref))))
        worst[kind] = max(worst[kind], err)
        assert err <= ULP_BOUND[kind], (kind, arg, val, err)
    print("largest ulp error:", {k: round(v, 3) for k, v in worst.items()}, "over", len(set(CALLS)), "values")
