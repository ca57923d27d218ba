"""Constructed frames for the pose-optimisation tests: each scene names the paths of Optimizer::PoseOptimization (and of the
kernel that restates it) it must reach, and `paths_reached` reads them back from the oracle's replay log, so a test can check
both that a scene still reaches what it was built for and that the scenes together reach every path in PATHS.

  rotations   input poses swept over 0 .. pi about x, y, z and (1, 1, 1); exact float matrices with trace 0 (the 120 degree cyclic
              permutation) and the three diagonal half turns, which tie on the diagonal and have w = 0; half turns approached from
              one side, so that an accepted step carries w through 0 and oplus's normalizeRotation flips the sign.
  scale       camera positions 100 .. 600 m from the origin with world points of that size stored as float.
  fixed       dyadic points at power-of-two depths seen from the identity, every error exactly 0: b = 0, x = 0, the trial is the
              current pose and rho = 0 ends the iteration at once.  Mirrored pairs (one point, one octave, observed at +e and -e)
              keep b = 0 while holding a chosen chi2 exactly (`pair_errors`).
  counts      3, 9, 10 and 11 edges; mono-only and stereo-only frames; every stereo edge gross, so rounds 1 - 3 have no edge; every
              point on the camera plane, so every edge is invalid.
  extremes    large finite intrinsics and near-zero depths (chi2 near 1e107, lambda near 1e238).

Also the seeded frames of the pose tests (`scene`, and `exact_scene` at the identity), and `embed`, which lays a frame out per
entry of a semantic-key map (oracle/keymap.py) for the device form.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
from scipy.linalg import expm

from oracle import pose_oracle as P
from sivo_b200.orb import KP_DTYPE

F32, F64 = np.float32, np.float64
INV_SIGMA2 = (F32(1) / np.array([F32(1.2 ** (2 * l)) for l in range(8)], F32)).astype(F32)  # ORBextractor(.., 1.2, 8, ..)
KITTI = (718.856, 718.856, 498.1928, 174.2157, 386.1448)
CAM = P.Camera(*KITTI)
EXACT = (512.0, 512.0, 0.0, 0.0, 256.0)  # the fixed-point scenes' camera: cx = cy = 0, so a point on the axis projects to 0
DSQR_MONO, DSQR_STEREO = P.DELTA_MONO * P.DELTA_MONO, P.DELTA_STEREO * P.DELTA_STEREO

PATHS = (
    "quat_trace_pos", "quat_i0", "quat_i1", "quat_i2", "quat_tie", "input_w_zero", "input_flip", "oplus_flip",
    "kitti_scale", "fixed_point", "chol_fail", "stale_x", "rho_zero", "ten_trials", "accepted", "rejected",
    "dead_round", "all_invalid_round", "sigma_invalid",
    "chi2_7815f", "chi2_7815f_next", "chi2_dsqr_stereo", "chi2_dsqr_stereo_pm", "chi2_dsqr_mono",
    "chi2_dsqr_mono_pm", "ne_3", "ne_9", "ne_10", "ne_11", "mono_only", "stereo_only",
)


@dataclass
class Scene:
    name: str
    kps: np.ndarray
    ur: np.ndarray
    X: np.ndarray
    Tin: np.ndarray
    cam: tuple
    paths: set = field(default_factory=set)

    def camera(self) -> P.Camera:
        return P.Camera(*self.cam)


def axis_rotation(axis, angle) -> np.ndarray:
    """Rodrigues' formula in double."""
    a = np.asarray(axis, F64) / np.linalg.norm(axis)
    K = P.skew(a)
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * (K @ K)


def pose34(R, t) -> np.ndarray:
    return np.concatenate([np.asarray(R, F64), np.asarray(t, F64).reshape(3, 1)], 1).astype(F32)


def posed_scene(seed, R, C, n=120, mode="mixed", noise=0.5, outliers=0.0, motion=(0.01, 0.05), cam=KITTI, depth=(3, 40)):
    """Keys at random pixels and depths seen from the true pose [R | -R C] (camera centre C), points stored as float, pixel noise,
    a fraction of gross outliers and an input pose moved by `motion`.  Returns (kps, ur, X, Tin)."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy, bf = cam
    R = np.asarray(R, F64)
    t = -R @ np.asarray(C, F64)
    u, v = rng.uniform(0, 1024, n), rng.uniform(0, 352, n)
    z = rng.uniform(*depth, n)
    Pc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    X = ((Pc - t) @ R).astype(F32)
    oct_ = rng.integers(0, 8, n)
    sc = 1.2 ** oct_
    kps = np.zeros(n, KP_DTYPE)
    kps["x"] = u + noise * sc * rng.standard_normal(n)
    kps["y"] = v + noise * sc * rng.standard_normal(n)
    kps["octave"] = oct_
    ur = (u - bf / z + noise * sc * rng.standard_normal(n)).astype(F32)
    stereo = {"mono": np.zeros(n, bool), "stereo": np.ones(n, bool), "mixed": rng.uniform(size=n) < 0.6}[mode]
    ur = np.where(stereo, np.maximum(ur, F32(0)), F32(-1)).astype(F32)
    bad = rng.permutation(n)[:int(round(outliers * n))]
    X[bad] = (X[bad] + rng.uniform(-5, 5, (len(bad), 3)) * (1 + np.abs(X[bad]) / 50)).astype(F32)
    dR = axis_rotation(rng.standard_normal(3), rng.uniform(0, motion[0]))
    dt = rng.uniform(-motion[1], motion[1], 3)
    return kps, ur, X, pose34(dR @ R, t + dt)


# ---------------------------------------------------------------------------------------------------------- seeded frames
def rotation(ax, ay, az):
    return expm(np.array([[0, -az, ay], [az, 0, -ax], [-ay, ax, 0]], float))


def scene(seed, n=300, mode="mixed", outliers=0.0, noise=0.5, motion=(0.01, 0.05), cam=CAM, size=(1024, 352)):
    """A frame seen from a true pose: keys at random pixels and depths, their points placed in the world exactly, pixel noise
    (sigma `noise` times the octave's scale), a fraction of the points replaced by gross outliers, and an initial pose moved by
    `motion` (rotation rad, translation m).  mode: "mono" (u_right < 0), "stereo" or "mixed".  Returns (kps, u_right, xw,
    Tcw_in, Tcw_true)."""
    rng = np.random.default_rng(seed)
    R = rotation(*rng.uniform(-0.2, 0.2, 3))
    t = rng.uniform(-2, 2, 3)
    u = rng.uniform(0, size[0], n)
    v = rng.uniform(0, size[1], n)
    z = rng.uniform(3, 40, n)
    Pc = np.stack([(u - cam.cx) * z / cam.fx, (v - cam.cy) * z / cam.fy, z], 1)
    X = ((Pc - t) @ R).astype(F32)
    oct_ = rng.integers(0, 8, n)
    sc = 1.2 ** oct_
    kps = np.zeros(n, KP_DTYPE)
    kps["x"] = u + noise * sc * rng.standard_normal(n)
    kps["y"] = v + noise * sc * rng.standard_normal(n)
    kps["octave"] = oct_
    ur = (u - cam.mbf / z + noise * sc * rng.standard_normal(n)).astype(F32)
    stereo = {"mono": np.zeros(n, bool), "stereo": np.ones(n, bool), "mixed": rng.uniform(size=n) < 0.6}[mode]
    ur = np.where(stereo, np.maximum(ur, F32(0)), F32(-1)).astype(F32)
    bad = rng.permutation(n)[:int(round(outliers * n))]
    X[bad] = (X[bad] + rng.uniform(-5, 5, (len(bad), 3))).astype(F32)
    dR = rotation(*rng.uniform(-motion[0], motion[0], 3))
    dt = rng.uniform(-motion[1], motion[1], 3)
    return kps, ur, X, pose34(dR @ R, t + dt), pose34(R, t)


def exact_scene(mode):
    """Observations that are exact floats of exact projections at the identity pose (fx = 512, power-of-two depths), so the
    optimum is the identity."""
    cam = P.Camera(512.0, 512.0, 320.0, 240.0, 256.0)
    rng = np.random.default_rng(7)
    n = 64
    z = 2.0 ** rng.integers(1, 5, n)
    x = rng.integers(-200, 200, n) / 64.0
    y = rng.integers(-150, 150, n) / 64.0
    kps = np.zeros(n, KP_DTYPE)
    kps["x"] = (x / z) * 512 + 320
    kps["y"] = (y / z) * 512 + 240
    kps["octave"] = rng.integers(0, 8, n)
    ur = (kps["x"] - 256 / z).astype(F32)
    if mode == "mono":
        ur[:] = -1
    elif mode == "mixed":
        ur[::3] = -1
    X = np.stack([x, y, z], 1).astype(F32)
    return cam, kps, ur, X


def embed(km, kps, ur, X):
    """Keys, u_right and points per entry of the map km (oracle/keymap.py): the real keys at their entries; a rejected entry holds
    a point but no key, so it has no edge."""
    K, U, W = np.zeros(km.n_keep, KP_DTYPE), np.zeros(km.n_keep, F32), np.ones((km.n_keep, 3), F32)
    K[km.real], U[km.real], W[km.real] = kps, ur, X
    return K, U, W


# ---------------------------------------------------------------------------------------------------------- fixed points
def exact_base(n=48, seed=7, mode="mixed"):
    """Dyadic points at power-of-two depths observed exactly from the identity with the EXACT camera (every error 0).  Stereo
    keys have u_right = u - 256 / z >= 0; mode "mono" makes every key mono."""
    rng = np.random.default_rng(seed)
    z = 2.0 ** rng.integers(1, 5, n)
    x = rng.integers(64, 400, n) / 64.0 * np.where(rng.uniform(size=n) < 0.5, 1, -1)
    y = rng.integers(-150, 150, n) / 64.0
    kps = np.zeros(n, KP_DTYPE)
    kps["x"] = (x / z) * 512
    kps["y"] = (y / z) * 512
    kps["octave"] = rng.integers(0, 8, n)
    ur = (kps["x"] - 256 / z).astype(F32)
    ur[ur < 0] = -1
    if mode == "mono":
        ur[:] = -1
    elif mode == "stereo":
        keep = ur >= 0
        kps, ur, x, y, z = kps[keep], ur[keep], x[keep], y[keep], z[keep]
    return kps, ur, np.stack([x, y, z], 1).astype(F32)


def chi2_of(e, info, stereo):
    """The oracle's chi2 formula for errors e (3,) and information info."""
    e0, e1, e2 = (float(v) for v in e)
    c = e0 * (info * e0) + e1 * (info * e1)
    return c + e2 * (info * e2) if stereo else c


def three_squares(N):
    """(k0, k1, k2) with k0^2 + k1^2 + k2^2 == N, k0 as large as possible, or None."""
    k0 = math.isqrt(N)
    for a in range(k0, -1, -1):
        r = N - a * a
        for b in range(math.isqrt(r), -1, -1):
            c2 = r - b * b
            if c2 > b * b:
                break
            c = math.isqrt(c2)
            if c * c == c2:
                return a, b, c
    return None


# A mirrored pair: two keys of one octave on one point, observed at proj + e and proj - e, so that their terms of b cancel
# exactly; information 1 (octave 0), so chi2 is the exact sum of the squares.  Three placements of the point (EXACT camera):
#   "mid"   (3, 3, 4): u = v = 384, u_right = 320, where floats are 2^-15 apart: e on the 2^-15 grid, chi2 = N 2^-30.
#   "axis"  (0, 0, 4), mono: u = v = 0, so e may be any float.
#   "far"   (0.5, 0, 2^11), stereo: u = 2^-3, v = 0, u_right = 0: e_u on the 2^-26 grid with |e_u| < 2^-4, e_v any float, e_r = 0.
PAIR_POINT = {"mid": (3.0, 3.0, 4.0), "axis": (0.0, 0.0, 4.0), "far": (0.5, 0.0, 2.0 ** 11)}


def pair_errors(target):
    """name -> (placement, stereo, (e_u, e_v, e_r)) for each chi2 target the pairs reach exactly."""
    t = float(P.CHI2_STEREO)
    out = {}
    for name, T in (("chi2_7815f", t), ("chi2_7815f_next", f32_next(t))):
        k = three_squares(int(T * 2.0 ** 30))
        out[name] = ("mid", True, tuple(v * 2.0 ** -15 for v in k))
    ds, dm = float(P.DELTA_STEREO), float(P.DELTA_MONO)
    out["chi2_dsqr_stereo"] = ("far", True, (0.0, ds, 0.0))
    out["chi2_dsqr_stereo_up"] = ("far", True, (2.0 ** -25, ds, 0.0))
    out["chi2_dsqr_mono"] = ("axis", False, (dm, 0.0, 0.0))
    out["chi2_dsqr_mono_up"] = ("axis", False, (dm, 2.0 ** -25, 0.0))
    return out if target is None else out[target]


def chi2_targets():
    """name -> the chi2 each pair holds.  Two targets have no mirrored pair: (7.815f + next) / 2 and delta^2 - 1 ulp.  With
    information 1 both are 4^a (8 b + 7) on any dyadic grid (7.815f's mantissa is odd, and delta^2 = m^2 2^-44 gives 64 m^2 - 1
    in ulps), so no three dyadic squares sum to them; at other octaves the information's rounding does not reach a given ulp
    either: the coarse term's steps leave a remainder that the fine term, on the grid its placement allows, cannot close."""
    up = lambda x: float(np.nextafter(x, np.inf))
    t = float(P.CHI2_STEREO)
    return {"chi2_7815f": t, "chi2_7815f_next": f32_next(t), "chi2_dsqr_stereo": DSQR_STEREO, "chi2_dsqr_stereo_up": up(DSQR_STEREO),
            "chi2_dsqr_mono": DSQR_MONO, "chi2_dsqr_mono_up": up(DSQR_MONO)}


def add_pair(base, where, stereo, e):
    """The base frame plus a mirrored pair at the placement `where` with errors +e and -e (octave 0)."""
    kps, ur, X = base
    x, y, z = PAIR_POINT[where]
    u0, v0 = x / z * 512, y / z * 512
    r0 = u0 - 256 / z
    add = np.zeros(2, KP_DTYPE)
    add["x"] = [u0 + e[0], u0 - e[0]]
    add["y"] = [v0 + e[1], v0 - e[1]]
    ur2 = np.array([r0 + e[2], r0 - e[2]], F32) if stereo else np.full(2, -1, F32)
    for k, (p0, d) in enumerate(((u0, e[0]), (v0, e[1]))):
        col = add["x" if k == 0 else "y"]
        assert float(col[0]) - p0 == d and float(col[1]) - p0 == -d, "a pair's observation is not a float"
    if stereo:
        assert (ur2 >= 0).all()
    return np.concatenate([kps, add]), np.concatenate([ur, ur2]), np.concatenate([X, np.array([[x, y, z]] * 2, F32)])


def f32_next(x) -> float:
    return float(np.nextafter(F32(x), F32(np.inf)))


def pair_scenes():
    out = []
    base = exact_base()
    for name, (where, stereo, e) in pair_errors(None).items():
        kps, ur, X = add_pair(base, where, stereo, e)
        path = name.replace("_up", "_pm")
        out.append(Scene("pair_" + name, kps, ur, X, pose34(np.eye(3), np.zeros(3)), EXACT, {path, "fixed_point", "rho_zero"}))
    return out


# ---------------------------------------------------------------------------------------------------------- the scene list
def _rot_special():
    return {"cyclic120": np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]], F64), "diag_x": np.diag([1.0, -1, -1]),
            "diag_y": np.diag([-1.0, 1, -1]), "diag_z": np.diag([-1.0, -1, 1])}


def rotation_scenes():
    out = []
    axes = {"x": (1, 0, 0), "y": (0, 1, 0), "z": (0, 0, 1), "xyz": (1, 1, 1)}
    for k, (an, ax) in enumerate(axes.items()):
        for j, ang in enumerate(np.linspace(0, math.pi, 7)):
            R = axis_rotation(ax, ang)
            kps, ur, X, Tin = posed_scene(100 + 10 * k + j, R, np.array([0.5, -0.3, 1.0]) * (j + 1), n=80, outliers=0.1)
            out.append(Scene(f"sweep_{an}_{j}", kps, ur, X, Tin, KITTI))
    for j, (name, R) in enumerate(_rot_special().items()):
        kps, ur, X, _ = posed_scene(200 + j, R, (1.0, 2.0, -3.0), n=60, noise=0.3)
        Tin = pose34(R, -R @ np.array([1.0, 2.0, -3.0]))  # the exact float matrix as the input pose
        paths = {"cyclic120": {"quat_i0"}, "diag_x": {"quat_i0", "input_w_zero"}, "diag_y": {"quat_i1", "input_w_zero"},
                 "diag_z": {"quat_i2", "quat_tie", "input_w_zero"}}[name]
        out.append(Scene(f"special_{name}", kps, ur, X, Tin, KITTI, paths))
    # half turns approached from below: the solution lies past pi about the same axis, so w crosses 0 during the optimisation
    for j, ax in enumerate([(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1), (0.3, -1, 0.2)]):
        R_true = axis_rotation(ax, math.pi + 0.004)
        kps, ur, X, _ = posed_scene(300 + j, R_true, (2.0, -1.0, 0.5), n=100, noise=0.3, motion=(0, 0))
        R_in = axis_rotation(ax, math.pi - 0.004)
        Tin = pose34(R_in, -R_in @ np.array([2.0, -1.0, 0.5]))
        out.append(Scene(f"halfturn_{j}", kps, ur, X, Tin, KITTI, {"oplus_flip"}))
    return out


def scale_scenes():
    out = []
    for j, dist in enumerate((100, 250, 400, 600)):
        rng = np.random.default_rng(400 + j)
        C = rng.standard_normal(3)
        C = C / np.linalg.norm(C) * dist
        R = axis_rotation(rng.standard_normal(3), rng.uniform(0, math.pi))
        kps, ur, X, Tin = posed_scene(400 + j, R, C, n=150, outliers=0.1)
        out.append(Scene(f"kitti_{dist}m", kps, ur, X, Tin, KITTI, {"kitti_scale"}))
    return out


def count_scenes():
    out = []
    for ne in (3, 9, 10, 11):
        kps, ur, X, Tin = posed_scene(500 + ne, axis_rotation((0, 1, 0), 0.3), (0.5, 0, 1), n=ne, noise=0.5)
        out.append(Scene(f"ne_{ne}", kps, ur, X, Tin, KITTI, {f"ne_{ne}"}))
    for mode in ("mono", "stereo"):
        kps, ur, X, Tin = posed_scene(520, axis_rotation((1, 0, 0), 2.0), (1, 1, 1), n=120, mode=mode, outliers=0.2)
        out.append(Scene(f"{mode}_only", kps, ur, X, Tin, KITTI, {f"{mode}_only"}))
    # every stereo edge gross: round 0 flags them all, rounds 1 - 3 have no edge, the pose stays the input and Sigma is invalid
    rng = np.random.default_rng(530)
    kps, ur, X, Tin = posed_scene(530, np.eye(3), (0, 0, 0), n=40, mode="stereo")
    X = rng.uniform(-50, 50, (40, 3)).astype(F32)
    X[:, 2] = rng.uniform(-30, -2, 40)  # behind the camera: invalid at every pose near the input
    out.append(Scene("stereo_all_gross", kps, ur, X, Tin, KITTI, {"dead_round", "sigma_invalid"}))
    # every point on the camera plane at the input pose: every edge invalid, H = 0, lambda = 0, every factorisation fails
    for mode in ("mono", "mixed"):
        kps, ur, X = exact_base(n=24, seed=531, mode=mode)
        X = X.copy()
        X[:, 2] = 0
        out.append(Scene(f"plane_{mode}", kps, ur, X, pose34(np.eye(3), np.zeros(3)), EXACT,
                         {"all_invalid_round", "chol_fail", "ten_trials", "sigma_invalid"}))
    # stereo edges far off their projections and mono points on the camera plane: round 0 solves on the stereo edges and flags
    # them all, so round 1's factorisations fail (H = 0) and its trials reuse round 0's last, nonzero x
    kps, ur, X = exact_base(n=40, seed=532, mode="mixed")
    X = X.copy()
    mono = ur < 0
    X[mono, 2] = 0
    kps["x"][~mono] += 300
    kps["y"][~mono] -= 200
    ur[~mono] += 300
    out.append(Scene("stale_x", kps, ur, X, pose34(np.eye(3), np.zeros(3)), EXACT, {"chol_fail", "stale_x"}))
    return out


# Not reached: a lambda that turns non-finite ("lambda_nonfinite").  Every edge here is mono and robust, and Huber's weight
# delta / sqrt(chi2) cancels one power of the error: with float inputs (|x| <= 3.4e38, z >= 1.4e-45, fx <= 3.4e38) H stays
# below 1e289, so lambda = 1e-5 max|H_jj| is finite; the scene below keeps such extreme values as a plain comparison.
def overflow_scenes():
    """fx = fy = 3e38, points at x = 1e38 and depths near 1e-30: chi2 near 1e107, H near 1e235, lambda near 1e238."""
    n = 12
    kps = np.zeros(n, KP_DTYPE)
    kps["octave"] = np.arange(n) % 8
    X = np.zeros((n, 3), F32)
    X[:, 0] = F32(1e38)
    X[:, 1] = F32(1e37) * np.arange(n)
    X[:, 2] = F32(1e-30) * (1 + np.arange(n))
    return [Scene("overflow", kps, np.full(n, -1, F32), X, pose34(np.eye(3), np.zeros(3)), (3e38, 3e38, 0.0, 0.0, 256.0))]


def fixed_scenes():
    out = []
    for mode in ("mono", "stereo", "mixed"):
        kps, ur, X = exact_base(mode=mode)
        out.append(Scene(f"fixed_{mode}", kps, ur, X, pose34(np.eye(3), np.zeros(3)), EXACT, {"fixed_point", "rho_zero"}))
    return out


def constructed_scenes():
    return rotation_scenes() + scale_scenes() + fixed_scenes() + pair_scenes() + count_scenes() + overflow_scenes()


# ---------------------------------------------------------------------------------------------------------- paths
def quat_branch(m) -> str:
    """Which branch quat_from_matrix takes on m: "trace_pos" or "i0" / "i1" / "i2"; "+tie" when the i choice met a tie."""
    m = np.asarray(m, F64)
    if (m[0, 0] + m[1, 1]) + m[2, 2] > 0:
        return "trace_pos"
    i = 1 if m[1, 1] > m[0, 0] else 0
    i = 2 if m[2, 2] > m[i, i] else i
    tie = m[1, 1] == m[0, 0] or m[2, 2] == m[i, i]
    return f"i{i}" + ("+tie" if tie else "")


def paths_reached(s: Scene, r: P.Result, log) -> set:
    """The paths of PATHS this run reached, read from the scene's input, the Result and the replay log."""
    out = set()
    T = np.asarray(s.Tin, F32).reshape(-1, 4)[:3].astype(F64)
    br = quat_branch(T[:, :3])
    out.add("quat_" + br.split("+")[0])
    if "+tie" in br:
        out.add("quat_tie")
    q = P.quat_from_matrix(T[:, :3])
    if q[3] == 0:
        out.add("input_w_zero")
    if q[3] < 0:
        out.add("input_flip")
    if np.linalg.norm(T[:, 3]) >= 100:
        out.add("kitti_scale")
    E = r.edges
    if len(E) in (3, 9, 10, 11):
        out.add(f"ne_{len(E)}")
    if len(E) >= 3 and not E.stereo.any():
        out.add("mono_only")
    if len(E) >= 3 and E.stereo.all():
        out.add("stereo_only")
    if r.rounds_run and not r.sigma_valid:
        out.add("sigma_invalid")
    trials = [e for e in log if e["kind"] == "trial"]
    rounds = [e for e in log if e["kind"] == "round"]
    T_in = P.to_se3quat(s.Tin)
    cur, last = T_in, None
    for e in trials:
        if (e["round"], e["iteration"]) != last and e["iteration"] == 0 and e["trial"] == 0:
            cur = T_in
        last = (e["round"], e["iteration"])
        raw = P.quat_mul(P.se3_exp(e["x"]).q, cur.q)
        if raw[3] < 0:
            out.add("oplus_flip")
        if not e["ok2"]:
            out.add("chol_fail")
            if np.any(e["x"] != 0):
                out.add("stale_x")
        if not e["accepted"] and not math.isfinite(e["lam_after"]):
            out.add("lambda_nonfinite")
        if e["rho"] == 0:
            out.add("rho_zero")
        if e["trial"] == P.MAX_TRIALS - 1:
            out.add("ten_trials")
        out.add("accepted" if e["accepted"] else "rejected")
        if e["accepted"]:
            cur = P.Pose(np.asarray(e["q"]), np.asarray(e["t"]))
    if any(t["n_active"] > 0 for t in rounds) and any(b["n_active"] == 0 and b["round"] > a["round"] and a["n_active"] > 0
                                                      for a in rounds for b in rounds):
        out.add("dead_round")
    for rd in rounds:
        first = [e for e in trials if e["round"] == rd["round"]][:1]
        if first and first[0]["current"] == 0 and first[0]["lam_before"] == 0 and not first[0]["ok2"]:
            out.add("all_invalid_round")
    if trials and all(np.all(e["x"] == 0) for e in trials) and np.array_equal(r.Tcw, np.asarray(s.Tin, F32).reshape(-1, 4)[:3]) \
            and all(e["rho"] == 0 for e in trials):
        out.add("fixed_point")
    # the chi2 each edge has at the final estimate, against the constructed targets
    if len(E) >= 3:
        ev = P.evaluate(E, P.Pose(r.q, r.t), s.camera(), np.ones(len(E), bool))
        c = ev.chi2
        st = E.stereo
        t = float(P.CHI2_STEREO)
        with np.errstate(invalid="ignore"):
            if (st & (c == t)).any():
                out.add("chi2_7815f")
            if (st & (c == f32_next(t))).any():
                out.add("chi2_7815f_next")
            for name, d, sel in (("stereo", DSQR_STEREO, st), ("mono", DSQR_MONO, ~st)):
                if (sel & (c == d)).any():
                    out.add(f"chi2_dsqr_{name}")
                if (sel & ((c == np.nextafter(d, np.inf)) | (c == np.nextafter(d, -np.inf)))).any():
                    out.add(f"chi2_dsqr_{name}_pm")
    return out
