"""Optimizer::PoseOptimization (src/orbslam/Optimizer.cc:273-491) and the g2o code it runs, restated literally in numpy float64.
Test infrastructure only: the product path is sivo_b200/csrc/pose.cu.

The g2o sources restated (dependencies/g2o/g2o/):
  core/optimization_algorithm_levenberg.cpp   solve(): the trial loop, computeLambdaInit, computeScale
  core/sparse_optimizer.cpp                   initializeOptimization(level), sortVectorContainers, optimize, activeRobustChi2
  core/base_unary_edge.hpp                    constructQuadraticForm (b -= rho1 A^T Omega e, H += A^T (rho1 Omega) A)
  core/robust_kernel_impl.cpp                 RobustKernelHuber::robustify
  core/base_edge.h                            robustInformation (rho1 Omega only), chi2
  core/marginal_covariance_cholesky.cpp       computeEntry / computeCovariance
  types/sba/types_six_dof_expmap.{h,cpp}      the two pose-only edges: computeError, cam_project, linearizeOplus
  types/slam3d/se3quat.h                      SE3Quat: exp, operator*, map, normalizeRotation
and Eigen 3's quaternion formulas (quaternion from a rotation matrix, the quaternion product, q * v, toRotationMatrix).

Reference facts kept as they are, not fixed:
  edges      one per semantic key with a map point (xw[j, 0] not NaN), created in key order; stereo iff mvRight[j] >= 0 (so a NaN
             mvRight makes a stereo edge).  sortVectorContainers orders the active edges by insertion id, so every sum over
             edges runs in key order ("sequential"; the kernel's fixed tree is "device", below).
  info       Omega = I * mvInvLevelSigma2[octave], the float widened to double.  Huber deltas sqrt(5.991f) (mono) and sqrt(7.815f)
             (stereo) in float, widened: delta^2 is neither 5.991 nor 7.815 exactly.
  robust     robustInformation uses rho1 Omega only; g = ((rho1 A[i][k]) info) e[i] summed over i, b = -sum over edges of g;
             h[k][l] = (A[i][k] (rho1 info)) A[i][l] summed over i; activeRobustChi2 sums rho0 (chi2 for an edge without kernel).
             chi2 = ((e0 (info e0) + e1 (info e1)) + e2 (info e2)).
  project    mono: u = (x / z) fx + cx in double.  Stereo: invz = (float)(1.0 / z) (`const float invz = 1.0f / z`,
             types_six_dof_expmap.cpp:575-582), u = ((x invz) fx) + cx, ur = u - bf invz.  Jacobians as linearizeOplus writes them
             (:543-565, :610-641), update order [omega, upsilon].
  oplus      SE3Quat::exp(delta) * T with the theta < 1e-5 branch; the product renormalises the quaternion (normalizeRotation:
             negate if w < 0, then divide by the norm).
  LM         tau = 1e-5, lambda re-initialised at iteration 0 of every optimize(); at most 10 trials after a failure; scale =
             x . (lambda x + b) + 1e-3; Terminate when qmax == 10 || rho == 0 || !isfinite(lambda).  A failed factorisation sets
             tempChi = DBL_MAX and leaves x as the last successful solve of the call left it (g2o's solver buffer; its first
             contents are uninitialised memory in a release build, taken as zeros here).
  rounds     4 rounds of optimize(10), each from the INPUT pose (pFrame->mTcw is not updated between rounds); a round whose level-0
             edge set is empty does nothing (optimize() returns -1) and leaves the input pose.
  classify   only stereo edges are classified (SIVO: mono edges never become outliers and keep their kernel).  Outlier iff
             (float) chi2 > 7.815f.  After round 2's classification the stereo kernels are removed.  The loop breaks after a round
             when the total edge count is below 10.
  stale      an inlier's chi2 is the one the last computeActiveErrors left, possibly at a rejected trial's estimate (pop() does
             not recompute errors); only edges already flagged outlier call computeError() at the round's final estimate.
  early      below 3 edges the function returns 0 at once, with the flags of the added edges false and the pose untouched.
  result     the pose is Converter::toCvMat(SE3Quat): toRotationMatrix in double, rounded to float.  nGood = nInitial - nBad of
             the last round run.  Ow = -Rcw^T tcw by camera_centre (Frame::UpdatePoseMatrices).
  marginals  Sigma = the inverse of the last buildSystem's H (diagonal restored) of the last round run: its level-0 edges and that
             round's kernels.  LL^T factor (natural order here), then MarginalCovarianceCholesky's recursion.  A factorisation that
             meets a pivot that is not > 0, or a last round without level-0 edges, means no covariance (sigma_valid 0).

The NaN rule (the reference feeds such an edge on, with undefined effect): an edge is valid at a pose iff its chi2 is finite and
1 / z^2 is finite (z the camera-frame depth; z = 0 included).  An invalid edge contributes nothing to H, b or the robust chi2 of
that pass, its stored chi2 is NaN, and a classified (stereo) invalid edge is an outlier: outlier iff not ((float) chi2 <= 7.815f).

Unpinned (the order of operations of code that is not built here): CHOLMOD's AMD permutation and supernodal / simplicial choice
(natural order here); Eigen's quaternion-from-matrix, quaternion product, cross product, q * v and toRotationMatrix operation
orders, its 3-term sums and its product kernels (Eigen 3's scalar formulas here); sin / cos / pow.

Replay: se3_exp's sin(theta), cos(theta), pow(theta, 3) and the lambda update's pow(2 rho - 1, 3) come from a Transcendentals
source, Python's math by default.  pose_optimization(..., replay=calls) takes them from calls instead, in call order, each after
asserting that the argument computed here has the bits of the one recorded; with the device's own values (sivo_dbg_pose_trace)
every other operation is restated, so the whole optimisation is comparable bit for bit.  The log it returns holds one record per
transcendental call, per trial and per round, with sivo_pose_trace_rec's field names.

Reductions over edges, `order`:
  "sequential"  s = 0; s = s + v_e in key order (g2o).
  "device"      the kernel's fixed tree: 256 threads, thread t sums the edges t, t + 256, t + 512, ... in order from 0; each warp
                of 32 folds by xor shuffles (lane l + lane l ^ s for s = 16, 8, 4, 2, 1); the 8 warp totals fold as w[i] + w[i + s]
                for s = 4, 2, 1.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

F32, F64 = np.float32, np.float64
THREADS, WARP = 256, 32
DELTA_MONO = F64(np.sqrt(F32(5.991)))
DELTA_STEREO = F64(np.sqrt(F32(7.815)))
CHI2_STEREO = F32(7.815)
TAU = 1e-5
MAX_TRIALS = 10
ITERATIONS = 10
DBL_MAX = np.finfo(F64).max


# ---------------------------------------------------------------------------------------------------------- quaternions (Eigen 3)
def normalize_rotation(q):
    """SE3Quat::normalizeRotation: q = (x, y, z, w)."""
    x, y, z, w = (float(v) for v in q)
    if w < 0:
        x, y, z, w = -x, -y, -z, -w
    n2 = ((x * x + y * y) + z * z) + w * w
    if n2 > 0:
        n = math.sqrt(n2)
        x, y, z, w = x / n, y / n, z / n, w / n
    return np.array([x, y, z, w], F64)


def quat_from_matrix(m):
    """Eigen's quaternionbase_assign_impl<Matrix3>: (x, y, z, w)."""
    m = np.asarray(m, F64)
    q = [0.0, 0.0, 0.0, 0.0]
    t = (float(m[0, 0]) + float(m[1, 1])) + float(m[2, 2])
    if t > 0:
        t = math.sqrt(t + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0] = (float(m[2, 1]) - float(m[1, 2])) * t
        q[1] = (float(m[0, 2]) - float(m[2, 0])) * t
        q[2] = (float(m[1, 0]) - float(m[0, 1])) * t
    else:
        i = 0
        if m[1, 1] > m[0, 0]:
            i = 1
        if m[2, 2] > m[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = math.sqrt(((float(m[i, i]) - float(m[j, j])) - float(m[k, k])) + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (float(m[k, j]) - float(m[j, k])) * t
        q[j] = (float(m[j, i]) + float(m[i, j])) * t
        q[k] = (float(m[k, i]) + float(m[i, k])) * t
    return np.array(q, F64)


def quat_mul(a, b):
    """Eigen's quat_product: a * b."""
    ax, ay, az, aw = (float(v) for v in a)
    bx, by, bz, bw = (float(v) for v in b)
    return np.array([((aw * bx + ax * bw) + ay * bz) - az * by,
                     ((aw * by + ay * bw) + az * bx) - ax * bz,
                     ((aw * bz + az * bw) + ax * by) - ay * bx,
                     ((aw * bw - ax * bx) - ay * by) - az * bz], F64)


def _cross(a, b):
    """a x b with a (3,) and b (..., 3)."""
    b = np.asarray(b, F64)
    return np.stack([a[1] * b[..., 2] - a[2] * b[..., 1], a[2] * b[..., 0] - a[0] * b[..., 2], a[0] * b[..., 1] - a[1] * b[..., 0]], -1)


def transform(q, v):
    """Eigen's q * v (_transformVector): uv = q.vec x v; uv += uv; v + w uv + q.vec x uv.  v (..., 3)."""
    qv = np.asarray(q[:3], F64)
    v = np.asarray(v, F64)
    uv = _cross(qv, v)
    uv = uv + uv
    return (v + F64(q[3]) * uv) + _cross(qv, uv)


def rotation_matrix(q):
    """Eigen's toRotationMatrix."""
    x, y, z, w = (float(v) for v in q)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy)]], F64)


@dataclass
class Pose:
    q: np.ndarray  # (x, y, z, w)
    t: np.ndarray

    def map(self, X):
        """SE3Quat::map: q * X + t."""
        return transform(self.q, X) + self.t


def to_se3quat(Tcw) -> Pose:
    """Converter::toSE3Quat: the float 3 x 4 (or 4 x 4) pose widened; SE3Quat(R, t) normalises."""
    T = np.asarray(Tcw, F32).reshape(-1, 4)[:3].astype(F64)
    return Pose(normalize_rotation(quat_from_matrix(T[:, :3])), T[:, 3].copy())


def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]], F64)


def _mat3(a, b):
    """3 x 3 product, each entry ((a0 b0 + a1 b1) + a2 b2)."""
    return np.array([[(a[i, 0] * b[0, j] + a[i, 1] * b[1, j]) + a[i, 2] * b[2, j] for j in range(3)] for i in range(3)], F64)


def _same_bits(a, b) -> bool:
    a, b = float(a), float(b)
    return (a != a and b != b) or np.float64(a).view(np.int64) == np.float64(b).view(np.int64)


TRANSCENDENTAL_KINDS = ("sin", "cos", "pow_theta", "pow_rho")


class Transcendentals:
    """The source of sin(theta), cos(theta), pow(theta, 3) ("pow_theta") and pow(2 rho - 1, 3) ("pow_rho"): Python's math, or
    `replay`, a sequence of {"kind", "arg", "value"} taken in call order (other kinds skipped) after checking the kind and the
    argument's bits.  Every call is appended to `log` (when given) with the current `where` (round, iteration, trial)."""

    def __init__(self, replay=None, log=None):
        self.calls = None if replay is None else [c for c in replay if c["kind"] in TRANSCENDENTAL_KINDS]
        self.used = 0
        self.log = log
        self.where = (0, 0, 0)

    def __call__(self, kind, arg):
        arg = float(arg)
        if self.calls is None:
            value = math.sin(arg) if kind == "sin" else math.cos(arg) if kind == "cos" else math.pow(arg, 3)
        else:
            assert self.used < len(self.calls), f"replay: no recorded value left for {kind}({arg!r})"
            c = self.calls[self.used]
            assert c["kind"] == kind and _same_bits(c["arg"], arg), \
                f"replay call {self.used}: {kind}({arg.hex()}) here, {c['kind']}({float(c['arg']).hex()}) recorded"
            value = float(c["value"])
            self.used += 1
        if self.log is not None:
            r, it, q = self.where
            self.log.append({"kind": kind, "round": r, "iteration": it, "trial": q, "arg": arg, "value": value})
        return value


MATH = Transcendentals()


def se3_exp(delta, tx: Transcendentals = MATH) -> Pose:
    """SE3Quat::exp(update): update = [omega, upsilon]."""
    d = [float(v) for v in delta]
    omega, upsilon = d[:3], d[3:]
    theta = math.sqrt((omega[0] * omega[0] + omega[1] * omega[1]) + omega[2] * omega[2])
    O = skew(omega)
    I3 = np.eye(3)
    if theta < 0.00001:
        R = (I3 + O) + _mat3(O, O)
        V = R
    else:
        O2 = _mat3(O, O)
        s, c = tx("sin", theta), tx("cos", theta)
        R = (I3 + (s / theta) * O) + ((1 - c) / (theta * theta)) * O2
        V = (I3 + ((1 - c) / (theta * theta)) * O) + ((theta - s) / tx("pow_theta", theta)) * O2
    t = np.array([(V[i, 0] * upsilon[0] + V[i, 1] * upsilon[1]) + V[i, 2] * upsilon[2] for i in range(3)], F64)
    return Pose(normalize_rotation(quat_from_matrix(R)), t)


def oplus(delta, T: Pose, tx: Transcendentals = MATH) -> Pose:
    """VertexSE3Expmap::oplusImpl: exp(delta) * T (SE3Quat::operator*)."""
    E = se3_exp(delta, tx)
    return Pose(normalize_rotation(quat_mul(E.q, T.q)), E.t + transform(E.q, T.t))


def camera_centre(Rcw, tcw) -> np.ndarray:
    """mOw = -Rcw^T tcw: each entry the double sum of the three products, rounded to float (as sivo_b200.track computes it)."""
    R = np.asarray(Rcw, F32).reshape(3, 3).astype(F64)
    t = np.asarray(tcw, F32).reshape(3).astype(F64)
    return np.array([-F32((R[0, r] * t[0] + R[1, r] * t[1]) + R[2, r] * t[2]) for r in range(3)], F32)


# ---------------------------------------------------------------------------------------------------------- edges
@dataclass
class Camera:
    fx: float
    fy: float
    cx: float
    cy: float
    mbf: float

    def __post_init__(self):
        for k in ("fx", "fy", "cx", "cy", "mbf"):
            setattr(self, k, F64(F32(getattr(self, k))))


@dataclass
class Edges:
    key: np.ndarray     # semantic-key index of each edge, ascending
    obs: np.ndarray     # (n, 3): u, v, u_right (0 for mono)
    X: np.ndarray       # (n, 3) world position
    info: np.ndarray    # (n,) mvInvLevelSigma2[octave]
    stereo: np.ndarray  # (n,) bool

    def __len__(self):
        return len(self.key)


def make_edges(kps, u_right, xw, inv_sigma2) -> Edges:
    """One edge per key j whose xw[j, 0] is not NaN, in key order."""
    xw = np.asarray(xw, F32).reshape(-1, 3)
    ur = np.asarray(u_right, F32)
    inv = np.asarray(inv_sigma2, F32)
    key = np.flatnonzero(~np.isnan(xw[:, 0]))
    stereo = ~(ur[key] < 0)
    obs = np.zeros((len(key), 3), F64)
    obs[:, 0] = kps["x"][key]
    obs[:, 1] = kps["y"][key]
    obs[:, 2] = np.where(stereo, ur[key], F32(0))
    return Edges(key, obs, xw[key].astype(F64), inv[kps["octave"][key]].astype(F64), stereo)


def huber(chi2, delta):
    """RobustKernelHuber::robustify: (rho0, rho1) for chi2 = e and the (double) delta."""
    chi2 = np.asarray(chi2, F64)
    dsqr = np.asarray(delta, F64) * delta
    with np.errstate(invalid="ignore"):
        sqrte = np.sqrt(chi2)
        inl = chi2 <= dsqr
        return np.where(inl, chi2, (2 * sqrte) * delta - dsqr), np.where(inl, 1.0, delta / sqrte)


@dataclass
class EdgeEval:
    err: np.ndarray    # (n, 3)
    chi2: np.ndarray   # (n,), NaN for an invalid edge
    rho0: np.ndarray
    rho1: np.ndarray
    valid: np.ndarray
    J: np.ndarray | None = None  # (n, 3, 6)


def evaluate(E: Edges, T: Pose, cam: Camera, robust, jacobian=False) -> EdgeEval:
    """computeError, chi2 and the Huber weights of every edge at T (robust: bool per edge), plus linearizeOplus."""
    P = T.map(E.X)
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    st = E.stereo
    with np.errstate(all="ignore"):
        u_m = (x / z) * cam.fx + cam.cx
        v_m = (y / z) * cam.fy + cam.cy
        invz_f = (F64(1.0) / z).astype(F32).astype(F64)
        u_s = (x * invz_f) * cam.fx + cam.cx
        v_s = (y * invz_f) * cam.fy + cam.cy
        r_s = u_s - cam.mbf * invz_f
        err = np.zeros((len(E), 3), F64)
        err[:, 0] = E.obs[:, 0] - np.where(st, u_s, u_m)
        err[:, 1] = E.obs[:, 1] - np.where(st, v_s, v_m)
        err[:, 2] = np.where(st, E.obs[:, 2] - r_s, 0.0)
        info = E.info
        chi2 = err[:, 0] * (info * err[:, 0]) + err[:, 1] * (info * err[:, 1])
        chi2 = np.where(st, chi2 + err[:, 2] * (info * err[:, 2]), chi2)
        invz = F64(1.0) / z
        invz_2 = invz * invz
        valid = np.isfinite(chi2) & np.isfinite(invz_2)
        chi2 = np.where(valid, chi2, np.nan)
        rho0, rho1 = huber(chi2, np.where(st, DELTA_STEREO, DELTA_MONO))
        robust = np.asarray(robust, bool)
        rho0 = np.where(robust, rho0, chi2)
        rho1 = np.where(robust, rho1, 1.0)
        J = None
        if jacobian:
            fx, fy, bf = cam.fx, cam.fy, cam.mbf
            J = np.zeros((len(E), 3, 6), F64)
            J[:, 0, 0] = ((x * y) * invz_2) * fx
            J[:, 0, 1] = (-(1 + ((x * x) * invz_2))) * fx
            J[:, 0, 2] = (y * invz) * fx
            J[:, 0, 3] = (-invz) * fx
            J[:, 0, 5] = (x * invz_2) * fx
            J[:, 1, 0] = (1 + ((y * y) * invz_2)) * fy
            J[:, 1, 1] = (((-x) * y) * invz_2) * fy
            J[:, 1, 2] = ((-x) * invz) * fy
            J[:, 1, 4] = (-invz) * fy
            J[:, 1, 5] = (y * invz_2) * fy
            s = st.astype(F64)
            J[:, 2, 0] = np.where(st, J[:, 0, 0] - ((bf * y) * invz_2), 0.0)
            J[:, 2, 1] = np.where(st, J[:, 0, 1] + ((bf * x) * invz_2), 0.0)
            J[:, 2, 2] = J[:, 0, 2] * s
            J[:, 2, 3] = J[:, 0, 3] * s
            J[:, 2, 5] = np.where(st, J[:, 0, 5] - (bf * invz_2), 0.0)
    return EdgeEval(err, chi2, rho0, rho1, valid, J)


UPPER = [(k, l) for k in range(6) for l in range(k, 6)]  # the 21 entries of H the kernel sums, row by row


def edge_terms(E: Edges, ev: EdgeEval) -> np.ndarray:
    """(n, 28): per edge h[k][l] for the 21 upper entries, then g[0..5] (b = -sum g), then rho0."""
    st = E.stereo
    w = ev.rho1 * E.info
    out = np.zeros((len(E), 28), F64)
    with np.errstate(all="ignore"):
        for q, (k, l) in enumerate(UPPER):
            s = (ev.J[:, 0, k] * w) * ev.J[:, 0, l] + (ev.J[:, 1, k] * w) * ev.J[:, 1, l]
            out[:, q] = np.where(st, s + (ev.J[:, 2, k] * w) * ev.J[:, 2, l], s)
        for k in range(6):
            s = ((ev.rho1 * ev.J[:, 0, k]) * E.info) * ev.err[:, 0] + ((ev.rho1 * ev.J[:, 1, k]) * E.info) * ev.err[:, 1]
            out[:, 21 + k] = np.where(st, s + ((ev.rho1 * ev.J[:, 2, k]) * E.info) * ev.err[:, 2], s)
    out[:, 27] = ev.rho0
    return out


def tree_sum(acc):
    """The device's fixed reduction tree over per-thread sums acc (THREADS, ...) of a THREADS-thread block: xor shuffles
    16 .. 1 within each warp (lane 0's sum adds the halves, w[i] + w[i + s] for s = 16 .. 1), then the warp totals folded as
    w[i] + w[i + s] for s = 4, 2, 1."""
    w = np.asarray(acc, F64).reshape(THREADS // WARP, WARP, *np.shape(acc)[1:])
    s = WARP // 2
    while s:
        w = w[:, :s] + w[:, s:2 * s]
        s //= 2
    t = w[:, 0]
    s = THREADS // WARP // 2
    while s:
        t = t[:s] + t[s:2 * s]
        s //= 2
    return t[0]


def reduce_edges(v, order: str) -> np.ndarray:
    """Sum the rows of v (n, m) in the given order (rows in key order; rows of edges left out must be zero)."""
    v = np.asarray(v, F64)
    m = v.shape[1]
    if len(v) == 0:
        return np.zeros(m, F64)
    if order == "sequential":
        return np.add.accumulate(v, axis=0)[-1] + 0.0
    if order != "device":
        raise ValueError(order)
    n_pad = -(-len(v) // THREADS) * THREADS
    p = np.zeros((n_pad, m), F64)
    p[:len(v)] = v
    acc = np.zeros((THREADS, m), F64)
    for k in range(0, n_pad, THREADS):
        acc = acc + p[k:k + THREADS]
    return tree_sum(acc)


@dataclass
class System:
    H: np.ndarray
    b: np.ndarray
    chi: float
    ev: EdgeEval


def system(E: Edges, T: Pose, cam: Camera, robust, active, order: str) -> System:
    """computeActiveErrors + activeRobustChi2 + buildSystem over the active (level-0) edges."""
    ev = evaluate(E, T, cam, robust, jacobian=True)
    terms = edge_terms(E, ev)
    use = np.asarray(active, bool) & ev.valid
    terms[~use] = 0.0
    s = reduce_edges(terms, order)
    H = np.zeros((6, 6), F64)
    for q, (k, l) in enumerate(UPPER):
        H[k, l] = H[l, k] = s[q]
    return System(H, -s[21:27], float(s[27]), ev)


def robust_chi(E: Edges, T: Pose, cam: Camera, robust, active, order: str):
    """computeActiveErrors + activeRobustChi2 only: (sum, EdgeEval)."""
    ev = evaluate(E, T, cam, robust)
    use = np.asarray(active, bool) & ev.valid
    v = np.where(use, ev.rho0, 0.0)[:, None]
    return float(reduce_edges(v, order)[0]), ev


# ---------------------------------------------------------------------------------------------------------- dense 6 x 6 algebra
def cholesky(A):
    """LL^T in natural order; None when a pivot is not > 0."""
    n = len(A)
    L = np.zeros((n, n), F64)
    for j in range(n):
        d = float(A[j, j])
        for k in range(j):
            d = d - L[j, k] * L[j, k]
        if not d > 0:
            return None
        L[j, j] = math.sqrt(d)
        for i in range(j + 1, n):
            s = float(A[i, j])
            for k in range(j):
                s = s - L[i, k] * L[j, k]
            L[i, j] = s / L[j, j]
    return L


def cholesky_solve(L, b):
    n = len(L)
    y = [0.0] * n
    for i in range(n):
        s = float(b[i])
        for k in range(i):
            s = s - L[i, k] * y[k]
        y[i] = s / L[i, i]
    x = [0.0] * n
    for i in range(n - 1, -1, -1):
        s = y[i]
        for k in range(i + 1, n):
            s = s - L[k, i] * x[k]
        x[i] = s / L[i, i]
    return np.array(x, F64)


def marginal_covariance(L):
    """MarginalCovarianceCholesky::computeCovariance for the whole matrix, natural order: entries (r <= c) by decreasing c, then
    decreasing r (the order its sort gives), each by computeEntry's recursion."""
    n = len(L)
    diag = [1.0 / L[r, r] for r in range(n)]
    C = np.zeros((n, n), F64)
    for c in range(n - 1, -1, -1):
        for r in range(c, -1, -1):
            s = 0.0
            for rr in range(r + 1, n):
                val = C[rr, c] if rr < c else C[c, rr]
                s += val * L[rr, r]
            C[r, c] = diag[r] * (diag[r] - s) if r == c else -s * diag[r]
    return np.triu(C) + np.triu(C, 1).T


# ---------------------------------------------------------------------------------------------------------- Levenberg-Marquardt
@dataclass
class LMState:
    """The solver state that outlives one optimize(): x (the solver's buffer)."""
    x: np.ndarray = field(default_factory=lambda: np.zeros(6, F64))


@dataclass
class Optimized:
    pose: Pose
    chi2: np.ndarray          # per edge, as the last computeActiveErrors left it (NaN for edges not computed)
    H: np.ndarray | None      # the last buildSystem's H
    log: list                 # (iteration, trial, accepted, currentChi, tempChi, lambda, trial pose)


def optimize(E: Edges, T0: Pose, cam: Camera, robust, active, order: str, state: LMState, iterations=ITERATIONS,
             tx: Transcendentals = MATH, trace=None, round_=0) -> Optimized:
    """SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg over the active edges, from T0.  tx: the
    transcendentals' source; trace: a list that receives one record per trial (sivo_pose_trace_rec's fields)."""
    T = T0
    chi2 = np.full(len(E), np.nan)
    log = []
    H = None
    lam, ni = 0.0, 2.0
    for it in range(iterations):
        S = system(E, T, cam, robust, active, order)
        chi2 = np.where(active, S.ev.chi2, chi2)
        H = S.H
        current = S.chi
        if it == 0:
            m = 0.0
            for j in range(6):
                a = abs(float(H[j, j]))
                m = m if a < m else a
            lam, ni = TAU * m, 2.0
        rho, qmax = 0.0, 0
        while True:
            A = H.copy()
            for j in range(6):
                A[j, j] = A[j, j] + lam
            L = cholesky(A)
            if L is not None:
                state.x = cholesky_solve(L, S.b)
            tx.where = (round_, it, qmax)
            lam0, ni0, current0 = lam, ni, current
            trial = oplus(state.x, T, tx)
            temp, ev = robust_chi(E, trial, cam, robust, active, order)
            chi2 = np.where(active, ev.chi2, chi2)
            if L is None:
                temp = DBL_MAX
            rho = current - temp
            scale = 0.0
            for j in range(6):
                scale += state.x[j] * (lam * state.x[j] + S.b[j])
            scale += 1e-3
            rho /= scale
            accepted = rho > 0 and math.isfinite(temp)
            if accepted:
                alpha = 1.0 - tx("pow_rho", 2 * rho - 1)
                alpha = 2.0 / 3.0 if 2.0 / 3.0 < alpha else alpha
                lam *= alpha if 1.0 / 3.0 < alpha else 1.0 / 3.0
                ni = 2.0
                log.append((it, qmax, True, current, temp, lam, trial))
                current = temp
                T = trial
            else:
                lam *= ni
                ni *= 2
                log.append((it, qmax, False, current, temp, lam, trial))
            if trace is not None:
                trace.append({"kind": "trial", "round": round_, "iteration": it, "trial": qmax, "ok2": int(L is not None),
                              "accepted": int(accepted), "current": current0, "temp": float(temp), "lam_before": lam0,
                              "ni_before": ni0, "lam_after": lam, "ni_after": ni, "rho": rho, "x": state.x.copy(),
                              "q": trial.q.copy(), "t": trial.t.copy()})
            if not accepted and not math.isfinite(lam):
                break
            qmax += 1
            if not (rho < 0 and qmax < MAX_TRIALS):
                break
        if qmax == MAX_TRIALS or rho == 0 or not math.isfinite(lam):
            break
    return Optimized(T, chi2, H, log)


@dataclass
class Result:
    Tcw: np.ndarray           # float32 3 x 4
    q: np.ndarray             # double (x, y, z, w)
    t: np.ndarray
    Rcw: np.ndarray
    tcw: np.ndarray
    Rwc: np.ndarray
    Ow: np.ndarray
    sigma: np.ndarray         # 6 x 6 (zeros when not valid)
    sigma_valid: bool
    n_initial: int
    n_bad: int
    n_good: int
    rounds_run: int
    outlier: np.ndarray       # bool per semantic key
    chi2: np.ndarray          # per edge: the chi2 the last classification tested (NaN where none)
    edges: Edges
    logs: list               # per round: robust, active, the LM log and the round's final pose
    H: np.ndarray | None = None  # the last buildSystem's H


def _result(Tcw, T: Pose, n_keys, E, outlier, sigma, valid, n_bad, n_good, rounds, chi2, logs) -> Result:
    Tcw = np.asarray(Tcw, F32).reshape(-1, 4)[:3].copy()
    R = Tcw[:, :3].copy()
    out = np.zeros(n_keys, bool)
    out[E.key] = outlier
    return Result(Tcw, T.q.copy(), T.t.copy(), R, Tcw[:, 3].copy(), R.T.copy(), camera_centre(R, Tcw[:, 3]),
                  sigma if valid else np.zeros((6, 6), F64), bool(valid), len(E), n_bad, n_good, rounds, out, chi2, E, logs)


def pose_optimization(kps, u_right, xw, Tcw, inv_sigma2, cam: Camera, order: str = "sequential", replay=None, log=False):
    """Optimizer::PoseOptimization for the semantic keys kps (mvKeysSemantic), mvRight, the matched points' positions (NaN x: no
    map point) and the frame's pose (float 3 x 4 or 4 x 4).  Returns the Result; with `replay` (the recorded transcendental
    calls, see Transcendentals) or `log`, (Result, log): the transcendental, trial and round records in the device's order."""
    if replay is None and not log:
        return _pose_optimization(kps, u_right, xw, Tcw, inv_sigma2, cam, order, MATH, None)
    trace = []
    tx = Transcendentals(replay, trace)
    r = _pose_optimization(kps, u_right, xw, Tcw, inv_sigma2, cam, order, tx, trace)
    if replay is not None:
        assert tx.used == len(tx.calls), f"replay: {len(tx.calls) - tx.used} recorded calls left over"
    return r, trace


def _pose_optimization(kps, u_right, xw, Tcw, inv_sigma2, cam, order, tx, trace) -> Result:
    E = make_edges(kps, u_right, xw, inv_sigma2)
    n_keys = len(np.asarray(u_right))
    T_in = to_se3quat(Tcw)
    outlier = np.zeros(len(E), bool)
    if len(E) < 3:
        return _result(Tcw, T_in, n_keys, E, outlier, None, False, 0, 0, 0, np.full(len(E), np.nan), [])
    robust = np.ones(len(E), bool)
    state = LMState()
    n_bad, rounds, logs = 0, 0, []
    chi2_last = np.full(len(E), np.nan)
    T, H = T_in, None
    for r in range(4):
        active = ~outlier
        T, H = T_in, None
        chi2 = np.full(len(E), np.nan)
        log = []
        if active.any():
            o = optimize(E, T_in, cam, robust, active, order, state, tx=tx, trace=trace, round_=r)
            T, H, chi2, log = o.pose, o.H, o.chi2, o.log
        logs.append({"robust": robust.copy(), "active": active.copy(), "lm": log, "pose": T})
        redo = E.stereo & outlier
        if redo.any():
            chi2 = np.where(redo, evaluate(E, T, cam, robust).chi2, chi2)
        with np.errstate(invalid="ignore"):
            bad = E.stereo & ~(chi2.astype(F32) <= CHI2_STEREO)
        outlier = bad
        n_bad = int(bad.sum())
        if trace is not None:
            trace.append({"kind": "round", "round": r, "n_active": int(active.sum()), "n_bad": n_bad, "robust_stereo": int(r < 3)})
        chi2_last = np.where(E.stereo, chi2, np.nan)
        if r == 2:
            robust = ~E.stereo
        rounds = r + 1
        if len(E) < 10:
            break
    L = None if H is None else cholesky(H)
    sigma = None if L is None else marginal_covariance(L)
    R = rotation_matrix(T.q)
    Tout = np.concatenate([R, T.t[:, None]], 1).astype(F32)
    r = _result(Tout, T, n_keys, E, outlier, sigma, L is not None, n_bad, len(E) - n_bad, rounds, chi2_last, logs)
    r.H = H
    return r
