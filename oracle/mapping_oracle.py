"""Scalar restatement of LocalMapping::CreateNewMapPoints (LocalMapping.cc:198-472) as SIVO runs it (stereo), with
ORBmatcher::SearchForTriangulation (ORBmatcher.cc:631-785), CheckDistEpipolarLine (:137-159), LocalMapping::ComputeF12 (:639-654)
and SIVO's LocalMapping::CheckSemantics (:474-545).

Reference facts kept:
- SearchForTriangulation declares vbMatched2 and never sets it, and its only caller builds ORBmatcher(0.6, false): no orientation
  histogram.  A neighbour key can be matched by several current keys; no current key's result depends on another's.
- Candidates of current key idx1 (no map point at that moment) are the neighbour's keys in idx1's FeatureVector node, ascending
  index (a node's entry lists its features in index order), without the ones that have a map point on entry.  A key of the
  current keyframe that gets a point at neighbour i has one for every later neighbour (GetMapPoint(idx1)); a neighbour's own
  points change only in its own pair, after its search.
- The fold: bestDist starts at TH_LOW = 50; `dist > TH_LOW || dist > bestDist` skips, so a later candidate at an equal distance
  replaces the best.  The epipole gate applies only when both keys are mono: distex^2 + distey^2 < 100 * mvScaleFactors[octave2]
  (the scale factor, not squared) rejects.
- CheckDistEpipolarLine: a, b, c, num, den, dsqr in float as written; den == 0 rejects; dsqr < 3.84 * sigma2 compares in double
  (the literal is double).
- Baseline: (float) cv::norm(Ow2 - Ow1) < mb skips the neighbour (stereo).  CheckNewKeyFrames() between neighbours is not
  emulated: the caller chooses the neighbours.  The monocular branch is not ported.
- Parallax: cosParallaxRays = (float)(ray1.dot(ray2) / (norm(ray1) * norm(ray2))) in double; cosParallaxStereo2 is set only in
  the `else if (bStereo2)` branch; cos(2 * atan2(mb / 2, depth)) are the float overloads (`using namespace std` reaches
  LocalMapping.cc through DBoW2's TemplatedVocabulary.h, as for PredictScale's log in track_oracle), restated as the correctly
  rounded float functions: float32(atan2 / cos in float64).  glibc's atan2f / cosf are within an ulp of them.
- The checks in order: parallax (else UnprojectStereo of the key with the smaller stereo cosine, else no point), w == 0, z1 <= 0,
  z2 <= 0, reprojection in the current keyframe (5.991 / 7.8 * sigma2 in double), in the neighbour (its stereo error uses the
  CURRENT keyframe's mbf), dist == 0, scale consistency with ratioFactor = 1.5f * mfScaleFactor.
- CheckSemantics(current): depth > 0, class <= max_static_class, (double) confidence >= (float) thConfidence; then MI of the
  triangulated WORLD point (info_oracle's rule: the Jacobian gets world coordinates), sigma2 of the key's octave and the
  keyframe's mSigmacw; VOID iff MI - H < (float) thEntropyReduction, so a NaN reduction passes.  CheckSemantics(neighbour)
  returns its class.  The point is created iff the classes are equal and not VOID (255).

cv::Mat forms (tests/test_oracle_mapping.py pins each against cv2 4.13):
- A * x, A * B (3 x 3 floats, no transpose): ((a0 b0 + a1 b1) + a2 b2) in float (+ c in float for gemm's C term).
- A * B^T (GEMM_2_T): each entry the double sum of the three products, rounded to float.
- Mat::inv of a 3 x 3 float: the closed form, cofactors times 1 / det in double, rounded to float.
- s * T.row(i) - T.row(j): addWeighted in double, rounded to float.
- cv::norm of three floats: sqrt of the double sum of squares.
- Mat::dot of three floats: ((0 + a0 b0) + a1 b1) + a2 b2 in double (Mat::dot has no Python binding: unpinned, as in track_oracle).
- Mat / w: the division of the float vt row by its float fourth entry, in float (unpinned: a MatExpr).

Triangulation (a documented rule; cv::SVD's float Jacobi is not restated): svd_null_vector below, in double, then rounded to float.
Keys whose octave is outside the extractor's levels never take part.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from oracle.info_oracle import stereo_covariance, stereo_jacobian_pose, det3_cofactor, det_lu
from oracle.orb_oracle import descriptor_distance

F32, F64 = np.float32, np.float64
TH_LOW = 50
VOID = 255
MAX_SWEEPS = 30
(HAS_POINT, BASELINE, NO_MATCH, PARALLAX, W_ZERO, Z1, Z2, REPROJ1, REPROJ2, SCALE, SEMANTIC, CREATED) = range(12)


@dataclass
class Camera:
    fx: float
    fy: float
    cx: float
    cy: float
    mbf: float

    def __post_init__(self):
        self.fx, self.fy, self.cx, self.cy, self.mbf = (F32(v) for v in (self.fx, self.fy, self.cx, self.cy, self.mbf))
        self.invfx, self.invfy = F32(1) / self.fx, F32(1) / self.fy
        self.mb = self.mbf / self.fx


@dataclass
class KeyFrame:
    """One keyframe's semantic keys (numpy arrays of one entry per key) and pose."""
    kps: np.ndarray            # KP_DTYPE
    desc: np.ndarray           # (n, 32) uint8
    u_right: np.ndarray
    depth: np.ndarray
    kp_class: np.ndarray
    kp_conf: np.ndarray
    kp_entropy: np.ndarray
    node: np.ndarray
    has_point: np.ndarray
    Rcw: np.ndarray
    tcw: np.ndarray
    Ow: np.ndarray = field(default=None)

    def __post_init__(self):
        self.Rcw = np.asarray(self.Rcw, F32).reshape(3, 3)
        self.tcw = np.asarray(self.tcw, F32).reshape(3)
        if self.Ow is None:
            R = self.Rcw.astype(F64)
            t = self.tcw.astype(F64)
            self.Ow = np.array([-F32((R[0, r] * t[0] + R[1, r] * t[1]) + R[2, r] * t[2]) for r in range(3)], F32)
        self.Ow = np.asarray(self.Ow, F32).reshape(3)
        self.Rwc = np.ascontiguousarray(self.Rcw.T)


# ---------------------------------------------------------------------------------------------------------- cv::Mat forms
def gemm(A, B, C=None) -> np.ndarray:
    """cv::gemm(A, B[, C]) for float matrices without transposes: ((a0 b0 + a1 b1) + a2 b2) [+ c] in float."""
    A = np.asarray(A, F32)
    B = np.asarray(B, F32)
    out = np.empty((A.shape[0], B.shape[1]), F32)
    for i in range(A.shape[0]):
        for j in range(B.shape[1]):
            s = A[i, 0] * B[0, j]
            for k in range(1, A.shape[1]):
                s = s + A[i, k] * B[k, j]
            out[i, j] = s if C is None else s + F32(np.asarray(C, F32)[i, j])
    return out


def gemm_bt(A, B) -> np.ndarray:
    """A * B^T (cv::gemm with GEMM_2_T): each entry the double sum, rounded to float."""
    A = np.asarray(A, F32).astype(F64)
    B = np.asarray(B, F32).astype(F64)
    out = np.empty((A.shape[0], B.shape[0]), F32)
    for i in range(A.shape[0]):
        for j in range(B.shape[0]):
            s = A[i, 0] * B[j, 0]
            for k in range(1, A.shape[1]):
                s = s + A[i, k] * B[j, k]
            out[i, j] = F32(s)
    return out


def inv3(K) -> np.ndarray:
    """Mat::inv of a 3 x 3 float matrix (DECOMP_LU's closed form for 3 x 3)."""
    a = np.asarray(K, F32).astype(F64)
    d = (a[0, 0] * (a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1]) - a[0, 1] * (a[1, 0] * a[2, 2] - a[1, 2] * a[2, 0])
         + a[0, 2] * (a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0]))
    d = 1.0 / d
    b = [[(a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1]) * d, (a[0, 2] * a[2, 1] - a[0, 1] * a[2, 2]) * d, (a[0, 1] * a[1, 2] - a[0, 2] * a[1, 1]) * d],
         [(a[1, 2] * a[2, 0] - a[1, 0] * a[2, 2]) * d, (a[0, 0] * a[2, 2] - a[0, 2] * a[2, 0]) * d, (a[0, 2] * a[1, 0] - a[0, 0] * a[1, 2]) * d],
         [(a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0]) * d, (a[0, 1] * a[2, 0] - a[0, 0] * a[2, 1]) * d, (a[0, 0] * a[1, 1] - a[0, 1] * a[1, 0]) * d]]
    return np.array(b, F64).astype(F32)


def add_weighted_row(s, ri, rj) -> np.ndarray:
    """s * T.row(i) - T.row(j): addWeighted(ri, s, rj, -1, 0) in double, rounded to float."""
    ri = np.asarray(ri, F32).astype(F64)
    rj = np.asarray(rj, F32).astype(F64)
    return (ri * F64(F32(s)) + rj * -1.0 + 0.0).astype(F32)


def norm3(a) -> float:
    """cv::norm of three floats (double)."""
    s = 0.0
    for v in np.asarray(a, F32):
        s = s + float(v) * float(v)
    return math.sqrt(s)


def dot3(a, b) -> float:
    s = 0.0
    for x, y in zip(np.asarray(a, F32), np.asarray(b, F32)):
        s = s + float(x) * float(y)
    return s


def cos_parallax_stereo(mb, depth) -> F32:
    half = F32(mb) / F32(2)
    a = F32(math.atan2(float(half), float(F32(depth))))
    return F32(math.cos(float(F32(2) * a)))


def float_ulps(a, b) -> int:
    """Distance in float32 ulps between two finite floats."""
    def key(x):
        i = int(np.array(F32(x)).view(np.int32))
        return i if i >= 0 else -(i & 0x7FFFFFFF)
    return abs(key(a) - key(b))


def svd_null_vector(A) -> list:
    """The right singular vector of A (4 x 4, float64) for its smallest singular value: one-sided Jacobi on the columns, pairs
    (0,1) (0,2) (0,3) (1,2) (1,3) (2,3) per sweep, a pair rotated only while |gamma| > 2^-52 sqrt(alpha beta), at most 30 sweeps,
    stopping after a sweep without a rotation; the column of least norm (the first on ties).  Python floats are IEEE doubles and
    math.sqrt is correctly rounded, as the device's sqrt and division."""
    a = [[float(A[r][c]) for c in range(4)] for r in range(4)]
    v = [[1.0 if r == c else 0.0 for c in range(4)] for r in range(4)]
    for _ in range(MAX_SWEEPS):
        rotated = False
        for p in range(3):
            for q in range(p + 1, 4):
                alpha = beta = gamma = 0.0
                for r in range(4):
                    alpha = alpha + a[r][p] * a[r][p]
                    beta = beta + a[r][q] * a[r][q]
                    gamma = gamma + a[r][p] * a[r][q]
                if not abs(gamma) > 2.0 ** -52 * math.sqrt(alpha * beta):
                    continue
                zeta = (beta - alpha) / (2.0 * gamma)
                t = (1.0 if zeta >= 0.0 else -1.0) / (abs(zeta) + math.sqrt(1.0 + zeta * zeta))
                c = 1.0 / math.sqrt(1.0 + t * t)
                s = c * t
                for r in range(4):
                    ap, aq = a[r][p], a[r][q]
                    a[r][p] = c * ap - s * aq
                    a[r][q] = s * ap + c * aq
                    vp, vq = v[r][p], v[r][q]
                    v[r][p] = c * vp - s * vq
                    v[r][q] = s * vp + c * vq
                rotated = True
        if not rotated:
            break
    best, best_n = 0, 0.0
    for c in range(4):
        n = 0.0
        for r in range(4):
            n = n + a[r][c] * a[r][c]
        if c == 0 or n < best_n:
            best, best_n = c, n
    return [v[r][best] for r in range(4)]


# ---------------------------------------------------------------------------------------------------------- per neighbour
def compute_f12(kf1: KeyFrame, kf2: KeyFrame, cam: Camera) -> np.ndarray:
    """LocalMapping::ComputeF12: K1^-T [t12]x R12 K2^-1 with R12 = R1w R2w^T, t12 = -R1w R2w^T t2w + t1w."""
    R12 = gemm_bt(kf1.Rcw, kf2.Rcw)
    t12 = gemm(-R12, kf2.tcw.reshape(3, 1), kf1.tcw.reshape(3, 1)).reshape(3)
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]], F32)
    K = np.array([[cam.fx, 0, cam.cx], [0, cam.fy, cam.cy], [0, 0, 1]], F32)
    return gemm(gemm(gemm(inv3(K.T), tx), R12), inv3(K))


def epipole(kf1: KeyFrame, kf2: KeyFrame, cam: Camera):
    C2 = gemm(kf2.Rcw, kf1.Ow.reshape(3, 1), kf2.tcw.reshape(3, 1)).reshape(3)
    invz = F32(1) / C2[2]
    return cam.fx * C2[0] * invz + cam.cx, cam.fy * C2[1] * invz + cam.cy


def below_baseline(kf1: KeyFrame, kf2: KeyFrame, cam: Camera) -> bool:
    return bool(F32(norm3(kf2.Ow - kf1.Ow)) < cam.mb)


def check_dist_epipolar_line(kp1, kp2, F, sigma2) -> bool:
    x1, y1 = F32(kp1["x"]), F32(kp1["y"])
    a = (x1 * F[0, 0] + y1 * F[1, 0]) + F[2, 0]
    b = (x1 * F[0, 1] + y1 * F[1, 1]) + F[2, 1]
    c = (x1 * F[0, 2] + y1 * F[1, 2]) + F[2, 2]
    num = (a * F32(kp2["x"]) + b * F32(kp2["y"])) + c
    den = a * a + b * b
    if den == 0:
        return False
    dsqr = num * num / den
    return float(dsqr) < 3.84 * float(F32(sigma2[kp2["octave"]]))


def search_key(kf1: KeyFrame, j, kf2: KeyFrame, F, ex, ey, scale, sigma2, groups) -> int:
    """SearchForTriangulation's loop for current key j: the matched neighbour key or -1."""
    nl = len(scale)
    kp1 = kf1.kps[j]
    stereo1 = F32(kf1.u_right[j]) >= 0
    best_d, best = TH_LOW, -1
    for i2 in groups.get(int(kf1.node[j]), ()):
        kp2 = kf2.kps[i2]
        if not 0 <= kp2["octave"] < nl:
            continue
        d = descriptor_distance(kf1.desc[j], kf2.desc[i2])
        if d > TH_LOW or d > best_d:
            continue
        if not stereo1 and not F32(kf2.u_right[i2]) >= 0:
            dex, dey = ex - F32(kp2["x"]), ey - F32(kp2["y"])
            if dex * dex + dey * dey < F32(100) * F32(scale[kp2["octave"]]):
                continue
        if check_dist_epipolar_line(kp1, kp2, F, sigma2):
            best, best_d = i2, d
    return best


def unproject(kf: KeyFrame, i, cam: Camera) -> np.ndarray:
    z = F32(kf.depth[i])
    x = (F32(kf.kps[i]["x"]) - cam.cx) * z * cam.invfx
    y = (F32(kf.kps[i]["y"]) - cam.cy) * z * cam.invfy
    return gemm(kf.Rwc, np.array([[x], [y], [z]], F32), kf.Ow.reshape(3, 1)).reshape(3)


def reproj_ok(kf: KeyFrame, x3, z, kp, stereo, ur, cam: Camera, sigma2) -> bool:
    s2 = F32(sigma2[kp["octave"]])
    x = F32(dot3(kf.Rcw[0], x3) + float(kf.tcw[0]))
    y = F32(dot3(kf.Rcw[1], x3) + float(kf.tcw[1]))
    invz = F32(1) / z
    u = cam.fx * x * invz + cam.cx
    v = cam.fy * y * invz + cam.cy
    ex, ey = u - F32(kp["x"]), v - F32(kp["y"])
    if not stereo:
        return not float(ex * ex + ey * ey) > 5.991 * float(s2)
    er = (u - cam.mbf * invz) - F32(ur)
    return not float(ex * ex + ey * ey + er * er) > 7.8 * float(s2)


def mi_reduction(x3, octave, entropy, sigma2, cam: Camera, sigma_cw) -> float:
    """CheckSemantics' MI - H (info_oracle's rule with the triangulated world point)."""
    J = stereo_jacobian_pose(cam.fx, cam.fy, cam.mb, np.array([F64(x3[0])]), np.array([F64(x3[1])]), np.array([F64(x3[2])]))
    M = stereo_covariance(np.asarray(sigma_cw, F64).reshape(6, 6), J, np.array([F64(F32(sigma2[octave]))]))
    ds = det_lu(np.asarray(sigma_cw, F64).reshape(1, 6, 6))[0]
    dm = det3_cofactor(M[:, 6:, 6:])[0]
    dj = det_lu(M)[0]
    with np.errstate(all="ignore"):
        mi = 0.5 * np.log2(ds * dm / dj)
    return float(mi - F64(entropy))


def triangulate_pair(kf1, j, kf2, m, cam, scale, sigma2, scale_factor, sigma_cw, max_class, th_conf, th_red):
    """LocalMapping.cc:281-469 for the pair (j, m) -> (stage, world point or None, reduction, parallax margin in float ulps)."""
    kp1, kp2 = kf1.kps[j], kf2.kps[m]
    ur1, ur2 = F32(kf1.u_right[j]), F32(kf2.u_right[m])
    z1d, z2d = F32(kf1.depth[j]), F32(kf2.depth[m])
    stereo1, stereo2 = bool(ur1 >= 0), bool(ur2 >= 0)
    xn1 = np.array([(F32(kp1["x"]) - cam.cx) * cam.invfx, (F32(kp1["y"]) - cam.cy) * cam.invfy, F32(1)], F32)
    xn2 = np.array([(F32(kp2["x"]) - cam.cx) * cam.invfx, (F32(kp2["y"]) - cam.cy) * cam.invfy, F32(1)], F32)
    ray1 = gemm(kf1.Rwc, xn1.reshape(3, 1)).reshape(3)
    ray2 = gemm(kf2.Rwc, xn2.reshape(3, 1)).reshape(3)
    cos_rays = F32(dot3(ray1, ray2) / (norm3(ray1) * norm3(ray2)))
    cs1 = cs2 = cos_rays + F32(1)
    if stereo1:
        cs1 = cos_parallax_stereo(cam.mb, z1d)
    elif stereo2:
        cs2 = cos_parallax_stereo(cam.mb, z2d)
    cs = cs2 if cs2 < cs1 else cs1
    # the decisions that read cos(2 atan2(...)): how far they are from flipping, in float ulps
    par_ulps = min(float_ulps(cos_rays, cs), float_ulps(cs1, cs2)) if stereo1 or stereo2 else 1 << 30
    nan = float("nan")
    if cos_rays < cs and cos_rays > 0 and (stereo1 or stereo2 or float(cos_rays) < 0.9998):
        T1 = np.hstack([kf1.Rcw, kf1.tcw.reshape(3, 1)])
        T2 = np.hstack([kf2.Rcw, kf2.tcw.reshape(3, 1)])
        A = np.stack([add_weighted_row(xn1[0], T1[2], T1[0]), add_weighted_row(xn1[1], T1[2], T1[1]),
                      add_weighted_row(xn2[0], T2[2], T2[0]), add_weighted_row(xn2[1], T2[2], T2[1])]).astype(F64)
        v = np.array(svd_null_vector(A), F64).astype(F32)
        if v[3] == 0:
            return W_ZERO, None, nan, par_ulps
        x3 = v[:3] / v[3]
    elif stereo1 and cs1 < cs2 and z1d > 0:
        x3 = unproject(kf1, j, cam)
    elif stereo2 and cs2 < cs1 and z2d > 0:
        x3 = unproject(kf2, m, cam)
    else:
        return PARALLAX, None, nan, par_ulps
    z1 = F32(dot3(kf1.Rcw[2], x3) + float(kf1.tcw[2]))
    if z1 <= 0:
        return Z1, None, nan, par_ulps
    z2 = F32(dot3(kf2.Rcw[2], x3) + float(kf2.tcw[2]))
    if z2 <= 0:
        return Z2, None, nan, par_ulps
    if not reproj_ok(kf1, x3, z1, kp1, stereo1, ur1, cam, sigma2):
        return REPROJ1, None, nan, par_ulps
    if not reproj_ok(kf2, x3, z2, kp2, stereo2, ur2, cam, sigma2):
        return REPROJ2, None, nan, par_ulps
    dist1 = F32(norm3(x3 - kf1.Ow))
    dist2 = F32(norm3(x3 - kf2.Ow))
    if dist1 == 0 or dist2 == 0:
        return SCALE, None, nan, par_ulps
    ratio_dist = dist2 / dist1
    ratio_octave = F32(scale[kp1["octave"]]) / F32(scale[kp2["octave"]])
    ratio_factor = F32(1.5) * F32(scale_factor)
    if ratio_dist * ratio_factor < ratio_octave or ratio_dist > ratio_octave * ratio_factor:
        return SCALE, None, nan, par_ulps
    c1 = VOID
    red = nan
    if z1d > 0 and int(kf1.kp_class[j]) <= max_class and float(kf1.kp_conf[j]) >= float(F32(th_conf)):
        red = mi_reduction(x3, kp1["octave"], kf1.kp_entropy[j], sigma2, cam, sigma_cw)
        c1 = VOID if red < float(F32(th_red)) else int(kf1.kp_class[j])
    if c1 == int(kf2.kp_class[m]) and c1 != VOID:
        return CREATED, x3.astype(F32), red, par_ulps
    return SEMANTIC, None, red, par_ulps


def create_new_map_points(kf1: KeyFrame, neighbours, cam: Camera, scale, sigma2, scale_factor, sigma_cw, max_class, th_conf, th_red):
    """CreateNewMapPoints -> dict with per (neighbour, key) match / stage / reduction / parallax_ulps (n_nb x n1), per key created_nb /
    created_idx / world, and the created list (neighbour, key) in the reference's order."""
    n1, nn = len(kf1.kps), len(neighbours)
    nl = len(scale)
    match = np.full((nn, n1), -1, np.int32)
    stage = np.full((nn, n1), NO_MATCH, np.int32)
    red = np.full((nn, n1), np.nan, F64)
    par = np.full((nn, n1), 1 << 30, np.int64)
    created_nb = np.full(n1, -1, np.int32)
    created_idx = np.full(n1, -1, np.int32)
    world = np.full((n1, 3), np.nan, F32)
    has = np.asarray(kf1.has_point, bool).copy()
    created = []
    for i, kf2 in enumerate(neighbours):
        if below_baseline(kf1, kf2, cam):
            stage[i, :] = BASELINE
            continue
        F = compute_f12(kf1, kf2, cam)
        ex, ey = epipole(kf1, kf2, cam)
        groups = {}
        for i2 in range(len(kf2.kps)):
            if kf2.node[i2] >= 0 and not kf2.has_point[i2]:
                groups.setdefault(int(kf2.node[i2]), []).append(i2)
        for j in range(n1):
            if has[j]:
                stage[i, j] = HAS_POINT
                continue
            if kf1.node[j] < 0 or not 0 <= kf1.kps[j]["octave"] < nl:
                continue
            m = search_key(kf1, j, kf2, F, ex, ey, scale, sigma2, groups)
            match[i, j] = m
            if m < 0:
                continue
            st, x3, r, par[i, j] = triangulate_pair(kf1, j, kf2, m, cam, scale, sigma2, scale_factor, sigma_cw, max_class, th_conf, th_red)
            stage[i, j] = st
            red[i, j] = r
            if st == CREATED:
                has[j] = True
                created_nb[j], created_idx[j] = i, m
                world[j] = x3
                created.append((i, j))
    return dict(match=match, stage=stage, reduction=red, parallax_ulps=par, created_nb=created_nb, created_idx=created_idx, world=world,
                created=np.array(created, np.int32).reshape(-1, 2))
