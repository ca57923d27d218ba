"""Scalar restatement of the Frame's grid and the two per-frame projection searches of ORB-SLAM2 as SIVO runs them:
Frame::AssignFeaturesToGrid / PosInGrid / GetFeaturesInArea (Frame.cc:205-223, 326-404), Frame::isInFrustum (Frame.cc:267-324),
MapPoint::PredictScale (MapPoint.cc:439-453), ORBmatcher::RadiusByViewingCos, SearchByProjection(F, vpMapPoints, th)
(ORBmatcher.cc:44-127), SearchByProjection(CurrentFrame, LastFrame, th) for stereo (ORBmatcher.cc:1278-1418) and
ComputeThreeMaxima (ORBmatcher.cc:1545-1577).

Arithmetic: every float operation is one numpy float32 operation on float32 scalars, every double one a float64 operation, in the
order the reference writes it (no fused multiply-add).  The rules the reference leaves to its libraries:
- round (PosInGrid, the rotation bin) rounds half away from zero; Python's round and np.round round half to even and are not used.
- cv::gemm: Rcw P + tcw (3 x 3 float) is ((R0 x + R1 y) + R2 z) + t in float (info_oracle.unproject's form); -Rcw^T tcw
  (GEMM_1_T, alpha -1) is each entry's double sum of the three products, rounded to float and negated.  tests/test_oracle_track.py
  pins both against cv2.gemm.
- cv::norm of three floats: sqrt of ((0 + a0 a0) + a1 a1) + a2 a2 in double (pinned against cv2.norm).
- Mat::dot of three floats: ((0 + a0 n0) + a1 n1) + a2 n2 in double, OpenCV 4's scalar path (Mat::dot has no Python binding, so
  this order is not pinned; only a viewCos within an ulp of 0.5 or 0.998 can depend on it).
- PredictScale's log is the float overload (MapPoint.cc sees `using namespace std` through DBoW2's TemplatedVocabulary.h); here the
  correctly rounded float logarithm, float32(log(float64(ratio))).  mfLogScaleFactor likewise.
- A point whose u, v, viewCos or level quotient is NaN is not in view (the reference converts the NaN to int).
- Angles: a key or last-frame point angle takes part only if it is finite and in [0, 360] (angle_ok).  A key with another angle
  goes in no cell; a last-frame point with one is not searched.  Within the rule the rotation bin is in 0..12; the reference
  asserts bin in [0, HISTO_LENGTH) (ORBmatcher.cc:1390) and has no rule for angles that would break it.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle.orb_oracle import descriptor_distance

F32, F64 = np.float32, np.float64
COLS, ROWS = 64, 48  # FRAME_GRID_COLS / FRAME_GRID_ROWS
TH_HIGH = 100
HISTO_LENGTH = 30


def round_half_away(x) -> float:
    """C's round / roundf: half away from zero (exact for float32 inputs in float64)."""
    a = np.floor(abs(F64(x)) + 0.5)
    return float(-a if x < 0 else a)


@dataclass
class Frame:
    """The current Frame's members (bounds = mnMinX, mnMaxX, mnMinY, mnMaxY)."""
    fx: float
    fy: float
    cx: float
    cy: float
    mbf: float
    bounds: tuple
    Rcw: np.ndarray
    tcw: np.ndarray

    def __post_init__(self):
        self.fx, self.fy, self.cx, self.cy, self.mbf = (F32(v) for v in (self.fx, self.fy, self.cx, self.cy, self.mbf))
        self.mb = self.mbf / self.fx
        self.min_x, self.max_x, self.min_y, self.max_y = (F32(v) for v in self.bounds)
        self.w_inv = F32(COLS) / (self.max_x - self.min_x)
        self.h_inv = F32(ROWS) / (self.max_y - self.min_y)
        self.Rcw = np.asarray(self.Rcw, F32).reshape(3, 3)
        self.tcw = np.asarray(self.tcw, F32).reshape(3)
        self.Ow = gemm_neg_t(self.Rcw, self.tcw)


# ---------------------------------------------------------------------------------------------------------- OpenCV forms
def gemm_pc(R, P, t) -> np.ndarray:
    """cv::gemm(R, P, 1, t, 1) for 3 x 3 floats: ((R0 x + R1 y) + R2 z) + t per row, in float."""
    R = np.asarray(R, F32).reshape(3, 3)
    P = np.asarray(P, F32).reshape(3)
    t = np.asarray(t, F32).reshape(3)
    return np.array([((R[r, 0] * P[0] + R[r, 1] * P[1]) + R[r, 2] * P[2]) + t[r] for r in range(3)], F32)


def gemm_neg_t(R, t) -> np.ndarray:
    """-R^T t as cv::gemm(R, t, -1, noArray(), 0, GEMM_1_T) computes it: the double sum, rounded to float, negated."""
    R = np.asarray(R, F32).reshape(3, 3).astype(F64)
    t = np.asarray(t, F32).reshape(3).astype(F64)
    return np.array([-F32((R[0, r] * t[0] + R[1, r] * t[1]) + R[2, r] * t[2]) for r in range(3)], F32)


def norm3(a) -> F32:
    """(float) cv::norm of a 3-float vector."""
    s = F64(0)
    for v in np.asarray(a, F32):
        s = s + F64(v) * F64(v)
    return F32(np.sqrt(s))


def dot3(a, b) -> F64:
    """Mat::dot of two 3-float vectors (OpenCV 4's scalar path)."""
    s = F64(0)
    for x, y in zip(np.asarray(a, F32), np.asarray(b, F32)):
        s = s + F64(x) * F64(y)
    return s


def logf(x) -> F32:
    return F32(np.log(F64(x)))


# ---------------------------------------------------------------------------------------------------------- grid
def pos_in_grid(x, y, f: Frame):
    """Frame::PosInGrid -> (ix, iy) or None."""
    gx = round_half_away((F32(x) - f.min_x) * f.w_inv)
    gy = round_half_away((F32(y) - f.min_y) * f.h_inv)
    if not (0 <= gx < COLS and 0 <= gy < ROWS):  # also keeps a NaN out of the int conversion
        return None
    return int(gx), int(gy)


def angle_ok(a) -> bool:
    """The angle rule: finite and in [0, 360] (-0.0 included)."""
    return bool(F32(0) <= F32(a) <= F32(360))


def assign_features_to_grid(kps, f: Frame):
    """Frame::AssignFeaturesToGrid -> grid[ix][iy] = ascending key indices; a key breaking the angle rule goes in no cell."""
    grid = [[[] for _ in range(ROWS)] for _ in range(COLS)]
    for j in range(len(kps)):
        if not angle_ok(kps["angle"][j]):
            continue
        c = pos_in_grid(kps["x"][j], kps["y"][j], f)
        if c is not None:
            grid[c[0]][c[1]].append(j)
    return grid


def get_features_in_area(grid, kps, f: Frame, x, y, r, min_level=-1, max_level=-1) -> list:
    """Frame::GetFeaturesInArea, in its walk order."""
    x, y, r = F32(x), F32(y), F32(r)
    out = []
    min_cx = max(0, int(np.floor(((x - f.min_x) - r) * f.w_inv)))
    if min_cx >= COLS:
        return out
    max_cx = min(COLS - 1, int(np.ceil(((x - f.min_x) + r) * f.w_inv)))
    if max_cx < 0:
        return out
    min_cy = max(0, int(np.floor(((y - f.min_y) - r) * f.h_inv)))
    if min_cy >= ROWS:
        return out
    max_cy = min(ROWS - 1, int(np.ceil(((y - f.min_y) + r) * f.h_inv)))
    if max_cy < 0:
        return out
    check = min_level > 0 or max_level >= 0
    for ix in range(min_cx, max_cx + 1):
        for iy in range(min_cy, max_cy + 1):
            for j in grid[ix][iy]:
                o = int(kps["octave"][j])
                if check and (o < min_level or (max_level >= 0 and o > max_level)):
                    continue
                if abs(F32(kps["x"][j]) - x) < r and abs(F32(kps["y"][j]) - y) < r:
                    out.append(j)
    return out


# ---------------------------------------------------------------------------------------------------------- projection
def predict_scale(max_distance, dist, log_scale, nlevels):
    """MapPoint::PredictScale(dist, F) -> level, or None for a NaN quotient."""
    lq = logf(F32(max_distance) / F32(dist)) / F32(log_scale)
    if np.isnan(lq):
        return None
    c = np.ceil(lq)
    return 0 if c < 0 else (nlevels - 1 if c >= nlevels else int(c))


def radius_by_viewing_cos(view_cos) -> F32:
    return F32(2.5) if F64(view_cos) > 0.998 else F32(4.0)


def is_in_frustum(mp, f: Frame, log_scale, nlevels, viewing_cos_limit=0.5):
    """Frame::isInFrustum(pMP, 0.5) -> None, or (u, v, projXR, level, viewCos)."""
    P = np.asarray(mp["pos"], F32)
    pc = gemm_pc(f.Rcw, P, f.tcw)
    if pc[2] < F32(0):
        return None
    with np.errstate(all="ignore"):
        invz = F32(1) / pc[2]
        u = f.fx * pc[0] * invz + f.cx
        v = f.fy * pc[1] * invz + f.cy
    if np.isnan(u) or np.isnan(v):
        return None
    if u < f.min_x or u > f.max_x or v < f.min_y or v > f.max_y:
        return None
    max_d = F32(1.2) * F32(mp["max_distance"])
    min_d = F32(0.8) * F32(mp["min_distance"])
    PO = P - f.Ow
    dist = norm3(PO)
    if dist < min_d or dist > max_d:
        return None
    with np.errstate(all="ignore"):
        view_cos = F32(dot3(PO, mp["normal"]) / F64(dist))
        if np.isnan(view_cos) or view_cos < F32(viewing_cos_limit):
            return None
        level = predict_scale(mp["max_distance"], dist, log_scale, nlevels)
        if level is None:
            return None
        return u, v, u - f.mbf * invz, level, view_cos


# ---------------------------------------------------------------------------------------------------------- the searches
def search_local_points(kps, desc, u_right, points, f: Frame, scale, th, nnratio=0.8, blocked=None, per_point=None):
    """SearchLocalPoints' isInFrustum loop + SearchByProjection(F, vpMapPoints, th) -> (in_view bool, match int32, n_matches).
    blocked[j]: key j held by an observed point on entry.  A point takes its key for every later point iff it is observed.
    per_point (a list, optional) receives the key each point took, or -1."""
    scale = np.asarray(scale, F32)
    nlevels = len(scale)
    log_scale = logf(scale[1]) if nlevels > 1 else F32(0)
    th = F32(th)
    nnratio = F32(nnratio)
    n = len(kps)
    grid = assign_features_to_grid(kps, f)
    held = np.zeros(n, bool) if blocked is None else np.asarray(blocked).astype(bool).copy()
    match = np.full(n, -1, np.int32)
    in_view = np.zeros(len(points), bool)
    nmatches = 0
    for i, mp in enumerate(points):
        if per_point is not None:
            per_point.append(-1)
        proj = is_in_frustum(mp, f, log_scale, nlevels)
        if proj is None:
            continue
        in_view[i] = True
        u, v, xr, level, view_cos = proj
        r = radius_by_viewing_cos(view_cos)
        if th != F32(1):
            r = r * th
        rad = r * scale[level]
        best_dist, best_level, best_dist2, best_level2, best_idx = 256, -1, 256, -1, -1
        for j in get_features_in_area(grid, kps, f, u, v, rad, level - 1, level):
            if held[j]:
                continue
            if F32(u_right[j]) > F32(0) and abs(xr - F32(u_right[j])) > rad:
                continue
            d = descriptor_distance(mp["desc"], desc[j])
            if d < best_dist:
                best_dist2, best_dist, best_level2 = best_dist, d, best_level
                best_level, best_idx = int(kps["octave"][j]), j
            elif d < best_dist2:
                best_level2, best_dist2 = int(kps["octave"][j]), d
        if best_dist <= TH_HIGH:
            if best_level == best_level2 and F32(best_dist) > nnratio * F32(best_dist2):
                continue
            match[best_idx] = i
            if mp["observed"] > 0:
                held[best_idx] = True
            nmatches += 1
            if per_point is not None:
                per_point[i] = best_idx
    return in_view, match, nmatches


def compute_three_maxima(counts):
    """ORBmatcher::ComputeThreeMaxima over the bin sizes -> (ind1, ind2, ind3)."""
    max1 = max2 = max3 = 0
    ind1 = ind2 = ind3 = -1
    for i, s in enumerate(counts):
        if s > max1:
            max3, max2, max1 = max2, max1, s
            ind3, ind2, ind1 = ind2, ind1, i
        elif s > max2:
            max3, max2 = max2, s
            ind3, ind2 = ind2, i
        elif s > max3:
            max3, ind3 = s, i
    if F32(max2) < F32(0.1) * F32(max1):
        ind2 = ind3 = -1
    elif F32(max3) < F32(0.1) * F32(max1):
        ind3 = -1
    return ind1, ind2, ind3


def rotation_bin(angle_last, angle_cur) -> int:
    """The histogram bin of a match; both angles must satisfy the angle rule (the bin is then in 0..12)."""
    if not (angle_ok(angle_last) and angle_ok(angle_cur)):
        raise ValueError(f"angle outside [0, 360]: {angle_last}, {angle_cur}")
    rot = F32(angle_last) - F32(angle_cur)
    if rot < F32(0):
        rot = rot + F32(360)
    b = int(round_half_away(rot * (F32(1) / F32(HISTO_LENGTH))))
    return 0 if b == HISTO_LENGTH else b


def search_last_frame(kps, desc, u_right, points, f: Frame, Rlw, tlw, scale, th):
    """SearchByProjection(CurrentFrame, LastFrame, th, bMono = false) with the orientation check -> (match int32, n_matches).
    points carry the last frame's key octave and angle."""
    scale = np.asarray(scale, F32)
    nlevels = len(scale)
    th = F32(th)
    n = len(kps)
    grid = assign_features_to_grid(kps, f)
    twc = gemm_neg_t(f.Rcw, f.tcw)
    tlc = gemm_pc(Rlw, twc, tlw)
    forward = tlc[2] > f.mb
    backward = -tlc[2] > f.mb
    owner = [None] * n  # (point, observed)
    hist = [[] for _ in range(HISTO_LENGTH)]
    nmatches = 0
    for i, mp in enumerate(points):
        if not angle_ok(mp["angle"]):
            continue
        pc = gemm_pc(f.Rcw, mp["pos"], f.tcw)
        with np.errstate(all="ignore"):
            invzc = F32(F64(1.0) / F64(pc[2]))
            if invzc < 0:
                continue
            u = f.fx * pc[0] * invzc + f.cx
            v = f.fy * pc[1] * invzc + f.cy
        if np.isnan(u) or np.isnan(v):
            continue
        if u < f.min_x or u > f.max_x or v < f.min_y or v > f.max_y:
            continue
        o = int(mp["octave"])
        if not 0 <= o < nlevels:
            raise ValueError("octave out of range")
        radius = th * scale[o]
        if forward:
            cand = get_features_in_area(grid, kps, f, u, v, radius, o)
        elif backward:
            cand = get_features_in_area(grid, kps, f, u, v, radius, 0, o)
        else:
            cand = get_features_in_area(grid, kps, f, u, v, radius, o - 1, o + 1)
        best_dist, best_idx = 256, -1
        for j in cand:
            if owner[j] is not None and owner[j][1]:
                continue
            if F32(u_right[j]) > F32(0):
                ur = u - f.mbf * invzc
                if abs(ur - F32(u_right[j])) > radius:
                    continue
            d = descriptor_distance(mp["desc"], desc[j])
            if d < best_dist:
                best_dist, best_idx = d, j
        if best_dist <= TH_HIGH:
            owner[best_idx] = (i, mp["observed"] > 0)
            nmatches += 1
            hist[rotation_bin(mp["angle"], kps["angle"][best_idx])].append(best_idx)
    keep = compute_three_maxima([len(h) for h in hist])
    for b in range(HISTO_LENGTH):
        if b not in keep:
            for j in hist[b]:
                owner[j] = None
                nmatches -= 1
    match = np.array([-1 if o is None else o[0] for o in owner], np.int32)
    return match, nmatches


# ---------------------------------------------------------------------------------------------------------- test inputs
def map_points_from_keys(kps, depth, Rwc, Ow, fx, fy, cx, cy, scale):
    """Map points made from stereo keys the way a keyframe creates them: the position by Frame::UnprojectStereo at the pose (Rwc,
    Ow), then MapPoint::UpdateNormalAndDepth with that camera as the only observer: maxDist = dist scale[octave], minDist =
    maxDist / scale[nlevels - 1], normal = the unit vector from the camera centre.  Returns a dict of arrays (pos, normal,
    min_distance, max_distance) for the keys with depth > 0, and their indices."""
    from .info_oracle import Camera, unproject
    scale = np.asarray(scale, F32)
    z = np.asarray(depth, F32)
    idx = np.flatnonzero(z > 0)
    cam = Camera(fx, fy, cx, cy, 1.0, Rwc, Ow, np.eye(6))
    pos = unproject(kps["x"][idx], kps["y"][idx], z[idx], cam)
    normal = np.empty_like(pos)
    dmax = np.empty(len(idx), F32)
    for i in range(len(idx)):
        a = pos[i] - cam.Ow
        dist = norm3(a)
        normal[i] = [F32(F64(c) * (1.0 / F64(dist))) for c in a]
        dmax[i] = dist * scale[int(kps["octave"][idx[i]])]
    return {"pos": pos, "normal": normal, "max_distance": dmax, "min_distance": dmax / scale[-1]}, idx
