"""Scalar restatement of ORBmatcher::Fuse(pKF, vpMapPoints, th) (ORBmatcher.cc:787-930) and of LocalMapping::SearchInNeighbors'
two Fuse phases (LocalMapping.cc:586-621), over a small literal model of the map objects they touch (KeyFrame's mvpMapPoints,
MapPoint's observations, nObs, mbBad, mpReplaced and descriptor), and the replay that drives the same bookkeeping from the
device's decision matrices.

The decision of one (target keyframe, map point) pair, as include/sivo_b200.h states it:
- Pc in the projection searches' gemm form (track_oracle.gemm_pc); out (DEPTH) if Pc_z < 0.0f.
- invz = 1 / Pc_z, x = Pc_x invz, u = fx x + cx (v likewise), float; out (IMAGE) unless KeyFrame::IsInImage, min <= u < max with
  the strict upper bound (KeyFrame.cc:638-640); a NaN is out.  ur = u - mbf invz.
- dist3D = track_oracle.norm3(pos - Ow); out (DISTANCE) if dist3D < 0.8f min_distance or > 1.2f max_distance.
- out (ANGLE) if track_oracle.dot3(PO, normal) < 0.5 * dist3D in double (a NaN dot passes, as in the reference).
- level = track_oracle.predict_scale (KeyFrame::mfLogScaleFactor is the Frame's); a NaN quotient searches nothing
  (NO_CANDIDATE).  radius = th scale[level] in float.
- window = track_oracle.get_features_in_area with no level filter (KeyFrame::GetFeaturesInArea has none); empty: NO_CANDIDATE.
- candidate iff level - 1 <= octave <= level and 0 <= octave < nlevels (new: the reference would read mvInvLevelSigma2[-1] for
  an octave -1 key at level 0), and (double)(e2 * invSigma2[octave]) is not above 7.8 (stereo: u_right >= 0, e2 = (ex^2 + ey^2)
  + er^2) or 5.99 (mono, a NaN u_right included; e2 = ex^2 + ey^2).
- best = the first strictly smaller Hamming distance in walk order from 256; MATCHED iff best <= TH_LOW (50).

Reference facts kept by the map model:
- MapPoint::AddObservation returns when the keyframe is already observed; nObs += 2 for a key with mvRight >= 0, else 1.
- MapPoint::Replace returns for the same point; else it clears its observations, sets mbBad and mpReplaced, and for each former
  observation (pKF, idx) either moves it to the survivor (ReplaceMapPointMatch + AddObservation) or, when the survivor already
  observes pKF, erases pKF's match at idx; then the survivor's ComputeDistinctiveDescriptors.  The replaced point's nObs is left
  as it was.
- ComputeDistinctiveDescriptors: nothing for a bad point or one without observations; the observed descriptors of good keyframes,
  the pairwise distances, each row's sorted median at index (int)(0.5 (N - 1)), the least median, the first on ties.
- Observations iterate in keyframe-id order.  The reference's std::map<KeyFrame*, size_t> iterates in pointer order, which
  follows allocation; id order stands in for it, and the replay uses the same model, so the two agree whatever the order.
- Fuse's bookkeeping: pMPinKF = pKF->GetMapPoint(bestIdx); a good pMPinKF with strictly more observations absorbs pMP
  (pMP->Replace(pMPinKF)), otherwise pMPinKF->Replace(pMP) (equal counts included); a bad pMPinKF leaves everything as it is; no
  point: AddObservation + AddMapPoint.
- SearchInNeighbors: phase 1 fuses a copy of the current keyframe's mvpMapPoints into each target in order; phase 2 fuses the
  targets' points (in target order, then key order; NULL, bad and already collected points skipped via mnFuseCandidateForKF)
  into the current keyframe.  The update of the points and connections that follows is not modelled.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle import track_oracle as T
from oracle.orb_oracle import descriptor_distance

F32, F64 = np.float32, np.float64
TH_LOW = 50
DEPTH, IMAGE, DISTANCE, ANGLE, NO_CANDIDATE, ABOVE_TH_LOW, MATCHED = range(7)  # SIVO_FUSE_STAGE_*
NEGATIVE = -1  # a target whose count is negative (device and host forms only)


@dataclass
class Camera:
    """sivo_fuse_camera: the keyframes' shared members; bounds = (mnMinX, mnMaxX, mnMinY, mnMaxY)."""
    fx: float
    fy: float
    cx: float
    cy: float
    mbf: float
    bounds: tuple

    def __post_init__(self):
        self.fx, self.fy, self.cx, self.cy, self.mbf = (F32(v) for v in (self.fx, self.fy, self.cx, self.cy, self.mbf))
        self.min_x, self.max_x, self.min_y, self.max_y = (F32(v) for v in self.bounds)


@dataclass
class Tables:
    """The keyframes' scale tables (mvScaleFactors, mvInvLevelSigma2)."""
    scale: np.ndarray
    inv_sigma2: np.ndarray

    def __post_init__(self):
        self.scale = np.asarray(self.scale, F32)
        self.inv_sigma2 = np.asarray(self.inv_sigma2, F32)
        self.nlevels = len(self.scale)
        self.log_scale = T.logf(self.scale[1]) if self.nlevels > 1 else F32(0)


class KeyFrame:
    """A keyframe: its semantic keys (KP_DTYPE records), descriptors (n x 32), mvRight, pose (Rcw row-major, tcw, Ow) and
    mvpMapPoints (one entry per key, a MapPoint or None)."""

    def __init__(self, kf_id, kps, desc, u_right, Rcw, tcw, Ow, cam: Camera):
        self.id = kf_id
        self.kps = kps
        self.desc = np.asarray(desc, np.uint8).reshape(-1, 32)
        self.u_right = np.asarray(u_right, F32)
        self.Rcw = np.asarray(Rcw, F32).reshape(3, 3)
        self.tcw = np.asarray(tcw, F32).reshape(3)
        self.Ow = np.asarray(Ow, F32).reshape(3)
        self.bad = False
        self.points = [None] * len(kps)
        geo = T.Frame(cam.fx, cam.fy, cam.cx, cam.cy, cam.mbf, cam.bounds, self.Rcw, self.tcw)
        self.geo = geo
        self.grid = T.assign_features_to_grid(kps, geo)

    # KeyFrame.cc:260-279
    def add_map_point(self, mp, idx):
        self.points[idx] = mp

    def erase_map_point_match(self, idx):
        self.points[idx] = None

    def replace_map_point_match(self, idx, mp):
        self.points[idx] = mp


@dataclass(eq=False)
class MapPoint:
    id: int
    pos: np.ndarray
    normal: np.ndarray
    min_distance: float  # mfMinDistance (the rule applies 0.8f)
    max_distance: float  # mfMaxDistance (the rule applies 1.2f)
    desc: np.ndarray
    obs: dict = field(default_factory=dict)  # keyframe -> key index
    nobs: int = 0
    bad: bool = False
    replaced: "MapPoint" = None

    def observations(self):
        """mObservations in the model's iteration order: keyframe id."""
        return sorted(self.obs.items(), key=lambda e: e[0].id)

    def is_in_keyframe(self, kf) -> bool:
        return kf in self.obs

    # MapPoint.cc:149-162
    def add_observation(self, kf, idx):
        if kf in self.obs:
            return
        self.obs[kf] = idx
        self.nobs += 2 if kf.u_right[idx] >= F32(0) else 1

    # MapPoint.cc:225-261
    def replace(self, mp):
        if mp.id == self.id:
            return
        obs = self.observations()
        self.obs = {}
        self.bad = True
        self.replaced = mp
        for kf, idx in obs:
            if not mp.is_in_keyframe(kf):
                kf.replace_map_point_match(idx, mp)
                mp.add_observation(kf, idx)
            else:
                kf.erase_map_point_match(idx)
        mp.compute_distinctive_descriptors()

    # MapPoint.cc:284-347
    def compute_distinctive_descriptors(self):
        if self.bad or not self.obs:
            return
        descs = [kf.desc[idx] for kf, idx in self.observations() if not kf.bad]
        if not descs:
            return
        n = len(descs)
        dist = np.zeros((n, n), np.int64)
        for i in range(n):
            for j in range(i + 1, n):
                dist[i, j] = dist[j, i] = descriptor_distance(descs[i], descs[j])
        best_median, best = None, 0
        for i in range(n):
            median = int(np.sort(dist[i])[int(0.5 * (n - 1))])
            if best_median is None or median < best_median:
                best_median, best = median, i
        self.desc = descs[best].copy()


def point_record(mp: MapPoint) -> dict:
    """The fields of a sivo_map_point the rule reads."""
    return {"pos": mp.pos, "normal": mp.normal, "min_distance": mp.min_distance, "max_distance": mp.max_distance, "desc": mp.desc}


# ---------------------------------------------------------------------------------------------------------- the decision
def decide(kf: KeyFrame, mp, cam: Camera, tables: Tables, th) -> tuple:
    """One pair's decision (ORBmatcher.cc:814-909): (key index or -1, best distance, stage).  mp: a MapPoint or a dict with pos,
    normal, min_distance, max_distance and desc."""
    if isinstance(mp, MapPoint):
        mp = point_record(mp)
    th = F32(th)
    P = np.asarray(mp["pos"], F32)
    pc = T.gemm_pc(kf.Rcw, P, kf.tcw)
    if pc[2] < F32(0):
        return -1, 256, DEPTH
    with np.errstate(all="ignore"):
        invz = F32(1) / pc[2]
        x = pc[0] * invz
        y = pc[1] * invz
        u = cam.fx * x + cam.cx
        v = cam.fy * y + cam.cy
        if not (cam.min_x <= u < cam.max_x and cam.min_y <= v < cam.max_y):
            return -1, 256, IMAGE
        ur = u - cam.mbf * invz
        max_d = F32(1.2) * F32(mp["max_distance"])
        min_d = F32(0.8) * F32(mp["min_distance"])
        PO = P - kf.Ow
        dist3 = T.norm3(PO)
        if dist3 < min_d or dist3 > max_d:
            return -1, 256, DISTANCE
        if T.dot3(PO, mp["normal"]) < 0.5 * F64(dist3):
            return -1, 256, ANGLE
        level = T.predict_scale(mp["max_distance"], dist3, tables.log_scale, tables.nlevels)
    if level is None:
        return -1, 256, NO_CANDIDATE
    radius = th * tables.scale[level]
    window = T.get_features_in_area(kf.grid, kf.kps, kf.geo, u, v, radius)
    if not window:
        return -1, 256, NO_CANDIDATE
    best_dist, best_idx = 256, -1
    for j in window:
        o = int(kf.kps["octave"][j])
        if o < level - 1 or o > level or not 0 <= o < tables.nlevels:
            continue
        with np.errstate(all="ignore"):
            ex = u - F32(kf.kps["x"][j])
            ey = v - F32(kf.kps["y"][j])
            kr = F32(kf.u_right[j])
            if kr >= F32(0):
                er = ur - kr
                e2 = (ex * ex + ey * ey) + er * er
                if F64(e2 * tables.inv_sigma2[o]) > 7.8:
                    continue
            else:
                e2 = ex * ex + ey * ey
                if F64(e2 * tables.inv_sigma2[o]) > 5.99:
                    continue
        d = descriptor_distance(mp["desc"], kf.desc[j])
        if d < best_dist:
            best_dist, best_idx = d, j
    if best_dist <= TH_LOW:
        return best_idx, best_dist, MATCHED
    return -1, best_dist, ABOVE_TH_LOW


def decide_all(targets, points, cam: Camera, tables: Tables, th, counts=None):
    """The (n_targets, n_points) match, dist and stage matrices of the device call.  counts[k] < 0: row k is -1 / 256 / -1."""
    nt, npt = len(targets), len(points)
    match = np.full((nt, npt), -1, np.int32)
    dist = np.full((nt, npt), 256, np.int32)
    stage = np.full((nt, npt), NEGATIVE, np.int32)
    for k, kf in enumerate(targets):
        if counts is not None and counts[k] < 0:
            continue
        for i, mp in enumerate(points):
            match[k, i], dist[k, i], stage[k, i] = decide(kf, mp, cam, tables, th)
    return match, dist, stage


# ---------------------------------------------------------------------------------------------------------- bookkeeping
def apply_match(kf: KeyFrame, mp: MapPoint, best_idx, events=None, position=None, points=None):
    """ORBmatcher.cc:911-925 for a decided pair (best_idx -1: nothing).  events (a set, optional) records which branch ran."""
    if best_idx < 0:
        return
    in_kf = kf.points[best_idx]
    if in_kf is not None:
        if not in_kf.bad:
            if events is not None:
                if in_kf.nobs == mp.nobs:
                    events.add("equal_obs")
            if in_kf.nobs > mp.nobs:
                if events is not None:
                    events.add("replace_into_inkf")
                    if points is not None and position is not None and any(p is in_kf for p in points[position + 1:]):
                        events.add("survivor_later")
                mp.replace(in_kf)
            else:
                if events is not None:
                    events.add("replace_into_mp")
                in_kf.replace(mp)
        elif events is not None:
            events.add("bad_inkf")
    else:
        if events is not None:
            events.add("add")
        mp.add_observation(kf, best_idx)
        kf.add_map_point(mp, best_idx)


def fuse(kf: KeyFrame, points, cam: Camera, tables: Tables, th=3.0, events=None) -> int:
    """ORBmatcher::Fuse(pKF, vpMapPoints, th), literally: the points in order, each decided with its descriptor of the moment."""
    n_fused = 0
    taken = {}
    for i, mp in enumerate(points):
        if mp is None:
            continue
        if mp.bad or mp.is_in_keyframe(kf):
            continue
        best_idx, _, stage = decide(kf, mp, cam, tables, th)
        if stage == MATCHED:
            if events is not None:
                if best_idx in taken:
                    events.add("same_key")
                taken[best_idx] = mp
            apply_match(kf, mp, best_idx, events, i, points)
            n_fused += 1
    return n_fused


def fuse_candidates(targets) -> list:
    """Phase 2's vpFuseCandidates: the targets' points in order, NULL, bad and repeated points skipped (mnFuseCandidateForKF)."""
    seen, out = set(), []
    for kf in targets:
        for mp in list(kf.points):
            if mp is None or mp.bad or id(mp) in seen:
                continue
            seen.add(id(mp))
            out.append(mp)
    return out


def search_in_neighbors(current: KeyFrame, targets, cam: Camera, tables: Tables, th=3.0, events=None):
    """Both Fuse phases of LocalMapping::SearchInNeighbors, literally."""
    matches = list(current.points)
    for kf in targets:
        fuse(kf, matches, cam, tables, th, events)
    fuse(current, fuse_candidates(targets), cam, tables, th, events)


def replay(current: KeyFrame, targets, fuse_rows, research=True, events=None) -> dict:
    """Both phases driven by decision matrices.  fuse_rows(keyframes, records) -> the (len(keyframes), len(records)) match matrix
    (the device call, or decide_all).  Phase 1 decides the current keyframe's points (non-NULL, key order) in every target at once,
    phase 2 the candidates in the current keyframe.  The walk follows the reference's order: a point that is bad now or already in
    the target is skipped; a point whose descriptor differs from the one it was decided with is searched again (research=False
    leaves that rule out, to show it is needed).  Returns counts of the re-searches per phase."""
    stats = {"researched": [0, 0], "changed": [0, 0]}

    def run(phase, kfs, points):
        if not kfs or not points:
            return
        m = fuse_rows(kfs, [point_record(mp) for mp in points])
        searched = [mp.desc.copy() for mp in points]
        for k, kf in enumerate(kfs):
            for i, mp in enumerate(points):
                if mp.bad or mp.is_in_keyframe(kf):
                    continue
                best = int(m[k, i])
                if research and not np.array_equal(mp.desc, searched[i]):
                    again = int(fuse_rows([kf], [point_record(mp)])[0, 0])
                    stats["researched"][phase] += 1
                    if again != best:
                        stats["changed"][phase] += 1
                        if events is not None:
                            events.add("research_changed")
                    best = again
                apply_match(kf, mp, best)

    run(0, list(targets), [mp for mp in current.points if mp is not None])
    run(1, [current], fuse_candidates(targets))
    return stats


def oracle_rows(cam: Camera, tables: Tables, th=3.0):
    """fuse_rows for replay from the oracle's own decision."""
    return lambda kfs, records: decide_all(kfs, records, cam, tables, th)[0]


def map_state(keyframes, points) -> list:
    """The final map state compared bit for bit: every keyframe's point per key (id or -1), and per point its bad flag,
    mpReplaced, observations (keyframe id, key), nObs and descriptor."""
    out = [[-1 if p is None else p.id for p in kf.points] for kf in keyframes]
    for mp in points:
        out.append((mp.id, mp.bad, None if mp.replaced is None else mp.replaced.id,
                    tuple((kf.id, idx) for kf, idx in mp.observations()), mp.nobs, bytes(mp.desc)))
    return out
