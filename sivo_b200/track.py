"""Map points matched to a frame's semantic keys by projection over the C-ABI: the local-map search (Tracking::SearchLocalPoints:
Frame::isInFrustum + ORBmatcher::SearchByProjection(F, vpMapPoints, th)) and the last-frame search (TrackWithMotionModel:
SearchByProjection(CurrentFrame, LastFrame, th)), with the Frame's grid.  The rules are spelled out in include/sivo_b200.h and
oracle/track_oracle.py."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from .orb import KP_DTYPE, ORBextractor

# sivo_map_point
MAP_POINT_DTYPE = np.dtype([("desc", np.uint8, 32), ("pos", np.float32, 3), ("normal", np.float32, 3), ("min_distance", np.float32),
                            ("max_distance", np.float32), ("observed", np.int32), ("octave", np.int32), ("angle", np.float32),
                            ("reserved", np.int32)])


class TrackFrame(C.Structure):
    """sivo_track_frame: the current Frame's members (Rcw row-major)."""
    _fields_ = [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "mb", "mbf", "min_x", "max_x", "min_y", "max_y")] + \
               [("Rcw", C.c_float * 9), ("tcw", C.c_float * 3), ("Ow", C.c_float * 3)]


def camera_centre(Rcw, tcw) -> np.ndarray:
    """mOw = -mRcw^T mtcw as cv::gemm computes it (each entry the double sum of the three products, rounded to float)."""
    R = np.asarray(Rcw, np.float32).reshape(3, 3).astype(np.float64)
    t = np.asarray(tcw, np.float32).reshape(3).astype(np.float64)
    return np.array([-np.float32((R[0, r] * t[0] + R[1, r] * t[1]) + R[2, r] * t[2]) for r in range(3)], np.float32)


def make_frame(fx, fy, cx, cy, mbf, bounds, Rcw, tcw) -> TrackFrame:
    """bounds = (mnMinX, mnMaxX, mnMinY, mnMaxY); mb = mbf / fx in float (Frame.cc:172); Ow from the pose."""
    f = TrackFrame()
    f32 = np.float32
    f.fx, f.fy, f.cx, f.cy, f.mbf = f32(fx), f32(fy), f32(cx), f32(cy), f32(mbf)
    f.mb = f32(mbf) / f32(fx)
    f.min_x, f.max_x, f.min_y, f.max_y = (f32(v) for v in bounds)
    f.Rcw[:] = [float(v) for v in np.asarray(Rcw, np.float32).reshape(9)]
    f.tcw[:] = [float(v) for v in np.asarray(tcw, np.float32).reshape(3)]
    f.Ow[:] = [float(v) for v in camera_centre(Rcw, tcw)]
    return f


def map_points(desc, pos, normal, min_distance, max_distance, observed=1, octave=0, angle=0.0) -> np.ndarray:
    """The sivo_map_point array: one row per point (scalars broadcast)."""
    desc = np.asarray(desc, np.uint8).reshape(-1, 32)
    pts = np.zeros(len(desc), MAP_POINT_DTYPE)
    pts["desc"] = desc
    pts["pos"] = np.asarray(pos, np.float32).reshape(-1, 3)
    pts["normal"] = np.asarray(normal, np.float32).reshape(-1, 3)
    pts["min_distance"], pts["max_distance"] = min_distance, max_distance
    pts["observed"], pts["octave"], pts["angle"] = observed, octave, angle
    return pts


def _keys(kps, desc, u_right):
    k = np.ascontiguousarray(kps, KP_DTYPE)
    d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    u = np.ascontiguousarray(u_right, np.float32)
    if len(d) != len(k) or len(u) != len(k):
        raise ValueError("kps, desc and u_right need one entry per semantic key")
    return k, d, u


def search_local_points(left: ORBextractor, kps, desc, u_right, points, frame: TrackFrame, th: float, nnratio: float = 0.8, blocked=None):
    """Host form: keys gathered per semantic key (mvKeysSemantic, mDescriptorsSemantic, mvRight), blocked[j] = key j held by an
    observed point on entry (None: none).  Returns (in_view bool per point, match int32 per key (-1: none), n_matches)."""
    k, d, u = _keys(kps, desc, u_right)
    pts = np.ascontiguousarray(points, MAP_POINT_DTYPE)
    b = None if blocked is None else np.ascontiguousarray(blocked, np.uint8)
    if b is not None and len(b) != len(k):
        raise ValueError("blocked needs one entry per semantic key")
    view = np.empty(max(len(pts), 1), np.uint8)
    match = np.empty(max(len(k), 1), np.int32)
    nm = C.c_int(0)
    L.check(L.lib().sivo_search_local_points(left._h, L.ptr(k), L.ptr(d), L.ptr(u), L.ptr(b), len(k), L.ptr(pts), len(pts),
                                             C.byref(frame), th, nnratio, L.ptr(view), L.ptr(match), C.byref(nm)))
    return view[:len(pts)].astype(bool), match[:len(k)].copy(), nm.value


def search_last_frame(left: ORBextractor, kps, desc, u_right, points, frame: TrackFrame, Rlw, tlw, th: float):
    """Host form of the last-frame search; points carry their last-frame key's octave and angle.  Returns (match, n_matches)."""
    k, d, u = _keys(kps, desc, u_right)
    pts = np.ascontiguousarray(points, MAP_POINT_DTYPE)
    R = np.ascontiguousarray(Rlw, np.float32).reshape(9)
    t = np.ascontiguousarray(tlw, np.float32).reshape(3)
    match = np.empty(max(len(k), 1), np.int32)
    nm = C.c_int(0)
    L.check(L.lib().sivo_search_last_frame(left._h, L.ptr(k), L.ptr(d), L.ptr(u), len(k), L.ptr(pts), len(pts), C.byref(frame),
                                           L.ptr(R), L.ptr(t), th, L.ptr(match), C.byref(nm)))
    return match[:len(k)].copy(), nm.value


def search_local_points_device(left: ORBextractor, kps_ptr: int, desc_ptr: int, keep_idx_ptr: int, n_keep_ptr: int, u_right_ptr: int,
                               blocked_ptr: int, points_ptr: int, n_points: int, frame: TrackFrame, th: float, nnratio: float,
                               in_view_ptr: int, match_ptr: int, n_matches_ptr: int, stream: int = 0):
    """sivo_search_local_points_device on device pointers (0 for an optional one).  Runs on `stream` (0 = the left extractor's)
    without waits of its own and without a host synchronisation."""
    L.check(L.lib().sivo_search_local_points_device(left._h, kps_ptr, desc_ptr, keep_idx_ptr, n_keep_ptr, u_right_ptr, blocked_ptr,
                                                    points_ptr, n_points, C.byref(frame), th, nnratio, in_view_ptr, match_ptr,
                                                    n_matches_ptr, stream))


def search_last_frame_device(left: ORBextractor, kps_ptr: int, desc_ptr: int, keep_idx_ptr: int, n_keep_ptr: int, u_right_ptr: int,
                             points_ptr: int, n_points: int, frame: TrackFrame, Rlw, tlw, th: float, match_ptr: int, n_matches_ptr: int,
                             stream: int = 0):
    """sivo_search_last_frame_device on device pointers; Rlw / tlw are host arrays."""
    R = np.ascontiguousarray(Rlw, np.float32).reshape(9)
    t = np.ascontiguousarray(tlw, np.float32).reshape(3)
    L.check(L.lib().sivo_search_last_frame_device(left._h, kps_ptr, desc_ptr, keep_idx_ptr, n_keep_ptr, u_right_ptr, points_ptr,
                                                  n_points, C.byref(frame), L.ptr(R), L.ptr(t), th, match_ptr, n_matches_ptr, stream))


def features_in_area(left: ORBextractor, kps, bounds, queries):
    """Test hook: GetFeaturesInArea on the device grid; queries = rows (x, y, r, minLevel, maxLevel).  Returns one int32 array
    of semantic-key indices per query."""
    k = np.ascontiguousarray(kps, KP_DTYPE)
    q = list(queries)
    xyr = np.array([[a[0], a[1], a[2]] for a in q], np.float32).reshape(-1)
    lv = np.array([[a[3], a[4]] for a in q], np.int32).reshape(-1)
    off = np.zeros(len(q) + 1, np.int32)
    cap = 1 << 16
    while True:
        idx = np.empty(cap, np.int32)
        rc = L.lib().sivo_dbg_features_in_area(left._h, L.ptr(k), len(k), *bounds, L.ptr(xyr), L.ptr(lv), len(q), L.ptr(off),
                                               L.ptr(idx), cap)
        if rc == L.ERANGE and off[-1] > cap:
            cap = int(off[-1])
            continue
        L.check(rc)
        return [idx[off[i]:off[i + 1]].copy() for i in range(len(q))]
