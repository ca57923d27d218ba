"""A keyframe's new map points over the C-ABI: LocalMapping::CreateNewMapPoints with ORBmatcher::SearchForTriangulation and SIVO's
CheckSemantics, the KeyFrame's copy of a Frame's semantic keys, and SearchInNeighbors' ORBmatcher::Fuse over every target keyframe
at once.  The rules are spelled out in include/sivo_b200.h, oracle/mapping_oracle.py and oracle/fuse_oracle.py."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from .orb import KP_DTYPE, ORBextractor

FUSE_STAGES = ("depth", "image", "distance", "angle", "no_candidate", "above_th_low", "matched")  # SIVO_FUSE_STAGE_*
STAGES = ("has_point", "baseline", "no_match", "parallax", "w_zero", "z1", "z2", "reproj1", "reproj2", "scale", "semantic", "created")


class KeyframeKeys(C.Structure):
    """sivo_keyframe_keys: one keyframe's semantic-key arrays (all host or all device pointers) and its pose."""
    _fields_ = [(n, C.c_void_p) for n in ("kps", "desc", "u_right", "depth", "kp_class", "kp_conf", "kp_entropy", "node", "has_point",
                                          "count")] + \
               [("Rcw", C.c_float * 9), ("tcw", C.c_float * 3), ("Ow", C.c_float * 3)]


class MappingParams(C.Structure):
    """sivo_mapping_params: the keyframes' camera, the current keyframe's mSigmacw and SIVO's thresholds."""
    _fields_ = [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "invfx", "invfy", "mb", "mbf")] + \
               [("sigma_cw", C.c_double * 36), ("max_static_class", C.c_int32), ("th_confidence", C.c_float),
                ("th_entropy_reduction", C.c_float), ("reserved", C.c_int32)]


def make_params(fx, fy, cx, cy, mbf, sigma_cw, max_static_class=8, th_confidence=0.0, th_entropy_reduction=0.0) -> MappingParams:
    """invfx = 1.0f / fx and mb = mbf / fx in float, as Frame.cc computes them."""
    f32 = np.float32
    p = MappingParams()
    p.fx, p.fy, p.cx, p.cy, p.mbf = f32(fx), f32(fy), f32(cx), f32(cy), f32(mbf)
    p.invfx, p.invfy = f32(1) / f32(fx), f32(1) / f32(fy)
    p.mb = f32(mbf) / f32(fx)
    p.sigma_cw[:] = [float(v) for v in np.asarray(sigma_cw, np.float64).reshape(36)]
    p.max_static_class = int(max_static_class)
    p.th_confidence = f32(th_confidence)
    p.th_entropy_reduction = f32(th_entropy_reduction)
    return p


def set_pose(k: KeyframeKeys, Rcw, tcw, Ow):
    k.Rcw[:] = [float(v) for v in np.asarray(Rcw, np.float32).reshape(9)]
    k.tcw[:] = [float(v) for v in np.asarray(tcw, np.float32).reshape(3)]
    k.Ow[:] = [float(v) for v in np.asarray(Ow, np.float32).reshape(3)]


class HostKeyframe:
    """Host arrays of one keyframe (kept alive here) and their sivo_keyframe_keys."""

    def __init__(self, kps, desc, u_right, depth, kp_class, kp_conf, kp_entropy, node, has_point, Rcw, tcw, Ow, count=None):
        self.arrays = [np.ascontiguousarray(kps, KP_DTYPE), np.ascontiguousarray(desc, np.uint8).reshape(-1, 32),
                       np.ascontiguousarray(u_right, np.float32), np.ascontiguousarray(depth, np.float32),
                       np.ascontiguousarray(kp_class, np.uint8), np.ascontiguousarray(kp_conf, np.float64),
                       np.ascontiguousarray(kp_entropy, np.float64), np.ascontiguousarray(node, np.int32),
                       np.ascontiguousarray(has_point, np.uint8)]
        n = len(self.arrays[0])
        if any(len(a) != n for a in self.arrays):
            raise ValueError("every keyframe array needs one entry per key")
        self.n = n
        self.count = np.array([n if count is None else count], np.int64)
        self.keys = KeyframeKeys(*[a.ctypes.data for a in self.arrays], self.count.ctypes.data)
        set_pose(self.keys, Rcw, tcw, Ow)


def _nb_array(neighbours):
    arr = (KeyframeKeys * max(len(neighbours), 1))()
    for i, k in enumerate(neighbours):
        arr[i] = k
    return arr


def create_map_points(left: ORBextractor, kf1: HostKeyframe, neighbours, params: MappingParams, debug=False):
    """Host form (debug: the test hook, every key searched).  Returns a dict: created_nb, created_idx, world (n1, 3), created
    (m, 2) pairs (neighbour, key), n_created; with debug also match / stage / reduction (n_neighbours, n1)."""
    n1 = kf1.n
    nn = len(neighbours)
    out = dict(created_nb=np.empty(n1, np.int32), created_idx=np.empty(n1, np.int32), world=np.empty((n1, 3), np.float32),
               created=np.empty((max(n1, 1), 2), np.int32))
    nc = C.c_longlong(0)
    nbs = _nb_array([k.keys for k in neighbours])
    common = (left._h, C.byref(kf1.keys), nbs, nn, C.byref(params))
    tail = (L.ptr(out["created_nb"]), L.ptr(out["created_idx"]), L.ptr(out["world"]), L.ptr(out["created"]), C.byref(nc))
    if debug:
        for k, dt in (("match", np.int32), ("stage", np.int32), ("reduction", np.float64)):
            out[k] = np.empty((nn, n1), dt)
        L.check(L.lib().sivo_dbg_create_map_points(*common, L.ptr(out["match"]), L.ptr(out["stage"]), L.ptr(out["reduction"]), *tail))
    else:
        L.check(L.lib().sivo_create_map_points(*common, *tail))
    out["n_created"] = nc.value
    out["created"] = out["created"][:max(nc.value, 0)].copy()
    return out


def create_map_points_device(left: ORBextractor, kf1: KeyframeKeys, neighbours, params: MappingParams, created_nb_ptr: int = 0,
                             created_idx_ptr: int = 0, world_ptr: int = 0, created_list_ptr: int = 0, n_created_ptr: int = 0,
                             stream: int = 0):
    """sivo_create_map_points_device: kf1 / neighbours hold device pointers; outputs of left.capacity() keys (0: not wanted).
    Enqueued on `stream` (0 = the left extractor's stream) with no waits and no host synchronisation."""
    L.check(L.lib().sivo_create_map_points_device(left._h, C.byref(kf1), _nb_array(neighbours), len(neighbours), C.byref(params),
                                                  created_nb_ptr, created_idx_ptr, world_ptr, created_list_ptr, n_created_ptr, stream))


def keyframe_gather_device(left: ORBextractor, kps_ptr, desc_ptr, keep_idx_ptr, n_keep_ptr, u_right_ptr, depth_ptr, class_ptr, conf_ptr,
                           entropy_ptr, out: dict, stream: int = 0):
    """sivo_keyframe_gather_device into the caller's device buffers out[kps, desc, u_right, depth, kp_class, kp_conf, kp_entropy,
    count] (torch tensors or raw pointers of left.capacity() keys)."""
    ptr = [int(out[k].data_ptr()) if hasattr(out[k], "data_ptr") else int(out[k])
           for k in ("kps", "desc", "u_right", "depth", "kp_class", "kp_conf", "kp_entropy", "count")]
    L.check(L.lib().sivo_keyframe_gather_device(left._h, kps_ptr, desc_ptr, keep_idx_ptr, n_keep_ptr, u_right_ptr, depth_ptr,
                                                class_ptr, conf_ptr, entropy_ptr, *ptr, stream))


class FuseCamera(C.Structure):
    """sivo_fuse_camera: the keyframes' shared camera and image bounds."""
    _fields_ = [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "mbf", "min_x", "max_x", "min_y", "max_y")]


def make_fuse_camera(fx, fy, cx, cy, mbf, bounds) -> FuseCamera:
    """bounds = (mnMinX, mnMaxX, mnMinY, mnMaxY)."""
    c = FuseCamera()
    c.fx, c.fy, c.cx, c.cy, c.mbf = (np.float32(v) for v in (fx, fy, cx, cy, mbf))
    c.min_x, c.max_x, c.min_y, c.max_y = (np.float32(v) for v in bounds)
    return c


class FuseTarget:
    """Host arrays of one Fuse target (kept alive here): its semantic keys, descriptors, mvRight and pose; count defaults to the
    number of keys (a negative count: the target's row is all -1)."""

    def __init__(self, kps, desc, u_right, Rcw, tcw, Ow, count=None):
        self.arrays = [np.ascontiguousarray(kps, KP_DTYPE), np.ascontiguousarray(desc, np.uint8).reshape(-1, 32),
                       np.ascontiguousarray(u_right, np.float32)]
        n = len(self.arrays[0])
        if any(len(a) != n for a in self.arrays):
            raise ValueError("kps, desc and u_right need one entry per key")
        self.n = n
        self.count = np.array([n if count is None else count], np.int64)
        k, d, u = (a.ctypes.data for a in self.arrays)
        self.keys = KeyframeKeys(k, d, u, None, None, None, None, None, None, self.count.ctypes.data)
        set_pose(self.keys, Rcw, tcw, Ow)


def _points(points):
    from .track import MAP_POINT_DTYPE
    return np.ascontiguousarray(points, MAP_POINT_DTYPE)


def fuse(left: ORBextractor, targets, cam: FuseCamera, points, th: float = 3.0, debug: bool = False):
    """Host form of sivo_fuse (debug: sivo_dbg_fuse).  targets: FuseTarget list; points: sivo_map_point records.  Returns (match,
    dist) as (n_targets, n_points) int32 arrays, with debug also stage (SIVO_FUSE_STAGE_*, -1 for a negative count)."""
    pts = _points(points)
    nt, npt = len(targets), len(pts)
    match = np.empty((nt, npt), np.int32)
    dist = np.empty((nt, npt), np.int32)
    common = (left._h, _nb_array([t.keys for t in targets]), nt, C.byref(cam), L.ptr(pts), npt, th, L.ptr(match), L.ptr(dist))
    if not debug:
        L.check(L.lib().sivo_fuse(*common))
        return match, dist
    stage = np.empty((nt, npt), np.int32)
    L.check(L.lib().sivo_dbg_fuse(*common, L.ptr(stage)))
    return match, dist, stage


def dbg_fuse(left: ORBextractor, targets, cam: FuseCamera, points, th: float = 3.0):
    """The test hook sivo_dbg_fuse: (match, dist, stage)."""
    return fuse(left, targets, cam, points, th, debug=True)


def fuse_device(left: ORBextractor, targets, cam: FuseCamera, points_ptr: int, n_points: int, th: float, match_ptr: int, dist_ptr: int = 0,
                stream: int = 0):
    """sivo_fuse_device: targets are KeyframeKeys holding device pointers (kps, desc, u_right, count) and poses; points_ptr a
    device array of n_points sivo_map_point records; match_ptr / dist_ptr device int32 arrays of len(targets) x n_points (dist 0:
    not wanted).  Enqueued on `stream` (0 = the left extractor's stream) with no waits and no host synchronisation."""
    L.check(L.lib().sivo_fuse_device(left._h, _nb_array(targets), len(targets), C.byref(cam), points_ptr, n_points, th, match_ptr,
                                      dist_ptr, stream))
