"""SIVO's information-based map-point selection (Tracking::StereoInitialization / CreateNewKeyFrame) over the C-ABI: per semantic
key, the mutual information between the pose and the key's stereo measurement minus its classification entropy, against a
threshold.  The rule is spelled out in include/sivo_b200.h and oracle/info_oracle.py."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from ._lib import InfoCamera
from .orb import KP_DTYPE, ORBextractor


def make_camera(fx, fy, cx, cy, mb, Rwc, Ow, sigma_cw) -> InfoCamera:
    """The Frame's members: invfx / invfy = 1.0f / fx as Frame.cc:170-171 computes them, in float."""
    cam = InfoCamera()
    f32 = np.float32
    cam.fx, cam.fy, cam.cx, cam.cy, cam.mb = f32(fx), f32(fy), f32(cx), f32(cy), f32(mb)
    cam.invfx, cam.invfy = f32(1) / f32(fx), f32(1) / f32(fy)
    cam.Rwc[:] = [float(v) for v in np.asarray(Rwc, np.float32).reshape(9)]
    cam.Ow[:] = [float(v) for v in np.asarray(Ow, np.float32).reshape(3)]
    cam.sigma_cw[:] = [float(v) for v in np.asarray(sigma_cw, np.float64).reshape(36)]
    return cam


def info_select(left: ORBextractor, kps, depth, entropy, camera: InfoCamera, threshold: float):
    """Host form: kps / depth / entropy gathered per semantic key (mvKeysSemantic, mvDepth, mEntropy at the key).
    Returns (world (n, 3) float32, reduction float64, selected int32 ascending)."""
    k = np.ascontiguousarray(kps, KP_DTYPE)
    z = np.ascontiguousarray(depth, np.float32)
    h = np.ascontiguousarray(entropy, np.float64)
    n = len(k)
    if len(z) != n or len(h) != n:
        raise ValueError("kps, depth and entropy need one entry per semantic key")
    world = np.empty((n, 3), np.float32)
    red = np.empty(n, np.float64)
    sel = np.empty(max(n, 1), np.int32)
    ns = C.c_int(0)
    L.check(L.lib().sivo_info_select(left._h, L.ptr(k), L.ptr(z), L.ptr(h), n, C.byref(camera), threshold, L.ptr(world), L.ptr(red),
                                     L.ptr(sel), C.byref(ns)))
    return world, red, sel[:ns.value].copy()


def info_select_device(left: ORBextractor, kps_ptr: int, kp_entropy_ptr: int, keep_idx_ptr: int, n_keep_ptr: int, depth_ptr: int,
                       camera: InfoCamera, threshold: float, world_ptr: int, reduction_ptr: int, selected_ptr: int, n_selected_ptr: int,
                       stream: int = 0):
    """info_select on device buffers (sivo_info_select_device): semantic key j is extractor key keep_idx[j] (keep_idx_ptr 0: key j)
    for j < the int64 count at n_keep_ptr; outputs of left.capacity() keys (any pointer may be 0), *n_selected int64.  Runs on
    `stream` (0 = the left extractor's stream) without waits of its own and without a host synchronisation."""
    L.check(L.lib().sivo_info_select_device(left._h, kps_ptr, kp_entropy_ptr, keep_idx_ptr, n_keep_ptr, depth_ptr, C.byref(camera),
                                            threshold, world_ptr, reduction_ptr, selected_ptr, n_selected_ptr, stream))


def info_terms(left: ORBextractor, kps, depth, camera: InfoCamera):
    """Test hook: (world (n, 3) float32, det S, det M33, det M) per key as the kernel computes them."""
    k = np.ascontiguousarray(kps, KP_DTYPE)
    z = np.ascontiguousarray(depth, np.float32)
    n = len(k)
    world = np.empty((n, 3), np.float32)
    dets = [np.empty(n, np.float64) for _ in range(3)]
    L.check(L.lib().sivo_dbg_info_terms(left._h, L.ptr(k), L.ptr(z), n, C.byref(camera), L.ptr(world), *(L.ptr(d) for d in dets)))
    return (world, *dets)
