"""The frame pose over the C-ABI: Optimizer::PoseOptimization (g2o Levenberg-Marquardt over the frame's map-point matches, four
rounds of outlier classification) and its marginal covariance, as Tracking runs it after each projection search.  The rules are
spelled out in include/sivo_b200.h and oracle/pose_oracle.py.

A frame's chain reads as Tracking does: last-frame search -> pose_gather_device -> pose_optimize_device -> (read the small
result) -> local-map search with frame_from_result -> pose_gather_device -> pose_optimize_device -> information selection with
camera_from_result."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from ._lib import InfoCamera
from .info import make_camera
from .orb import KP_DTYPE, ORBextractor
from .track import TrackFrame, make_frame


class PoseResult(C.Structure):
    """sivo_pose_result: Tcw (3 x 4 row-major, the next call's initial pose), the SE3Quat (q = x, y, z, w; t), the Frame's pose
    matrices, mSigmacw (row-major 6 x 6) and the counts."""
    _fields_ = [("Tcw", C.c_float * 12), ("q", C.c_double * 4), ("t", C.c_double * 3), ("Rcw", C.c_float * 9), ("tcw", C.c_float * 3),
                ("Rwc", C.c_float * 9), ("Ow", C.c_float * 3), ("sigma_cw", C.c_double * 36), ("sigma_valid", C.c_int32),
                ("n_initial", C.c_int32), ("n_bad", C.c_int32), ("n_good", C.c_int32), ("rounds_run", C.c_int32),
                ("reserved", C.c_int32)]

    def pose(self) -> np.ndarray:
        return np.array(self.Tcw, np.float32).reshape(3, 4)

    def sigma(self) -> np.ndarray:
        return np.array(self.sigma_cw, np.float64).reshape(6, 6)


def frame_from_result(res: PoseResult, fx, fy, cx, cy, mbf, bounds) -> TrackFrame:
    """The sivo_track_frame of the optimised pose (Rcw, tcw and Ow copied from the result)."""
    f = make_frame(fx, fy, cx, cy, mbf, bounds, np.array(res.Rcw, np.float32), np.array(res.tcw, np.float32))
    f.Ow[:] = list(res.Ow)
    return f


def camera_from_result(res: PoseResult, fx, fy, cx, cy, mb, prior_sigma) -> InfoCamera:
    """The sivo_info_camera of the optimised pose: Rwc, Ow and Sigma_cw from the result, or prior_sigma when the result has no
    covariance (sigma_valid 0: the frame keeps the prior its caller set)."""
    S = res.sigma() if res.sigma_valid else np.asarray(prior_sigma, np.float64)
    cam = make_camera(fx, fy, cx, cy, mb, np.array(res.Rwc, np.float32), np.array(res.Ow, np.float32), S)
    return cam


def _host_keys(kps, u_right, xw):
    k = np.ascontiguousarray(kps, KP_DTYPE)
    u = np.ascontiguousarray(u_right, np.float32)
    x = np.ascontiguousarray(xw, np.float32).reshape(-1, 3)
    if len(u) != len(k) or len(x) != len(k):
        raise ValueError("kps, u_right and xw need one entry per semantic key")
    return k, u, x


def pose_optimize(left: ORBextractor, kps, u_right, xw, Tcw, fx, fy, cx, cy, mbf):
    """Host form: keys gathered per semantic key (mvKeysSemantic, mvRight, the matched point's world position or NaN x 3), Tcw
    the frame's pose (3 x 4 or 4 x 4).  Returns (PoseResult, outlier bool per key)."""
    k, u, x = _host_keys(kps, u_right, xw)
    T = np.ascontiguousarray(np.asarray(Tcw, np.float32).reshape(-1, 4)[:3]).reshape(12)
    res = PoseResult()
    out = np.zeros(max(len(k), 1), np.uint8)
    L.check(L.lib().sivo_pose_optimize(left._h, L.ptr(k), L.ptr(u), L.ptr(x), len(k), fx, fy, cx, cy, mbf, L.ptr(T), C.byref(res),
                                       L.ptr(out)))
    return res, out[:len(k)].astype(bool)


def pose_optimize_device(left: ORBextractor, kps_ptr: int, keep_idx_ptr: int, n_keep_ptr: int, u_right_ptr: int, xw_ptr: int, fx, fy, cx,
                         cy, mbf, Tcw_in_ptr: int, result_ptr: int, outlier_ptr: int, stream: int = 0):
    """sivo_pose_optimize_device on device pointers (keep_idx_ptr / outlier_ptr may be 0); result_ptr points to a device
    sivo_pose_result (512 bytes).  Runs on `stream` (0 = the left extractor's) without waits of its own and without a host
    synchronisation."""
    L.check(L.lib().sivo_pose_optimize_device(left._h, kps_ptr, keep_idx_ptr, n_keep_ptr, u_right_ptr, xw_ptr, fx, fy, cx, cy, mbf,
                                              Tcw_in_ptr, result_ptr, outlier_ptr, stream))


def pose_gather_device(left: ORBextractor, match_ptr: int, n_keep_ptr: int, points_ptr: int, n_points: int, xw_ptr: int, stream: int = 0):
    """sivo_pose_gather_device: xw[j] = points[match[j]].pos for the keys with a match, other entries untouched."""
    L.check(L.lib().sivo_pose_gather_device(left._h, match_ptr, n_keep_ptr, points_ptr, n_points, xw_ptr, stream))


def result_from_bytes(b) -> PoseResult:
    """A PoseResult from the 512 bytes of a device result copied to the host."""
    return PoseResult.from_buffer_copy(np.ascontiguousarray(b, np.uint8).tobytes())


def pose_system(left: ORBextractor, kps, u_right, xw, pose7, fx, fy, cx, cy, mbf, robust_stereo=True, level1=None):
    """Test hook: one linearisation pass at pose7 = (qx, qy, qz, qw, tx, ty, tz).  Returns a dict of per-key err (n, 3), chi2, rho
    (n, 2), jac (n, 3, 6) and H (6, 6), b (6,), chi."""
    k, u, x = _host_keys(kps, u_right, xw)
    n = len(k)
    p7 = np.ascontiguousarray(pose7, np.float64).reshape(7)
    l1 = None if level1 is None else np.ascontiguousarray(level1, np.uint8)
    out = {"err": np.empty((n, 3)), "chi2": np.empty(n), "rho": np.empty((n, 2)), "jac": np.empty((n, 3, 6)), "H": np.empty((6, 6)),
           "b": np.empty(6)}
    chi = C.c_double(0)
    L.check(L.lib().sivo_dbg_pose_system(left._h, L.ptr(k), L.ptr(u), L.ptr(x), n, fx, fy, cx, cy, mbf, L.ptr(p7),
                                         int(bool(robust_stereo)), L.ptr(l1),
                                         *(L.ptr(out[key]) for key in ("err", "chi2", "rho", "jac", "H", "b")), C.byref(chi)))
    out["chi"] = chi.value
    return out


# sivo_pose_trace_rec and its kinds (include/sivo_b200.h)
TRACE_TRIAL, TRACE_ROUND, TRACE_SIN, TRACE_COS, TRACE_POW_THETA, TRACE_POW_RHO = range(6)
TRACE_MAX = 4 + 4 * 10 * 10 * 5
TRACE_DTYPE = np.dtype([(k, "<i4") for k in ("kind", "round", "iteration", "trial", "ok2", "accepted", "n_active", "n_bad",
                                             "robust_stereo", "reserved")]
                       + [(k, "<f8") for k in ("current", "temp", "lam_before", "ni_before", "lam_after", "ni_after", "rho")]
                       + [("x", "<f8", 6), ("q", "<f8", 4), ("t", "<f8", 3), ("arg", "<f8"), ("value", "<f8")])


def pose_trace(left: ORBextractor, kps, u_right, xw, Tcw, fx, fy, cx, cy, mbf):
    """Test hook: pose_optimize run by the traced kernel.  Returns (PoseResult, outlier bool per key, the TRACE_DTYPE records:
    per trial its transcendental calls then its state, per round its counts)."""
    k, u, x = _host_keys(kps, u_right, xw)
    T = np.ascontiguousarray(np.asarray(Tcw, np.float32).reshape(-1, 4)[:3]).reshape(12)
    res = PoseResult()
    out = np.zeros(max(len(k), 1), np.uint8)
    rec = np.zeros(TRACE_MAX, TRACE_DTYPE)
    n = L.check(L.lib().sivo_dbg_pose_trace(left._h, L.ptr(k), L.ptr(u), L.ptr(x), len(k), fx, fy, cx, cy, mbf, L.ptr(T), C.byref(res),
                                            L.ptr(out), L.ptr(rec), TRACE_MAX))
    if n > TRACE_MAX:
        raise RuntimeError(f"pose_trace: {n} records, more than the bound {TRACE_MAX}")
    return res, out[:len(k)].astype(bool), rec[:n]


def pose_se3(T, d, device: int = 0):
    """Test hook: the kernel's to_se3quat, oplus and result rounding on n entries (T (n, 12) float, d (n, 6) double).  Returns
    (se3 (n, 7), up (n, 7), tv (n, 4): theta, sin, cos, pow(theta, 3) or NaN, results: a PoseResult array of n)."""
    T = np.ascontiguousarray(T, np.float32).reshape(-1, 12)
    d = np.ascontiguousarray(d, np.float64).reshape(-1, 6)
    n = len(T)
    if len(d) != n:
        raise ValueError("T and d need one row per entry")
    se3, up, tv = np.empty((n, 7)), np.empty((n, 7)), np.empty((n, 4))
    res = (PoseResult * n)()
    L.check(L.lib().sivo_dbg_pose_se3(device, n, L.ptr(T), L.ptr(d), L.ptr(se3), L.ptr(up), L.ptr(tv), res))
    return se3, up, tv, res
