"""Tracking::Relocalization's pose hypotheses over the C-ABI: PnPsolver's EPnP RANSAC batched over the candidate keyframes
(sivo_pnp_*), fed by search_by_bow_device's outputs.  The caller keeps Relocalization's loop.  The rule is spelled out in
include/sivo_b200.h and oracle/pnp_oracle.py."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from .orb import ORBextractor


class PoseDebug(C.Structure):
    """sivo_pnp_pose_debug."""
    _fields_ = [("cws", C.c_double * 12), ("d", C.c_double * 12), ("ut", C.c_double * 144), ("l_6x10", C.c_double * 60),
                ("rho", C.c_double * 6), ("betas", C.c_double * 12), ("Rs", C.c_double * 27), ("ts", C.c_double * 9),
                ("rep_errors", C.c_double * 3), ("R", C.c_double * 9), ("t", C.c_double * 3), ("best", C.c_int32),
                ("reserved", C.c_int32)]


class PnpSolver:
    """One PnPsolver per candidate keyframe (at most max_candidates), on the extractor's device.  The extractor must outlive it."""

    def __init__(self, left: ORBextractor, max_candidates: int, seed: int = 0):
        self._h = C.c_void_p()
        self.left = left
        L.check(L.lib().sivo_pnp_create(left._h, max_candidates, seed, C.byref(self._h)))
        self.n_kf = 0

    def setup_device(self, kps_ptr: int, keep_idx_ptr: int, n_keep_ptr: int, match_ptr: int, n_matches_ptr: int, points_ptr: int,
                     n_points: int, kf_ids, frame_id: int, fx: float, fy: float, cx: float, cy: float, stream: int = 0):
        """sivo_pnp_setup_device on device pointers (keep_idx 0: identity); kf_ids one id per candidate (host)."""
        ids = np.ascontiguousarray(kf_ids, np.uint32)
        self.n_kf = len(ids)
        L.check(L.lib().sivo_pnp_setup_device(self._h, kps_ptr, keep_idx_ptr, n_keep_ptr, match_ptr, n_matches_ptr, points_ptr,
                                              n_points, L.ptr(ids), len(ids), frame_id, fx, fy, cx, cy, stream))

    def iterate_device(self, n_iterations: int, active, Tcw_ptr: int, has_pose_ptr: int, no_more_ptr: int, inlier_match_ptr: int,
                       n_inliers_ptr: int, stream: int = 0):
        """sivo_pnp_iterate_device: iterate(n_iterations) on the candidates with active[k] set (host array of n_kf)."""
        act = np.ascontiguousarray(active, np.uint8)
        if len(act) != self.n_kf:
            raise ValueError("active needs one entry per candidate of the last setup")
        L.check(L.lib().sivo_pnp_iterate_device(self._h, n_iterations, L.ptr(act), Tcw_ptr, has_pose_ptr, no_more_ptr,
                                                inlier_match_ptr, n_inliers_ptr, stream))

    def state(self) -> dict:
        """Test hook: per candidate N, min_inliers, max_its, iterations, best, refine_failed, dead and eps (synchronises the device)."""
        out = np.zeros((max(self.n_kf, 1), 7), np.int32)
        eps = np.zeros(max(self.n_kf, 1), np.float32)
        L.check(L.lib().sivo_dbg_pnp_state(self._h, L.ptr(out), L.ptr(eps)))
        names = ("N", "min_inliers", "max_its", "iterations", "best", "refine_failed", "dead")
        d = {k: out[:self.n_kf, i].copy() for i, k in enumerate(names)}
        d["eps"] = eps[:self.n_kf].copy()
        return d

    def hypotheses(self, k: int, first: int, n_hyp: int) -> dict:
        """Test hook: k_pnp_hyp's hypotheses first .. first + n_hyp - 1 of candidate k, the state untouched -> dict(draws (n_hyp, 4),
        R (n_hyp, 3, 3), t (n_hyp, 3) float64, counts (n_hyp), masks (n_hyp, capacity) bool)."""
        words = (self.left.capacity() + 31) // 32
        dr = np.zeros((n_hyp, 4), np.int32)
        rt = np.zeros((n_hyp, 12), np.float64)
        cnt = np.zeros(n_hyp, np.int32)
        masks = np.zeros((n_hyp, max(words, 1)), np.uint32)
        L.check(L.lib().sivo_dbg_pnp_hypotheses(self._h, k, first, n_hyp, L.ptr(dr), L.ptr(rt), L.ptr(cnt), L.ptr(masks)))
        bits = np.unpackbits(masks.view(np.uint8), axis=1, bitorder="little").astype(bool)
        return dict(draws=dr, R=rt[:, :9].reshape(-1, 3, 3), t=rt[:, 9:], counts=cnt, masks=bits)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            L.lib().sivo_pnp_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def compute_pose(p3d, p2d, max_err, fx, fy, cx, cy, device: int = 0):
    """Test hook: Refine's kernel path on n host correspondences, all selected -> (alphas (n, 4), inlier mask (n, bool),
    n_inliers, PoseDebug)."""
    p = np.ascontiguousarray(p3d, np.float32).reshape(-1, 3)
    u = np.ascontiguousarray(p2d, np.float32).reshape(-1, 2)
    e = np.ascontiguousarray(max_err, np.float32).reshape(-1)
    if not (len(p) == len(u) == len(e)):
        raise ValueError("p3d, p2d and max_err need one row per correspondence")
    n = len(p)
    alphas = np.zeros((max(n, 1), 4), np.float64)
    mask = np.zeros(max((n + 31) // 32, 1), np.uint32)
    cnt = C.c_int(0)
    dbg = PoseDebug()
    L.check(L.lib().sivo_dbg_pnp_compute_pose(device, L.ptr(p), L.ptr(u), L.ptr(e), n, fx, fy, cx, cy, L.ptr(alphas), L.ptr(mask),
                                              C.byref(cnt), C.byref(dbg)))
    bits = np.unpackbits(mask.view(np.uint8), bitorder="little")[:n].astype(bool)
    return alphas[:n], bits, cnt.value, dbg


def draws(seed: int, kf_id: int, frame_id: int, first: int, n_hyp: int, N: int, device: int = 0) -> np.ndarray:
    """Test hook: the minimal sets of hypotheses first .. first + n_hyp - 1 -> (n_hyp, 4) int32."""
    out = np.zeros((max(n_hyp, 1), 4), np.int32)
    L.check(L.lib().sivo_dbg_pnp_draws(device, seed, kf_id, frame_id, first, n_hyp, N, L.ptr(out)))
    return out[:n_hyp]
