"""Python mirror of `SIVO::ORBextractor` (include/orbslam/ORBextractor.h:46-125) and of the Hamming stage
of `Frame::ComputeStereoMatches` over the C-ABI."""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional

import numpy as np

from . import _lib as L

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])


class ORBextractor:
    def __init__(self, nfeatures: int, scaleFactor: float, nlevels: int, iniThFAST: int, minThFAST: int, device: int = 0):
        self._h = C.c_void_p()
        L.check(L.lib().sivo_orb_create(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, device, C.byref(self._h)))
        self.nfeatures, self.nlevels = nfeatures, nlevels
        self._scale = np.empty(nlevels, np.float32)
        self._inv = np.empty(nlevels, np.float32)
        self._s2 = np.empty(nlevels, np.float32)
        self._is2 = np.empty(nlevels, np.float32)
        self._per = np.empty(nlevels, np.int32)
        L.check(L.lib().sivo_orb_tables(self._h, *(L.ptr(a) for a in (self._scale, self._inv, self._s2, self._is2, self._per))))
        self.mvImagePyramid: List[np.ndarray] = []
        self._scale_factor = scaleFactor

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value and L is not None and getattr(L, "lib", None):
            try:
                L.lib().sivo_orb_destroy(self._h)
            except Exception:  # interpreter shutdown: module globals may already be gone
                pass
            self._h = C.c_void_p()

    def GetLevels(self): return self.nlevels
    def GetScaleFactor(self): return float(np.float32(self._scale_factor))
    def GetScaleFactors(self): return self._scale.copy()
    def GetInverseScaleFactors(self): return self._inv.copy()
    def GetScaleSigmaSquares(self): return self._s2.copy()
    def GetInverseScaleSigmaSquares(self): return self._is2.copy()
    def features_per_level(self): return self._per.copy()

    def __call__(self, image: np.ndarray, mask=None, want_pyramid: bool = True, pyramid_buffers=None):
        """Returns (keypoints structured array KP_DTYPE, descriptors u8 [N,32]); fills mvImagePyramid with
        views at offset (19,19) into the bordered level buffers, like the reference's public member."""
        if image is None or image.size == 0:
            return np.empty(0, KP_DTYPE), np.empty((0, 32), np.uint8)
        if image.dtype != np.uint8 or image.ndim != 2:
            raise ValueError("ORBextractor expects a single-channel uint8 image")  # assert(type == CV_8UC1)
        if image.strides[1] != 1:
            image = np.ascontiguousarray(image)
        rows, cols = image.shape
        cap = self.nfeatures + 4 * self.nlevels + 64
        kps = np.empty(cap, KP_DTYPE)
        desc = np.empty((cap, 32), np.uint8)
        n = C.c_int(0)
        ptrs = strides = None
        bufs = []
        if want_pyramid:
            # the marshalled pointer / stride arrays of caller-owned level buffers are cached per buffer set: the per-call
            # Python work of the mirror (a dozen ctypes calls) would otherwise rival the operator's own latency
            key = (rows, cols, id(pyramid_buffers)) if pyramid_buffers is not None else None
            cached = getattr(self, "_pyr_cache", None)
            if key is not None and cached is not None and cached[0] == key:
                _, ptrs, strides, bufs, views = cached
            else:
                ptrs = (C.c_void_p * self.nlevels)()
                strides = (C.c_size_t * self.nlevels)()
                shapes = self.level_shapes(rows, cols)
                for l in range(self.nlevels):
                    if pyramid_buffers is not None:  # caller-owned (e.g. page-locked) storage, reused across frames
                        b = pyramid_buffers[l]
                        assert b.shape == shapes[l] and b.dtype == np.uint8
                    else:
                        b = np.empty(shapes[l], np.uint8)
                    bufs.append(b)
                    ptrs[l] = b.ctypes.data
                    strides[l] = b.strides[0]
                views = [b[19:-19, 19:-19] for b in bufs]
                if key is not None:
                    self._pyr_cache = (key, ptrs, strides, bufs, views)
            self._bordered = bufs
            self.mvImagePyramid = views
        else:
            self._bordered = []
            self.mvImagePyramid = []
        L.check(L.lib().sivo_orb_run(self._h, L.ptr(image), rows, cols, image.strides[0], L.ptr(kps), cap, C.byref(n), L.ptr(desc),
                                     ptrs, strides))
        return kps[:n.value], desc[:n.value]

    def level_shapes(self, rows: int, cols: int):
        """Bordered level buffer shapes (h + 38, w + 38) for a rows x cols image."""
        cache = self.__dict__.setdefault("_shape_cache", {})
        if (rows, cols) not in cache:
            out = []
            for l in range(self.nlevels):
                w, h = C.c_int(), C.c_int()
                L.check(L.lib().sivo_orb_level_size(self._h, rows, cols, l, C.byref(w), C.byref(h)))
                out.append((h.value + 38, w.value + 38))
            cache[(rows, cols)] = out
        return list(cache[(rows, cols)])

    def run_device_input(self, gray_ptr: int, rows: int, cols: int, pitch: int):
        cap = self.nfeatures + 4 * self.nlevels + 64
        kps = np.empty(cap, KP_DTYPE)
        desc = np.empty((cap, 32), np.uint8)
        n = C.c_int(0)
        L.check(L.lib().sivo_orb_run_device_input(self._h, gray_ptr, rows, cols, pitch, L.ptr(kps), cap, C.byref(n), L.ptr(desc)))
        return kps[:n.value], desc[:n.value]

    def has_device_tree(self) -> bool:
        """True if this handle distributes on the device (no host round trip; the asynchronous form is available)."""
        y = C.c_int()
        L.check(L.lib().sivo_orb_has_device_tree(self._h, C.byref(y)))
        return bool(y.value)

    def capacity(self) -> int:
        n = C.c_int()
        L.check(L.lib().sivo_orb_capacity(self._h, C.byref(n)))
        return n.value

    def enqueue_device(self, gray_ptr: int, rows: int, cols: int, pitch: int, kps_ptr: int, desc_ptr: int, count_ptr: int):
        """Asynchronous operator on device-resident buffers (sivo_orb_enqueue_device): returns after the launches are enqueued on
        the handle's stream; kps / desc / count (int64) stay on the device."""
        L.check(L.lib().sivo_orb_enqueue_device(self._h, gray_ptr, rows, cols, pitch, kps_ptr, desc_ptr, count_ptr))

    def stream_wait(self, consumer_stream: int):
        L.check(L.lib().sivo_orb_stream_wait(self._h, consumer_stream))

    def wait_for_stream(self, producer_stream: int):
        L.check(L.lib().sivo_orb_wait_for_stream(self._h, producer_stream))

    def wait_event(self, cuda_event: int):
        L.check(L.lib().sivo_orb_wait_event(self._h, cuda_event))

    def device_status(self) -> int:
        m = C.c_int()
        L.check(L.lib().sivo_orb_device_status(self._h, C.byref(m)))
        return m.value

    def candidates(self, level: int):
        n = C.c_int()
        cap = 1 << 16
        xs, ys, rs = (np.empty(cap, np.int32) for _ in range(3))
        L.check(L.lib().sivo_orb_candidates(self._h, level, L.ptr(xs), L.ptr(ys), L.ptr(rs), cap, C.byref(n)))
        return xs[:n.value].copy(), ys[:n.value].copy(), rs[:n.value].copy()

    def last_timing(self):
        a, b, n = C.c_float(), C.c_float(), C.c_int()
        L.check(L.lib().sivo_orb_last_timing(self._h, C.byref(a), C.byref(b), C.byref(n)))
        return {"device_ms": a.value, "tree_ms": b.value, "launches": n.value}


def distribute_octtree(xs, ys, resp, min_x, max_x, min_y, max_y, n_target) -> np.ndarray:
    """Host-only DistributeOctTree of the library (no GPU needed)."""
    xs = np.ascontiguousarray(xs, np.float32)
    ys = np.ascontiguousarray(ys, np.float32)
    resp = np.ascontiguousarray(resp, np.float32)
    keep = np.empty(max(len(xs), 1), np.int32)
    n = L.check(L.lib().sivo_orb_distribute(L.ptr(xs), L.ptr(ys), L.ptr(resp), len(xs), min_x, max_x, min_y, max_y, n_target,
                                            L.ptr(keep), len(keep)))
    return keep[:n].copy()


def stereo_hamming(kp_left, desc_left, kp_right, desc_right, scale_factors, rows, min_d, max_d, device: int = 0):
    kl = np.ascontiguousarray(kp_left, KP_DTYPE)
    kr = np.ascontiguousarray(kp_right, KP_DTYPE)
    dl = np.ascontiguousarray(desc_left, np.uint8)
    dr = np.ascontiguousarray(desc_right, np.uint8)
    sf = np.ascontiguousarray(scale_factors, np.float32)
    idx = np.empty(len(kl), np.int32)
    dist = np.empty(len(kl), np.int32)
    L.check(L.lib().sivo_stereo_hamming(device, L.ptr(kl), L.ptr(dl), len(kl), L.ptr(kr), L.ptr(dr), len(kr), L.ptr(sf), len(sf), rows,
                                        min_d, max_d, L.ptr(idx), L.ptr(dist)))
    return idx, dist


def stereo_match(left: ORBextractor, right: ORBextractor, kp_left, desc_left, kp_right, desc_right, mb: float, mbf: float):
    """Frame::ComputeStereoMatches on the device pyramids of the two extractors' last runs -> (mvRight, mvDepth)."""
    kl = np.ascontiguousarray(kp_left, KP_DTYPE)
    kr = np.ascontiguousarray(kp_right, KP_DTYPE)
    dl = np.ascontiguousarray(desc_left, np.uint8)
    dr = np.ascontiguousarray(desc_right, np.uint8)
    u = np.empty(len(kl), np.float32)
    z = np.empty(len(kl), np.float32)
    L.check(L.lib().sivo_stereo_match(left._h, right._h, L.ptr(kl), L.ptr(dl), len(kl), L.ptr(kr), L.ptr(dr), len(kr), mb, mbf,
                                      L.ptr(u), L.ptr(z)))
    return u, z


def stereo_match_device(left: ORBextractor, right: ORBextractor, kp_left_ptr: int, desc_left_ptr: int, keep_idx_ptr: int,
                        n_left_ptr: int, kp_right_ptr: int, desc_right_ptr: int, n_right_ptr: int, mb: float, mbf: float,
                        u_right_ptr: int, depth_ptr: int, stream: int = 0):
    """stereo_match on device buffers (sivo_stereo_match_device): output j belongs to left keypoint keep_idx[j] (keep_idx_ptr 0:
    keypoint j) for j < the int64 count at n_left_ptr; float32 outputs of left.capacity() entries.  `stream` (0 = the left
    extractor's stream) first waits for both extractors' work; the next enqueue_device on either must be ordered after this call
    (wait_for_stream).  No host synchronisation."""
    L.check(L.lib().sivo_stereo_match_device(left._h, right._h, kp_left_ptr, desc_left_ptr, keep_idx_ptr, n_left_ptr, kp_right_ptr,
                                             desc_right_ptr, n_right_ptr, mb, mbf, u_right_ptr, depth_ptr, stream))


def stereo_median_cut(sad, u, z, device: int = 0):
    """Test hook: the median-based outlier cut of stereo_match alone (sivo_dbg_stereo_median_cut) over int SAD distances (< 0 =
    unmatched).  Returns copies of u and z with the cut keys set to -1."""
    s = np.ascontiguousarray(sad, np.int32)
    u = np.array(u, np.float32)
    z = np.array(z, np.float32)
    L.check(L.lib().sivo_dbg_stereo_median_cut(device, L.ptr(s), len(s), L.ptr(u), L.ptr(z)))
    return u, z


def hamming_best2(query_desc, train_desc, cand_offsets, cand_idx, train_level=None, device: int = 0) -> np.ndarray:
    """Inner loop of ORBmatcher::SearchByProjection & co (ORBmatcher.cc:79-113) for all queries at once.
    Returns int32 [n_query, 5] = (bestIdx, bestDist, bestLevel, bestDist2, bestLevel2)."""
    q = np.ascontiguousarray(query_desc, np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(train_desc, np.uint8).reshape(-1, 32)
    off = np.ascontiguousarray(cand_offsets, np.int32)
    idx = np.ascontiguousarray(cand_idx, np.int32)
    if len(off) != len(q) + 1:
        raise ValueError("cand_offsets must have n_query + 1 entries")
    lvl = None if train_level is None else np.ascontiguousarray(train_level, np.int32)
    out = np.empty((len(q), 5), np.int32)
    L.check(L.lib().sivo_hamming_best2(device, L.ptr(q), len(q), L.ptr(t), len(t), L.ptr(off), L.ptr(idx), L.ptr(lvl), L.ptr(out)))
    return out
