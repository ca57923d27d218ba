"""The bag of words over the C-ABI: the DBoW2 vocabulary (text file or arrays), Frame::ComputeBoW / KeyFrame::ComputeBoW
(TemplatedVocabulary::transform) and ORBmatcher::SearchByBoW(KeyFrame*, Frame&) batched over keyframes.  The rules are spelled out in
include/sivo_b200.h and oracle/bow_oracle.py."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from .mapping import KeyframeKeys
from .orb import KP_DTYPE, ORBextractor

WEIGHTINGS = ("TF_IDF", "TF", "IDF", "BINARY")
SCORINGS = ("L1_NORM", "L2_NORM", "CHI_SQUARE", "KL", "BHATTACHARYYA", "DOT_PRODUCT")


class Vocabulary:
    """A vocabulary on one device (read-only: any thread may use it)."""

    def __init__(self, handle: C.c_void_p, device: int):
        self._h = handle
        self.device = device

    @classmethod
    def from_text(cls, path: str, device: int = 0) -> "Vocabulary":
        h = C.c_void_p()
        L.check(L.lib().sivo_vocabulary_load_text(str(path).encode(), device, C.byref(h)))
        return cls(h, device)

    @classmethod
    def from_arrays(cls, k, L_, scoring, weighting, parent, is_leaf, desc, weight, device: int = 0) -> "Vocabulary":
        """Arrays indexed by node id, the root at 0 (its entries are ignored)."""
        par = np.ascontiguousarray(parent, np.int32)
        leaf = np.ascontiguousarray(is_leaf, np.uint8)
        d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        w = np.ascontiguousarray(weight, np.float64)
        if not (len(par) == len(leaf) == len(d) == len(w)):
            raise ValueError("every node array needs one entry per node")
        h = C.c_void_p()
        L.check(L.lib().sivo_vocabulary_create(device, k, L_, scoring, weighting, L.ptr(par), L.ptr(leaf), L.ptr(d), L.ptr(w),
                                               len(par), C.byref(h)))
        return cls(h, device)

    def info(self) -> dict:
        v = [C.c_int(0) for _ in range(6)]
        L.check(L.lib().sivo_vocabulary_info(self._h, *(C.byref(x) for x in v)))
        return dict(zip(("k", "L", "scoring", "weighting", "nodes", "words"), (x.value for x in v)))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            L.lib().sivo_vocabulary_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def parse_text(path: str) -> dict:
    """Test hook: the library's text parser and checks without a device -> dict(k, L, scoring, weighting, parent, is_leaf, desc,
    weight); raises SivoError (SIVO_EFORMAT / SIVO_ENOENT) as the loader would."""
    hdr = np.zeros(4, np.int32)
    n = C.c_int(0)
    rc = L.lib().sivo_dbg_vocabulary_parse(str(path).encode(), L.ptr(hdr), C.byref(n), None, None, None, None, 0)
    if rc != L.ERANGE:
        L.check(rc)
    par, leaf = np.empty(n.value, np.int32), np.empty(n.value, np.uint8)
    desc, w = np.empty((n.value, 32), np.uint8), np.empty(n.value, np.float64)
    L.check(L.lib().sivo_dbg_vocabulary_parse(str(path).encode(), L.ptr(hdr), C.byref(n), L.ptr(par), L.ptr(leaf), L.ptr(desc),
                                              L.ptr(w), n.value))
    return dict(k=int(hdr[0]), L=int(hdr[1]), scoring=int(hdr[2]), weighting=int(hdr[3]), parent=par, is_leaf=leaf, desc=desc, weight=w)


def compute_bow(voc: Vocabulary, desc, levelsup: int = 4) -> dict:
    """Host form over n descriptors -> dict(node, word (n, int32, -1: not in the vectors), bow_words (int32 ascending),
    bow_weights (float64))."""
    d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    n = len(d)
    node, word = np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.int32)
    bw, bwt = np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.float64)
    m = C.c_int(0)
    L.check(L.lib().sivo_compute_bow(voc._h, L.ptr(d), n, levelsup, L.ptr(node), L.ptr(word), L.ptr(bw), L.ptr(bwt), C.byref(m)))
    return dict(node=node[:n].copy(), word=word[:n].copy(), bow_words=bw[:m.value].copy(), bow_weights=bwt[:m.value].copy())


def compute_bow_device(voc: Vocabulary, left: ORBextractor, desc_ptr: int, keep_idx_ptr: int, n_keep_ptr: int, levelsup: int,
                       node_ptr: int = 0, word_ptr: int = 0, bow_word_ptr: int = 0, bow_weight_ptr: int = 0, bow_len_ptr: int = 0,
                       stream: int = 0):
    """sivo_compute_bow_device on device pointers (0: not wanted / identity keep_idx); outputs of left.capacity() keys.  Enqueued
    on `stream` (0 = the left extractor's stream) with no waits and no host synchronisation."""
    L.check(L.lib().sivo_compute_bow_device(voc._h, left._h, desc_ptr, keep_idx_ptr, n_keep_ptr, levelsup, node_ptr, word_ptr,
                                            bow_word_ptr, bow_weight_ptr, bow_len_ptr, stream))


def keyframe_keys(kps_ptr: int, desc_ptr: int, node_ptr: int, count_ptr: int) -> KeyframeKeys:
    """The sivo_keyframe_keys members SearchByBoW reads (host or device pointers)."""
    k = KeyframeKeys()
    k.kps, k.desc, k.node, k.count = kps_ptr, desc_ptr, node_ptr, count_ptr
    return k


def _kf_table(keys, points):
    arr = (KeyframeKeys * max(len(keys), 1))()
    for i, k in enumerate(keys):
        arr[i] = k
    pts = (C.c_void_p * max(len(points), 1))(*[int(p) for p in points])
    return arr, pts


def search_by_bow(left: ORBextractor, kps, desc, node, keyframes, nnratio: float = 0.7, check_orientation: bool = True):
    """Host form.  keyframes: a list of dicts with kps, desc, node, point (host arrays of one entry per key) and optionally count
    (default: the array length; negative: that keyframe's n_matches is -1).  Returns (match (n_kf, n) int32, n_matches int64)."""
    k = np.ascontiguousarray(kps, KP_DTYPE)
    d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    nd = np.ascontiguousarray(node, np.int32)
    n = len(k)
    if len(d) != n or len(nd) != n:
        raise ValueError("kps, desc and node need one entry per frame key")
    hold, keys, points = [], [], []
    for kf in keyframes:
        a = [np.ascontiguousarray(kf["kps"], KP_DTYPE), np.ascontiguousarray(kf["desc"], np.uint8).reshape(-1, 32),
             np.ascontiguousarray(kf["node"], np.int32), np.ascontiguousarray(kf["point"], np.int32)]
        cnt = np.array([len(a[0]) if kf.get("count") is None else kf["count"]], np.int64)
        hold += a + [cnt]
        keys.append(keyframe_keys(a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, cnt.ctypes.data))
        points.append(a[3].ctypes.data)
    arr, pts = _kf_table(keys, points)
    nk = len(keys)
    match = np.full((max(nk, 1), max(n, 1)), -1, np.int32)
    nm = np.zeros(max(nk, 1), np.int64)
    L.check(L.lib().sivo_search_by_bow(left._h, L.ptr(k), L.ptr(d), L.ptr(nd), n, arr, pts, nk, nnratio, int(bool(check_orientation)),
                                       L.ptr(match), L.ptr(nm)))
    return match[:nk, :n].copy(), nm[:nk].copy()


def search_by_bow_device(left: ORBextractor, kps_ptr: int, desc_ptr: int, keep_idx_ptr: int, n_keep_ptr: int, node_ptr: int, keyframes,
                         kf_point_ptrs, nnratio: float, check_orientation: bool, match_ptr: int, n_matches_ptr: int, stream: int = 0):
    """sivo_search_by_bow_device: keyframes = KeyframeKeys with device pointers (keyframe_keys()), kf_point_ptrs one device int
    array per keyframe; match_ptr holds len(keyframes) rows of left.capacity() ints, n_matches_ptr one int64 per keyframe."""
    arr, pts = _kf_table(list(keyframes), list(kf_point_ptrs))
    L.check(L.lib().sivo_search_by_bow_device(left._h, kps_ptr, desc_ptr, keep_idx_ptr, n_keep_ptr, node_ptr, arr, pts, len(keyframes),
                                              nnratio, int(bool(check_orientation)), match_ptr, n_matches_ptr, stream))
