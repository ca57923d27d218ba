"""TEST INFRASTRUCTURE -- CPU oracle for `SIVO::ORBextractor::operator()` and the stereo Hamming
match; never imported by the product path.

numpy restatement of src/orbslam/ORBextractor.cc (ctor :412-475, ComputePyramid :1085-1122,
ComputeKeyPointsOctTree :752-847, DistributeOctTree :544-750, DivideNode :488-542, IC_Angle :75-100,
computeOrbDescriptor :104-150, operator() :1019-1083).

The arithmetic that lives in un-vendored OpenCV (`find_package(OpenCV 3.0)`, CMakeLists.txt:37-43 --
version not pinned, sources not in the reference tree) is restated from OpenCV's published algorithms:
  cv::FAST (9_16, cornerScore, 3x3 NMS)      -> fast_score_map / cell_keypoints
  cv::resize INTER_LINEAR 8-bit fixed point   -> resize_linear_u8
  cv::copyMakeBorder BORDER_REFLECT_101       -> reflect101
  cv::GaussianBlur 7x7 sigma 2, 8.8 fixed pt  -> gaussian_blur7
  cv::fastAtan2                               -> fast_atan2
  cvRound                                     -> round-half-even
PARITY STATUS: the reference holds no ORB test or fixture (SURVEY 4), so these are pinned against the
operational oracle cv2 (tests/test_oracle_orb.py compares every function above with cv2 on the KITTI
fixture and seeded images, bit for bit, and records cv2.__version__); parity with an OpenCV-3.x build of
the reference is UNPINNED.  Two places where the reference itself is not a function of its input are
given a documented rule here and in the product:
  * DistributeOctTree's last-round ordering sorts (size, ExtractorNode*) pairs (:671-676): ties between
    equal-size nodes are decided by heap addresses.  Rule: ties by creation order (later-created first
    when walking from the back), i.e. what monotonically growing heap addresses would give.
  * computeOrbDescriptor reads the blurred *clone* (no border, :1060) up to 18 px from keypoints that may
    sit 16 px from the edge; the read lands in the adjacent row of the continuous buffer or outside it
    (undefined).  Rule: flat index into the w*h buffer as the reference computes it; outside -> 0.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np

PATCH_SIZE = 31
HALF_PATCH_SIZE = 15
EDGE_THRESHOLD = 19

# radius-3 Bresenham ring, (dx, dy), in OpenCV's order (fast_score.cpp makeOffsets)
RING16 = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3),
          (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3)]


def load_pattern() -> np.ndarray:
    """256x4 int8 test-pair table (x0,y0,x1,y1): data, shipped as sivo_b200/csrc/orb_pattern.inc."""
    import os
    import re
    p = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "sivo_b200", "csrc", "orb_pattern.inc")
    nums = re.findall(r"-?\d+", re.sub(r"//[^\n]*", "", open(p).read()))
    a = np.array(nums, dtype=np.int32).reshape(256, 4)
    return a


def cv_round(x):
    return np.rint(x).astype(np.int32)


@dataclass
class ExtractorParams:
    nfeatures: int = 2000
    scale_factor: float = 1.2
    nlevels: int = 8
    ini_th: int = 20
    min_th: int = 7


class Tables:
    """ORBextractor::ORBextractor (:412-475)."""

    def __init__(self, p: ExtractorParams):
        n = p.nlevels
        sf_d = float(np.float32(p.scale_factor))  # member is double, initialised from the float arg
        self.scale = np.ones(n, dtype=np.float32)
        self.sigma2 = np.ones(n, dtype=np.float32)
        for i in range(1, n):
            self.scale[i] = np.float32(float(self.scale[i - 1]) * sf_d)
            self.sigma2[i] = self.scale[i] * self.scale[i]
        self.inv_scale = (np.float32(1.0) / self.scale).astype(np.float32)
        self.inv_sigma2 = (np.float32(1.0) / self.sigma2).astype(np.float32)
        factor = np.float32(1.0 / sf_d)
        denom = np.float32(1.0) - np.float32(math.pow(float(factor), float(n)))
        desired = np.float32(np.float32(np.float32(p.nfeatures) * (np.float32(1) - factor)) / denom)
        self.per_level = [0] * n
        s = 0
        for lvl in range(n - 1):
            self.per_level[lvl] = int(np.rint(desired))
            s += self.per_level[lvl]
            desired = np.float32(desired * factor)
        self.per_level[n - 1] = max(p.nfeatures - s, 0)
        # umax
        umax = [0] * (HALF_PATCH_SIZE + 1)
        sq2 = np.float32(math.sqrt(np.float32(2.0)))  # sqrt(2.f) is float
        vmax = int(math.floor(np.float32(np.float32(HALF_PATCH_SIZE * sq2) / np.float32(2)) + np.float32(1)))
        vmin = int(math.ceil(np.float32(np.float32(HALF_PATCH_SIZE * sq2) / np.float32(2))))
        hp2 = float(HALF_PATCH_SIZE * HALF_PATCH_SIZE)
        for v in range(vmax + 1):
            umax[v] = int(np.rint(math.sqrt(hp2 - v * v)))
        v0 = 0
        for v in range(HALF_PATCH_SIZE, vmin - 1, -1):
            while umax[v0] == umax[v0 + 1]:
                v0 += 1
            umax[v] = v0
            v0 += 1
        self.umax = umax


# ---------------------------------------------------------------------------------- image ops
def reflect101(img: np.ndarray, b: int) -> np.ndarray:
    return np.pad(img, b, mode="reflect")


def resize_linear_u8(src: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """cv::resize(..., INTER_LINEAR) for CV_8UC1: 11-bit fixed-point coefficients."""
    sh, sw = src.shape

    def coeffs(dn, sn):
        scale = float(sn) / float(dn)
        d = np.arange(dn, dtype=np.float64)
        f = ((d + 0.5) * scale - 0.5).astype(np.float32)
        s0 = np.floor(f).astype(np.int32)
        frac = (f - s0.astype(np.float32)).astype(np.float32)
        lo = s0 < 0
        frac = np.where(lo, np.float32(0), frac)
        s0 = np.where(lo, 0, s0)
        hi = s0 >= sn - 1
        frac = np.where(hi, np.float32(0), frac)
        s0 = np.where(hi, sn - 1, s0)
        s1 = np.minimum(s0 + 1, sn - 1)
        # cvRound of the float product, as saturate_cast<short>(float)
        a1 = np.rint(frac * np.float32(2048)).astype(np.int32)
        a0 = np.rint((np.float32(1) - frac) * np.float32(2048)).astype(np.int32)
        return s0, s1, a0, a1

    x0, x1, ax0, ax1 = coeffs(dw, sw)
    y0, y1, by0, by1 = coeffs(dh, sh)
    s = src.astype(np.int32)
    rows = s[:, x0] * ax0[None, :] + s[:, x1] * ax1[None, :]  # [sh, dw]
    r0 = rows[y0]
    r1 = rows[y1]
    out = (((by0[:, None] * (r0 >> 4)) >> 16) + ((by1[:, None] * (r1 >> 4)) >> 16) + 2) >> 2
    return out.astype(np.uint8)


GAUSS7 = np.array([18, 34, 48, 56, 48, 34, 18], dtype=np.int64)  # getGaussianKernel(7, 2) in 8.8 fixed point


def gaussian_blur7(img: np.ndarray) -> np.ndarray:
    """cv::GaussianBlur(img, 7x7, sigma 2, BORDER_REFLECT_101) for CV_8UC1 (fixed-point path)."""
    h, w = img.shape
    p = reflect101(img, 3).astype(np.int64)
    hor = np.zeros((h + 6, w), dtype=np.int64)
    for k in range(7):
        hor += GAUSS7[k] * p[:, k:k + w]
    ver = np.zeros((h, w), dtype=np.int64)
    for k in range(7):
        ver += GAUSS7[k] * hor[k:k + h]
    return ((ver + 32768) >> 16).astype(np.uint8)


def fast_atan2(y: np.ndarray, x: np.ndarray) -> np.ndarray:
    """cv::fastAtan2 (degrees, float32 polynomial, no FMA contraction)."""
    y = np.asarray(y, dtype=np.float32)
    x = np.asarray(x, dtype=np.float32)
    ax, ay = np.abs(x), np.abs(y)
    scale = np.float32(180.0 / math.pi)
    p1 = np.float32(0.9997878412794807) * scale
    p3 = np.float32(-0.3258083974640975) * scale
    p5 = np.float32(0.1555786518463281) * scale
    p7 = np.float32(-0.04432655554792128) * scale
    eps = np.float32(2.220446049250313e-16)
    with np.errstate(divide="ignore", invalid="ignore"):
        big = ax >= ay
        c = np.where(big, ay / (ax + eps), ax / (ay + eps)).astype(np.float32)
        c2 = (c * c).astype(np.float32)
        a = ((((p7 * c2 + p5).astype(np.float32) * c2 + p3).astype(np.float32) * c2 + p1).astype(np.float32) * c)
        a = a.astype(np.float32)
        a = np.where(big, a, np.float32(90.0) - a).astype(np.float32)
        a = np.where(x < 0, np.float32(180.0) - a, a).astype(np.float32)
        a = np.where(y < 0, np.float32(360.0) - a, a).astype(np.float32)
    return a


def fast_score_map(img: np.ndarray) -> np.ndarray:
    """S(p) = max over the 16 contiguous 9-arcs of min_k(+-(ring_k - p)) - 1 for every pixel with a
    3-px margin, 0 elsewhere.  `p is a FAST-9/16 corner at threshold t  <=>  S(p) >= t`, and S is the
    response cv::FAST reports (cornerScore<16>)."""
    h, w = img.shape
    s = img.astype(np.int16)
    c = s[3:h - 3, 3:w - 3]
    d = np.stack([s[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] - c for dx, dy in RING16], axis=0)  # ring - p
    d = np.concatenate([d, d[:8]], axis=0)  # 24 entries, circular
    best = np.full(c.shape, -32768, dtype=np.int16)
    for sgn in (1, -1):
        e = d * sgn
        for i in range(16):
            m = e[i:i + 9].min(axis=0)
            best = np.maximum(best, m)
    out = np.zeros((h, w), dtype=np.int32)
    out[3:h - 3, 3:w - 3] = np.maximum(best.astype(np.int32) - 1, 0)
    return out


def cell_keypoints(score: np.ndarray, x0: int, y0: int, x1: int, y1: int, th: int):
    """cv::FAST(sub-image [y0:y1, x0:x1], th, nonmaxSuppression=true) from a global score map:
    returns (xs, ys, responses) in sub-image row-major order, coordinates relative to (x0, y0)."""
    if x1 - x0 < 7 or y1 - y0 < 7:
        return np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int32)
    sub = np.zeros((y1 - y0, x1 - x0), dtype=np.int32)
    sub[3:-3, 3:-3] = score[y0 + 3:y1 - 3, x0 + 3:x1 - 3]
    sub[sub < th] = 0
    p = np.pad(sub, 1)
    keep = sub > 0
    hh, ww = sub.shape
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx == 0 and dy == 0:
                continue
            keep &= sub > p[1 + dy:1 + dy + hh, 1 + dx:1 + dx + ww]
    ys, xs = np.nonzero(keep)
    return xs.astype(np.int32), ys.astype(np.int32), sub[ys, xs]


# ---------------------------------------------------------------------------------- quad tree
class _Node:
    __slots__ = ("ulx", "uly", "urx", "blx", "bly", "brx", "bry", "ury", "keys", "no_more", "prev", "next", "seq")

    def __init__(self):
        self.keys: List[int] = []
        self.no_more = False
        self.prev = None
        self.next = None
        self.seq = 0


class _List:
    def __init__(self):
        self.head = _Node()
        self.tail = _Node()
        self.head.next = self.tail
        self.tail.prev = self.head
        self.size = 0

    def push_front(self, n):
        n.prev, n.next = self.head, self.head.next
        self.head.next.prev = n
        self.head.next = n
        self.size += 1

    def push_back(self, n):
        n.prev, n.next = self.tail.prev, self.tail
        self.tail.prev.next = n
        self.tail.prev = n
        self.size += 1

    def erase(self, n):
        n.prev.next = n.next
        n.next.prev = n.prev
        self.size -= 1
        return n.next

    def __iter__(self):
        n = self.head.next
        while n is not self.tail:
            yield n
            n = n.next


def _divide(node: _Node, xs, ys):
    half_x = int(math.ceil(np.float32(node.urx - node.ulx) / np.float32(2)))
    half_y = int(math.ceil(np.float32(node.bry - node.uly) / np.float32(2)))
    n = [_Node() for _ in range(4)]
    mx, my = node.ulx + half_x, node.uly + half_y
    n[0].ulx, n[0].uly, n[0].urx, n[0].bry = node.ulx, node.uly, mx, my
    n[1].ulx, n[1].uly, n[1].urx, n[1].bry = mx, node.uly, node.urx, my
    n[2].ulx, n[2].uly, n[2].urx, n[2].bry = node.ulx, my, mx, node.bry
    n[3].ulx, n[3].uly, n[3].urx, n[3].bry = mx, my, node.urx, node.bry
    for k in node.keys:
        if xs[k] < mx:
            (n[0] if ys[k] < my else n[2]).keys.append(k)
        elif ys[k] < my:
            n[1].keys.append(k)
        else:
            n[3].keys.append(k)
    for c in n:
        if len(c.keys) == 1:
            c.no_more = True
    return n


def distribute_octtree(xs: np.ndarray, ys: np.ndarray, resp: np.ndarray, min_x: int, max_x: int,
                       min_y: int, max_y: int, n_target: int) -> List[int]:
    """Indices (into xs/ys/resp) of the retained keypoints, in the reference's output order."""
    xs = np.asarray(xs, dtype=np.float32)
    ys = np.asarray(ys, dtype=np.float32)
    n_ini = int(np.float32(max_x - min_x) / np.float32(max_y - min_y) + np.float32(0.5))  # round(), positive
    n_ini = max(n_ini, 1)
    hx = np.float32(np.float32(max_x - min_x) / np.float32(n_ini))
    lst = _List()
    ini = []
    for i in range(n_ini):
        nd = _Node()
        nd.ulx = int(np.float32(hx * np.float32(i)))
        nd.urx = int(np.float32(hx * np.float32(i + 1)))
        nd.uly = 0
        nd.bry = max_y - min_y
        lst.push_back(nd)
        ini.append(nd)
    for k in range(len(xs)):
        ini[int(np.float32(xs[k] / hx))].keys.append(k)
    nd = lst.head.next
    while nd is not lst.tail:
        if len(nd.keys) == 1:
            nd.no_more = True
            nd = nd.next
        elif len(nd.keys) == 0:
            nd = lst.erase(nd)
        else:
            nd = nd.next
    seq = 0
    finish = False
    pending: List[_Node] = []

    def add_children(children):
        nonlocal seq
        added = 0
        for c in children:
            if len(c.keys) > 0:
                lst.push_front(c)
                if len(c.keys) > 1:
                    added += 1
                    seq += 1
                    c.seq = seq
                    pending.append(c)
        return added

    while not finish:
        prev_size = lst.size
        n_expand = 0
        pending = []
        nd = lst.head.next
        while nd is not lst.tail:
            if nd.no_more:
                nd = nd.next
                continue
            n_expand += add_children(_divide(nd, xs, ys))
            nd = lst.erase(nd)
        if lst.size >= n_target or lst.size == prev_size:
            finish = True
        elif lst.size + n_expand * 3 > n_target:
            while not finish:
                prev_size = lst.size
                prev = sorted(pending, key=lambda c: (len(c.keys), c.seq))
                pending = []
                for c in reversed(prev):
                    add_children(_divide(c, xs, ys))
                    lst.erase(c)
                    if lst.size >= n_target:
                        break
                if lst.size >= n_target or lst.size == prev_size:
                    finish = True
    out = []
    for nd in lst:
        best = nd.keys[0]
        for k in nd.keys[1:]:
            if resp[k] > resp[best]:
                best = k
        out.append(best)
    return out


# ---------------------------------------------------------------------------------- extractor
@dataclass
class OrbResult:
    keypoints: np.ndarray     # [N, 7] float64 columns: x, y, size, angle, response, octave, class_id(-1)
    descriptors: np.ndarray   # [N, 32] uint8
    pyramid: List[np.ndarray]  # bordered level buffers (level image = [19:-19, 19:-19])
    level_counts: List[int]
    candidates: List[Tuple[np.ndarray, np.ndarray, np.ndarray]]  # per level (x, y, response) before the quad tree


def level_sizes(w: int, h: int, tables: Tables) -> List[Tuple[int, int]]:
    out = []
    for s in tables.inv_scale:
        out.append((int(np.rint(np.float32(w) * s)), int(np.rint(np.float32(h) * s))))
    return out


def compute_pyramid(image: np.ndarray, tables: Tables) -> List[np.ndarray]:
    h, w = image.shape
    levels = []
    prev = image
    for lvl, (lw, lh) in enumerate(level_sizes(w, h, tables)):
        cur = image if lvl == 0 else resize_linear_u8(prev, lw, lh)
        levels.append(reflect101(cur, EDGE_THRESHOLD))
        prev = cur
    return levels


def level_cells(lw: int, lh: int):
    """Cell rectangles of ComputeKeyPointsOctTree (:759-805) in level-image coordinates."""
    min_bx = min_by = EDGE_THRESHOLD - 3
    max_bx = lw - EDGE_THRESHOLD + 3
    max_by = lh - EDGE_THRESHOLD + 3
    width = np.float32(max_bx - min_bx)
    height = np.float32(max_by - min_by)
    n_cols = int(width / np.float32(30))
    n_rows = int(height / np.float32(30))
    w_cell = int(math.ceil(width / np.float32(n_cols)))
    h_cell = int(math.ceil(height / np.float32(n_rows)))
    cells = []
    for i in range(n_rows):
        ini_y = min_by + i * h_cell
        max_y = ini_y + h_cell + 6
        if ini_y >= max_by - 3:
            continue
        max_y = min(max_y, max_by)
        for j in range(n_cols):
            ini_x = min_bx + j * w_cell
            max_x = ini_x + w_cell + 6
            if ini_x >= max_bx - 6:
                continue
            max_x = min(max_x, max_bx)
            cells.append((ini_x, ini_y, max_x, max_y))
    return cells, (min_bx, min_by, max_bx, max_by)


def ic_angle(bordered: np.ndarray, x: int, y: int, umax: List[int]) -> np.float32:
    cx, cy = x + EDGE_THRESHOLD, y + EDGE_THRESHOLD
    img = bordered.astype(np.int64)
    m01 = 0
    m10 = 0
    for u in range(-HALF_PATCH_SIZE, HALF_PATCH_SIZE + 1):
        m10 += u * int(img[cy, cx + u])
    for v in range(1, HALF_PATCH_SIZE + 1):
        d = umax[v]
        u = np.arange(-d, d + 1)
        plus = img[cy + v, cx - d:cx + d + 1]
        minus = img[cy - v, cx - d:cx + d + 1]
        m01 += v * int((plus - minus).sum())
        m10 += int((u * (plus + minus)).sum())
    return fast_atan2(np.float32(m01), np.float32(m10))


def orb_descriptor(blur: np.ndarray, x: int, y: int, angle_deg: np.float32, pattern: np.ndarray) -> np.ndarray:
    h, w = blur.shape
    flat = blur.reshape(-1)
    factor_pi = np.float32(math.pi / np.float32(180.0))
    ang = np.float32(np.float32(angle_deg) * factor_pi)
    a = np.float32(math.cos(float(ang)))
    b = np.float32(math.sin(float(ang)))
    px = pattern[:, [0, 2]].astype(np.float32)  # [256, 2]
    py = pattern[:, [1, 3]].astype(np.float32)
    ry = cv_round((px * b).astype(np.float32) + (py * a).astype(np.float32))
    rx = cv_round((px * a).astype(np.float32) - (py * b).astype(np.float32))
    idx = (y + ry) * w + (x + rx)
    ok = (idx >= 0) & (idx < w * h)
    val = np.where(ok, flat[np.clip(idx, 0, w * h - 1)], 0).astype(np.int32)
    bits = (val[:, 0] < val[:, 1]).astype(np.uint8).reshape(32, 8)
    return (bits << np.arange(8, dtype=np.uint8)).sum(axis=1).astype(np.uint8)


def extract(image: np.ndarray, params: ExtractorParams = ExtractorParams()) -> OrbResult:
    assert image.dtype == np.uint8 and image.ndim == 2
    tables = Tables(params)
    pattern = load_pattern()
    pyr = compute_pyramid(image, tables)
    all_kps = []
    cands = []
    for lvl in range(params.nlevels):
        bordered = pyr[lvl]
        lh, lw = bordered.shape[0] - 2 * EDGE_THRESHOLD, bordered.shape[1] - 2 * EDGE_THRESHOLD
        lvl_img = bordered[EDGE_THRESHOLD:-EDGE_THRESHOLD, EDGE_THRESHOLD:-EDGE_THRESHOLD]
        score = fast_score_map(np.ascontiguousarray(lvl_img))
        cells, (min_bx, min_by, max_bx, max_by) = level_cells(lw, lh)
        cx, cy, cr = [], [], []
        for (x0, y0, x1, y1) in cells:
            xs, ys, rs = cell_keypoints(score, x0, y0, x1, y1, params.ini_th)
            if len(xs) == 0:
                xs, ys, rs = cell_keypoints(score, x0, y0, x1, y1, params.min_th)
            cx.append(xs + (x0 - min_bx))
            cy.append(ys + (y0 - min_by))
            cr.append(rs)
        cx = np.concatenate(cx) if cx else np.zeros(0, np.int32)
        cy = np.concatenate(cy) if cy else np.zeros(0, np.int32)
        cr = np.concatenate(cr) if cr else np.zeros(0, np.int32)
        cands.append((cx, cy, cr))
        sel = distribute_octtree(cx, cy, cr.astype(np.float32), min_bx, max_bx, min_by, max_by,
                                 tables.per_level[lvl]) if len(cx) else []
        size = np.float32(int(np.float32(PATCH_SIZE) * tables.scale[lvl]))
        kps = []
        for k in sel:
            x, y = int(cx[k]) + min_bx, int(cy[k]) + min_by
            ang = ic_angle(bordered, x, y, tables.umax)
            kps.append([x, y, size, ang, np.float32(cr[k]), lvl])
        all_kps.append(kps)
    out_k = []
    out_d = []
    counts = []
    for lvl in range(params.nlevels):
        kps = all_kps[lvl]
        counts.append(len(kps))
        if not kps:
            continue
        bordered = pyr[lvl]
        lvl_img = np.ascontiguousarray(bordered[EDGE_THRESHOLD:-EDGE_THRESHOLD, EDGE_THRESHOLD:-EDGE_THRESHOLD])
        blur = gaussian_blur7(lvl_img)
        sc = tables.scale[lvl]
        for (x, y, size, ang, resp, octave) in kps:
            out_d.append(orb_descriptor(blur, x, y, ang, pattern))
            fx, fy = np.float32(x), np.float32(y)
            if lvl != 0:
                fx, fy = np.float32(fx * sc), np.float32(fy * sc)
            out_k.append([fx, fy, size, ang, resp, octave, -1])
    kp = np.array(out_k, dtype=np.float64).reshape(-1, 7)
    desc = np.array(out_d, dtype=np.uint8).reshape(-1, 32)
    return OrbResult(kp, desc, pyr, counts, cands)


# ---------------------------------------------------------------------------------- Hamming
def descriptor_distance(a: np.ndarray, b: np.ndarray) -> int:
    """ORBmatcher::DescriptorDistance (src/orbslam/ORBmatcher.cc:1582-1596): popcount of a XOR b."""
    return int(np.unpackbits(np.bitwise_xor(a, b)).sum())


def compute_stereo_matches(kl, dl, kr, dr, pyr_l, pyr_r, scale, inv_scale, mb, mbf):
    """Frame::ComputeStereoMatches (src/orbslam/Frame.cc:444-629) restated: row table, Hamming search with the octave
    and disparity gates, 11x11 SAD slide on the keypoint's pyramid level, parabola fit, median-based outlier cut.
    kl / kr: structured keypoint arrays (x, y, octave), dl / dr: [N, 32] u8, pyr_*: bordered level buffers.
    Returns (mvRight, mvDepth) float32 arrays."""
    f32 = np.float32
    n_l = len(kl)
    u_right = np.full(n_l, -1.0, f32)
    depth = np.full(n_l, -1.0, f32)
    rows = pyr_l[0].shape[0] - 2 * EDGE_THRESHOLD
    table = [[] for _ in range(rows)]
    for i in range(len(kr)):
        r = f32(2.0) * scale[kr["octave"][i]]
        lo, hi = int(np.floor(f32(kr["y"][i] - r))), int(np.ceil(f32(kr["y"][i] + r)))
        for y in range(lo, hi + 1):
            table[y].append(i)
    th_orb = (100 + 50) // 2
    min_d, max_d = f32(0), f32(f32(mbf) / f32(mb))
    cand = []

    def c_round(v):
        return f32(np.floor(v + f32(0.5))) if v >= 0 else f32(-np.floor(-v + f32(0.5)))
    for il in range(n_l):
        ul, vl, lv = f32(kl["x"][il]), f32(kl["y"][il]), int(kl["octave"][il])
        cands = table[int(vl)]
        if not cands:
            continue
        min_u, max_u = f32(ul - max_d), f32(ul - min_d)
        if max_u < 0:
            continue
        best, best_i = 100, 0
        for j in cands:
            if kr["octave"][j] < lv - 1 or kr["octave"][j] > lv + 1:
                continue
            if min_u <= kr["x"][j] <= max_u:
                d = descriptor_distance(dl[il], dr[j])
                if d < best:
                    best, best_i = d, j
        if best >= th_orb:
            continue
        sf = inv_scale[lv]
        su_l, sv_l, su_r0 = c_round(f32(ul * sf)), c_round(f32(vl * sf)), c_round(f32(kr["x"][best_i] * sf))
        img_l = pyr_l[lv][EDGE_THRESHOLD:-EDGE_THRESHOLD, EDGE_THRESHOLD:-EDGE_THRESHOLD].astype(np.int64)
        img_r = pyr_r[lv][EDGE_THRESHOLD:-EDGE_THRESHOLD, EDGE_THRESHOLD:-EDGE_THRESHOLD].astype(np.int64)
        w = 5
        cy, cxl, cxr = int(sv_l), int(su_l), int(su_r0)
        if su_r0 + 5 - 5 < 0 or su_r0 + 5 + 5 + 1 >= img_r.shape[1]:
            continue
        il_win = img_l[cy - w:cy + w + 1, cxl - w:cxl + w + 1]
        il_win = il_win - il_win[w, w]
        dists = []
        for inc in range(-5, 6):
            ir_win = img_r[cy - w:cy + w + 1, cxr + inc - w:cxr + inc + w + 1]
            ir_win = ir_win - ir_win[w, w]
            dists.append(int(np.abs(il_win - ir_win).sum()))
        bd, binc = 2 ** 31 - 1, 0
        for k, d in enumerate(dists):
            if d < bd:
                bd, binc = d, k - 5
        if binc in (-5, 5):
            continue
        d1, d2, d3 = f32(dists[binc + 4]), f32(dists[binc + 5]), f32(dists[binc + 6])
        with np.errstate(divide="ignore", invalid="ignore"):
            delta = f32(f32(d1 - d3) / f32(f32(2.0) * f32(f32(d1 + d3) - f32(f32(2.0) * d2))))
        if delta < -1 or delta > 1 or np.isnan(delta):
            continue
        best_u = f32(scale[lv] * f32(f32(su_r0 + f32(binc)) + delta))
        disp = f32(ul - best_u)
        if min_d <= disp < max_d:
            if disp <= 0:
                disp = f32(0.01)
                best_u = f32(float(ul) - 0.01)
            depth[il] = f32(f32(mbf) / disp)
            u_right[il] = best_u
            cand.append((bd, il))
    if cand:
        cand.sort()
        median = f32(cand[len(cand) // 2][0])
        th = f32(1.5) * f32(1.4) * median
        for d, il in reversed(cand):
            if f32(d) < th:
                break
            u_right[il] = -1
            depth[il] = -1
    return u_right, depth


def select_semantic_keys(kps_xy, classes, confidence=None, entropy=None, max_static_class=8):
    """Frame::SelectSemanticKeys (Frame.cc:177-203): col = int(pt.x), row = int(pt.y) (C++ truncation), keep the keypoint
    iff mClasses(row, col) <= Classes::TERRAIN (= 8, bayesian_segnet.hpp:67-83), in keypoint order.  Also returns the per-keypoint
    reads of the maps (what Tracking.cc:487,538 / LocalMapping.cc:483-485 look up later).  kps_xy: [n, 2] float32 (x, y)."""
    kps_xy = np.asarray(kps_xy, np.float32)
    col = np.trunc(kps_xy[:, 0]).astype(np.int64)
    row = np.trunc(kps_xy[:, 1]).astype(np.int64)
    cls = classes[row, col]
    keep = np.nonzero(cls <= max_static_class)[0].astype(np.int32)
    conf = confidence[row, col] if confidence is not None else None
    ent = entropy[row, col] if entropy is not None else None
    return cls, conf, ent, keep


def hamming_best2(query_desc, train_desc, cand_offsets, cand_idx, train_level=None):
    """The candidate loop of ORBmatcher::SearchByProjection (ORBmatcher.cc:79-113; the same loop body recurs at :1278-, :1420-,
    :631-) as written: strict '<' on both tests, levels carried with the distances.  DescriptorDistance (:1582-1596) is the
    popcount of the XOR of the two 256-bit descriptors.  Returns int32 [n_query, 5] = bestIdx, bestDist, bestLevel, bestDist2,
    bestLevel2 (256 / -1 defaults)."""
    q = np.asarray(query_desc, np.uint8).reshape(-1, 32)
    t = np.asarray(train_desc, np.uint8).reshape(-1, 32)
    out = np.empty((len(q), 5), np.int32)
    for i in range(len(q)):
        best_dist, best_level, best_dist2, best_level2, best_idx = 256, -1, 256, -1, -1
        for idx in cand_idx[cand_offsets[i]:cand_offsets[i + 1]]:
            dist = int(np.unpackbits(q[i] ^ t[idx]).sum())
            lvl = 0 if train_level is None else int(train_level[idx])
            if dist < best_dist:
                best_dist2, best_level2 = best_dist, best_level
                best_dist, best_level, best_idx = dist, lvl, int(idx)
            elif dist < best_dist2:
                best_level2, best_dist2 = lvl, dist
        out[i] = (best_idx, best_dist, best_level, best_dist2, best_level2)
    return out
