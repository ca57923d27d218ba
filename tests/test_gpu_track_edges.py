"""-m gpu: the projection searches (sivo_search_local_points / _last_frame, host and device forms) on constructed worst cases
against oracle/track_oracle.py bit for bit.  The device folds every point once without claims and then re-searches, in order,
only the points whose recorded best (local: or second-best) key an earlier point took; these cases put that argument where it
can fail: crowded windows whose column ranges span several 32-key chunks, exact distance ties, long chains of claims, every
decision boundary hit exactly, the grid's bounds, the level clamps, the size limits and a seeded differential fuzz.

Every comparison is the same: in_view, match and n_matches of both forms equal the oracle's.  The device form runs on
extractor-sized buffers through an oracle/keymap.py map whose rejected entries are keys in no cell, with decoy records and a
blocked mask; the host form on the gathered keys."""
import numpy as np
import pytest
import torch

from frame_support import extractor, i64, sentinel, upload
from oracle import track_oracle as T
from oracle.keymap import SLACK, keymap, scatter
from oracle.track_scene import MP, RESERVED, desc_with, keys, point_at
from sivo_b200 import _lib as L
from sivo_b200 import (KP_DTYPE, make_frame, search_last_frame, search_last_frame_device,
                       search_local_points, search_local_points_device)
from sivo_b200.track import features_in_area

pytestmark = pytest.mark.gpu

F32 = np.float32
FX, CX, CY, MBF = 700.0, 512.0, 176.0, 380.0
BOUNDS = (0.0, 1024.0, 0.0, 352.0)
UP, DOWN = F32(np.inf), F32(-np.inf)
DIRECTIONS = {"forward": (0.0, 0.0, 1.0), "backward": (0.0, 0.0, -1.0), "neither": (0.0, 0.0, 0.0)}  # tlw; mb = 380 / 700


def ulp(x, toward):
    return np.nextafter(F32(x), toward)


def oframe(bounds=BOUNDS, R=np.eye(3), t=(0, 0, 0)):
    return T.Frame(FX, FX, CX, CY, MBF, bounds, R, t)


def point(pos, desc, observed=1, octave=0, angle=0.0, normal=None, max_distance=None):
    """A map point at world position pos (seen head-on from the origin unless a normal is given)."""
    p = np.zeros((), MP)
    p["pos"] = np.asarray(pos, F32)
    d = T.norm3(p["pos"])
    p["normal"] = p["pos"] / d if normal is None else np.asarray(normal, F32)
    p["max_distance"] = d if max_distance is None else max_distance
    p["min_distance"] = p["max_distance"] / F32(1.2) ** 7
    p["desc"], p["observed"], p["octave"], p["angle"], p["reserved"] = desc, observed, octave, angle, RESERVED
    return p


def flip(desc, bits):
    d = desc.copy()
    for b in bits:
        d[b // 8] ^= np.uint8(1 << (b % 8))
    return d


class Scene:
    """One search input: keys (oracle records), descriptors, mvRight, points, the current pose and bounds, th, nnratio,
    blocked on entry (local search) and the last frame's pose (last-frame search)."""

    def __init__(self, k, d, pts, ur=None, th=1.0, nnratio=0.8, blocked=None, R=np.eye(3), t=np.zeros(3), bounds=BOUNDS,
                 Rlw=np.eye(3), tlw=np.zeros(3)):
        self.k = k
        self.d = np.ascontiguousarray(np.asarray(d, np.uint8).reshape(-1, 32))
        self.pts = np.array(pts, MP) if isinstance(pts, list) else np.asarray(pts).astype(MP)
        self.ur = np.full(len(k), -1, F32) if ur is None else np.asarray(ur, F32)
        self.th, self.nnratio = F32(th), F32(nnratio)
        self.blocked = None if blocked is None else np.asarray(blocked, np.uint8)
        self.R, self.t, self.bounds = np.asarray(R, F32), np.asarray(t, F32), bounds
        self.Rlw, self.tlw = np.asarray(Rlw, F32), np.asarray(tlw, F32)

    def frames(self):
        return make_frame(FX, FX, CX, CY, MBF, self.bounds, self.R, self.t), oframe(self.bounds, self.R, self.t)


class Searcher:
    """Runs a scene through the oracle, the host form and the device form of one extractor and asserts bit identity."""

    def __init__(self, el, seed):
        self.el, self.cap, self.scale = el, el.capacity(), el.GetScaleFactors()
        self.rng = np.random.default_rng(seed)

    def device(self, sc, last):
        """The device form: semantic key j sits at its slot of an oracle/keymap.py map, in capacity-sized buffers whose other
        records are decoys (copies of the scene's keys); the map's rejected entries must stay unmatched, and blocked marks them."""
        n, m, cap = len(sc.k), len(sc.pts), self.cap
        km = keymap(n, cap, self.rng)
        nk, real, rejected = km.n_keep, km.real, km.src < 0
        decoy = sc.k[self.rng.integers(0, n, cap + SLACK)] if n else np.zeros(1, KP_DTYPE)
        kps = scatter(sc.k, km.slots, cap, decoy)
        desc = scatter(sc.d, km.slots, cap, self.rng.integers(0, 256, (cap + SLACK, 32), dtype=np.uint8))
        ur = self.rng.uniform(-5, 1030, len(km.keep)).astype(F32)
        ur[real] = sc.ur
        blocked = np.zeros(len(km.keep), np.uint8)
        blocked[np.flatnonzero(rejected)] = 1
        if sc.blocked is not None:
            blocked[real] = sc.blocked
        bufs = [upload(kps), upload(desc), upload(km.keep), i64(nk), upload(ur), upload(blocked)]
        pts = upload(sc.pts) if m else None
        view, match, nm = sentinel(max(m, 1), 7, torch.uint8), sentinel(cap, -7, torch.int32), sentinel(1, -7, torch.int64)
        frame, _ = sc.frames()
        p = [b.data_ptr() for b in bufs]
        pp = pts.data_ptr() if m else 0
        torch.cuda.synchronize()
        if last:
            search_last_frame_device(self.el, p[0], p[1], p[2], p[3], p[4], pp, m, frame, sc.Rlw, sc.tlw, sc.th, match.data_ptr(),
                                     nm.data_ptr())
        else:
            search_local_points_device(self.el, p[0], p[1], p[2], p[3], p[4], p[5], pp, m, frame, sc.th, sc.nnratio, view.data_ptr(),
                                       match.data_ptr(), nm.data_ptr())
        torch.cuda.synchronize()
        mt, v = match.cpu().numpy(), view.cpu().numpy()
        assert (mt[:nk][rejected] == -1).all() and (mt[nk:] == -7).all()
        assert (v == 7).all() if last else set(np.unique(v[:m])) <= {0, 1}
        return v[:m].astype(bool), mt[real].copy(), int(nm.cpu()[0])

    def local(self, sc, per_point=None):
        frame, of = sc.frames()
        ov, om, on = T.search_local_points(sc.k, sc.d, sc.ur, sc.pts, of, self.scale, sc.th, sc.nnratio, sc.blocked, per_point)
        hv, hm, hn = search_local_points(self.el, sc.k, sc.d, sc.ur, sc.pts, frame, sc.th, sc.nnratio,
                                         sc.blocked)
        assert np.array_equal(hv, ov) and np.array_equal(hm, om) and hn == on, "host form"
        dv, dm, dn = self.device(sc, False)
        assert np.array_equal(dv, ov) and np.array_equal(dm, om) and dn == on, "device form"
        return ov, om, on

    def last(self, sc):
        frame, of = sc.frames()
        om, on = T.search_last_frame(sc.k, sc.d, sc.ur, sc.pts, of, sc.Rlw, sc.tlw, self.scale, sc.th)
        hm, hn = search_last_frame(self.el, sc.k, sc.d, sc.ur, sc.pts, frame, sc.Rlw, sc.tlw, sc.th)
        assert np.array_equal(hm, om) and hn == on, "host form"
        _, dm, dn = self.device(sc, True)
        assert np.array_equal(dm, om) and dn == on, "device form"
        return om, on


@pytest.fixture(scope="module")
def s8():
    return Searcher(extractor(1000, 1.2, 8), 1)


@pytest.fixture(scope="module")
def s4():
    return Searcher(extractor(500, 1.5, 4), 2)


def per_point_changes(s, sc):
    """Points whose accepted key differs between the sequential search and the same points searched without claims: the
    ordered pass had to search each of them again."""
    per, free = [], []
    T.search_local_points(sc.k, sc.d, sc.ur, sc.pts, oframe(sc.bounds, sc.R, sc.t), s.scale, sc.th, sc.nnratio, sc.blocked, per)
    lone = sc.pts.copy()
    lone["observed"] = 0
    T.search_local_points(sc.k, sc.d, sc.ur, lone, oframe(sc.bounds, sc.R, sc.t), s.scale, sc.th, sc.nnratio, None, free)
    return sum(a != b for a, b in zip(per, free))


# ---------------------------------------------------------------------------------------------------------- hand-built cases
def test_oracle_hand_built_cases_on_both_forms(s8):
    """The cases of test_oracle_track.py, with their expected outcomes, through both forms."""
    f = oframe()
    # claims: an observed point blocks its key for later points, an unobserved one does not; keys blocked on entry
    k = keys([(500, 100), (501, 100)])
    d = [desc_with([]), desc_with([1])]
    pts = [point_at(f, 500.2, 100, 10, desc_with([])), point_at(f, 500.3, 100, 10, desc_with([]))]
    assert list(s8.local(Scene(k, d, pts))[1]) == [0, 1]
    m, n = s8.last(Scene(k, d, pts, th=7))
    assert list(m) == [0, 1] and n == 2
    pts[0]["observed"] = 0
    _, m, n = s8.local(Scene(k, d, pts))
    assert list(m) == [1, -1] and n == 2
    m, n = s8.last(Scene(k, d, pts, th=7))
    assert list(m) == [1, -1] and n == 2
    _, m, n = s8.local(Scene(k, d, pts[1:], blocked=[1, 0]))
    assert list(m) == [-1, 0] and n == 1
    # the ratio test applies only on equal levels
    k = keys([(500, 100), (501, 100)], 0)
    d = [desc_with(range(10)), desc_with(range(11))]
    q = [point_at(f, 500.5, 100, 10, desc_with([]))]
    assert s8.local(Scene(k, d, q))[2] == 0
    k["octave"][1] = 1
    assert list(s8.local(Scene(k, d, q))[1]) == [0, -1]
    k["octave"][1] = 0
    assert s8.local(Scene(k, [desc_with(range(10)), desc_with(range(13))], q))[2] == 1
    # frustum edges: behind the camera, Pc = 0, NaN, the 0.8 / 1.2 distance limits exactly
    p = point_at(f, 500, 100, 10, desc_with([]))
    dist = T.norm3(p["pos"] - f.Ow)
    edge = [p.copy() for _ in range(7)]
    edge[1]["pos"] = -p["pos"]
    edge[2]["pos"] = (0, 0, 0)
    edge[3]["pos"] = (np.nan, 0, 5)
    edge[4]["max_distance"], edge[4]["min_distance"] = dist / F32(1.2), 0
    edge[5]["max_distance"], edge[5]["min_distance"] = dist, dist / F32(0.8)
    edge[6]["max_distance"] = dist * F32(0.5)
    for e in edge:
        e["observed"] = 0
    want = [True, False, False, False] + [F32(0.8) * e["min_distance"] <= dist <= F32(1.2) * e["max_distance"] for e in edge[4:6]] + [False]
    view, m, n = s8.local(Scene(keys([(500, 100)]), [desc_with([])], edge))
    assert list(view) == want and n == sum(want)
    s8.last(Scene(keys([(500, 100)]), [desc_with([])], edge, th=7))
    # ComputeThreeMaxima: ties (the first of equals wins each rank) and the tenth rule exactly at max2 == 0.1f * max1
    row = keys([(100 + 20 * i, 100) for i in range(40)], 0, 0.0)
    rd = [desc_with([i]) for i in range(40)]
    for counts, keep in (({3: 10, 5: 10, 7: 10}, (3, 5, 7)), ({3: 10, 5: 10, 7: 10, 9: 10}, (3, 5, 7)), ({2: 20, 4: 2, 6: 1}, (2, 4)),
                         ({2: 20, 4: 1, 6: 1}, (2,)), ({0: 30, 1: 3, 2: 2}, (0, 1)), ({12: 4, 0: 4, 6: 1}, (0, 6, 12)), ({12: 40}, (12,))):
        bins = [b for b, c in sorted(counts.items()) for _ in range(c)]
        pts = [point_at(f, 100 + 20 * i, 100, 10, desc_with([i]), angle=30.0 * b) for i, b in enumerate(bins)]
        m, n = s8.last(Scene(row, rd, pts, th=7))
        assert n == sum(counts[b] for b in keep) and [m[i] >= 0 for i in range(len(bins))] == [b in keep for b in bins], counts
    # the culling of duplicates: the losing bin's entry frees the key, every entry counts
    a = point_at(f, 100, 100, 10, desc_with([0]), observed=0, angle=0.0)
    b = point_at(f, 100, 100, 10, desc_with([0]), observed=0, angle=100.0)
    m, n = s8.last(Scene(row, rd, [a] * 5 + [b], th=7))
    assert n == 6 and m[0] == 5
    m, n = s8.last(Scene(row, rd, [a] * 11 + [b] + [a], th=7))
    assert n == 12 and m[0] == -1


# ---------------------------------------------------------------------------------------------------------- dense contention
def dense_scene(seed, n_keys=600, n_points=160, n_desc=4):
    """n_keys keys inside a 36 x 36 px square (three grid columns of about 200 keys), n_desc distinct descriptors, points of
    level 1 over the square whose best keys coincide, observed and unobserved alternating."""
    rng = np.random.default_rng(seed)
    f = oframe()
    xy = np.c_[rng.uniform(482, 518, n_keys), rng.uniform(132, 168, n_keys)]
    xy[: n_keys // 4] = np.round(xy[: n_keys // 4] * 2) / 2  # repeated positions
    k = keys(xy, 0, 0.0)
    k["octave"] = rng.integers(0, 2, n_keys)
    k["angle"] = rng.choice([0.0, 10.0, 100.0, 250.0, 359.0], n_keys)
    base = rng.integers(0, 256, (n_desc, 32), dtype=np.uint8)
    d = base[rng.integers(0, n_desc, n_keys)]
    pts = []
    for i in range(n_points):
        c = rng.integers(n_desc)
        q = base[c] if i % 3 else flip(base[c], rng.choice(256, rng.integers(1, 3), replace=False))
        p = point_at(f, rng.uniform(496, 504), rng.uniform(146, 154), 10, q, observed=i % 2, octave=1, angle=float(rng.choice([0, 100, 250])))
        p["max_distance"] *= F32(1.1)  # PredictScale: ceil(log(1.1) / log(1.2)) = level 1
        pts.append(p)
    return Scene(k, d, pts, th=8), k


def test_dense_windows_span_several_chunks_and_columns(s8):
    changed = 0
    for seed in range(2):
        sc, k = dense_scene(seed)
        _, of = sc.frames()
        # the window of a point at the square's centre: some column's walk holds more than 32 candidates
        got = features_in_area(s8.el, k, BOUNDS, [(500.0, 150.0, 24.0, 0, 1)])[0]
        per_col = np.bincount([T.pos_in_grid(k["x"][j], k["y"][j], of)[0] for j in got])
        assert per_col.max() > 64, per_col
        view, m, n = s8.local(sc)
        assert view.all() and n > 20
        changed += per_point_changes(s8, sc)
        m, n = s8.last(sc)
        assert n > 20
        sc.th = F32(20)
        s8.last(sc)
    assert changed > 50  # a long chain: most points were searched again


def test_second_best_ties_change_the_ratio_test(s8):
    """Point 1's recorded best is key A and its second is key B (tied with key C, walked later); point 0 takes B, so point 1's
    new second-best is C, on the other level: the ratio test's outcome flips and only a re-search triggered by the taken second
    key finds it."""
    f = oframe()
    changed = 0
    for lv_a, lv_b, lv_c in ((1, 1, 0), (0, 1, 0)):
        k = keys([(500, 100), (501, 100), (501.5, 100)])
        k["octave"] = lv_a, lv_b, lv_c
        d = [desc_with(range(9)), desc_with(range(20, 30)), desc_with(range(40, 50))]
        p0 = point_at(f, 501, 100, 10, d[1])
        p1 = point_at(f, 500.5, 100, 10, desc_with([]))
        for p in (p0, p1):
            p["max_distance"] *= F32(1.1)  # level 1: the window holds levels 0 and 1
        sc = Scene(k, d, [p0, p1])
        _, m, n = s8.local(sc)
        assert m[1] == 0 and (m[0] == 1) == (lv_a != lv_c)
        changed += per_point_changes(s8, sc)
    assert changed == 2


# ---------------------------------------------------------------------------------------------------------- decision boundaries
def test_th_high_at_100_and_101(s8):
    f = oframe()
    k = keys([(500, 100), (600, 100)])
    d = [desc_with(range(100)), desc_with(range(101))]
    pts = [point_at(f, 500, 100, 10, desc_with([])), point_at(f, 600, 100, 10, desc_with([]))]
    assert list(s8.local(Scene(k, d, pts))[1]) == [0, -1]
    assert list(s8.last(Scene(k, d, pts, th=7))[0]) == [0, -1]


def test_ratio_test_at_equality_and_one_ulp_either_side(s8):
    f = oframe()
    k = keys([(500, 100), (501, 100)])
    q = [point_at(f, 500.5, 100, 10, desc_with([]))]
    d = [desc_with(range(8)), desc_with(range(8, 18))]  # 8 vs 10: 0.8f * 10 rounds to 8.0f
    assert F32(0.8) * F32(10) == F32(8)
    for nn, accepted in ((0.8, True), (ulp(0.8, DOWN), False), (ulp(0.8, UP), True)):
        assert (s8.local(Scene(k, d, q, nnratio=nn))[2] == 1) == accepted, nn
    assert s8.local(Scene(k, [desc_with(range(9)), d[1]], q))[2] == 0


def test_stereo_gate_at_the_radius(s8):
    """Point on the optical axis at z = 2: u = 512, projXR = 512 - 380 / 2 = 322, radius 2.5 (local, th 1, level 0, head-on)
    and th 2.5 (last frame, octave 0).  A key with u_right > 0 stays a candidate iff |projXR - u_right| <= radius."""
    f = oframe()
    p = [point_at(f, 512, 176, 2, desc_with([]))]
    k = keys([(512.5, 176)])
    for ur, kept in ((324.5, True), (ulp(324.5, UP), False), (319.5, True), (ulp(319.5, DOWN), False), (0.0, True), (-0.0, True),
                     (-3.0, True), (-330.0, True)):
        sc = Scene(k, [desc_with([])], p, ur=[ur])
        assert (s8.local(sc)[2] == 1) == kept, ur
        sc.th = F32(2.5)
        assert (s8.last(sc)[1] == 1) == kept, ur


def test_viewing_cosine_and_th_boundaries(s8):
    """On the optical axis viewCos is the normal's z exactly.  0.5 is in view, the float below is not; F32(0.998) > 0.998 in
    double gives radius 2.5, the float below 4.  th == 1 leaves the radius alone; one ulp either side multiplies it."""
    z = 10.0
    pos = (0.0, 0.0, z)

    def axis_point(c):
        return point(pos, desc_with([]), normal=(np.sqrt(1 - F32(c) ** 2), 0, c))
    k = keys([(512, 176)])
    view, _, _ = s8.local(Scene(k, [desc_with([])], [axis_point(F32(0.5)), axis_point(ulp(0.5, DOWN))]))
    assert list(view) == [True, False]
    far = keys([(515, 176)])  # 3 px off: inside radius 4, outside 2.5
    assert s8.local(Scene(far, [desc_with([])], [axis_point(F32(0.998))]))[2] == 0
    assert s8.local(Scene(far, [desc_with([])], [axis_point(ulp(0.998, DOWN))]))[2] == 1
    edge = keys([(514.5, 176)])  # 2.5 px off: |dx| < r needs r > 2.5
    for th, hit in ((1.0, False), (ulp(1.0, UP), True), (ulp(1.0, DOWN), False)):
        assert s8.local(Scene(edge, [desc_with([])], [axis_point(1.0)], th=th))[2] == int(hit), th


# ---------------------------------------------------------------------------------------------------------- grid and levels
ODD = (3.75, 1019.3, 2.125, 349.6)  # ComputeImageBounds after undistortion: non-integer, non-zero


def solve(fn, target, x0):
    """The float x near x0 with fn(x) == target exactly (fn increasing), or None."""
    x = F32(x0)
    first = None
    for _ in range(100000):
        y = fn(x)
        if y == target:
            return x
        step = UP if y < target else DOWN
        if first is not None and step != first:
            return None  # stepped over the target
        first = step
        x = np.nextafter(x, step)
    return None


def beyond(fn, x, step):
    """The first float past x in direction step at which fn changes."""
    y = fn(x)
    while fn(x) == y:
        x = np.nextafter(x, step)
    return x


def on_axis_u(of, x, z):
    pc = T.gemm_pc(of.Rcw, (x, 0.0, z), of.tcw)
    return of.fx * pc[0] * (F32(1) / pc[2]) + of.cx


def on_axis_v(of, y, z):
    pc = T.gemm_pc(of.Rcw, (0.0, y, z), of.tcw)
    return of.fy * pc[1] * (F32(1) / pc[2]) + of.cy


def test_grid_at_half_cells_bounds_and_clipped_corners(s8):
    of = oframe(ODD)
    rng = np.random.default_rng(7)
    xs = [of.min_x + (F32(c) + F32(0.5)) / of.w_inv for c in (-1, 0, 5, 31, 62, 63)]
    ys = [of.min_y + (F32(c) + F32(0.5)) / of.h_inv for c in (-1, 0, 7, 23, 46, 47)]
    xs = [v for x in xs + [of.min_x, of.max_x] for v in (x, ulp(x, DOWN), ulp(x, UP))]
    ys = [v for y in ys + [of.min_y, of.max_y] for v in (y, ulp(y, DOWN), ulp(y, UP))]
    xy = [(x, y) for x in xs for y in ys]
    xy += list(np.c_[rng.uniform(0, 1024, 600), rng.uniform(0, 352, 600)])
    k = keys(xy, 0)
    k["octave"] = rng.integers(0, 8, len(k))
    # the half-cell keys round away from zero and the keys on or past the bounds are placed as PosInGrid places them
    grid = T.assign_features_to_grid(k, of)
    assert grid[0][0] and any(grid[63]) and any(T.pos_in_grid(x, ys[3], of) is None for x in xs)
    q = [(float(x), float(y), float(r), *lv) for x in (of.min_x, of.max_x, 500.3, ulp(of.min_x, DOWN), -30.0, 1060.0)
         for y in (of.min_y, of.max_y, 171.9, ulp(of.max_y, UP)) for r in (0.5, 7.9, 40.0) for lv in ((-1, -1), (0, 0), (2, -1))]
    q += [(float(x), float(y), float(rng.uniform(0.5, 50)), -1, -1) for x, y in xy[:200]]
    got = features_in_area(s8.el, k, ODD, q)
    total = 0
    for a, g in zip(q, got):
        want = T.get_features_in_area(grid, k, of, F32(a[0]), F32(a[1]), F32(a[2]), a[3], a[4])
        assert list(g) == want, a
        total += len(want)
    assert total > 1000
    # points projecting exactly onto each bound and one ulp outside, at every corner; windows clipped there
    for z in (4.0, 8.0, 2.0, 16.0, 1.0, 32.0):
        fu, fv = (lambda x: on_axis_u(of, x, z)), (lambda y: on_axis_v(of, y, z))
        us = {b: solve(fu, b, (b - CX) * z / FX) for b in (of.min_x, of.max_x)}
        vs = {b: solve(fv, b, (b - CY) * z / FX) for b in (of.min_y, of.max_y)}
        if None not in us.values() and None not in vs.values():
            break
    assert None not in us.values() and None not in vs.values()
    pts, inside = [], []
    for bu, x in us.items():
        for bv, y in vs.items():
            for dx, dy in ((0, 0), (1, 0), (0, 1)):
                xx = x if not dx else beyond(fu, x, DOWN if bu == of.min_x else UP)
                yy = y if not dy else beyond(fv, y, DOWN if bv == of.min_y else UP)
                assert (fu(xx) == bu) == (not dx) and (fv(yy) == bv) == (not dy)
                pts.append(point((xx, yy, z), desc_with([len(pts)]), observed=len(pts) % 2, angle=float(rng.uniform(0, 360))))
                inside.append(not (dx or dy))
    corner = keys([(x, y) for x in (of.min_x + 1, of.max_x - 1, of.min_x, of.max_x) for y in (of.min_y + 1, of.max_y - 1, of.min_y, of.max_y)])
    cd = [desc_with([i % len(pts)]) for i in range(len(corner))]
    for th in (1.0, 5.0):
        view, m, n = s8.local(Scene(corner, cd, pts, th=th, bounds=ODD))
        assert list(view) == inside
    assert n > 0
    for th in (1.0, 10.0):
        m, n = s8.last(Scene(corner, cd, pts, th=th, bounds=ODD))
    assert n > 0
    # a mixed scene on the odd bounds
    pts = [point_at(of, u, v, float(rng.uniform(3, 30)), flip(desc_with([]), rng.choice(256, 3, replace=False)),
                    observed=int(rng.integers(2)), octave=int(rng.integers(8)), angle=float(rng.uniform(0, 360)))
           for u, v in xy[:150]]
    km = k[:1000]  # within the extractor's capacity
    d = [flip(desc_with([]), rng.choice(256, 4, replace=False)) for _ in range(len(km))]
    assert s8.local(Scene(km, d, pts, th=3, bounds=ODD))[2] > 0
    assert s8.last(Scene(km, d, pts, th=7, bounds=ODD))[1] > 10


def level_scene(s, rng):
    """Per case one point, with the keys of every octave around it whose distance grows with the octave: the match shows the
    predicted level's window.  max_distance = dist * scale^e and one ulp either side, for e from -1 to nlevels + 1 (clamped
    below 0 and at nlevels - 1), 0 and +inf."""
    f = oframe()
    nl = len(s.scale)
    sf = s.scale[1]
    factors = [F32(1) / sf] + [s.scale[e] for e in range(nl)] + [s.scale[-1] * sf, s.scale[-1] * sf * sf]
    xy, kd, ko, pts = [], [], [], []
    for c, fac in enumerate(factors):
        for delta in (DOWN, None, UP):
            i = len(pts)
            u, v = 60 + 90 * (i % 11), 40 + 90 * (i // 11)
            p = point_at(f, u, v, float(rng.uniform(4, 20)), desc_with([]), observed=int(rng.integers(2)))
            md = T.norm3(p["pos"] - f.Ow) * fac
            p["max_distance"] = md if delta is None else ulp(md, delta)
            p["min_distance"] = 0
            pts.append(p)
            for o in range(nl):
                xy.append((u + 1.5 * np.cos(o), v + 1.5 * np.sin(o)))
                kd.append(desc_with(range(1 + o)))
                ko.append(o)
    for md in (0.0, np.inf):
        p = point_at(f, 500, 300, 10, desc_with([]))
        p["max_distance"], p["min_distance"] = md, 0
        pts.append(p)
    k = keys(xy)
    k["octave"] = ko
    return Scene(k, kd, pts), f


def test_predict_scale_at_exact_powers_and_clamps(s8, s4):
    rng = np.random.default_rng(11)
    for s in (s8, s4):
        sc, f = level_scene(s, rng)
        nl = len(s.scale)
        levels = [None if r is None else r[3] for r in (T.is_in_frustum(p, f, T.logf(s.scale[1]), nl) for p in sc.pts)]
        assert levels[-2] is None and levels[-1] == nl - 1  # max_distance 0: out of view; +inf: clamped
        assert {0, nl - 1} <= set(levels) and levels.count(nl - 1) > 3
        view, m, n = s.local(sc)
        assert n > len(sc.pts) // 2
        sc.th = F32(2.0)
        s.local(sc)


def test_last_frame_windows_at_the_end_octaves(s8, s4):
    f = oframe()
    for s in (s8, s4):
        nl = len(s.scale)
        xy, kd, ko = [], [], []
        for c, u in enumerate((300, 700)):
            for o in range(nl):
                xy.append((u + 1.5 * np.cos(o), 200 + 1.5 * np.sin(o)))
                kd.append(desc_with(range(1 + (o if c == 0 else nl - 1 - o))))
                ko.append(o)
        k = keys(xy)
        k["octave"] = ko
        for o in (0, nl - 1):
            outcomes = set()
            for direction, tlw in DIRECTIONS.items():
                pts = [point_at(f, u, 200, 10, desc_with([]), octave=o) for u in (300, 700)]
                m, n = s.last(Scene(k, kd, pts, th=3, tlw=tlw))
                outcomes.add(tuple(m))
            assert len(outcomes) > 1, o


# ---------------------------------------------------------------------------------------------------------- limits
def random_keys(rng, n, nlevels, region=(0, 1024, 0, 352)):
    k = keys(np.c_[rng.uniform(region[0], region[1], n), rng.uniform(region[2], region[3], n)])
    k["octave"] = rng.integers(0, nlevels, n)
    k["angle"] = rng.uniform(0, 360, n)
    return k


def points_from_keys(rng, k, d, idx, f, scale, flips=(0, 6)):
    """Points near keys idx with perturbed descriptors, predicted at the key's octave."""
    pts = []
    for j in idx:
        z = float(rng.uniform(3, 40))
        q = flip(d[j], rng.choice(256, rng.integers(*flips), replace=False))
        o = int(k["octave"][j])
        p = point_at(f, float(k["x"][j]) + rng.uniform(-1, 1), float(k["y"][j]) + rng.uniform(-1, 1), z, q, observed=int(rng.random() < 0.7),
                     octave=o, angle=float(np.clip(k["angle"][j] + rng.uniform(-40, 40), 0, 360)))
        p["max_distance"] *= scale[o] * F32(rng.uniform(0.97, 1.0))
        pts.append(p)
    return pts


def test_host_form_key_limit(s8):
    """40,960 keys fill the ordered pass's 200 KB of shared memory exactly; one more is refused."""
    rng = np.random.default_rng(5)
    f = oframe()
    n = 40960
    k = random_keys(rng, n, 8)
    d = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    ur = np.where(rng.random(n) < 0.5, k["x"] - rng.uniform(0, 60, n), -1).astype(F32)
    pts = np.array(points_from_keys(rng, k, d, rng.choice(n, 300, replace=False), f, s8.scale), MP)
    sc = Scene(k, d, pts, ur=ur, th=1)
    frame, of = sc.frames()
    ov, om, on = T.search_local_points(k, d, ur, pts, of, s8.scale, 1, 0.8)
    hv, hm, hn = search_local_points(s8.el, k, d, ur, pts, frame, 1)
    assert np.array_equal(hv, ov) and np.array_equal(hm, om) and hn == on > 100
    om, on = T.search_last_frame(k, d, ur, pts, of, np.eye(3), np.zeros(3), s8.scale, 7)
    hm, hn = search_last_frame(s8.el, k, d, ur, pts, frame, np.eye(3), np.zeros(3), 7)
    assert np.array_equal(hm, om) and hn == on > 100
    k1, d1, u1 = np.concatenate([k, k[:1]]), np.concatenate([d, d[:1]]), np.concatenate([ur, ur[:1]])
    for call in (lambda: search_local_points(s8.el, k1, d1, u1, pts, frame, 1),
                 lambda: search_last_frame(s8.el, k1, d1, u1, pts, frame, np.eye(3), np.zeros(3), 7)):
        with pytest.raises(L.SivoError) as e:
            call()
        assert e.value.code == L.EINVAL


def test_device_count_equal_to_the_capacity(s8):
    rng = np.random.default_rng(6)
    f = oframe()
    n = s8.cap
    k = random_keys(rng, n, 8, (300, 700, 50, 300))
    d = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    pts = points_from_keys(rng, k, d, rng.choice(n, 400, replace=False), f, s8.scale)
    _, m, nm = s8.local(Scene(k, d, pts, th=2))
    assert nm > 100
    m, nm = s8.last(Scene(k, d, pts, th=7))
    assert nm > 100


def test_fifty_thousand_points_on_a_handful_of_keys(s8):
    """Device form = host form on all of them; the oracle on all in_view values and on the first 3,000 points' search."""
    rng = np.random.default_rng(8)
    f = oframe()
    k = random_keys(rng, 6, 8, (400, 600, 100, 250))
    d = rng.integers(0, 256, (6, 32), dtype=np.uint8)
    pts = points_from_keys(rng, k, d, rng.integers(0, 6, 50000), f, s8.scale, (0, 40))
    pts = np.array(pts, MP)
    pts["pos"][::3, 2] *= -1  # a third behind the camera
    sc = Scene(k, d, pts, th=3)
    frame, of = sc.frames()
    hv, hm, hn = search_local_points(s8.el, k, d, sc.ur, pts, frame, 3)
    dv, dm, dn = s8.device(sc, False)
    assert np.array_equal(dv, hv) and np.array_equal(dm, hm) and dn == hn
    lg = T.logf(s8.scale[1])
    sample = rng.choice(len(pts), 3000, replace=False)
    assert [T.is_in_frustum(pts[i], of, lg, 8) is not None for i in sample] == list(hv[sample])
    assert 0.4 < hv.mean() < 0.8
    s8.local(Scene(k, d, pts[:3000], th=3))
    hm, hn = search_last_frame(s8.el, k, d, sc.ur, pts, frame, np.eye(3), np.zeros(3), 7)
    _, dm, dn = s8.device(Scene(k, d, pts, th=7), True)
    assert np.array_equal(dm, hm) and dn == hn and hn > 0
    s8.last(Scene(k, d, pts[:3000], th=7))


# ---------------------------------------------------------------------------------------------------------- the angle rule
def test_angle_rule_on_both_forms(s8):
    """Angles must be finite and in [0, 360]: the host forms refuse others with SIVO_ERANGE; the device forms put such a key
    in no cell and do not search such a last-frame point, as the oracle does."""
    f = oframe()
    bad = [np.nan, np.inf, -np.inf, -400.0, 720.0, ulp(360, UP), -F32(1e-45)]
    good = [-0.0, 0.0, 360.0, 359.99997, 1e-45]
    angles = bad + good + bad
    n = len(angles)
    k = keys([(100 + 20 * i, 100) for i in range(n)], 0)
    d = [desc_with([i]) for i in range(n)]
    pts = [point_at(f, 100 + 20 * i, 100, 10, desc_with([i]), angle=30.0) for i in range(n)]
    frame, _ = Scene(k, d, pts).frames()
    for a in bad:
        kb = k.copy()
        kb["angle"] = 0.0
        kb["angle"][3] = a
        for call in (lambda: search_local_points(s8.el, kb, d, np.full(n, -1, F32), np.array(pts, MP), frame, 1),
                     lambda: search_last_frame(s8.el, kb, d, np.full(n, -1, F32), np.array(pts, MP), frame,
                                               np.eye(3), np.zeros(3), 7)):
            with pytest.raises(L.SivoError) as e:
                call()
            assert e.value.code == L.ERANGE, a
        pb = np.array(pts, MP)
        pb["angle"][3] = a
        with pytest.raises(L.SivoError) as e:
            search_last_frame(s8.el, k, d, np.full(n, -1, F32), pb, frame, np.eye(3), np.zeros(3), 7)
        assert e.value.code == L.ERANGE, a
        s8.local(Scene(k, d, pb))  # the local search does not read point angles
    # device forms: keys with bad angles are no candidates; last-frame points with bad angles are not searched
    k["angle"] = angles
    for last, sc in ((False, Scene(k, d, pts)), (True, Scene(k, d, pts, th=7))):
        _, of = sc.frames()
        if last:
            om, on = T.search_last_frame(sc.k, sc.d, sc.ur, sc.pts, of, sc.Rlw, sc.tlw, s8.scale, sc.th)
        else:
            _, om, on = T.search_local_points(sc.k, sc.d, sc.ur, sc.pts, of, s8.scale, sc.th, sc.nnratio)
        _, dm, dn = s8.device(sc, last)
        assert np.array_equal(dm, om) and dn == on == len(good)
    k["angle"] = 0.0
    for i, p in enumerate(pts):
        p["angle"] = angles[i]
    sc = Scene(k, d, pts, th=7)
    om, on = T.search_last_frame(sc.k, sc.d, sc.ur, sc.pts, sc.frames()[1], sc.Rlw, sc.tlw, s8.scale, sc.th)
    _, dm, dn = s8.device(sc, True)
    assert np.array_equal(dm, om) and dn == on == len(good)


# ---------------------------------------------------------------------------------------------------------- seeded fuzz
def fuzz_scene(seed, nlevels):
    """50-400 keys crowded into a 200 x 100 px region, 2-8 distinct descriptors with few-bit perturbations, random octaves,
    angles, mvRight, observed flags, a small random pose, th, and a last-frame pose moving forward, backward or neither."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(50, 401))
    x0, y0 = rng.uniform(0, 824), rng.uniform(0, 252)
    xy = np.c_[x0 + rng.uniform(0, 200, n), y0 + rng.uniform(0, 100, n)]
    snap = rng.random(n) < 0.3
    xy[snap] = np.round(xy[snap])  # shared positions and exact offsets
    k = keys(xy)
    k["octave"] = rng.integers(0, nlevels, n)
    k["angle"] = np.where(rng.random(n) < 0.1, rng.choice([0.0, 360.0], n), rng.uniform(0, 360, n))
    base = rng.integers(0, 256, (int(rng.integers(2, 9)), 32), dtype=np.uint8)
    d = np.stack([flip(base[rng.integers(len(base))], rng.choice(256, rng.integers(0, 4), replace=False)) for _ in range(n)])
    ur = np.where(rng.random(n) < 0.5, xy[:, 0] - rng.uniform(0, 80, n), rng.choice([-1.0, 0.0], n)).astype(F32)
    R = rotation(*rng.uniform(-0.01, 0.01, 3))
    t = rng.uniform(-0.05, 0.05, 3)
    f = oframe(BOUNDS, R, t)
    pts = []
    for _ in range(int(rng.integers(30, 180))):
        u, v = x0 + rng.uniform(-10, 210), y0 + rng.uniform(-10, 110)
        z = rng.uniform(2, 40)
        pc = np.array([(u - CX) * z / FX, (v - CY) * z / FX, z])
        pos = f.Rcw.astype(np.float64).T @ (pc - f.tcw)
        nflip = int(rng.choice([0, 1, 3, 8, 95, 100, 101, 105]))
        q = flip(base[rng.integers(len(base))], rng.choice(256, min(nflip, 256), replace=False))
        normal = pos - f.Ow + rng.normal(0, 0.3 * z, 3)
        p = point(pos, q, observed=int(rng.random() < 0.6), octave=int(rng.integers(nlevels)), angle=float(rng.uniform(0, 360)),
                  normal=normal / np.linalg.norm(normal))
        p["max_distance"] *= F32(rng.uniform(0.9, 4.0))
        p["min_distance"] = p["max_distance"] / F32(rng.uniform(1.0, 30.0))
        pts.append(p)
    blocked = (rng.random(n) < 0.1).astype(np.uint8) if rng.random() < 0.5 else None
    tlw = np.asarray(list(DIRECTIONS.values())[rng.integers(3)]) - T.gemm_neg_t(f.Rcw, f.tcw)  # tlc = Rlw twc + tlw, Rlw = I
    return (Scene(k, d, pts, ur=ur, th=float(rng.choice([1, 1, 2, 3.5, 5, 10])), blocked=blocked, R=R, t=t),
            Scene(k, d, pts, ur=ur, th=float(rng.choice([3, 7, 10, 15, 25])), R=R, t=t, tlw=tlw))


def rotation(a, b, c):
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1]])
    return (Rz @ Ry @ Rx).astype(np.float32)


def test_seeded_differential_fuzz(s8, s4):
    """200 scenes, one in five on the 4-level, 1.5x extractor.  The oracle's share of the run is about 15 s on one CPU core."""
    matched = [0, 0]
    for seed in range(200):
        s = s4 if seed % 5 == 4 else s8
        loc, last = fuzz_scene(seed, len(s.scale))
        matched[0] += s.local(loc)[2]
        matched[1] += s.last(last)[1]
    assert min(matched) > 1000, matched
