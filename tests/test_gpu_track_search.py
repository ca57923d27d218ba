"""-m gpu: the projection searches (sivo_search_local_points / _last_frame, host and device forms) and the device grid
(sivo_dbg_features_in_area) on the Frame tail's outputs -- SegNet -> extractors -> semantic keys -> stereo -- against
oracle/track_oracle.py bit for bit, and the device forms against the host forms."""
import ctypes as C

import numpy as np
import pytest
import torch

from frame_support import BOUNDS, CX, CY, FX, MB, MBF, H, W, ext, ptr, seg, synth, tails, upload  # noqa: F401
from oracle import track_oracle as T
from oracle.mapping_scene import rotation
from sivo_b200 import _lib as L
from sivo_b200 import (MAP_POINT_DTYPE, make_frame, map_points, search_last_frame, search_last_frame_device, search_local_points,
                       search_local_points_device, stereo_match)
from sivo_b200.frame import DeviceFrame
from sivo_b200.track import features_in_area

pytestmark = pytest.mark.gpu

POSES = {"identity": (np.eye(3), np.zeros(3)), "moved": (rotation(0.002, 0.01, -0.003), np.array([0.02, -0.01, 0.3])),
         "forward": (np.eye(3), np.array([0.0, 0.0, -1.0])), "backward": (np.eye(3), np.array([0.0, 0.0, 1.0]))}


def frames(pose):
    R, t = POSES[pose]
    return make_frame(FX, FX, CX, CY, MBF, BOUNDS, R, t), T.Frame(FX, FX, CX, CY, MBF, BOUNDS, R, t)


class Keys:
    """The semantic keys of one tail as host arrays: mvKeysSemantic, mDescriptorsSemantic, mvRight, mvDepth."""

    def __init__(self, t):
        self.t = t
        self.kps = t.kps
        self.desc = t.f.left.host()[1][t.keep]
        self.ur = t.ur
        self.depth = t.depth


def build_points(k: Keys, scale, seed):
    """Points from the keys with depth (unprojected at the identity pose), plus duplicates with 1-3 flipped descriptor bits,
    copies shifted by a sub-pixel to a few pixels and random distractors, in a shuffled order; about one in ten unobserved."""
    rng = np.random.default_rng(seed)
    f, idx = T.map_points_from_keys(k.kps, k.depth, np.eye(3), np.zeros(3), FX, FX, CX, CY, scale)
    base = map_points(k.desc[idx], f["pos"], f["normal"], f["min_distance"], f["max_distance"], 1, k.kps["octave"][idx], k.kps["angle"][idx])
    dup = base[rng.choice(len(base), len(base) // 2)].copy()
    for p in dup:
        for b in rng.choice(256, rng.integers(1, 4), replace=False):
            p["desc"][b // 8] ^= np.uint8(1 << (b % 8))
    shifted = base[rng.choice(len(base), len(base) // 3)].copy()
    shifted["pos"][:, 0] += (rng.uniform(-3, 3, len(shifted)) * shifted["pos"][:, 2] / FX).astype(np.float32)
    rnd = np.zeros(len(base) // 4, MAP_POINT_DTYPE)
    z = rng.uniform(2, 60, len(rnd))
    rnd["pos"] = np.c_[(rng.uniform(0, W, len(rnd)) - CX) * z / FX, (rng.uniform(0, H, len(rnd)) - CY) * z / FX, z]
    rnd["normal"] = rnd["pos"] / np.linalg.norm(rnd["pos"], axis=1, keepdims=True)
    d = np.linalg.norm(rnd["pos"], axis=1)
    rnd["max_distance"], rnd["min_distance"] = d * 1.5, d / 3
    rnd["desc"] = rng.integers(0, 256, (len(rnd), 32))
    rnd["octave"] = rng.integers(0, len(scale), len(rnd))
    rnd["angle"] = rng.uniform(0, 360, len(rnd))
    pts = np.concatenate([base, dup, shifted, rnd])
    pts = pts[rng.permutation(len(pts))]
    pts["observed"] = (rng.uniform(size=len(pts)) > 0.1).astype(np.int32)
    return pts


@pytest.fixture(scope="module")
def keysets(tails):
    return {f: Keys(t) for f, t in tails.items()}


class SearchOut:
    def __init__(self, cap, n_points):
        self.view = torch.full((max(n_points, 1),), 7, dtype=torch.uint8, device="cuda")
        self.match = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
        self.n = torch.full((1,), -7, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()

    def host(self, n_keep, n_points):
        return (self.view.cpu().numpy()[:n_points].copy(), self.match.cpu().numpy()[:max(n_keep, 0)].copy(), int(self.n.cpu()[0]))


def run_local_device(el, t, pts_dev, n_points, frame, th, stream, n=None, keep="sem", null=(), blocked=0):
    f = t.f
    out = SearchOut(f.left.cap, n_points)
    p = {k: (0 if k in null else ptr(getattr(out, k))) for k in ("view", "match", "n")}
    search_local_points_device(el, f.kps, f.desc, f.keep if keep == "sem" else 0, f.n_keep if n is None else ptr(n), f.u_right, blocked,
                               ptr(pts_dev), n_points, frame, th, 0.8, p["view"], p["match"], p["n"], stream.cuda_stream)
    stream.synchronize()
    return out


def run_last_device(el, t, pts_dev, n_points, frame, th, stream, null=()):
    f = t.f
    out = SearchOut(f.left.cap, n_points)
    p = {k: (0 if k in null else ptr(getattr(out, k))) for k in ("match", "n")}
    search_last_frame_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, ptr(pts_dev), n_points, frame, np.eye(3), np.zeros(3), th,
                             p["match"], p["n"], stream.cuda_stream)
    stream.synchronize()
    return out


# ---------------------------------------------------------------------------------------------------------- the grid
def test_features_in_area_equals_the_oracle(keysets, ext):
    el = ext[0]
    rng = np.random.default_rng(3)
    of = T.Frame(FX, FX, CX, CY, MBF, BOUNDS, np.eye(3), np.zeros(3))
    for f, k in keysets.items():
        grid = T.assign_features_to_grid(k.kps, of)
        q = [(rng.uniform(-20, W + 20), rng.uniform(-20, H + 20), rng.uniform(0.5, 60), *[(-1, -1), (0, -1), (-1, 0), (0, 0), (1, 2),
             (2, -1), (-1, 3)][rng.integers(7)]) for _ in range(400)]
        q += [(float(k.kps["x"][j]), float(k.kps["y"][j]), 4.0, -1, -1) for j in range(0, len(k.kps), 7)]
        got = features_in_area(el, k.kps, BOUNDS, q)
        total = 0
        for a, g in zip(q, got):
            want = T.get_features_in_area(grid, k.kps, of, np.float32(a[0]), np.float32(a[1]), np.float32(a[2]), a[3], a[4])
            assert list(g) == want, (f, a)
            total += len(want)
        assert total > 1000


# ---------------------------------------------------------------------------------------------------------- local-map search
@pytest.mark.parametrize("th", [1, 5])
@pytest.mark.parametrize("pose", ["identity", "moved"])
def test_local_search_is_bit_identical_to_the_oracle(keysets, tails, ext, pose, th):
    el = ext[0]
    frame, of = frames(pose)
    stream = torch.cuda.Stream()
    changed = 0
    for f, k in keysets.items():
        pts = build_points(k, el.GetScaleFactors(), 10 + th)
        view, match, n = search_local_points(el, k.kps, k.desc, k.ur, pts, frame, th)
        per, free = [], []
        ov, om, on = T.search_local_points(k.kps, k.desc, k.ur, pts, of, el.GetScaleFactors(), th, 0.8, per_point=per)
        assert np.array_equal(view, ov) and np.array_equal(match, om) and n == on, f
        assert n > 10 and view.sum() > n
        # the points searched alone (no claims): some final matches differ, so the ordered pass searched them again
        lone = pts.copy()
        lone["observed"] = 0
        T.search_local_points(k.kps, k.desc, k.ur, lone, of, el.GetScaleFactors(), th, 0.8, per_point=free)
        changed += sum(a != b and a >= 0 and b >= 0 for a, b in zip(per, free))
        # the device form on the tail's buffers equals the host form
        out = run_local_device(el, tails[f], upload(pts), len(pts), frame, th, stream)
        dv, dm, dn = out.host(k.t.n_keep, len(pts))
        assert np.array_equal(dv.astype(bool), view) and np.array_equal(dm, match) and dn == n, f
        assert (out.match.cpu().numpy()[k.t.n_keep:] == -7).all()
    assert changed > 0


def test_local_search_with_keys_blocked_on_entry(keysets, tails, ext):
    el = ext[0]
    frame, of = frames("moved")
    k = keysets[0]
    pts = build_points(k, el.GetScaleFactors(), 5)
    blocked = (np.arange(len(k.kps)) % 3 == 0).astype(np.uint8)
    view, match, n = search_local_points(el, k.kps, k.desc, k.ur, pts, frame, 1, blocked=blocked)
    ov, om, on = T.search_local_points(k.kps, k.desc, k.ur, pts, of, el.GetScaleFactors(), 1, 0.8, blocked)
    assert np.array_equal(view, ov) and np.array_equal(match, om) and n == on > 0 and (match[blocked == 1] == -1).all()
    stream = torch.cuda.Stream()
    b = torch.zeros(k.t.f.left.cap, dtype=torch.uint8, device="cuda")
    b[:len(blocked)] = torch.from_numpy(blocked).cuda()
    torch.cuda.synchronize()
    out = run_local_device(el, tails[0], upload(pts), len(pts), frame, 1, stream, blocked=ptr(b))
    dv, dm, dn = out.host(k.t.n_keep, len(pts))
    assert np.array_equal(dm, match) and dn == n


# ---------------------------------------------------------------------------------------------------------- last-frame search
@pytest.mark.parametrize("th", [7, 14])
@pytest.mark.parametrize("pose", ["identity", "moved", "forward", "backward"])
def test_last_frame_search_is_bit_identical_to_the_oracle(keysets, tails, ext, pose, th):
    el = ext[0]
    frame, of = frames(pose)
    stream = torch.cuda.Stream()
    for f, k in keysets.items():
        pts = build_points(k, el.GetScaleFactors(), 20 + th)
        match, n = search_last_frame(el, k.kps, k.desc, k.ur, pts, frame, np.eye(3), np.zeros(3), th)
        om, on = T.search_last_frame(k.kps, k.desc, k.ur, pts, of, np.eye(3), np.zeros(3), el.GetScaleFactors(), th)
        assert np.array_equal(match, om) and n == on, (f, pose)
        if pose in ("identity", "moved"):
            assert n > 50
        out = run_last_device(el, tails[f], upload(pts), len(pts), frame, th, stream)
        _, dm, dn = out.host(k.t.n_keep, len(pts))
        assert np.array_equal(dm, match) and dn == n, f


# ---------------------------------------------------------------------------------------------------------- edge cases
def test_edge_cases_and_error_codes(keysets, tails, ext):
    el = ext[0]
    t = tails[1]
    k = keysets[1]
    frame, of = frames("moved")
    pts = build_points(k, el.GetScaleFactors(), 9)
    pd = upload(pts)
    stream = torch.cuda.Stream()
    full = run_local_device(el, t, pd, len(pts), frame, 1, stream).host(t.n_keep, len(pts))

    def i64(v):
        x = torch.tensor([v], dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        return x

    # a negative count writes only n_matches = -1; zero keys match nothing; zero points
    out = run_local_device(el, t, pd, len(pts), frame, 1, stream, n=i64(-1))
    assert int(out.n.cpu()[0]) == -1 and (out.match.cpu().numpy() == -7).all() and (out.view.cpu().numpy() == 7).all()
    v, m, n = run_local_device(el, t, pd, len(pts), frame, 1, stream, n=i64(0)).host(0, len(pts))
    assert n == 0 and np.array_equal(v, full[0])
    v, m, n = run_local_device(el, t, pd, 0, frame, 1, stream).host(t.n_keep, 0)
    assert n == 0 and (m == -1).all()
    assert search_local_points(el, k.kps[:0], k.desc[:0], k.ur[:0], pts, frame, 1)[2] == 0
    assert search_last_frame(el, k.kps, k.desc, k.ur, pts[:0], frame, np.eye(3), np.zeros(3), 7)[1] == 0
    # NULL optional outputs
    for null in (("view",), ("match",), ("n",)):
        got = run_local_device(el, t, pd, len(pts), frame, 1, stream, null=null).host(t.n_keep, len(pts))
        for name, a, b in zip(("view", "match", "n"), got, full):
            if name not in null:
                assert np.array_equal(a, b), null
    _, lm, ln = run_last_device(el, t, pd, len(pts), frame, 7, stream).host(t.n_keep, len(pts))
    out = run_last_device(el, t, pd, len(pts), frame, 7, stream, null=("match",))
    assert int(out.n.cpu()[0]) == ln and (out.match.cpu().numpy() == -7).all()
    # a count above the capacity is clamped (keep_idx NULL: key j of the extractor, every one of the capacity's records)
    cap = t.f.left.cap
    u = torch.full((cap,), -1.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    out = SearchOut(cap, len(pts))
    search_local_points_device(el, t.f.kps, t.f.desc, 0, ptr(i64(cap + 1000)), ptr(u), 0, ptr(pd), len(pts), frame, 1, 0.8,
                               ptr(out.view), ptr(out.match), ptr(out.n), stream.cuda_stream)
    stream.synchronize()
    kall = t.f.left.kps.cpu().numpy().view(k.kps.dtype)[:cap]
    dall = t.f.left.desc.cpu().numpy().reshape(-1, 32)[:cap]
    hv, hm, hn = search_local_points(el, kall, dall, np.full(cap, -1, np.float32), pts, frame, 1)
    dv, dm, dn = out.host(cap, len(pts))
    assert np.array_equal(dm, hm) and dn == hn > 0
    # error codes
    lib = L.lib()
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    match, nm = np.empty(len(k.kps), np.int32), C.c_int()
    args = lambda: [el._h, P(k.kps), P(k.desc), P(k.ur), None, len(k.kps), P(pts), len(pts), C.byref(frame), 1.0, 0.8, None, P(match), C.byref(nm)]
    assert lib.sivo_search_local_points(*args()) == L.OK
    for i, v in ((0, None), (1, None), (5, -1), (7, -1), (8, None), (9, 0.0), (9, -1.0)):
        a = args()
        a[i] = v
        assert lib.sivo_search_local_points(*a) == L.EINVAL, i
    bad = make_frame(FX, FX, CX, CY, MBF, (0.0, 0.0, 0.0, float(H)), np.eye(3), np.zeros(3))
    a = args()
    a[8] = C.byref(bad)
    assert lib.sivo_search_local_points(*a) == L.EINVAL
    R, tt = np.eye(3, dtype=np.float32).reshape(9), np.zeros(3, np.float32)
    largs = lambda p: [el._h, P(k.kps), P(k.desc), P(k.ur), len(k.kps), P(p), len(p), C.byref(frame), P(R), P(tt), 7.0, P(match), C.byref(nm)]
    assert lib.sivo_search_last_frame(*largs(pts)) == L.OK
    badp = pts.copy()
    badp["octave"][3] = 99
    assert lib.sivo_search_last_frame(*largs(badp)) == L.ERANGE
    a = largs(pts)
    a[8] = None
    assert lib.sivo_search_last_frame(*a) == L.EINVAL
    dargs = lambda: [el._h, t.f.kps, t.f.desc, t.f.keep, t.f.n_keep, t.f.u_right, None, ptr(pd), len(pts), C.byref(frame), 1.0, 0.8, None,
                     None, None, None]
    assert lib.sivo_search_local_points_device(*dargs()) == L.OK
    for i, v in ((0, None), (1, None), (2, None), (4, None), (5, None), (7, None), (8, -1), (9, None), (10, 0.0)):
        a = dargs()
        a[i] = v
        assert lib.sivo_search_local_points_device(*a) == L.EINVAL, i
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- asynchronous chain
def test_three_frames_in_flight_with_both_searches_equal_the_host_call_path(seg, ext):
    """SegNet -> two enqueue_device -> semantic keys -> stereo -> both searches for three frames on rotating buffers, the caller's
    wait before the next enqueue, one host synchronisation; each frame's results equal the host-call path's."""
    el, er = ext
    frames_in = [synth(30 + i) for i in range(3)]
    frame, _ = frames("moved")
    d_in = [[upload(x) for x in f] for f in frames_in]
    rng = np.random.default_rng(4)
    pts = np.zeros(3000, MAP_POINT_DTYPE)
    z = rng.uniform(3, 40, len(pts))
    pts["pos"] = np.c_[(rng.uniform(0, W, len(pts)) - CX) * z / FX, (rng.uniform(0, H, len(pts)) - CY) * z / FX, z]
    pts["normal"] = pts["pos"] / np.linalg.norm(pts["pos"], axis=1, keepdims=True)
    pts["max_distance"], pts["min_distance"] = z * 2, z / 4
    pts["desc"] = rng.integers(0, 256, (len(pts), 32))
    pts["octave"] = rng.integers(0, 8, len(pts))
    pts["observed"] = 1
    pd = upload(pts)
    bufs = [(DeviceFrame(el, er, H, W), SearchOut(el.capacity(), len(pts)), SearchOut(el.capacity(), len(pts))) for _ in frames_in]
    stream = torch.cuda.Stream()
    s = stream.cuda_stream

    def chain():
        for i, (f, loc, last) in enumerate(bufs):
            seg.set_frame(300 + i)
            f.extract(seg, *d_in[i], s)  # waits for the previous frame's stereo and searches
            f.tail(seg, MB, MBF, s)
            search_last_frame_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, ptr(pd), len(pts), frame, np.eye(3), np.zeros(3), 7,
                                     ptr(last.match), ptr(last.n), s)
            search_local_points_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, 0, ptr(pd), len(pts), frame, 1, 0.8, ptr(loc.view),
                                       ptr(loc.match), ptr(loc.n), s)

    chain()  # first use of the stream: the network's graph is captured here
    stream.synchronize()
    for _, loc, last in bufs:
        for o in (loc, last):
            o.match.fill_(-7)
            o.n.fill_(-7)
    torch.cuda.synchronize()
    chain()
    stream.synchronize()
    for i, (bgr, gl, gr) in enumerate(frames_in):
        seg.set_frame(300 + i)
        seg.segmentImage(bgr)
        kl, dl = el(gl, None)
        kr, dr = er(gr, None)
        _, _, _, keep = seg.semantic_keys(kl, 8)
        hu, _ = stereo_match(el, er, kl[keep], dl[keep], kr, dr, MB, MBF)
        hv, hm, hn = search_local_points(el, kl[keep], dl[keep], hu, pts, frame, 1)
        lm, ln = search_last_frame(el, kl[keep], dl[keep], hu, pts, frame, np.eye(3), np.zeros(3), 7)
        f, loc, last = bufs[i]
        n_keep = f.host()[0]
        v, m, n = loc.host(n_keep, len(pts))
        assert n_keep == len(keep) and np.array_equal(v.astype(bool), hv) and np.array_equal(m, hm) and n == hn
        _, m, n = last.host(n_keep, len(pts))
        assert np.array_equal(m, lm) and n == ln
        assert hv.sum() > 100
