"""CPU: the pieces of the stereo oracle (oracle/orb_oracle.py compute_stereo_matches) pinned one by one -- the rounding of the
scaled coordinates against libm's roundf, the window SAD against cv2.norm, the median cut against a literal sort and walk, the
parabola's delta bound -- and the constructed scenes of oracle/stereo_scene.py held to the stage every key names, so that the
GPU suite (test_gpu_stereo_edges.py) is known to test the boundaries it claims to."""
import ctypes
import ctypes.util

import cv2
import numpy as np
import pytest

from oracle import orb_oracle as O
from oracle import stereo_scene as S

f32 = np.float32


def libm_roundf():
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.roundf.restype = ctypes.c_float
    libm.roundf.argtypes = [ctypes.c_float]
    return libm.roundf


def test_round_half_away_equals_libm_roundf():
    roundf = libm_roundf()
    vals = []
    for h in np.arange(-4095.5, 4096.0, 1.0, dtype=np.float64):  # every half-integer in (-4096, 4096)
        v = f32(h)
        lo = hi = v
        vals.append(v)
        for _ in range(8):
            lo, hi = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
            vals += [lo, hi]
    rng = np.random.default_rng(0)
    vals += list(rng.uniform(-4096, 4096, 50_000).astype(np.float32))
    vals += [f32(0.49999997), f32(-0.49999997), f32(0.5), f32(-0.5), f32(-0.0), f32(2.0 ** 31), f32(3e38)]
    for v in vals:
        assert O.round_half_away(v) == f32(roundf(float(v))), v
    # floor(v + 0.5f) in float gives 1 here; roundf gives 0
    assert O.round_half_away(f32(0.49999997)) == 0


def test_window_sad_equals_cv2_norm_l1():
    rng = np.random.default_rng(1)
    for _ in range(300):
        a = rng.integers(0, 256, (40, 60)).astype(np.uint8)
        b = rng.integers(0, 256, (40, 60)).astype(np.uint8) if rng.random() < 0.5 else np.clip(a + rng.integers(-3, 4, a.shape), 0, 255).astype(np.uint8)
        cy, cxl, cxr = int(rng.integers(5, 35)), int(rng.integers(5, 55)), int(rng.integers(5, 55))
        il = a[cy - 5:cy + 6, cxl - 5:cxl + 6].astype(np.float32)
        ir = b[cy - 5:cy + 6, cxr - 5:cxr + 6].astype(np.float32)
        il = il - il[5, 5] * np.ones_like(il)
        ir = ir - ir[5, 5] * np.ones_like(ir)
        assert O.window_sad(a, b, cy, cxl, cxr) == int(np.float32(cv2.norm(il, ir, cv2.NORM_L1)))


def literal_cut(sad):
    """Frame.cc:617-628 as written: sort (dist, index) pairs, median at size / 2, walk from the back while dist >= th."""
    pairs = sorted((int(s), i) for i, s in enumerate(sad) if s >= 0)
    cut = np.zeros(len(sad), bool)
    if not pairs:
        return cut
    median = f32(pairs[len(pairs) // 2][0])
    th = f32(1.5) * f32(1.4) * median
    for d, i in reversed(pairs):
        if f32(d) < th:
            break
        cut[i] = True
    return cut


def test_median_cut_equals_the_literal_sort_and_walk():
    rng = np.random.default_rng(2)
    cases = [[], [-1, -1], [0], [0, 0, 0], [10, 20, 21, 10, 10], [61710, 0, 61710], [255, 256, 257], [511, 512, 512, 511, 1]]
    for n in (1, 2, 3, 4, 5, 17, 256, 1023, 1025, 3000):
        for hi in (3, 300, 61711):
            s = rng.integers(-1, hi, n)
            cases.append(list(s))
    for s in cases:
        s = np.array(s, np.int64)
        assert np.array_equal(O.median_cut(s), literal_cut(s)), s
    # the threshold of a median of 10 is exactly 21.0f: SAD 21 is cut, 20 kept
    assert f32(f32(1.5) * f32(1.4)) == f32(2.0999999) and f32(f32(2.0999999) * f32(10)) == f32(21.0)
    assert list(O.median_cut([10, 10, 10, 20, 21])) == [False, False, False, False, True]


def test_parabola_delta_lies_in_the_half_open_interval():
    """binc is the first strict minimum, so d1 > d2 <= d3 and delta = (d1 - d3) / (2 (d1 + d3 - 2 d2)) is in (-1/2, 1/2]: the
    reference's |delta| > 1 gate cannot fire.  delta = 1/2 exactly when d3 == d2."""
    rng = np.random.default_rng(3)
    hit_half = 0
    for _ in range(20000):
        d = rng.integers(0, int(rng.choice([4, 50, 61711])), 11)
        binc = int(np.argmin(d)) - 5
        if binc in (-5, 5):
            continue
        d1, d2, d3 = (f32(d[binc + 5 + j]) for j in (-1, 0, 1))
        delta = f32(f32(d1 - d3) / f32(f32(2) * f32(f32(d1 + d3) - f32(f32(2) * d2))))
        assert f32(-0.5) < delta <= f32(0.5)
        hit_half += bool(delta == f32(0.5))
        assert (delta == f32(0.5)) == (d3 == d2)
    assert hit_half > 100


@pytest.fixture(scope="module")
def traced():
    out = []
    for sc in S.constructed_scenes():
        trace = []
        u, z = sc.oracle(trace)
        out.append((sc, trace, u, z))
    return out


def test_constructed_keys_end_where_they_say(traced):
    for sc, trace, u, z in traced:
        for il, want in sc.want.items():
            assert trace[il]["stage"] in O.STAGE_GROUPS.get(want, (want,)), (sc.name, il, want, trace[il])
        for il, t in enumerate(trace):
            assert (u[il] >= 0) == (t["stage"] == "matched") and (z[il] >= 0) == (t["stage"] == "matched"), (sc.name, il)


def test_constructed_scenes_reach_every_stage_and_both_sides_of_every_gate(traced):
    """The coverage assertion: every stage but the unreachable delta gate, and each named boundary on both sides."""
    stages = {t["stage"] for _, trace, _, _ in traced for t in trace}
    assert stages == set(O.STAGES) - {"delta"}
    by = {sc.name: (sc, trace) for sc, trace, _, _ in traced}
    sc, tr = by["hamming"]
    best = [t.get("best") for t in tr]
    assert 74 in best and 75 in best
    sc, tr = by["sad"]
    bincs = {t["binc"] for t in tr if t["binc"] is not None}
    assert {-5, -4, 4, 5} <= bincs
    assert any(t["delta"] == f32(0.5) for t in tr)
    assert any(t["sad"] is not None and len(set(t["sad"])) == 1 for t in tr)  # a flat window
    sc, tr = by["disparity"]
    disps = {float(t["disp"]) for t in tr if t["disp"] is not None}
    assert {0.0, 40.0, float(S.ulp_down(40)), -float(np.spacing(f32(55)))} <= disps  # 0, maxD, maxD - ulp, -ulp
    sc, tr = by["median_th21"]
    assert [t["stage"] for t in tr][-2:] == ["matched", "cut"]
    for name in ("window0", "window3", "window7"):
        stages = {t["stage"] for t in by[name][1]}
        assert {"slide", "left_window"} <= stages and stages & set(O.STAGE_GROUPS["past_slide"]), name


def test_semantic_keys_rule_for_non_finite_and_outside_keys():
    rng = np.random.default_rng(4)
    H, W = 20, 30
    classes = rng.integers(0, 15, (H, W)).astype(np.uint8)
    conf, ent = rng.random((H, W)), rng.random((H, W))
    nan, inf = np.nan, np.inf
    xy = np.array([[0.5, 0.5], [-0.5, 3], [nan, 3], [3, nan], [inf, 3], [3, -inf], [-1, 3], [W, 3], [3, H], [W - 0.01, H - 0.01],
                   [3e9, 3], [-3e9, 3]], np.float32)
    cls, c, e, keep = O.select_semantic_keys(xy, classes, conf, ent, 14)
    inside = [0, 1, 9]
    assert (cls[[i for i in range(len(xy)) if i not in inside]] == 255).all()
    assert (c[cls == 255] == 0).all() and (e[cls == 255] == 0).all()
    assert cls[1] == classes[3, 0] and cls[9] == classes[H - 1, W - 1]
    assert list(keep) == inside
