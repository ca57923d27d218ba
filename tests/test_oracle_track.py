"""CPU: the projection-search oracle (oracle/track_oracle.py) against OpenCV's norm and gemm, a brute-force area filter, and
hand-built cases of the claim dependency, the ratio test, the rotation histogram and the frustum edges."""
import cv2
import numpy as np

from oracle import track_oracle as T
from oracle.track_scene import MP, SCALE, desc_with, keys, point_at

BOUNDS = (0.0, 1024.0, 0.0, 352.0)


def frame(R=np.eye(3), t=(0, 0, 0)):
    return T.Frame(700.0, 700.0, 512.0, 176.0, 380.0, BOUNDS, R, t)


def test_norm_and_pose_gemms_equal_cv2():
    rng = np.random.default_rng(0)
    for _ in range(10000):
        a = (rng.standard_normal(3) * rng.choice([1e-3, 1, 30, 1e3])).astype(np.float32)
        assert T.norm3(a) == np.float32(cv2.norm(a.reshape(3, 1)))
        R = (rng.standard_normal((3, 3)) * rng.choice([1e-2, 1, 10])).astype(np.float32)
        t = (rng.standard_normal((3, 1)) * rng.choice([1e-2, 1, 100])).astype(np.float32)
        assert T.gemm_neg_t(R, t).tobytes() == cv2.gemm(R, t, -1, None, 0, flags=cv2.GEMM_1_T).ravel().tobytes()
        P = (rng.standard_normal((3, 1)) * 50).astype(np.float32)
        assert T.gemm_pc(R, P, t).tobytes() == cv2.gemm(R, P, 1, t, 1).ravel().tobytes()


def test_grid_rounds_half_away_from_zero():
    f = frame()  # w_inv = 1 / 16, h_inv = 48 / 352
    assert f.w_inv == np.float32(1 / 16)
    for x, cell in ((8.0, 1), (24.0, 2), (40.0, 3), (7.99, 0), (1015.9, 63)):
        assert T.pos_in_grid(x, 0.0, f) == (cell, 0), x
    assert T.pos_in_grid(1016.0, 0.0, f) is None  # round(63.5) = 64 is outside
    assert T.pos_in_grid(-8.0, 0.0, f) is None  # round(-0.5) = -1
    assert T.pos_in_grid(-7.9, 0.0, f) == (0, 0)
    assert T.round_half_away(2.5) == 3 and T.round_half_away(-2.5) == -3 and T.round_half_away(np.float32(0.49999997)) == 0


def test_features_in_area_equals_a_brute_force_filter():
    rng = np.random.default_rng(1)
    f = frame()
    k = keys(np.c_[rng.uniform(-5, 1030, 3000), rng.uniform(-5, 360, 3000)], 0)
    k["octave"] = rng.integers(0, 8, len(k))
    k["x"][:50] = np.round(k["x"][:50] / 16) * 16 + 8  # exact .5 cell positions
    grid = T.assign_features_to_grid(k, f)
    cell = [T.pos_in_grid(k["x"][j], k["y"][j], f) for j in range(len(k))]
    for _ in range(300):
        x, y, r = np.float32(rng.uniform(-40, 1060)), np.float32(rng.uniform(-40, 390)), np.float32(rng.uniform(0.5, 80))
        lo, hi = [(-1, -1), (0, -1), (-1, 0), (0, 0), (2, 3), (3, -1)][rng.integers(6)]
        got = T.get_features_in_area(grid, k, f, x, y, r, lo, hi)
        cx0 = int(np.floor(((x - f.min_x) - r) * f.w_inv))
        cx1 = int(np.ceil(((x - f.min_x) + r) * f.w_inv))
        cy0 = int(np.floor(((y - f.min_y) - r) * f.h_inv))
        cy1 = int(np.ceil(((y - f.min_y) + r) * f.h_inv))
        check = lo > 0 or hi >= 0
        want = [j for j in range(len(k)) if cell[j] is not None and cx0 <= cell[j][0] <= cx1 and cy0 <= cell[j][1] <= cy1
                and not (check and (k["octave"][j] < lo or (hi >= 0 and k["octave"][j] > hi)))
                and abs(k["x"][j] - x) < r and abs(k["y"][j] - y) < r]
        want.sort(key=lambda j: (cell[j][0], cell[j][1], j))
        assert got == want


def local(points, k, d, ur=None, th=1.0, blocked=None, f=None):
    f = f or frame()
    ur = np.full(len(k), -1, np.float32) if ur is None else ur
    return T.search_local_points(k, d, ur, np.array(points, MP), f, SCALE, th, 0.8, blocked)


def test_claims_block_later_points_only_when_observed():
    f = frame()
    k = keys([(500, 100), (501, 100)])
    d = np.stack([desc_with([]), desc_with([1])])
    # two points wanting key 0: the first (observed) takes it, the second falls back to key 1
    pts = [point_at(f, 500.2, 100, 10, desc_with([])), point_at(f, 500.3, 100, 10, desc_with([]))]
    view, match, n = local(pts, k, d)
    assert view.all() and list(match) == [0, 1] and n == 2
    # an unobserved first point does not block: the second overwrites its claim, both count
    pts[0]["observed"] = 0
    view, match, n = local(pts, k, d)
    assert list(match) == [1, -1] and n == 2
    # a key blocked on entry is no candidate
    view, match, n = local(pts[1:], k, d, blocked=np.array([1, 0], np.uint8))
    assert list(match) == [-1, 0] and n == 1


def test_ratio_test_applies_only_on_equal_levels():
    f = frame()
    k = keys([(500, 100), (501, 100)], 0)
    d = np.stack([desc_with(range(10)), desc_with(range(11))])
    q = desc_with([])
    view, match, n = local([point_at(f, 500.5, 100, 10, q)], k, d)  # 10 > 0.8 * 11, same level: rejected
    assert n == 0 and (match == -1).all()
    k["octave"][1] = 1  # point predicts level 0: window levels [-1, 0] drop key 1 -> accepted
    view, match, n = local([point_at(f, 500.5, 100, 10, q)], k, d)
    assert n == 1 and match[0] == 0
    k["octave"][1] = 0
    d[1] = desc_with(range(13))  # 10 <= 0.8 * 13
    assert local([point_at(f, 500.5, 100, 10, q)], k, d)[2] == 1


def test_frustum_edges():
    f = frame()
    lg = T.logf(SCALE[1])
    p = point_at(f, 500, 100, 10, desc_with([]))
    assert T.is_in_frustum(p, f, lg, 8) is not None
    behind = p.copy()
    behind["pos"] = -p["pos"]
    assert T.is_in_frustum(behind, f, lg, 8) is None
    zero = p.copy()
    zero["pos"] = (0, 0, 0)  # PcZ = 0, PcX = 0: u is NaN
    assert T.is_in_frustum(zero, f, lg, 8) is None
    nan = p.copy()
    nan["pos"] = (np.nan, 0, 5)
    assert T.is_in_frustum(nan, f, lg, 8) is None
    # exactly on the distance-invariance limits: dist == 1.2f max and dist == 0.8f min are in view
    dist = T.norm3(p["pos"] - f.Ow)
    for mx, mn, ok in ((dist / np.float32(1.2), np.float32(0), None), (dist, dist / np.float32(0.8), None)):
        q = p.copy()
        q["max_distance"], q["min_distance"] = mx, mn
        lim_hi, lim_lo = np.float32(1.2) * q["max_distance"], np.float32(0.8) * q["min_distance"]
        expect = lim_lo <= dist <= lim_hi
        assert (T.is_in_frustum(q, f, lg, 8) is not None) == expect
    q = p.copy()
    q["max_distance"] = dist * np.float32(0.5)
    assert T.is_in_frustum(q, f, lg, 8) is None


def test_three_maxima_ties_and_the_tenth_rule():
    assert T.compute_three_maxima([0] * 30) == (-1, -1, -1)
    c = [0] * 30
    c[3], c[5], c[7] = 10, 10, 10  # ties: the first of equals wins each rank
    assert T.compute_three_maxima(c) == (3, 5, 7)
    c[9] = 10
    assert T.compute_three_maxima(c) == (3, 5, 7)
    c = [0] * 30
    c[2], c[4], c[6] = 100, 10, 9  # 9 < 0.1 * 100 drops the third, 10 is kept
    assert T.compute_three_maxima(c) == (2, 4, -1)
    c[4] = 9
    assert T.compute_three_maxima(c) == (2, -1, -1)


def test_rotation_bins_use_only_0_to_12():
    bins = {T.rotation_bin(a, 0.0) for a in np.arange(0, 360, 0.25, dtype=np.float32)}
    assert bins == set(range(13))
    assert T.rotation_bin(0.0, 15.0) == 12 and T.rotation_bin(0.0, 0.0) == 0 and T.rotation_bin(15.0, 0.0) == 1


BAD_ANGLES = (np.nan, np.inf, -np.inf, -400.0, 720.0, np.nextafter(np.float32(360), np.float32(400)), -np.float32(1e-45))
GOOD_ANGLES = (-0.0, 0.0, 360.0, 359.99997, 1e-45)


def test_angle_rule_keeps_every_rotation_bin_in_0_to_12():
    for a in BAD_ANGLES:
        assert not T.angle_ok(a), a
        for args in ((a, 0.0), (0.0, a), (a, a)):
            try:
                T.rotation_bin(*args)
            except ValueError:
                continue
            raise AssertionError(args)
    for a in GOOD_ANGLES:
        assert T.angle_ok(a), a
        for b in GOOD_ANGLES:
            assert 0 <= T.rotation_bin(a, b) <= 12, (a, b)
    assert T.rotation_bin(-0.0, 0.0) == 0 and T.rotation_bin(0.0, -0.0) == 0
    assert T.rotation_bin(360.0, 0.0) == 12 and T.rotation_bin(0.0, 360.0) == 0 and T.rotation_bin(360.0, 360.0) == 0


def test_angle_rule_drops_keys_and_last_frame_points():
    f = frame()
    n = 2 * len(BAD_ANGLES) + len(GOOD_ANGLES)
    angles = list(BAD_ANGLES) + list(GOOD_ANGLES) + list(BAD_ANGLES)
    k = keys([(100 + 20 * i, 100) for i in range(n)], 0)
    k["angle"] = angles
    d = np.stack([desc_with([i]) for i in range(n)])
    ur = np.full(n, -1, np.float32)
    grid = T.assign_features_to_grid(k, f)
    placed = sorted(j for col in grid for cell in col for j in cell)
    assert placed == [j for j in range(n) if T.angle_ok(angles[j])]
    # a key breaking the rule is no candidate of either search
    pts = [point_at(f, 100 + 20 * i, 100, 10, desc_with([i]), angle=0.0) for i in range(n)]
    view, match, nm = local(pts, k, d)
    assert view.all() and nm == len(GOOD_ANGLES) and list(np.flatnonzero(match >= 0)) == placed
    match, nm = T.search_last_frame(k, d, ur, np.array(pts, MP), f, np.eye(3), np.zeros(3), SCALE, 7)
    assert nm == len(GOOD_ANGLES) and list(np.flatnonzero(match >= 0)) == placed
    # a last-frame point breaking the rule is not searched; -0.0 and 360 are (bins 0 and 12, both kept)
    k["angle"] = 0.0
    for i, p in enumerate(pts):
        p["angle"] = angles[i]
    match, nm = T.search_last_frame(k, d, ur, np.array(pts, MP), f, np.eye(3), np.zeros(3), SCALE, 7)
    good = [i for i in range(n) if T.angle_ok(angles[i])]
    assert nm == len(good) and list(np.flatnonzero(match >= 0)) == good and [int(match[i]) for i in good] == good


def test_last_frame_histogram_culls_every_entry_of_a_losing_bin():
    f = frame()
    n = 40
    k = keys([(100 + 20 * i, 100) for i in range(n)], 0, 0.0)
    d = np.stack([desc_with([i]) for i in range(n)])
    ur = np.full(n, -1, np.float32)
    pts = []
    for i in range(n):
        angle = 0.0 if i < 30 else 30.0 * (i - 29)  # 30 in bin 0, then bins 1..10 with one entry each (< 0.1 * 30)
        pts.append(point_at(f, 100 + 20 * i, 100, 10, desc_with([i]), octave=0, angle=angle))
    match, nm = T.search_last_frame(k, d, ur, np.array(pts, MP), f, np.eye(3), np.zeros(3), SCALE, 7)
    assert nm == 30 and list(match[:30]) == list(range(30)) and (match[30:] == -1).all()
    # duplicates: two unobserved points claim key 0 from different bins; the losing entry frees the key and both entries count
    a = point_at(f, 100, 100, 10, desc_with([0]), observed=0, angle=0.0)
    b = point_at(f, 100, 100, 10, desc_with([0]), observed=0, angle=100.0)  # bin round(100 / 30) = 3
    match, nm = T.search_last_frame(k, d, ur, np.array([a] * 5 + [b], MP), f, np.eye(3), np.zeros(3), SCALE, 7)
    assert nm == 6 and match[0] == 5  # 1 >= 0.1 * 5: bin 3 is kept, the last writer holds the key
    match, nm = T.search_last_frame(k, d, ur, np.array([a] * 11 + [b] + [a], MP), f, np.eye(3), np.zeros(3), SCALE, 7)
    assert nm == 13 - 1 and match[0] == -1  # 1 < 0.1 * 12: bin 3's one entry frees key 0 although bin 0 won
