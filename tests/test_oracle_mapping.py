"""CPU: oracle/mapping_oracle.py -- its cv::Mat forms pinned against cv2, the triangulation rule against cv2.SVDecomp and a float64
SVD, and hand-built cases for the reference facts it keeps."""
import copy
import math

import cv2
import numpy as np
import pytest

from oracle import mapping_scene as S
from oracle import mapping_oracle as MO
from sivo_b200.orb import KP_DTYPE

F32, F64 = np.float32, np.float64
N_PIN = 10000


def _rot(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], F32)


def test_cv_forms_pinned():
    rng = np.random.default_rng(0)
    for _ in range(N_PIN):
        R1, R2 = _rot(rng), _rot(rng)
        x = (rng.normal(size=(3, 1)) * 10).astype(F32)
        t = rng.normal(size=(3, 1)).astype(F32)
        assert np.array_equal(cv2.gemm(R1, R2, 1, None, 0, flags=cv2.GEMM_2_T), MO.gemm_bt(R1, R2))
        assert np.array_equal(cv2.gemm(R1, R2, 1, None, 0), MO.gemm(R1, R2))
        assert np.array_equal(cv2.gemm(R1, x, 1, t, 1), MO.gemm(R1, x, t))
        assert np.array_equal(cv2.gemm(R1, x, 1, None, 0), MO.gemm(R1, x))
        K = np.array([[rng.uniform(300, 1000), 0, rng.uniform(200, 700)], [0, rng.uniform(300, 1000), rng.uniform(100, 400)], [0, 0, 1]],
                     F32)
        assert np.array_equal(cv2.invert(K)[1], MO.inv3(K))
        assert np.array_equal(cv2.invert(np.ascontiguousarray(K.T))[1], MO.inv3(K.T))
        r2, r0, s = rng.normal(size=(1, 4)).astype(F32), rng.normal(size=(1, 4)).astype(F32), F32(rng.normal())
        assert np.array_equal(cv2.addWeighted(r2, float(s), r0, -1.0, 0.0)[0], MO.add_weighted_row(s, r2[0], r0[0]))
        assert cv2.norm(x) == MO.norm3(x[:, 0])


def test_f12_is_the_cv_chain():
    rng = np.random.default_rng(1)
    cam = S.camera()
    K = np.array([[cam.fx, 0, cam.cx], [0, cam.fy, cam.cy], [0, 0, 1]], F32)
    for _ in range(300):
        kf1 = MO.KeyFrame(*([np.zeros(0)] * 9), Rcw=_rot(rng), tcw=rng.normal(size=3) * 5)
        kf2 = MO.KeyFrame(*([np.zeros(0)] * 9), Rcw=_rot(rng), tcw=rng.normal(size=3) * 5)
        R12 = cv2.gemm(kf1.Rcw, kf2.Rcw, 1, None, 0, flags=cv2.GEMM_2_T)
        t12 = cv2.gemm(-R12, kf2.tcw.reshape(3, 1), 1, kf1.tcw.reshape(3, 1), 1)[:, 0]
        tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]], F32)
        F = cv2.gemm(cv2.gemm(cv2.gemm(cv2.invert(np.ascontiguousarray(K.T))[1], tx, 1, None, 0), R12, 1, None, 0), cv2.invert(K)[1], 1, None, 0)
        assert np.array_equal(F, MO.compute_f12(kf1, kf2, cam))


def test_svd_rule_against_cv2_and_float64():
    """The documented rule's world point against what the reference computes (cv::SVD in float) and a float64 SVD, on triangulation
    systems of random stereo scenes.  Bound: 1e-4 relative on the point for well-conditioned systems."""
    rng = np.random.default_rng(2)
    worst_cv, worst_np = 0.0, 0.0
    for _ in range(3000):
        T1 = np.hstack([_rot(rng), rng.normal(size=(3, 1)).astype(F32)])
        T2 = np.hstack([_rot(rng) @ np.eye(3, dtype=F32), (T1[:, 3:] + rng.normal(size=(3, 1)) * 0.5).astype(F32)])
        X = rng.normal(size=3) * 5
        xs = []
        for T in (T1, T2):
            p = T[:, :3].astype(F64) @ X + T[:, 3]
            if p[2] <= 0.5:
                break
            xs.append((F32(p[0] / p[2]), F32(p[1] / p[2])))
        if len(xs) < 2:
            continue
        A = np.stack([MO.add_weighted_row(xs[0][0], T1[2], T1[0]), MO.add_weighted_row(xs[0][1], T1[2], T1[1]),
                      MO.add_weighted_row(xs[1][0], T2[2], T2[0]), MO.add_weighted_row(xs[1][1], T2[2], T2[1])])
        v = np.array(MO.svd_null_vector(A.astype(F64)), F64).astype(F32)
        rule = v[:3] / v[3]
        _, _, vt = cv2.SVDecomp(A.copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)
        cvp = vt[3, :3] / vt[3, 3]
        vt64 = np.linalg.svd(A.astype(F64))[2]
        npp = vt64[3, :3] / vt64[3, 3]
        s = np.linalg.svd(A.astype(F64), compute_uv=False)
        if s[2] < 1e3 * s[3] or s[2] < 1e-3:
            continue
        scale = max(1.0, float(np.abs(npp).max()))
        worst_cv = max(worst_cv, float(np.abs(rule - cvp).max()) / scale)
        worst_np = max(worst_np, float(np.abs(rule - npp).max()) / scale)
    assert worst_np < 1e-5, worst_np
    assert worst_cv < 1e-4, worst_cv


def test_svd_rule_decisions_against_cv2():
    """On every triangulation of constructed scenes (ill-conditioned systems included), the decisions that read the point -- w == 0,
    z1 > 0, z2 > 0 and the 5.991 sigma2 reprojection test in the current keyframe -- taken on the rule's point and on
    cv2.SVDecomp's.  The differing decisions are listed with their margins; they must be rare and close to their thresholds."""
    cam = S.camera()
    kf1, nbs = S.make_scene(600, 3, seed=21)
    n, diffs = 0, []
    for kf2 in nbs:
        F = MO.compute_f12(kf1, kf2, cam)
        ex, ey = MO.epipole(kf1, kf2, cam)
        groups = {}
        for i2 in range(len(kf2.kps)):
            if kf2.node[i2] >= 0:
                groups.setdefault(int(kf2.node[i2]), []).append(i2)
        T1 = np.hstack([kf1.Rcw, kf1.tcw.reshape(3, 1)])
        T2 = np.hstack([kf2.Rcw, kf2.tcw.reshape(3, 1)])
        for j in range(len(kf1.kps)):
            m = MO.search_key(kf1, j, kf2, F, ex, ey, S.TABLES.scale, S.TABLES.sigma2, groups) if kf1.node[j] >= 0 else -1
            if m < 0:
                continue
            xn1 = [(F32(kf1.kps["x"][j]) - cam.cx) * cam.invfx, (F32(kf1.kps["y"][j]) - cam.cy) * cam.invfy]
            xn2 = [(F32(kf2.kps["x"][m]) - cam.cx) * cam.invfx, (F32(kf2.kps["y"][m]) - cam.cy) * cam.invfy]
            A = np.stack([MO.add_weighted_row(xn1[0], T1[2], T1[0]), MO.add_weighted_row(xn1[1], T1[2], T1[1]),
                          MO.add_weighted_row(xn2[0], T2[2], T2[0]), MO.add_weighted_row(xn2[1], T2[2], T2[1])])
            v_rule = np.array(MO.svd_null_vector(A.astype(F64)), F64).astype(F32)
            v_cv = cv2.SVDecomp(A.copy(), flags=cv2.SVD_MODIFY_A | cv2.SVD_FULL_UV)[2][3]
            n += 1

            def decide(v):
                if v[3] == 0:
                    return (False,), (0.0,)
                x = v[:3] / v[3]
                z1 = MO.dot3(kf1.Rcw[2], x) + float(kf1.tcw[2])
                z2 = MO.dot3(kf2.Rcw[2], x) + float(kf2.tcw[2])
                u = cam.fx * F32(MO.dot3(kf1.Rcw[0], x) + float(kf1.tcw[0])) * (F32(1) / F32(z1)) + cam.cx
                e = float(u - F32(kf1.kps["x"][j]))
                lim = 5.991 * float(S.TABLES.sigma2[kf1.kps["octave"][j]])
                return (True, z1 > 0, z2 > 0, e * e <= lim), (1.0, z1, z2, e * e - lim)

            (dr, mr), (dc, _) = decide(v_rule), decide(v_cv)
            if dr != dc:
                diffs.append((j, dr, dc, mr))
    assert n > 300
    assert len(diffs) <= 0.01 * n, diffs
    for _, dr, dc, margin in diffs:  # a differing decision is one whose quantity is near its threshold
        assert len(dr) == len(dc) and min(abs(float(x)) for x in margin[1:]) < 1e-2, (dr, dc, margin)


def _kf(xs, octs, ur, node, desc, Rcw=np.eye(3), tcw=(0, 0, 0)):
    n = len(xs)
    kps = np.zeros(n, KP_DTYPE)
    kps["x"], kps["y"], kps["octave"] = [p[0] for p in xs], [p[1] for p in xs], octs
    return MO.KeyFrame(kps=kps, desc=np.asarray(desc, np.uint8).reshape(n, 32), u_right=np.asarray(ur, F32),
                       depth=np.full(n, 10, F32), kp_class=np.ones(n, np.uint8), kp_conf=np.ones(n), kp_entropy=np.zeros(n),
                       node=np.asarray(node, np.int32), has_point=np.zeros(n, np.uint8), Rcw=Rcw, tcw=tcw)


def test_tie_goes_to_the_later_candidate_and_duplicates_allowed():
    cam = S.camera()
    d = np.zeros((1, 32), np.uint8)
    kf1 = _kf([(500, 170), (500, 170)], [0, 0], [400, 400], [3, 3], np.vstack([d, d]))
    kf2 = _kf([(500, 170)] * 3, [0, 0, 0], [400] * 3, [3, 3, 3], np.vstack([d, d, d]), tcw=(-0.6, 0, 0))
    F = MO.compute_f12(kf1, kf2, cam)
    ex, ey = MO.epipole(kf1, kf2, cam)
    groups = {3: [0, 1, 2]}
    m0 = MO.search_key(kf1, 0, kf2, F, ex, ey, S.TABLES.scale, S.TABLES.sigma2, groups)
    m1 = MO.search_key(kf1, 1, kf2, F, ex, ey, S.TABLES.scale, S.TABLES.sigma2, groups)
    assert m0 == m1 == 2  # equal distances: the last candidate; both current keys match the same neighbour key


def test_epipole_gate_uses_the_scale_factor_not_squared():
    """Mono-mono pairs with the neighbour key at distance r from the epipole (the principal point: both centres on the z axis):
    inside sqrt(100 scale) the gate rejects, outside it the key matches, also inside sqrt(100 scale^2)."""
    s3 = float(S.TABLES.scale[3])
    radii = (0.99 * math.sqrt(100 * s3), 1.01 * math.sqrt(100 * s3), 0.99 * math.sqrt(100 * s3 * s3))
    kf1, kf2 = S.pair_scene([(0.0, 0.0, 30.0)] * 3, stereo1=False, stereo2=False, o2=3)
    for i, r in enumerate(radii):
        for kf in (kf1, kf2):
            kf.kps["x"][i], kf.kps["y"][i] = F32(S.CX + r), F32(S.CY)
    ex, ey = MO.epipole(kf1, kf2, S.camera())
    assert (ex, ey) == (F32(S.CX), F32(S.CY))
    r = S.oracle_run(kf1, [kf2], 0.5, -1e9)
    assert list(r["match"][0]) == [-1, 1, 2]
    # the same pairs with a stereo neighbour key: no gate
    kf2.u_right[:] = 100.0
    assert (S.oracle_run(kf1, [kf2], 0.5, -1e9)["match"][0] >= 0).all()


def test_second_keyframes_stereo_branch():
    """A mono current key and a stereo neighbour key at low ray parallax: cosParallaxStereo2 is set (the `else if`), and the point
    is the neighbour's UnprojectStereo; with both keys stereo the first keyframe's branch wins and cosParallaxStereo2 stays
    cosParallaxRays + 1."""
    cam = S.camera()
    k1, k2 = S.pair_scene([S.P0], stereo1=False, stereo2=True, o2=3)
    st, x3, _, _ = MO.triangulate_pair(k1, 0, k2, 0, cam, S.TABLES.scale, S.TABLES.sigma2, F32(1.2), S.sigma_cw(), 8, 0.5, -1e9)
    assert st == MO.CREATED and np.array_equal(x3, MO.unproject(k2, 0, cam))
    k1, k2 = S.pair_scene([S.P0], stereo1=True, stereo2=True, o2=3)
    k1.depth[0] = F32(3000.0)  # the first keyframe's stereo cosine near 1: the rays triangulate
    st, x3, _, _ = MO.triangulate_pair(k1, 0, k2, 0, cam, S.TABLES.scale, S.TABLES.sigma2, F32(1.2), S.sigma_cw(), 8, 0.5, -1e9)
    assert st == MO.CREATED and not np.array_equal(x3, MO.unproject(k2, 0, cam))


def test_nan_reduction_passes():
    kf1, nbs = S.make_scene(400, 1, seed=9)
    kf1.kp_entropy[:] = np.nan
    r = S.oracle_run(kf1, nbs)
    made = r["stage"] == MO.CREATED
    assert made.any() and np.isnan(r["reduction"][made]).all()


@pytest.fixture(scope="module")
def constructed():
    return [(sc, sc.run()) for sc in S.constructed_scenes()]


def test_constructed_pairs_end_where_they_say(constructed):
    for sc, r in constructed:
        for k, st in sc.want.items():
            assert r["stage"][k] == st, (sc.name, k, int(r["stage"][k]), st)
        for k, m in sc.match.items():
            assert r["match"][k] == m, (sc.name, k, int(r["match"][k]), m)
        if sc.flip is not None:  # one ulp apart, pairs 1 and 2 fall on either side of the flip
            st = r["stage"][0]
            assert (st[1] == sc.flip) != (st[2] == sc.flip) and st[0] == st[1] and st[2] == st[3], (sc.name, st)


def test_constructed_scenes_reach_every_stage(constructed):
    """Every stage of the rule is reached by some constructed pair, none named unreachable: W_ZERO needs a pose that is not a
    rotation (the `w_zero` scene) and dist == 0 a camera centre that is not -Rcw^T tcw (`dist_zero`); with true poses neither
    can happen (the reasons are in oracle/mapping_scene.py)."""
    reached = {int(s) for _, r in constructed for s in np.unique(r["stage"])}
    assert reached == set(range(MO.CREATED + 1))
    by = {sc.name: (sc, r) for sc, r in constructed}
    # dist_zero's SCALE is the dist1 == 0 branch: with the current keyframe's centre put back, the same pair creates the point
    # that the scene's centre sits on
    sc, _ = by["dist_zero"]
    kf1 = copy.copy(sc.kf1)
    kf1.Ow = np.zeros(3, F32)  # the current keyframe of a pair scene sits at the origin
    back = S.oracle_run(kf1, sc.nbs, sc.th_conf, sc.th_red)
    assert back["stage"][0, 0] == MO.CREATED and np.array_equal(back["world"][0], sc.kf1.Ow)
    # the epipole gate at octave 0 sits on distex^2 == 100 exactly
    sc, _ = by["epipole_o0"]
    assert (F32(S.CX) - sc.nbs[0].kps["x"][1]) ** 2 == F32(100)
    # the 4-level 1.5x extractor: ratioFactor 2.25, a key at octave nlevels (4) left out
    sc, r = by["four_levels"]
    assert F32(1.5) * F32(sc.ext.scale_factor) == F32(2.25) and sc.ext.nlevels == 4


def test_stereo_min_keeps_the_rays_cosine_over_a_nan_stereo_cosine():
    """std::min(cosParallaxStereo1, cosParallaxStereo2) is (b < a) ? b : a: a NaN stereo cosine of the neighbour key gives
    cosParallaxRays + 1, so a mono current key against a stereo neighbour key at depth NaN triangulates its rays."""
    k1, k2 = S.pair_scene([S.P0], stereo1=False, stereo2=True, o2=3)
    k2.depth[0] = np.nan
    st, x3, _, _ = MO.triangulate_pair(k1, 0, k2, 0, S.camera(), S.TABLES.scale, S.TABLES.sigma2, F32(1.2), S.sigma_cw(), 8, 0.5, -1e9)
    assert st == MO.CREATED and np.isfinite(x3).all()
