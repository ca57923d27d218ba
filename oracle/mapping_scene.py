"""Constructed keyframes for the map-point creation tests and tools/mapping_bench.py: world points seen from a short stereo trajectory, each keyframe's keys a
shuffled mix of the points' projections (descriptors a few bits off the point's own) and distractors sharing their vocabulary
nodes, with stereo and mono keys, keys that hold a point on entry and keys without a node."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle import mapping_oracle as MO
from oracle.orb_oracle import ExtractorParams, Tables
from sivo_b200.orb import KP_DTYPE

FX, FY, CX, CY, MBF = 718.856, 718.856, 498.19, 174.22, 386.1448
EXTRACTOR = ExtractorParams(nfeatures=2000, scale_factor=1.2, nlevels=8)
TABLES = Tables(EXTRACTOR)
W, H = 1000, 350


def rotation(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def camera():
    return MO.Camera(FX, FY, CX, CY, MBF)


def sigma_cw():
    a = np.random.default_rng(5).standard_normal((6, 6))
    return 1e-3 * (a @ a.T + 0.5 * np.eye(6))


def make_scene(n_keys=2000, n_neighbours=3, seed=0, n_nodes=300):
    """-> (kf1, [neighbour KeyFrames]) as oracle KeyFrames (one entry per key)."""
    rng = np.random.default_rng(seed)
    n_pts = int(n_keys * 0.8)
    P = np.stack([rng.uniform(-12, 12, n_pts), rng.uniform(-3, 2, n_pts), rng.uniform(4, 40, n_pts)], 1)
    pdesc = rng.integers(0, 256, (n_pts, 32), dtype=np.uint8)
    pnode = rng.integers(0, n_nodes, n_pts)
    pclass = np.where(rng.random(n_pts) < 0.85, rng.integers(0, 3, n_pts), rng.integers(0, 12, n_pts))
    kfs = []
    for k in range(n_neighbours + 1):
        R = rotation(0.004 * k, 0.02 * k * (-1) ** k, 0.002 * k).astype(np.float32)
        C = np.array([0.3 * k * (-1) ** k, 0.02 * k, 0.9 * k], np.float64)
        t = (-R.astype(np.float64) @ C).astype(np.float32)
        Pc = (R.astype(np.float64) @ P.T).T + t
        u = FX * Pc[:, 0] / Pc[:, 2] + CX
        v = FY * Pc[:, 1] / Pc[:, 2] + CY
        vis = np.flatnonzero((Pc[:, 2] > 0.5) & (u > 0) & (u < W) & (v > 0) & (v < H))
        vis = rng.permutation(vis)[: int(n_keys * 0.75)]
        n_dis = n_keys - len(vis)
        octave = rng.integers(0, 4, n_keys)
        scale = TABLES.scale[octave]
        x = np.concatenate([u[vis], rng.uniform(0, W, n_dis)]) + rng.normal(0, 0.6, n_keys) * scale
        y = np.concatenate([v[vis], rng.uniform(0, H, n_dis)]) + rng.normal(0, 0.6, n_keys) * scale
        z = np.concatenate([Pc[vis, 2], rng.uniform(3, 40, n_dis)]) * (1 + rng.normal(0, 0.01, n_keys))
        desc = np.concatenate([pdesc[vis], rng.integers(0, 256, (n_dis, 32), dtype=np.uint8)])
        flips = rng.integers(0, 256, (n_keys, 32), dtype=np.uint8) & rng.integers(0, 256, (n_keys, 32), dtype=np.uint8) \
            & rng.integers(0, 256, (n_keys, 32), dtype=np.uint8) & rng.integers(0, 256, (n_keys, 32), dtype=np.uint8)
        desc = desc ^ np.where(rng.random((n_keys, 1)) < 0.7, flips & (flips >> 1), flips)
        node = np.concatenate([pnode[vis], rng.integers(0, n_nodes, n_dis)])
        node[rng.random(n_keys) < 0.03] = -1
        cls = np.concatenate([pclass[vis], rng.integers(0, 12, n_dis)]).astype(np.uint8)
        stereo = rng.random(n_keys) < 0.6
        depth = np.where(stereo, z, np.where(rng.random(n_keys) < 0.5, -1.0, z)).astype(np.float32)
        ur = np.where(stereo, x - MBF / z, -1.0).astype(np.float32)
        order = rng.permutation(n_keys)
        kps = np.zeros(n_keys, KP_DTYPE)
        kps["x"], kps["y"], kps["octave"] = x[order], y[order], octave[order]
        kps["size"], kps["response"] = 31.0, 1.0
        kps["angle"] = rng.uniform(0, 360, n_keys)
        kfs.append(MO.KeyFrame(kps=kps, desc=desc[order], u_right=ur[order], depth=depth[order], kp_class=cls[order],
                               kp_conf=rng.uniform(0.2, 1.0, n_keys), kp_entropy=rng.uniform(0.0, 2.0, n_keys),
                               node=node[order].astype(np.int32), has_point=(rng.random(n_keys) < 0.1).astype(np.uint8),
                               Rcw=R, tcw=t))
    return kfs[0], kfs[1:]


def oracle_run(kf1, nbs, th_conf=0.5, th_red=9.5, max_class=8, ext=EXTRACTOR):
    t = TABLES if ext == EXTRACTOR else Tables(ext)
    return MO.create_new_map_points(kf1, nbs, camera(), t.scale, t.sigma2, np.float32(ext.scale_factor), sigma_cw(), max_class, th_conf,
                                    th_red)


def compare(got, want, th_red=9.5, max_exempt=5):
    """Bit-identical, except that a (neighbour, key) decision may differ where the oracle's reduction lies within 1e-12 of the
    threshold (log2) or a decision reading cos(2 atan2(...)) is within 2 float ulps of flipping; such a key is left out of every
    comparison from that pair on, and the number of such keys must stay small.  `got` without match / stage / reduction (the
    production and device forms) is compared on its outputs only.  Returns the number of exempt keys."""
    red_w = want["reduction"]
    with np.errstate(invalid="ignore"):
        near = (np.abs(red_w - np.float64(np.float32(th_red))) < 1e-12) | (want["parallax_ulps"] <= 2)
    exempt_key = near.any(axis=0)
    assert exempt_key.sum() <= max_exempt
    ok = ~exempt_key
    if "stage" in got:
        red_g = got["reduction"]
        both = ~np.isnan(red_w[:, ok])
        assert np.array_equal(np.isnan(red_g[:, ok]), ~both)
        np.testing.assert_allclose(red_g[:, ok][both], red_w[:, ok][both], rtol=0, atol=1e-12)
        np.testing.assert_array_equal(got["stage"][:, ok], want["stage"][:, ok])
        np.testing.assert_array_equal(got["match"][:, ok], want["match"][:, ok])
    np.testing.assert_array_equal(got["created_nb"][ok], want["created_nb"][ok])
    np.testing.assert_array_equal(got["created_idx"][ok], want["created_idx"][ok])
    np.testing.assert_array_equal(got["world"][ok].view(np.uint32), want["world"][ok].view(np.uint32))
    keep = lambda lst: lst[ok[lst[:, 1]]] if len(lst) else lst
    np.testing.assert_array_equal(keep(got["created"]), keep(want["created"]))
    if not exempt_key.any():
        assert got["n_created"] == len(want["created"])
    return int(exempt_key.sum())


# ---------------------------------------------------------------------------------------------------------- hand-built pairs
def _project(P, C, R=None):
    """Camera at centre C with rotation R (identity when None): (u, v, z) of world point P in float32."""
    X, Y, Z = (P[k] - C[k] for k in range(3))
    if R is not None:
        X, Y, Z = (float(R[r][0]) * X + float(R[r][1]) * Y + float(R[r][2]) * Z for r in range(3))
    return F32(FX * X / Z + CX), F32(FY * Y / Z + CY), F32(Z)


F32 = np.float32
C2_DEFAULT = (0.0, 0.0, 20.0)


def pair_scene(points, c2=C2_DEFAULT, o1=0, o2=0, stereo1=True, stereo2=True, R2=None):
    """One pair per world point: current key i and neighbour key i, both in node i, project the point exactly (kf1 at the origin
    with the identity rotation, the neighbour at c2 with rotation R2, identity when None); depths and right coordinates consistent,
    descriptors equal, class 1, confidence 1, entropy 0.  Returns (kf1, kf2); tests edit the per-key arrays."""
    n = len(points)
    kfs = []
    for C, o, stereo, R in (((0.0, 0.0, 0.0), o1, stereo1, None), (c2, o2, stereo2, R2)):
        kps = np.zeros(n, KP_DTYPE)
        ur = np.empty(n, np.float32)
        depth = np.empty(n, np.float32)
        for i, P in enumerate(points):
            u, v, z = _project(P, C, R)
            kps[i]["x"], kps[i]["y"], kps[i]["octave"] = u, v, o
            depth[i] = z
            ur[i] = u - F32(MBF) / z if stereo else -1.0
        kps["size"], kps["response"] = 31.0, 1.0
        Rf = np.eye(3, dtype=np.float32) if R is None else np.asarray(R, np.float32)
        kfs.append(MO.KeyFrame(kps=kps, desc=np.zeros((n, 32), np.uint8), u_right=ur, depth=depth, kp_class=np.ones(n, np.uint8),
                               kp_conf=np.ones(n), kp_entropy=np.zeros(n), node=np.arange(n, dtype=np.int32),
                               has_point=np.zeros(n, np.uint8), Rcw=Rf,
                               tcw=-(Rf.astype(np.float64) @ np.asarray(C, np.float64)).astype(np.float32)))
    return kfs[0], kfs[1]


def _bits(x) -> int:
    return int(np.array(F32(x)).view(np.int32))


def _float(b) -> np.float32:
    return np.array(b, np.int32).view(np.float32)[()]


def straddle(pred, lo, hi):
    """Positive floats lo < hi with pred(lo) != pred(hi): the four floats b - 1, b, b + 1, b + 2 ulps around the adjacent pair
    (b, b + 1) where pred flips."""
    a, b = _bits(lo), _bits(hi)
    pa = pred(_float(a))
    assert pred(_float(b)) != pa
    while b - a > 1:
        m = (a + b) // 2
        if pred(_float(m)) == pa:
            a = m
        else:
            b = m
    return [_float(a + k) for k in (-1, 0, 1, 2)]


P0 = (0.6, 0.3, 30.0)


def _set_point(kf1, kf2, i, P, c2=C2_DEFAULT):  # identity rotations
    for kf, C in ((kf1, (0.0, 0.0, 0.0)), (kf2, c2)):
        u, v, z = _project(P, C)
        kf.kps["x"][i], kf.kps["y"][i], kf.depth[i] = u, v, z
        if kf.u_right[i] >= 0:
            kf.u_right[i] = u - F32(MBF) / z


def boundary_cases():
    """Each geometric threshold of the rule at its flip: name -> (kf1, kf2, rejecting stage).  The four pairs of a scene differ only
    in the varied input, which steps by one float ulp across the flip; the oracle's stages on the two sides differ."""
    def stage_of(kf1, kf2):
        return oracle_run(kf1, [kf2], 0.5, -1e9)["stage"][0, 0]

    def case(setter, lo, hi, reject, P=P0, **kw):
        kw.setdefault("o2", 3)  # octaves 0 / 3 keep the pair's distance ratio (about 1 / 3) inside the scale test

        def one(v):
            kf1, kf2 = pair_scene([P], **kw)
            setter(kf1, kf2, 0, v)
            return kf1, kf2

        vals = straddle(lambda v: stage_of(*one(v)) == reject, lo, hi)
        kf1, kf2 = pair_scene([P] * 4, **kw)
        for i, v in enumerate(vals):
            setter(kf1, kf2, i, v)
        return kf1, kf2, reject

    k1, k2 = pair_scene([P0])
    y2, ur1, ur2 = float(k2.kps["y"][0]), float(k1.u_right[0]), float(k2.u_right[0])
    def set_y2(a, b, i, v):
        b.kps["y"][i] = v

    def set_ur1(a, b, i, v):
        a.u_right[i] = v

    def set_ur2(a, b, i, v):
        b.u_right[i] = v

    def set_z(a, b, i, v):
        _set_point(a, b, i, (P0[0], P0[1], float(v)))

    # forward motion by 1 along z and a point on the row through the principal point: the epipolar line is that row, so a key
    # moved along x stays on it while the other key's UnprojectStereo fixes the point
    Pr, cr = (0.6, 0.0, 30.0), (0.0, 0.0, 1.0)
    x1, x2 = float(_project(Pr, (0, 0, 0))[0]), float(_project(Pr, cr)[0])

    def set_x1(a, b, i, v):
        a.kps["x"][i] = v

    def set_x2(a, b, i, v):
        b.kps["x"][i] = v

    Pp, cp = (0.3, 0.1, 30.0), (0.6, 0.0, 1.0)

    def set_zp(a, b, i, v):
        _set_point(a, b, i, (Pp[0], Pp[1], float(v)), cp)

    def set_zu(a, b, i, v):
        _set_point(a, b, i, (P0[0], P0[1], float(v)), (0.0, 0.0, -20.0))

    def set_xe(a, b, i, v):  # both keys on the row through the epipole (the principal point), v pixels right of it
        for kf in (a, b):
            kf.kps["x"][i], kf.kps["y"][i] = F32(CX) + F32(v), F32(CY)

    return {
        # CheckDistEpipolarLine: dsqr < 3.84 sigma2 (the neighbour key moved off the epipolar line)
        "dsqr": case(set_y2, y2, y2 + 20, MO.NO_MATCH),
        # the stereo reprojection errors, 7.8 sigma2, in the current keyframe and in the neighbour
        "reproj1_stereo": case(set_ur1, ur1, ur1 + 20, MO.REPROJ1),
        "reproj2_stereo": case(set_ur2, ur2, ur2 + 20, MO.REPROJ2),
        # the mono reprojection errors, 5.991 sigma2: the mono key slides along its epipolar line, the stereo key's point stays
        "reproj1_mono": case(set_x1, x1, x1 + 6, MO.REPROJ1, Pr, c2=cr, o2=0, stereo1=False),
        "reproj2_mono": case(set_x2, x2, x2 + 6, MO.REPROJ2, Pr, c2=cr, o2=0, stereo2=False),
        # scale consistency: the point's depth moves the distance ratio across ratioOctave / ratioFactor (lower side) and, with the
        # neighbour behind the current keyframe, across ratioOctave * ratioFactor (upper side)
        "scale": case(set_z, 25.0, 40.0, MO.SCALE),
        "scale_upper": case(set_zu, 20.0, 25.0, MO.SCALE, c2=(0.0, 0.0, -20.0), o2=0),
        # mono-mono parallax: cosParallaxRays < 0.9998 as the point recedes (a lateral baseline of 0.6)
        "parallax_mono": case(set_zp, 30.0, 32.0, MO.PARALLAX, Pp, c2=cp, o2=0, stereo1=False, stereo2=False),
        # the epipole gate at octave 7: distex^2 + distey^2 < 100 scale[7] (3.58, not squared: 12.8)
        "epipole_o7": case(set_xe, 10.0, 40.0, MO.NO_MATCH, (0.0, 0.0, 30.0), o2=7, stereo1=False, stereo2=False),
    }


# ---------------------------------------------------------------------------------------------------------- constructed scenes
@dataclass
class Scene:
    """A constructed case: keyframes, the call's thresholds and extractor, and where named pairs must end in the oracle:
    want[(neighbour, key)] = stage, match[(neighbour, key)] = the neighbour key matched (-1: none)."""
    name: str
    kf1: MO.KeyFrame
    nbs: list
    want: dict
    match: dict = field(default_factory=dict)
    th_conf: float = 0.5
    th_red: float = -1e9
    max_class: int = 8
    ext: ExtractorParams = field(default_factory=lambda: EXTRACTOR)
    flip: int = None  # boundary_cases' stage on one side of the flip (pairs 1 and 2)

    def run(self):
        return oracle_run(self.kf1, self.nbs, self.th_conf, self.th_red, self.max_class, self.ext)


def desc_at(d) -> np.ndarray:
    """A 32-byte descriptor at Hamming distance d from the zero descriptor (the pair scenes' current keys)."""
    return np.packbits(np.arange(256) < d)


def crowd_scene(groups, o2=3):
    """Current key g (at P0's projection, node g) against the candidates groups[g]: neighbour keys in node g, all at P0's
    projection in the neighbour (every one passes the geometric gates), at descriptor distances groups[g][k] from key g, laid out
    group after group in the neighbour's key order."""
    kf1, _ = pair_scene([P0] * len(groups), o2=o2)
    sizes = [len(g) for g in groups]
    _, kf2 = pair_scene([P0] * sum(sizes), o2=o2)
    kf2.node[:] = np.repeat(np.arange(len(groups)), sizes).astype(np.int32)
    kf2.desc[:] = np.stack([desc_at(d) for g in groups for d in g])
    return kf1, kf2


def _next(x, toward):
    return np.nextafter(F32(x), F32(toward))


def constructed_scenes():
    """The matching, geometric and semantic decisions of the rule at their edges, each scene's named pairs ending at a named stage
    (tests/test_oracle_mapping.py holds the oracle to them; tests/test_gpu_mapping_edges.py runs them through every form)."""
    out = []
    add = lambda *a, **kw: out.append(Scene(*a, **kw))
    C, N, X = MO.CREATED, MO.NO_MATCH, MO.SEMANTIC
    # ---- matching
    # TH_LOW: distance 50 matches, 51 does not; a later 50 does not replace an earlier 49
    kf1, kf2 = crowd_scene([[50], [51], [49, 50]])
    add("th_low", kf1, [kf2], {(0, 0): C, (0, 1): N, (0, 2): C}, {(0, 0): 0, (0, 1): -1, (0, 2): 2})
    # exact ties: the later candidate.  Group 0: keys 3 / 20 (two lanes of one stride); group 1: keys 5 / 37 / 69 of the group
    # (one lane, three strides: groups of 64 and 96 keep the lanes); group 2: keys 10 / 33 (the later key in an earlier lane)
    g0, g1, g2 = [20] * 64, [20] * 96, [20] * 64
    g0[3] = g0[20] = 7
    g1[5] = g1[37] = g1[69] = 7
    g2[10] = g2[33] = 7
    kf1, kf2 = crowd_scene([g0, g1, g2])
    add("ties", kf1, [kf2], {(0, 0): C, (0, 1): C, (0, 2): C}, {(0, 0): 20, (0, 1): 64 + 69, (0, 2): 160 + 33})
    # a node of 330 candidates behind 17 keys of another node, the best in the last partial stride (keys 320-346)
    rng = np.random.default_rng(11)
    g = list(rng.integers(6, 51, 330))
    g[329] = 5
    kf1, kf2 = crowd_scene([[30] * 17, g])
    add("crowded_node", kf1, [kf2], {(0, 1): C}, {(0, 0): 16, (0, 1): 17 + 329})
    # the best candidates hold a point on entry (left out); so do neighbour keys at octave -1 and nlevels (they never take part)
    kf1, kf2 = crowd_scene([[10, 3, 12, 3, 8], [2, 2, 9, 11, 2]])
    kf2.has_point[[1, 3]] = 1
    kf2.kps["octave"][[5, 6, 9]] = [-1, EXTRACTOR.nlevels, 1 << 30]
    add("candidate_left_out", kf1, [kf2], {(0, 0): C, (0, 1): C}, {(0, 0): 4, (0, 1): 7})
    # current keys at octave -1 / nlevels and without a node: never searched (also by the debug form)
    kf1, kf2 = crowd_scene([[5]] * 4)
    kf1.kps["octave"][[0, 1]] = [-1, EXTRACTOR.nlevels]
    kf1.node[2] = -1
    add("current_left_out", kf1, [kf2], {(0, 0): N, (0, 1): N, (0, 2): N, (0, 3): C}, {(0, 0): -1, (0, 1): -1, (0, 2): -1, (0, 3): 3})
    # the epipole gate at octave 0 (threshold 100): distex = 10 - ulp rejected, 10 and 10 + ulp pass; both keys on the row of the
    # epipole (the principal point)
    kf1, kf2 = pair_scene([(0.0, 0.0, 30.0)] * 3, stereo1=False, stereo2=False, o2=0)
    x10 = F32(CX) + F32(10)
    for i, x in enumerate((_next(x10, 0), x10, _next(x10, 1e3))):
        for kf in (kf1, kf2):
            kf.kps["x"][i], kf.kps["y"][i] = x, F32(CY)
    add("epipole_o0", kf1, [kf2], {(0, 0): N}, {(0, 0): -1, (0, 1): 1, (0, 2): 2})
    # ---- geometry
    # the baseline: (float) norm(Ow2 - Ow1) < mb skips; at mb and one ulp above the neighbour is searched
    mb = camera().mb
    nbs = []
    for b in (_next(mb, 0), mb, _next(mb, 1)):
        _, k2 = pair_scene([P0], o2=3)
        k2.Ow = np.array([b, 0, 0], F32)
        nbs.append(k2)
    kf1, _ = pair_scene([P0], o2=3)
    add("baseline", kf1, nbs, {(0, 0): MO.BASELINE, (1, 0): C, (2, 0): MO.HAS_POINT})
    add("baseline_above", kf1, nbs[2:], {(0, 0): C})
    # rays at cos <= 0 (the neighbour faces the current keyframe from z = 60): mono-mono, no point; both stereo, the reference's
    # cosParallaxStereo2 stays cosParallaxRays + 1 < cosParallaxStereo1, so the neighbour's key is unprojected
    R180 = np.diag([-1.0, 1.0, -1.0])
    P = (3.0, 1.0, 30.0)
    kf1, kf2 = pair_scene([P] * 2, c2=(0.0, 0.0, 60.0), R2=R180, o2=0)
    kf1.u_right[0] = kf2.u_right[0] = -1
    add("rays_opposed", kf1, [kf2], {(0, 0): MO.PARALLAX, (0, 1): C}, {(0, 0): 0, (0, 1): 1})
    # the stereo branches at low parallax (forward motion by 1): both stereo and stereo1 only unproject the current key (cs1 <
    # cs2), stereo2 only the neighbour's; a stereo current key whose depth is 0, negative or NaN gives no point, as does a stereo
    # neighbour key at depth 0; at depth NaN its cosParallaxStereo2 is NaN, std::min keeps cosParallaxRays + 1 and the rays
    # triangulate (bStereo2 waives the 0.9998 test); a NaN u_right is mono
    Pf, cf = (0.6, 0.3, 30.0), (0.0, 0.0, 1.0)
    kf1, kf2 = pair_scene([Pf] * 9, c2=cf, o2=0)
    kf2.u_right[1] = -1
    kf1.u_right[2] = -1
    kf1.depth[3:6] = [0.0, -30.0, np.nan]
    kf2.depth[6:8] = [0.0, np.nan]
    kf1.u_right[6:8] = -1
    kf1.u_right[8] = np.nan
    add("stereo_branches", kf1, [kf2], {(0, 0): C, (0, 1): C, (0, 2): C, (0, 3): MO.PARALLAX, (0, 4): MO.PARALLAX,
                                        (0, 5): MO.PARALLAX, (0, 6): MO.PARALLAX, (0, 7): C, (0, 8): C})
    # points behind a camera: rays that meet behind the current keyframe (mono); a point between the keyframes (mono, behind the
    # neighbour); the current key's UnprojectStereo at depth 3, behind the neighbour at z = 20
    kf1, kf2 = pair_scene([(3.0, 1.0, 10.0), (3.0, 1.0, 10.0), P0], c2=(0.0, 0.0, 20.0), stereo1=False, stereo2=False, o2=0)
    kf1.kps["x"][0], kf2.kps["x"][0] = F32(CX + 300), F32(CX + 80)  # diverging rays on the row through the epipole
    kf1.kps["y"][0] = kf2.kps["y"][0] = F32(CY)
    kf1.u_right[2], kf1.depth[2] = kf1.kps["x"][2] - F32(MBF) / F32(3), F32(3)
    add("behind", kf1, [kf2], {(0, 0): MO.Z1, (0, 1): MO.Z2, (0, 2): MO.Z2})
    # the largest octave gaps, 0 against 7 and 7 against 0, with distance ratios inside the scale test
    kf1, kf2 = pair_scene([P0] * 2, o1=0, o2=7)
    add("octaves_0_7", kf1, [kf2], {(0, 0): C, (0, 1): C})
    kf1, kf2 = pair_scene([(0.6, 0.3, 20.0)] * 2, c2=(0.0, 0.0, -40.0), o1=7, o2=0)
    add("octaves_7_0", kf1, [kf2], {(0, 0): C, (0, 1): C})
    # w == 0: only a pose that is not a rotation reaches it.  The neighbour's Rcw is a shear whose third column cancels the key's
    # normalised x and y, so A's third column is exactly zero: the rule's null vector is (0, 0, 1, 0), while the rays (Rwc xn)
    # keep a parallax of about 0.1 rad.  A rotation cannot do this: w rounds to 0 only for |v3| < 2^-150, rays parallel to far
    # below the 2.4e-4 rad that cosParallaxRays < 1 needs.
    kf1, kf2 = pair_scene([(0.0, 0.0, 30.0)], c2=(1.0, 0.0, 0.0), stereo1=False, stereo2=False, o2=0)
    kf1.kps["x"][0], kf1.kps["y"][0] = F32(CX), F32(CY)  # xn1 = (0, 0): A's rows of the current keyframe have a zero third column
    kf2.kps["x"][0], kf2.kps["y"][0] = F32(CX) + F32(71.8856), F32(CY)
    a = (kf2.kps["x"][0] - F32(CX)) * (F32(1) / F32(FX))
    R2 = np.array([[1, 0, a], [0, 1, 0], [0, 0, 1]], F32)
    t12 = np.array([1.0, 0.0, 0.0])  # in the plane of the rays: the epipolar line passes through the key
    kf2.Rcw, kf2.tcw = R2, (-np.linalg.inv(R2.T.astype(np.float64)) @ t12).astype(F32)
    kf2.Rwc, kf2.Ow = np.ascontiguousarray(R2.T), np.array([5.0, 0.0, 0.0], F32)
    add("w_zero", kf1, [kf2], {(0, 0): MO.W_ZERO})
    # dist == 0: the Z1 check stops a point at a true camera centre, so only a centre that is not -Rcw^T tcw reaches it.  The
    # current keyframe's Ow is put on the point its stereo pair triangulates; its 7.8 sigma2 reprojection reads Rcw and tcw
    kf1, kf2 = pair_scene([P0], o2=3)
    x3 = MO.triangulate_pair(kf1, 0, kf2, 0, camera(), TABLES.scale, TABLES.sigma2, F32(1.2), sigma_cw(), 8, 0.5, -1e9)[1]
    kf1.Ow = x3.copy()
    add("dist_zero", kf1, [kf2], {(0, 0): MO.SCALE})
    # ---- semantics: classes 0 / 8 / 9 / 254 / 255 on both keys against max_static_class -1 / 8 / 254 / 255 (255 is VOID: never)
    cls = np.array([0, 8, 9, 254, 255], np.uint8)
    for mc, made in ((-1, ()), (8, (0, 1)), (254, (0, 1, 2, 3)), (255, (0, 1, 2, 3))):
        kf1, kf2 = pair_scene([P0] * 5, o2=3)
        kf1.kp_class[:] = kf2.kp_class[:] = cls
        add(f"max_class_{mc}", kf1, [kf2], {(0, j): C if j in made else X for j in range(5)}, max_class=mc)
    # a class mismatch, VOID on the neighbour's key, NaN confidence, a current key with depth <= 0 (mono: its class is VOID)
    kf1, kf2 = pair_scene([Pf] * 6, c2=cf, o2=0)
    kf2.kp_class[0], kf2.kp_class[1] = 2, 255
    kf1.kp_conf[2] = np.nan
    kf1.u_right[3:5], kf1.depth[3:5] = -1, [0.0, -1.0]
    add("semantic_keys", kf1, [kf2], {(0, 0): X, (0, 1): X, (0, 2): X, (0, 3): X, (0, 4): X, (0, 5): C})
    # NaN thresholds: confidence >= NaN fails; a reduction < NaN does not
    kf1, kf2 = pair_scene([P0] * 2, o2=3)
    add("nan_th_confidence", kf1, [kf2], {(0, 0): X, (0, 1): X}, th_conf=float("nan"))
    add("nan_th_reduction", kf1, [kf2], {(0, 0): C, (0, 1): C}, th_red=float("nan"))
    # ---- a 4-level 1.5x extractor (ratioFactor 2.25): keys at octave 3 take part, at octave 4 (nlevels) never
    four = ExtractorParams(nfeatures=2000, scale_factor=1.5, nlevels=4)
    kf1, kf2 = pair_scene([P0] * 4, o2=3)
    kf1.kps["octave"][1] = 4
    kf2.kps["octave"][2] = 4
    kf1.kps["octave"][3] = 3
    add("four_levels", kf1, [kf2], {(0, 0): C, (0, 1): N, (0, 2): N}, {(0, 1): -1, (0, 2): -1}, ext=four)
    # ---- the threshold flips of boundary_cases, one ulp apart
    for name, (kf1, kf2, reject) in boundary_cases().items():
        add(name, kf1, [kf2], {}, flip=reject)
    return out
