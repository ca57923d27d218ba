"""Constructed keyframes for the map-point creation tests and tools/mapping_bench.py: world points seen from a short stereo trajectory, each keyframe's keys a
shuffled mix of the points' projections (descriptors a few bits off the point's own) and distractors sharing their vocabulary
nodes, with stereo and mono keys, keys that hold a point on entry and keys without a node."""
from __future__ import annotations

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


def oracle_run(kf1, nbs, th_conf=0.5, th_red=9.5, max_class=8):
    return MO.create_new_map_points(kf1, nbs, camera(), TABLES.scale, TABLES.sigma2, np.float32(EXTRACTOR.scale_factor), sigma_cw(),
                                    max_class, th_conf, th_red)


# ---------------------------------------------------------------------------------------------------------- hand-built pairs
def _project(P, C):
    """Identity-rotation camera at centre C: (u, v, z) of world point P in float32."""
    X, Y, Z = (P[k] - C[k] for k in range(3))
    return F32(FX * X / Z + CX), F32(FY * Y / Z + CY), F32(Z)


F32 = np.float32
C2_DEFAULT = (0.0, 0.0, 20.0)


def pair_scene(points, c2=C2_DEFAULT, o1=0, o2=0, stereo1=True, stereo2=True):
    """One pair per world point: current key i and neighbour key i, both in node i, project the point exactly (kf1 at the origin,
    the neighbour at c2, identity rotations); depths and right coordinates consistent, descriptors equal, class 1, confidence 1,
    entropy 0.  Returns (kf1, kf2); tests edit the per-key arrays."""
    n = len(points)
    kfs = []
    for C, o, stereo in (((0.0, 0.0, 0.0), o1, stereo1), (c2, o2, stereo2)):
        kps = np.zeros(n, KP_DTYPE)
        ur = np.empty(n, np.float32)
        depth = np.empty(n, np.float32)
        for i, P in enumerate(points):
            u, v, z = _project(P, C)
            kps[i]["x"], kps[i]["y"], kps[i]["octave"] = u, v, o
            depth[i] = z
            ur[i] = u - F32(MBF) / z if stereo else -1.0
        kps["size"], kps["response"] = 31.0, 1.0
        kfs.append(MO.KeyFrame(kps=kps, desc=np.zeros((n, 32), np.uint8), u_right=ur, depth=depth, kp_class=np.ones(n, np.uint8),
                               kp_conf=np.ones(n), kp_entropy=np.zeros(n), node=np.arange(n, dtype=np.int32),
                               has_point=np.zeros(n, np.uint8), Rcw=np.eye(3), tcw=-np.asarray(C, np.float32)))
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


def _set_point(kf1, kf2, i, P, c2=C2_DEFAULT):
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

    return {
        # CheckDistEpipolarLine: dsqr < 3.84 sigma2 (the neighbour key moved off the epipolar line)
        "dsqr": case(set_y2, y2, y2 + 20, MO.NO_MATCH),
        # the stereo reprojection errors, 7.8 sigma2, in the current keyframe and in the neighbour
        "reproj1_stereo": case(set_ur1, ur1, ur1 + 20, MO.REPROJ1),
        "reproj2_stereo": case(set_ur2, ur2, ur2 + 20, MO.REPROJ2),
        # scale consistency: the point's depth moves the distance ratio across ratioOctave / ratioFactor
        "scale": case(set_z, 25.0, 40.0, MO.SCALE),
    }
