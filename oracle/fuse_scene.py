"""Constructed maps for the Fuse tests and tools/fuse_bench.py: landmarks seen from a short stereo trajectory, each keyframe's keys
the landmarks' projections (a few pixels and descriptor bits off) plus distractors, and map points that duplicate landmarks
across keyframes, so that SearchInNeighbors' two phases exercise every part of the replay contract:
- duplicate points near one 3-D position, so Fuse finds a key that already holds a point;
- Replace in both directions, equal observation counts among them (the strict > sends pMPinKF->Replace(pMP));
- bad points left in a target's mvpMapPoints;
- two points that pick the same key in one target;
- a landmark held twice by one keyframe, so a Replace survivor can come later in the phase-1 list;
- survivors whose new descriptor changes their match in a later target (the re-search rule).
oracle/fuse_oracle.py records which of these a map exercised (fuse(..., events=))."""
from __future__ import annotations

import numpy as np

from oracle import fuse_oracle as FO
from oracle.orb_oracle import ExtractorParams, Tables
from oracle.track_oracle import gemm_neg_t
from sivo_b200.orb import KP_DTYPE

FX, FY, CX, CY, MBF = 500.0, 500.0, 320.0, 240.0, 40.0
BOUNDS = (0.0, 640.0, 0.0, 480.0)
EXTRACTOR = ExtractorParams(nfeatures=2000, scale_factor=1.2, nlevels=8)
_T = Tables(EXTRACTOR)
TABLES = FO.Tables(_T.scale, _T.inv_sigma2)
CAMERA = FO.Camera(FX, FY, CX, CY, MBF, BOUNDS)


def rotation(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
            @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))


def pose(k, rng):
    R = rotation(*(rng.normal(0, 0.01, 3))).astype(np.float32)
    C = np.array([0.12 * k, 0.02 * rng.normal(), 0.05 * k], np.float64)
    t = (-R.astype(np.float64) @ C).astype(np.float32)
    return R, t, gemm_neg_t(R, t)


def flip(desc, n_bits, rng):
    d = desc.copy()
    for b in rng.choice(256, n_bits, replace=False):
        d[b >> 3] ^= np.uint8(1 << (b & 7))
    return d


def make_map(seed, n_landmarks=120, n_targets=5, n_distractors=40, dup=0.5, double=0.15, bad=0.05, max_flip=14):
    """-> (current KeyFrame, [target KeyFrames], [every MapPoint]).  The current keyframe is keyframe 0."""
    rng = np.random.default_rng(seed)
    L = np.stack([rng.uniform(-2.5, 2.5, n_landmarks), rng.uniform(-1.8, 1.8, n_landmarks), rng.uniform(4, 9, n_landmarks)], 1)
    ldesc = rng.integers(0, 256, (n_landmarks, 32), dtype=np.uint8)
    kfs, holders = [], []  # holders[k][l] = the keys of keyframe k that see landmark l
    for k in range(n_targets + 1):
        R, t, Ow = pose(k, rng)
        Pc = (R.astype(np.float64) @ L.T).T + t
        u = FX * Pc[:, 0] / Pc[:, 2] + CX
        v = FY * Pc[:, 1] / Pc[:, 2] + CY
        rec, desc, ur, hold = [], [], [], {}
        for l in range(n_landmarks):
            if not (Pc[l, 2] > 0.5 and 2 < u[l] < 638 and 2 < v[l] < 478) or rng.random() < 0.15:
                continue
            for _ in range(2 if rng.random() < double else 1):
                o = int(rng.integers(0, 3))
                rec.append((u[l] + rng.normal(0, 0.4), v[l] + rng.normal(0, 0.4), o))
                desc.append(flip(ldesc[l], int(rng.integers(0, max_flip)), rng))
                ur.append(u[l] - MBF / Pc[l, 2] + rng.normal(0, 0.4) if rng.random() < 0.7 else -1.0)
                hold.setdefault(l, []).append(len(rec) - 1)
        for _ in range(n_distractors):
            rec.append((rng.uniform(0, 640), rng.uniform(0, 480), int(rng.integers(0, 4))))
            desc.append(rng.integers(0, 256, 32, dtype=np.uint8))
            ur.append(-1.0)
        perm = rng.permutation(len(rec))  # keys in no particular order, as an extractor leaves them
        inv = np.argsort(perm)
        kps = np.zeros(len(rec), KP_DTYPE)
        kps["x"] = [rec[p][0] for p in perm]
        kps["y"] = [rec[p][1] for p in perm]
        kps["octave"] = [rec[p][2] for p in perm]
        kps["angle"] = rng.uniform(0, 360, len(rec))
        kps["size"] = 31
        kfs.append(FO.KeyFrame(k, kps, np.array(desc)[perm], np.array(ur, np.float32)[perm], R, t, Ow, CAMERA))
        holders.append({l: [int(inv[j]) for j in js] for l, js in hold.items()})
    points = []
    for l in range(n_landmarks):
        # one map point per landmark, a duplicate with probability dup; each key of the landmark goes to one of them at random
        n_copies = 2 if rng.random() < dup else 1
        copies = []
        for c in range(n_copies):
            mp = FO.MapPoint(len(points), (L[l] + rng.normal(0, 0.01, 3)).astype(np.float32), np.zeros(3, np.float32), 0.0, 0.0,
                             ldesc[l].copy())
            copies.append(mp)
            points.append(mp)
        for k, kf in enumerate(kfs):
            for j in holders[k].get(l, []):
                if rng.random() < 0.35:
                    continue
                mp = copies[int(rng.integers(0, n_copies))]
                if mp.is_in_keyframe(kf):
                    mp = copies[-1 - copies.index(mp)] if n_copies == 2 else None
                    if mp is None or mp.is_in_keyframe(kf):
                        continue
                mp.add_observation(kf, j)
                kf.add_map_point(mp, j)
        for mp in copies:
            obs = mp.observations()
            if not obs:
                mp.min_distance = mp.max_distance = np.float32(1.0)
                mp.normal = np.array([0, 0, 1], np.float32)
                continue
            mp.compute_distinctive_descriptors()
            # MapPoint::UpdateNormalAndDepth with the first observer as the reference keyframe
            n = np.zeros(3, np.float64)
            for kf, _ in obs:
                a = mp.pos.astype(np.float64) - kf.Ow
                n += a / np.linalg.norm(a)
            mp.normal = (n / len(obs)).astype(np.float32)
            ref, j = obs[0]
            dist = np.float32(np.linalg.norm(mp.pos.astype(np.float64) - ref.Ow))
            mp.max_distance = dist * TABLES.scale[int(ref.kps["octave"][j])]
            mp.min_distance = mp.max_distance / TABLES.scale[-1]
    # bad points left in a target's mvpMapPoints (their observations already cleared)
    for kf in kfs[1:]:
        for j, mp in enumerate(kf.points):
            if mp is not None and not mp.bad and rng.random() < bad:
                for okf, idx in mp.observations():
                    if okf is not kf:
                        okf.erase_map_point_match(idx)
                mp.obs, mp.bad = {}, True
    return kfs[0], kfs[1:], points


CONSTRUCTED = [dict(seed=s) for s in range(6)] + [dict(seed=100 + s, dup=0.9, double=0.4, max_flip=30) for s in range(6)]


def fuzz_params(seed):
    rng = np.random.default_rng(10_000 + seed)
    return dict(seed=seed, n_landmarks=int(rng.integers(20, 150)), n_targets=int(rng.integers(1, 8)),
                n_distractors=int(rng.integers(0, 60)), dup=float(rng.uniform(0, 1)), double=float(rng.uniform(0, 0.5)),
                bad=float(rng.uniform(0, 0.2)), max_flip=int(rng.integers(1, 40)))


# ---------------------------------------------------------------------------------------------------------- boundary cases
# A camera whose projections are exact at z = 1: u = 512 x + 320, v = 512 y + 256.
EDGE_CAMERA = FO.Camera(512.0, 512.0, 320.0, 256.0, 40.0, (0.0, 640.0, 0.0, 512.0))
F32, F64 = np.float32, np.float64


def _next(x, toward, n=1):
    x = F32(x)
    for _ in range(n):
        x = np.nextafter(x, F32(toward))
    return x


def desc_bits(n_bits) -> np.ndarray:
    """A descriptor at Hamming distance n_bits from the all-zero one (the edge points' descriptor)."""
    d = np.zeros(256, np.uint8)
    d[:n_bits] = 1
    return np.packbits(d, bitorder="little")


def edge_target(keys, kf_id=1, R=None, t=None, cam=EDGE_CAMERA):
    """keys: (x, y, octave, u_right, distance) tuples; identity pose by default."""
    kps = np.zeros(len(keys), KP_DTYPE)
    kps["x"] = [k[0] for k in keys]
    kps["y"] = [k[1] for k in keys]
    kps["octave"] = [k[2] for k in keys]
    kps["size"] = 31
    desc = np.array([desc_bits(k[4]) for k in keys], np.uint8).reshape(-1, 32)
    R = np.eye(3, dtype=np.float32) if R is None else np.asarray(R, np.float32)
    t = np.zeros(3, np.float32) if t is None else np.asarray(t, np.float32)
    return FO.KeyFrame(kf_id, kps, desc, np.array([k[3] for k in keys], np.float32), R, t, gemm_neg_t(R, t), cam)


def edge_point(pos, min_d=0.01, max_d=None, normal=None, bits=0):
    pos = np.asarray(pos, np.float32)
    if max_d is None:
        max_d = F32(np.linalg.norm(pos.astype(np.float64))) * TABLES.scale[2]  # predicts level 2 or 3
    if normal is None:
        n = pos.astype(np.float64)
        normal = (n / np.linalg.norm(n)).astype(np.float32) if np.all(np.isfinite(n)) and np.any(n) else np.array([0, 0, 1], np.float32)
    return {"pos": pos, "normal": np.asarray(normal, np.float32), "min_distance": F32(min_d), "max_distance": F32(max_d),
            "desc": desc_bits(bits)}


def level_of(p) -> int:
    from oracle.track_oracle import norm3, predict_scale
    lv = predict_scale(p["max_distance"], norm3(p["pos"]), TABLES.log_scale, TABLES.nlevels)
    return -1 if lv is None else lv


def _at(p, octave, ur=None, dist=10, dx=0.0, dy=0.0):
    """A key at p's projection (z = 1 camera) with the given octave, u_right (default: mono) and distance."""
    u = F32(512) * p["pos"][0] / p["pos"][2] + F32(320) if p["pos"][2] else F32(320)
    v = F32(512) * p["pos"][1] / p["pos"][2] + F32(256) if p["pos"][2] else F32(256)
    return (F32(u + F32(dx)), F32(v + F32(dy)), octave, -1.0 if ur is None else ur, dist)


def edge_cases():
    """-> [(name, [targets], [point records], th)] over the rule's boundaries; oracle.fuse_oracle.decide is the judge."""
    cases = []
    # depth: Pc_z at -0.0, +0.0 and one ulp either side (tcw = -0 keeps a -0 sum), x, y negative so that 0 x stays -0
    pts = [edge_point([-0.1, -0.1, z], max_d=100.0) for z in (F32(-0.0), F32(0.0), _next(0, 1), _next(0, -1), F32(1e-30), F32(-1e-30))]
    cases.append(("depth", [edge_target([(268.8, 204.8, 0, -1.0, 5)], t=np.array([-0.0, -0.0, -0.0], np.float32))], pts, 3.0))
    # image bounds: u and v at min (in) and max (out) and one ulp either side, at z = 1
    pts, keys = [], []
    for target_u, target_v in [(0, 100), (640, 100), (100, 0), (100, 512)]:
        for du in (-1, 0, 1):
            u = _next(target_u, np.inf if du > 0 else -np.inf, abs(du)) if du else F32(target_u)
            v = F32(target_v)
            if target_v in (0, 512):
                u, v = F32(target_u), (_next(target_v, np.inf if du > 0 else -np.inf, abs(du)) if du else F32(target_v))
            p = edge_point([(F64(u) - 320) / 512, (F64(v) - 256) / 512, 1.0])
            pts.append(p)
            keys += [(u, v, level_of(p), -1.0, 3), (u - F32(1), v - F32(1), level_of(p), -1.0, 4)]  # the first can fall off the grid
    cases.append(("image", [edge_target(keys)], pts, 3.0))
    # distance gates: dist3D = z exactly at 0.8f min and 1.2f max and one ulp either side
    pts = []
    for md in (F32(2.0), F32(3.3)):
        gate = F32(0.8) * md
        for z in (gate, _next(gate, 0), _next(gate, 9)):
            pts.append(edge_point([0, 0, z], min_d=md, max_d=F32(50.0)))
        gate = F32(1.2) * md
        for z in (gate, _next(gate, 0), _next(gate, 9)):
            pts.append(edge_point([0, 0, z], min_d=0.01, max_d=md))
    cases.append(("distance", [edge_target([(320.0, 256.0, o, -1.0, 7) for o in range(8)])], pts, 3.0))
    # viewing angle: PO . n against 0.5 dist3D (pos (0, 0, 2): dot = 2 n_z), NaN normals and positions
    pts = [edge_point([0, 0, 2], normal=[0, 0, nz]) for nz in (F32(0.5), _next(0.5, 0), _next(0.5, 1), F32(np.nan))]
    pts += [edge_point([0, 0, 2], normal=[F32(np.nan), 0, 0]), edge_point([F32(np.nan), 0, 2], max_d=10.0),
            edge_point([0, 0, F32(np.nan)], max_d=10.0), edge_point([0, 0, 2], max_d=F32(np.nan)), edge_point([0, 0, 2], min_d=F32(np.nan))]
    cases.append(("angle_nan", [edge_target([(320.0, 256.0, o, -1.0, 9) for o in range(8)])], pts, 3.0))
    # PredictScale at exact powers (max_distance / dist = scale[l]) and at both clamps
    pts = [edge_point([0, 0, 2], max_d=F32(2) * TABLES.scale[l]) for l in range(8)]
    pts += [edge_point([0, 0, 2], max_d=F32(2) * _next(TABLES.scale[l], 9)) for l in range(8)]
    pts += [edge_point([0, 0, 2], min_d=0.001, max_d=F32(1.7)), edge_point([0, 0, 2], max_d=F32(1e4))]
    cases.append(("scale", [edge_target([(320.0, 256.0, o, -1.0, 20 + o) for o in range(8)])], pts, 3.0))
    # octaves level - 2 .. level + 1 (each alone in its own target), and level 0 with an octave -1 key at the same place
    pts, targets = [], []
    p = edge_point([0.1, 0.05, 2.0], max_d=F32(2.0))
    for o in range(-1, 8):
        targets.append(edge_target([_at(p, o, dist=12)], kf_id=1 + len(targets)))
    pts.append(p)
    for lv in (1, 3, 7):
        pts.append(edge_point([0.1, 0.05, 2.0], max_d=F32(np.linalg.norm([0.1, 0.05, 2.0])) * TABLES.scale[lv] * F32(0.99)))
    cases.append(("octaves", targets, pts, 3.0))
    # u_right 0, -1, NaN, and a matching stereo key (z = 1: ur = u - 40)
    p = edge_point([0.05, 0.05, 1.0])
    lv = level_of(p)
    ur_p = _at(p, lv)[0] - F32(40)
    targets = [edge_target([_at(p, lv, ur=ur, dist=11)], kf_id=1 + i) for i, ur in enumerate((0.0, -1.0, np.nan, ur_p, ur_p + 2.5))]
    cases.append(("u_right", targets, [p], 3.0))
    # chi2: e2 invSigma2 at 5.99 (mono) and 7.8 (stereo), the floats either side of each in double
    p = edge_point([0.0, 0.0, 1.0], max_d=F32(1.0))  # projects at (320, 256), level 0, ur = 280
    targets = []
    for stereo, bound in ((False, 5.99), (True, 7.8)):
        ex = F32(np.sqrt(bound - 3e-4))
        kx = F32(320) - ex
        ex = F32(320) - kx
        base = []
        for step in range(-900, 900):
            ky = _next(256, np.inf if step > 0 else -np.inf, abs(step)) if step else F32(256)
            ey = F32(256) - ky
            if stereo:
                er = F32(0.0)
                e2 = (ex * ex + ey * ey) + er * er
            else:
                e2 = ex * ex + ey * ey
            base.append((abs(F64(e2) - bound), ky))
        for _, ky in sorted(base, key=lambda e: (e[0], e[1]))[:6]:
            targets.append(edge_target([(kx, ky, 0, F32(280) if stereo else -1.0, 4)], kf_id=1 + len(targets)))
    cases.append(("chi2", targets, [p], 3.0))
    # a crowded window: ties (the first in walk order wins), 50 against 51, over several cells and 32-key chunks
    rng = np.random.default_rng(3)
    p = edge_point([0.02, -0.01, 1.0], max_d=F32(1.0))  # level 0: radius 3 scale[0]
    u0, v0 = _at(p, 0)[:2]
    keys = [(u0 + F32(rng.uniform(-2.9, 2.9)), v0 + F32(rng.uniform(-2.9, 2.9)), int(rng.integers(0, 2)), -1.0, int(d))
            for d in rng.choice([50, 51, 52, 60], 90)]
    keys += [(u0 + F32(rng.uniform(-0.5, 0.5)), v0 + F32(rng.uniform(-0.5, 0.5)), 0, -1.0, 50) for _ in range(5)]
    pts = [p, edge_point([0.02, -0.01, 1.0], max_d=F32(1.0), bits=1), edge_point([0.02, -0.01, 1.0], max_d=F32(1.0), bits=256)]
    far = [k[:4] + (max(k[4], 51),) for k in keys]  # best 51: above TH_LOW
    cases.append(("crowd", [edge_target(keys), edge_target(far, kf_id=2)], pts, 3.0))
    cases.append(("crowd_th", [edge_target(keys), edge_target(far, kf_id=2)], pts, 1.5))
    # clipped corners: windows at the image corners
    corner_keys, pts = [], []
    for cu, cv in ((0.5, 0.5), (639.5, 0.5), (0.5, 511.5), (639.5, 511.5)):
        q = edge_point([(cu - 320) / 512, (cv - 256) / 512, 1.0])
        pts.append(q)
        corner_keys += [(F32(cu + dx), F32(cv + dy), level_of(q), -1.0, 30 + i) for i, (dx, dy) in enumerate(((0.4, 0.4), (-0.4, 0.2), (1.0, -0.3)))]
    cases.append(("corners", [edge_target(corner_keys)], pts, 4.0))
    return cases
