"""Constructed candidates for the PnP RANSAC tests: each scene names the paths of PnPsolver (and of k_pnp_setup / k_pnp_hyp /
k_pnp_decide, which restate it) it must reach, and `paths_reached` reads them back from the scene's inputs and the oracle's
per-hypothesis log, so a test can check both that a scene still reaches what it was built for and that the scenes together reach
every path in PATHS.

A scene is one candidate's correspondences (p2d, p3d, octave) with its draw keys (seed, kf_id, frame_id) and a schedule of
iterate(n) calls.  `embed` lays it out as sivo_pnp_setup_device's inputs: semantic keys in order, an oracle/keymap.py keep_idx
into the extractor's slots, a match row into a permuted point array, and (optionally) rejected entries of every kind in
between, so that the setup's compaction must return exactly the scene's correspondences.

  placed      every observation is computed from the pose it must agree with, in CheckInliers' own arithmetic: exact (error
              below 1e-3 px), at a chosen multiple of the threshold, or far off.  The hypothesis draws depend only on (seed,
              kf_id, frame_id, g, N), so a builder knows each hypothesis' minimal set before it places anything.
  searched    the RANSAC bookkeeping (a count at minInliers, ties, a failed Refine then a recovery, a pose on a call's last
              hypothesis) depends on every hypothesis' EPnP pose, which 4-point EPnP does not pin down; those scenes draw from a
              family of near-threshold observations and keep the first kf_id whose oracle run takes the named path.  The kf_ids
              are recorded in SEARCHED, and the CPU test holds every scene to its paths, so a change of rule that moves a path
              fails there first.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from oracle import pnp_oracle as P
from oracle.keymap import SLACK, keymap, scatter
from oracle.orb_oracle import ExtractorParams, Tables
from sivo_b200.orb import KP_DTYPE

F32, F64 = np.float32, np.float64
KITTI = (718.856, 718.856, 607.1928, 185.2157)
SEED, FRAME = 0x5EED5EED1234, 77
EXTRACTOR = ExtractorParams(nfeatures=2000, scale_factor=1.2, nlevels=8)
SIGMA2 = Tables(EXTRACTOR).sigma2


def capacity(ext=EXTRACTOR) -> int:
    """sivo_orb_capacity of an extractor with these parameters (nfeatures + 4 nlevels + 64)."""
    return ext.nfeatures + 4 * ext.nlevels + 64


PATHS = (
    # setup
    "keep_permuted", "keep_neg", "keep_cap", "match_neg5", "match_neg1", "match_np", "match_np1", "oct_neg", "oct_nlevels",
    "oct_127", "reject_255", "reject_256", "reject_511", "reject_512",
    "N_0", "N_4", "N_9", "N_10", "N_11", "N_14", "N_15", "N_cap",
    # iterate
    "below_at_min", "at_min", "improve", "tie", "worse", "refine_fail_at_min", "refine_ok_at_min1", "refine_skipped",
    "fail_then_recover", "ok_on_last", "no_more_pose", "no_more_none", "after_max_its", "pose_mid_schedule",
    # hypothesis
    "e2_eq_max", "e2_ulp_below", "zc_zero", "behind_camera", "xc_overflow", "coplanar", "collinear", "coincident", "duplicate",
    "best_1", "best_2", "best_3", "pcs_flip", "det_flip", "b1_neg", "b1_pos", "b2_neg", "b2_pos", "b2_x1_neg", "b3_neg",
    "b3_pos", "b3_x1_neg", "draw_swapped_r", "draw_swapped_back", "mask_31", "mask_32", "mask_33", "mask_255", "mask_256",
    "mask_257",
    # Refine's tree
    "refine_10", "refine_255", "refine_256", "refine_257", "refine_512", "refine_513", "refine_2000",
    # scale
    "kitti_scale", "frame_id_high", "kf_id_max", "seed_high",
)
# Targets no input reaches, with the reason; the CPU test checks that they are exactly the paths no scene reaches.
UNREACHED = {
    "zc_zero": "Zc == 0 exactly in CheckInliers: the depth is ((R20 x + R21 y) + R22 z) + t2 in double with R, t from EPnP and "
               "x, y, z floats; a float z moves R22 z in steps near 1e-6 while the sum must land on -t2 to the last of 53 bits, "
               "so a float point on a hypothesis' camera plane exists with probability near 1e-9 per pose, and no construction "
               "pins EPnP's t2 to a float grid",
}


@dataclass
class Scene:
    name: str
    p2d: np.ndarray          # N x 2 float32
    p3d: np.ndarray          # N x 3 float32
    octave: np.ndarray       # N int32
    kf_id: int = 1
    frame_id: int = FRAME
    seed: int = SEED
    cam: tuple = KITTI
    calls: tuple = (5, 5, 5, 5, 5, 5, 5, 5)
    paths: set = field(default_factory=set)
    junk: bool = True        # embed rejected entries between the correspondences
    targets: dict = field(default_factory=dict)  # hypothesis g -> (correspondence index, "e2_eq_max" / ...)

    @property
    def N(self):
        return len(self.p2d)

    def solver(self, sigma2=SIGMA2, log=True) -> P.Solver:
        return P.Solver(self.p2d, self.p3d, np.asarray(sigma2, F32)[self.octave], *self.cam, seed=self.seed, kf_id=self.kf_id,
                        frame_id=self.frame_id, log=log)


# ---------------------------------------------------------------------------------------------------------- geometry
def rotation(axis, angle) -> np.ndarray:
    a = np.asarray(axis, F64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * (K @ K)


def project(R, t, p3d, cam):
    """CheckInliers' (ue, ve) in double for float points (pnp_oracle.check_inliers' arithmetic)."""
    fu, fv, uc, vc = (float(F32(c)) for c in cam)
    p3 = np.asarray(p3d, F32).astype(F64)
    x, y, z = p3[:, 0], p3[:, 1], p3[:, 2]
    R = np.asarray(R, F64)
    t = np.asarray(t, F64)
    with np.errstate(all="ignore"):
        Xc = (R[0][0] * x + R[0][1] * y + R[0][2] * z + t[0]).astype(F32).astype(F64)
        Yc = (R[1][0] * x + R[1][1] * y + R[1][2] * z + t[1]).astype(F32).astype(F64)
        iz = (1.0 / (R[2][0] * x + R[2][1] * y + R[2][2] * z + t[2])).astype(F32).astype(F64)
        return uc + fu * Xc * iz, vc + fv * Yc * iz


def error2(R, t, p3d, p2d, cam):
    ue, ve = project(R, t, p3d, cam)
    p2 = np.asarray(p2d, F32).astype(F64)
    with np.errstate(all="ignore"):
        dx = (p2[:, 0] - ue).astype(F32)
        dy = (p2[:, 1] - ve).astype(F32)
        return dx * dx + dy * dy


def world_points(rng, n, R, C, depth=(6, 40), cam=KITTI):
    """n float points seen by the camera [R | -R C] at random pixels of a 1241 x 376 image and depths in `depth`."""
    fx, fy, cx, cy = cam
    u, v = rng.uniform(0, 1241, n), rng.uniform(0, 376, n)
    z = rng.uniform(*depth, n)
    Pc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    R = np.asarray(R, F64)
    return (Pc @ R + np.asarray(C, F64)).astype(F32)


def observe(R, C, X, cam, err=None):
    """Observations of X from [R | -R C]: the exact projection rounded to float, plus `err` pixels (n x 2)."""
    R = np.asarray(R, F64)
    ue, ve = project(R, -R @ np.asarray(C, F64), X, cam)
    p = np.stack([ue, ve], 1)
    if err is not None:
        p = p + err
    return p.astype(F32)


def family(rng, N, good, near, noise=0.3, R=None, C=(0.4, -0.2, 0.8), depth=(6, 40), cam=KITTI, octaves=8, radii=None):
    """N correspondences: `good` seen from the true pose with pixel noise `noise`, `near` of them moved to 0.6 .. 1.4 times
    their threshold distance (or to the given multiples `radii`), the rest far off.  Returns (p2d, p3d, octave)."""
    R = rotation((0.3, 1, 0.2), 0.4) if R is None else R
    X = world_points(rng, N, R, C, depth, cam)
    octave = rng.integers(0, octaves, N).astype(np.int32)
    err = rng.normal(size=(N, 2)) * noise
    idx = rng.permutation(N)
    nr = idx[:near]
    th = np.sqrt(SIGMA2[octave[nr]].astype(F64) * 5.991)
    ang = rng.uniform(0, 2 * np.pi, near)
    mult = rng.uniform(0.6, 1.4, near) if radii is None else np.asarray(radii, F64)
    err[nr] = np.stack([np.cos(ang), np.sin(ang)], 1) * (th * mult)[:, None]
    p2 = observe(R, C, X, cam, err)
    bad = idx[good:]
    p2[bad] = np.stack([rng.uniform(0, 1241, len(bad)), rng.uniform(0, 376, len(bad))], 1).astype(F32)
    return p2, X, octave


# ---------------------------------------------------------------------------------------------------------- the log
def draw_events(seed, kf_id, frame_id, g, N) -> set:
    """Whether hypothesis g's swap-remove read a position that an earlier draw had overwritten ("r"), and whether it moved a back
    slot that had been overwritten ("back") -- the two lookups of the device's draw4."""
    w = P.philox4x32_10(np.uint32(g), np.uint32(kf_id), np.uint32(frame_id & 0xFFFFFFFF), np.uint32(frame_id >> 32),
                        seed & 0xFFFFFFFF, seed >> 32)
    moved, out = set(), set()
    for i in range(P.MIN_SET):
        avail = N - i
        r = int(float(int(w[i])) / 4294967296.0 * float(avail))
        if r in moved:
            out.add("r")
        if avail - 1 in moved and avail - 1 != r:
            out.add("back")
        moved.add(r)
    return out


def run(scene: Scene, sigma2=SIGMA2):
    """The oracle over the scene's calls -> (solver, results, log)."""
    s = scene.solver(sigma2)
    res = [s.iterate(n) for n in scene.calls]
    return s, res, s.log


def hypothesis_paths(scene: Scene, s: P.Solver) -> set:
    out = set()
    for g, (idx, dbg, mask, cnt) in s.cache.items():
        out.add(f"best_{dbg.best}")
        if any(dbg.pcs_flip[1:]):
            out.add("pcs_flip")
        if any(dbg.det_flip[1:]):
            out.add("det_flip")
        out.add("b1_neg" if dbg.signs[1][0] else "b1_pos")
        out.add("b2_neg" if dbg.signs[2][0] else "b2_pos")
        out.add("b3_neg" if dbg.signs[3][0] else "b3_pos")
        if dbg.signs[2][1]:
            out.add("b2_x1_neg")
        if dbg.signs[3][1]:
            out.add("b3_x1_neg")
        ev = draw_events(scene.seed, scene.kf_id, scene.frame_id, g, s.N)
        out |= {"draw_swapped_" + e for e in ev}
        if s.N in (31, 32, 33, 255, 256, 257):
            out.add(f"mask_{s.N}")
        pts = np.asarray([s.p3d[i] for i in idx], F64)
        c = pts - pts.mean(0)
        rank = np.linalg.matrix_rank(c, tol=1e-9 * max(np.abs(c).max(), 1e-300)) if np.all(np.isfinite(c)) else 3
        if len({tuple(p) for p in pts}) == 1:
            out.add("coincident")
            if dbg.qr_early:
                out.add("qr_early")
        elif len({tuple(p) for p in pts}) < 4:
            out.add("duplicate")
        elif rank == 1:
            out.add("collinear")
        elif rank == 2:
            out.add("coplanar")
        R, t = np.asarray(dbg.R, F64), np.asarray(dbg.t, F64)
        if np.all(np.isfinite(R)):
            e2 = error2(R, t, s.p3d, s.p2d, scene.cam)
            with np.errstate(all="ignore"):
                if np.any(e2 == s.max_err):
                    out.add("e2_eq_max")
                below = np.nextafter(s.max_err, F32(0))
                if np.any((e2 == below) & mask):
                    out.add("e2_ulp_below")
                p3 = s.p3d.astype(F64)
                x, y, z = p3[:, 0], p3[:, 1], p3[:, 2]
                Zc = R[2][0] * x + R[2][1] * y + R[2][2] * z + t[2]  # CheckInliers' order
                Xc = R[0][0] * x + R[0][1] * y + R[0][2] * z + t[0]
                if np.any(Zc == 0):
                    out.add("zc_zero")
                if np.any((Zc < 0) & mask):
                    out.add("behind_camera")
                if np.any(np.abs(Xc) > float(np.finfo(F32).max)):
                    out.add("xc_overflow")
    return out


def paths_reached(scene: Scene, s: P.Solver, cap=None) -> set:
    """The paths of PATHS this run reached, read from the scene, the oracle's log and its hypothesis cache (cap: the
    extractor's capacity, by default that of EXTRACTOR)."""
    cap = capacity() if cap is None else cap
    out = hypothesis_paths(scene, s)
    N = s.N
    if N in (0, 4, 9, 10, 11, 14, 15):
        out.add(f"N_{N}")
    if N == cap:
        out.add("N_cap")
    log = s.log
    hyps = [e for e in log if e["kind"] != "call"]
    calls = [e for e in log if e["kind"] == "call"]
    failed = False
    for e in hyps:
        c, k = e["count"], e["kind"]
        if c == s.min_inl - 1:
            out.add("below_at_min")
        if c == s.min_inl and k != "below":
            out.add("at_min")
        if k in ("improve", "tie", "worse"):
            out.add(k)
        r = e.get("refine")
        if r == "failed":
            failed = True
            if e["refine_count"] == s.min_inl:
                out.add("refine_fail_at_min")
        if r == "skipped":
            out.add("refine_skipped")
        if r == "ok":
            if e["refine_count"] == s.min_inl + 1:
                out.add("refine_ok_at_min1")
            if failed and k == "improve":
                out.add("fail_then_recover")
            if e["last"]:
                out.add("ok_on_last")
        if r in ("ok", "failed") and e["refine_n"] in (10, 255, 256, 257, 512, 513, 2000):
            out.add(f"refine_{e['refine_n']}")
    for i, c in enumerate(calls):
        if c["no_more"] and N >= s.min_inl:
            out.add("no_more_pose" if c["pose"] else "no_more_none")
        start = c["end"] - c["ran"]
        if start >= s.max_its and c["ran"] == max(c["n"], 0) and c["no_more"]:
            out.add("after_max_its")
        if c["pose"] and not c["no_more"] and i + 1 < len(calls) and c["end"] < s.max_its:
            nxt = [e for e in hyps if e["call"] == i + 1]
            if nxt and nxt[0]["g"] == c["end"]:
                out.add("pose_mid_schedule")
    if np.linalg.norm(np.asarray(s.p3d, F64).mean(0)) > 300 if N else False:
        out.add("kitti_scale")
    if scene.frame_id >= 1 << 32:
        out.add("frame_id_high")
    if scene.kf_id == 0xFFFFFFFF:
        out.add("kf_id_max")
    if scene.seed >> 48:
        out.add("seed_high")
    return out


# ---------------------------------------------------------------------------------------------------------- embedding
@dataclass
class Frame:
    kps: np.ndarray          # cap + slack keypoint slots (x, y, octave set)
    keep_idx: np.ndarray     # n_keep + slack int32
    n_keep: int
    match: np.ndarray        # cap + slack int32 (candidate row)
    points: np.ndarray       # n_points + slack x 3 float32
    n_points: int
    paths: set


REJECTS = ("keep_neg", "keep_cap", "match_neg5", "match_neg1", "match_np", "match_np1", "oct_neg", "oct_nlevels", "oct_127")
FORCED = (255, 256, 511, 512)  # semantic keys whose entry is rejected: both sides of the 256-key chunk boundaries


def embed(scene: Scene, cap: int, nlevels: int, rng, junk=None) -> Frame:
    """sivo_pnp_setup_device's inputs for the scene: semantic key j's correspondences in order through an oracle/keymap.py map
    and a permuted point array, with rejected keys between them (junk), some at semantic keys 255, 256, 511 and 512.  The
    rejected entries cycle through REJECTS: the map's own rejected keep_idx (keep_neg or keep_cap by its sign), or a valid
    slot whose match is -5, -1, n_points or n_points + 1 or whose key's octave is -1, nlevels or 127.  Slack rows past cap,
    n_keep and n_points hold keys and points that would be accepted if a bound were off by one."""
    junk = scene.junk if junk is None else junk
    N = scene.N
    km = keymap(N, cap, rng, forced=FORCED, junk=junk)
    n_keep, keep = km.n_keep, km.keep
    n_points = N + 7
    perm_pts = rng.permutation(n_points)
    points = np.zeros((n_points + SLACK, 3), F32)
    points[n_points:] = [1.0, 2.0, 10.0]  # slack: a point a bound one too wide would read
    points[perm_pts[:N]] = scene.p3d
    points[perm_pts[N:]] = [3.0, -1.0, 20.0]
    p2 = np.asarray(scene.p2d, F32).reshape(N, 2)
    real = np.zeros(N, KP_DTYPE)
    real["x"], real["y"], real["octave"] = p2[:, 0], p2[:, 1], scene.octave
    kps = scatter(real, km.slots, cap, np.zeros(1, KP_DTYPE))
    kps["x"][cap:], kps["y"][cap:], kps["octave"][cap:] = 600.0, 180.0, 0  # slack: a key a bound one too wide would read
    # keep's entries past n_keep are valid slots, whose match entries are -1: a correct setup rejects them
    match = np.full(cap + SLACK, -1, np.int32)
    match[cap:] = 0
    match[km.real] = perm_pts[:N]
    free = np.setdiff1d(np.arange(cap), km.slots)
    paths = {"keep_permuted"} if cap > 1 else set()
    for r, j in enumerate(np.flatnonzero(km.src < 0)):
        kind = REJECTS[r % len(REJECTS)]
        match[j] = perm_pts[N + int(rng.integers(7))]
        if kind.startswith("keep"):
            kind = "keep_neg" if keep[j] < 0 else "keep_cap"
        else:
            keep[j] = s = free[r]
            kps[s]["x"], kps[s]["y"], kps[s]["octave"] = 600.0, 180.0, 0
            if kind.startswith("match"):
                match[j] = {"match_neg5": -5, "match_neg1": -1, "match_np": n_points, "match_np1": n_points + 1}[kind]
            else:
                kps[s]["octave"] = {"oct_neg": -1, "oct_nlevels": nlevels, "oct_127": 127}[kind]
        paths.add(kind)
        if j in FORCED:
            paths.add(f"reject_{j}")
    return Frame(kps, keep, n_keep, match, points, n_points, paths)


def frame_correspondences(fr: Frame, cap, sigma2):
    """pnp_oracle.correspondences over an embedded frame."""
    return P.correspondences(fr.kps, fr.match, min(max(fr.n_keep, 0), cap), fr.points[:fr.n_points], sigma2, keep_idx=fr.keep_idx,
                             cap=cap)


# ---------------------------------------------------------------------------------------------------------- placed scenes
def exact_scene(name, N, n_good, seed, paths, calls=(5, 5), R=None, C=(0.4, -0.2, 0.8), depth=(6, 40), **kw):
    """n_good exact observations (noise-free) and N - n_good far off."""
    rng = np.random.default_rng(seed)
    p2, X, oc = family(rng, N, n_good, 0, noise=0.0, R=R, C=C, depth=depth)
    return Scene(name, p2, X, oc, calls=calls, paths=set(paths), **kw)


def boundary_scene(name, target, g=0, N=30, seed=5):
    """Exact observations; correspondence i (outside hypothesis g's minimal set) is moved along x until error2 under hypothesis
    g's pose is exactly maxError (target "e2_eq_max") or the float below it ("e2_ulp_below")."""
    rng = np.random.default_rng(seed)
    p2, X, oc = family(rng, N, N, 0, noise=0.0)
    sc = Scene(name, p2, X, oc, calls=(5,), paths={target})
    s = sc.solver(log=False)
    idx, dbg, _, _ = s.hypothesis(g)
    R, t = np.asarray(dbg.R, F64), np.asarray(dbg.t, F64)
    want = s.max_err if target == "e2_eq_max" else np.nextafter(s.max_err, F32(0))
    steps = np.arange(-60, 61, dtype=np.int64)
    for i in [i for i in range(N) if i not in idx]:
        for trial in range(1500):  # nudge the point through floats until an observation on its row lands on the target
            ue, ve = project(R, t, X[i:i + 1], sc.cam)
            y = F32(ve[0])
            base = F32(ue[0] + math.sqrt(float(want[i])))
            xs = (np.array([base], F32).view(np.int32).astype(np.int64) + steps).astype(np.int32).view(F32)
            e2 = error2(R, t, np.repeat(X[i:i + 1], len(xs), 0), np.stack([xs, np.full(len(xs), y, F32)], 1), sc.cam)
            hit = np.nonzero(e2 == want[i])[0]
            if len(hit):
                p2[i] = [xs[hit[0]], y]
                sc.p2d = p2
                sc.targets[g] = (i, target)
                return sc
            X[i, 0] = np.nextafter(X[i, 0], F32(np.inf))
    raise RuntimeError(f"no float observation reaches {target}")


def degenerate_scene(name, kind, seed=11, N=24, g=0):
    """Exact observations; hypothesis g's minimal set made coplanar (z = 20 exactly), collinear, four copies of one point, or
    with one point twice (its observation too)."""
    rng = np.random.default_rng(seed)
    p2, X, oc = family(rng, N, N, 0, noise=0.0, R=np.eye(3), C=(0.0, 0.0, 0.0))
    sc = Scene(name, p2, X, oc, calls=(5, 5), paths={kind})
    idx = P.draws(sc.seed, sc.kf_id, sc.frame_id, g, N)
    if kind == "coplanar":
        X[idx, 2] = 20.0
    elif kind == "collinear":
        X[idx] = (np.array([1.0, -0.5, 12.0]) + np.outer([0.0, 1.0, 2.5, 4.0], [0.5, 0.25, 2.0])).astype(F32)
    elif kind == "coincident":
        X[idx] = X[idx[0]]
        p2[idx] = p2[idx[0]]
    else:
        X[idx[1]] = X[idx[0]]
        p2[idx[1]] = p2[idx[0]]
    sc.p2d, sc.p3d = p2, X
    if kind in ("coplanar", "collinear"):
        sc.p2d[idx] = observe(np.eye(3), (0, 0, 0), X[idx], sc.cam)
    return sc


def extremes_scene(name, seed=13, N=40):
    """Exact observations from a camera turned 45 degrees about its axis, plus points behind it observed at their projection,
    and points at 3e38 whose camera x (about 4.2e38) overflows float."""
    rng = np.random.default_rng(seed)
    Rz = rotation((0, 0, 1), math.pi / 4)
    p2, X, oc = family(rng, N, N, 0, noise=0.0, R=Rz, C=(0.0, 0.0, 0.0))
    X[:4, 2] = -X[:4, 2]  # behind: (x, y, -z) projects to the mirror image of (x, y, z) about the principal point
    p2[:4] = observe(Rz, (0, 0, 0), X[:4], KITTI)
    X[4:6] = [[3e38, -3e38, 20.0], [-3e38, 3e38, 25.0]]
    p2[4:6] = [[600.0, 180.0], [10.0, 10.0]]
    return Scene(name, p2, X, oc, calls=(5, 5), paths={"behind_camera", "xc_overflow"})


def kitti_scene(name, rng_seed, dist, angle, N=60, good=40, **kw):
    """The camera 350 m from the world origin (or `dist`), rotated by `angle` about a random axis, points 6 - 40 m ahead."""
    rng = np.random.default_rng(rng_seed)
    R = rotation(rng.standard_normal(3), angle)
    C = rng.standard_normal(3)
    C = C / np.linalg.norm(C) * dist
    p2, X, oc = family(rng, N, good, 4, noise=0.3, R=R, C=C)
    return Scene(name, p2, X, oc, **kw)


# ---------------------------------------------------------------------------------------------------------- searched scenes
def searched(name, kf_id):
    """The searched scenes, by name, at a given kf_id (their family is fixed; SEARCHED records the kf_id that reaches the
    paths)."""
    mk = SEARCH_FAMILIES[name]
    sc = mk(kf_id)
    sc.name = name
    return sc


def _fam(seed, N, good, near, noise, calls, paths, octaves=8, radii=None):
    def make(kf_id):
        rng = np.random.default_rng(seed)
        p2, X, oc = family(rng, N, good, near, noise=noise, octaves=octaves, radii=radii)
        return Scene("", p2, X, oc, kf_id=kf_id, calls=calls, paths=set(paths))
    return make


SEARCH_FAMILIES = {
    # counts straddling minInliers = 10 at N = 20: a count of 9, a count of 10 whose Refine fails at 10 (one near point inside
    # its threshold, two outside), no pose, then no_more with the best pose and calls after maxIts
    "at_min_fail": _fam(31, 20, 12, 3, 0.0, (5, 5, 5, 3, 0, -1),
                        {"below_at_min", "at_min", "refine_fail_at_min", "no_more_pose", "after_max_its"}, radii=(0.7, 1.2, 1.3)),
    # a failed Refine, a tie on a different set (skipped), a worse count, then an improvement whose Refine succeeds
    "tie_worse_recover": _fam(33, 22, 15, 6, 0.5, (5, 5, 5, 5),
                              {"refine_fail_at_min", "tie", "worse", "refine_skipped", "fail_then_recover"}),
    # Refine succeeding at exactly minInliers + 1
    "ok_at_min1": _fam(23, 20, 11, 2, 0.2, (5, 5, 5), {"refine_ok_at_min1"}),
    # a pose on the last hypothesis of a call (maxIts = 4 at N = 11, so the first call runs 5)
    "ok_on_last": _fam(24, 11, 11, 1, 0.2, (5, 5, 5), {"ok_on_last"}),
    # a pose mid-schedule, the next call continuing at g = mnIterations
    "mid_schedule": _fam(30, 24, 18, 4, 0.3, (5, 5, 5, 5), {"pose_mid_schedule", "improve"}),
    # no hypothesis reaches minInliers: no_more with no pose
    "no_pose": _fam(26, 30, 8, 4, 0.3, (5, 5, 40), {"no_more_none", "after_max_its"}),
}
SEARCHED = {"at_min_fail": 5, "tie_worse_recover": 5, "ok_at_min1": 1, "ok_on_last": 4, "mid_schedule": 1, "no_pose": 1}


def constructed_scenes():
    out = [searched(name, kf) for name, kf in SEARCHED.items()]
    for N in (0, 4, 9, 10, 11, 14, 15):
        out.append(exact_scene(f"N_{N}", N, N, 40 + N, {f"N_{N}"} | ({"refine_10"} if N == 10 else set())))
    for N in (31, 32, 33, 255, 256, 257):
        out.append(exact_scene(f"mask_{N}", N, N - 8, 60 + N, {f"mask_{N}"}))
    for n, k in ((255, 0), (256, 0), (257, 1), (512, 0), (513, 0), (2000, 0)):
        out.append(exact_scene(f"refine_{n}", n + 40, n, 80 + n + k, {f"refine_{n}"}, calls=(5,)))
    cap = capacity()
    out.append(exact_scene("N_cap", cap, cap - 50, 7, {"N_cap"}, calls=(5,), junk=False))
    out += [boundary_scene("e2_eq_max", "e2_eq_max"), boundary_scene("e2_ulp_below", "e2_ulp_below", seed=6)]
    out += [degenerate_scene(k, k, seed=11 + i) for i, k in enumerate(("coplanar", "collinear", "coincident", "duplicate"))]
    out.append(extremes_scene("extremes"))
    out.append(kitti_scene("kitti_350m", 90, 350.0, math.pi - 0.01, calls=(5, 5, 5), paths={"kitti_scale"}))
    out.append(kitti_scene("kitti_ids", 91, 350.0, 2.5, calls=(5, 5, 5), frame_id=(1 << 40) + 12345, kf_id=0xFFFFFFFF,
                           seed=0xFEDC_BA98_7654_3210, paths={"kitti_scale", "frame_id_high", "kf_id_max", "seed_high"}))
    return out


def find_searched(name, start=1, tries=400):
    """The first kf_id >= start whose oracle run takes the family's named paths (used to fill in SEARCHED)."""
    for kf in range(start, start + tries):
        sc = searched(name, kf)
        s, res, _ = run(sc)
        if sc.paths <= paths_reached(sc, s):
            return kf
    return None
