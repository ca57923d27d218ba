"""-m gpu: Relocalization's PnP RANSAC (k_pnp_setup / k_pnp_hyp / k_pnp_decide) on the constructed candidates of
oracle/pnp_scene.py, bit for bit against oracle/pnp_oracle.py with no tolerance: every call's Tcw bits, inlier row, counts and
flags, the state after every call (refine_failed included), the targeted hypotheses through sivo_dbg_pnp_hypotheses and Refine's
intermediates through sivo_dbg_pnp_compute_pose.  Every setup passes a permuted semantic-key map with rejected keys between the
correspondences, and the key, keep_idx and point buffers carry slack rows that a bound one too wide would accept.  Also: the
n_iterations schedule, the handle's lifetime, inputs overwritten on the stream right after setup, many candidates, the error
codes, a 4-level 1.5x extractor and 200 seeded fuzz scenes."""
import ctypes as C

import numpy as np
import pytest
import torch

from frame_support import extractor, i64, same_bits, sentinel, upload
from oracle import bow_oracle as BO
from oracle import bow_scene as BS
from oracle import pnp_bounds as PB
from oracle import pnp_oracle as P
from oracle import pnp_scene as S
from oracle.keymap import SLACK, keymap
from oracle.orb_oracle import ExtractorParams, Tables
from sivo_b200 import _lib as L
from sivo_b200 import reloc
from sivo_b200.bow import keyframe_keys, search_by_bow_device
from sivo_b200.track import map_points

pytestmark = pytest.mark.gpu
SCENES = {sc.name: sc for sc in S.constructed_scenes()}
class Setup:
    """One embedded scene as device buffers: n_kf candidates sharing the frame (the same match row), kf_ids as given."""

    def __init__(self, left, sc, kf_ids, rng_seed=0, n_matches=None, n_keep=None, junk=None):
        self.left, self.sc, self.cap = left, sc, left.capacity()
        self.fr = S.embed(sc, self.cap, left.nlevels, np.random.default_rng(rng_seed), junk=junk)
        self.kf_ids = np.asarray(kf_ids, np.int64) & 0xFFFFFFFF
        n_kf = len(self.kf_ids)
        self.n_keep = self.fr.n_keep if n_keep is None else n_keep
        rows = np.tile(self.fr.match[:self.cap], (n_kf, 1))
        self.rows = rows
        self.n_matches = np.full(n_kf, (self.fr.match[:self.fr.n_keep] >= 0).sum(), np.int64) if n_matches is None else \
            np.asarray(n_matches, np.int64)
        pts = map_points(np.zeros((len(self.fr.points), 32), np.uint8), self.fr.points, np.zeros_like(self.fr.points), 0.0, 1e9)
        self.t = dict(kps=upload(self.fr.kps), keep=torch.from_numpy(self.fr.keep_idx.copy()).cuda(), nk=i64(self.n_keep),
                      match=torch.from_numpy(np.concatenate([rows.reshape(-1), np.zeros(SLACK, np.int32)])).cuda(),
                      nm=torch.from_numpy(self.n_matches.copy()).cuda(), pts=upload(pts))

    def call(self, solver, stream=0):
        t = self.t
        solver.setup_device(t["kps"].data_ptr(), t["keep"].data_ptr(), t["nk"].data_ptr(), t["match"].data_ptr(), t["nm"].data_ptr(),
                            t["pts"].data_ptr(), self.fr.n_points, self.kf_ids.astype(np.uint32), self.sc.frame_id, *self.sc.cam,
                            stream=stream)

    def oracles(self):
        sigma2 = self.left._s2
        p2, p3, s2, key = P.correspondences(self.fr.kps, self.fr.match, min(max(self.n_keep, 0), self.cap),
                                            self.fr.points[:self.fr.n_points], sigma2, keep_idx=self.fr.keep_idx, cap=self.cap)
        out = []
        for k, kf in enumerate(self.kf_ids):
            dead = self.n_keep < 0 or self.n_matches[k] < 0
            s = P.Solver(p2, p3, s2, *self.sc.cam, seed=self.sc.seed, kf_id=int(kf), frame_id=self.sc.frame_id, dead=dead, log=True)
            out.append((s, key))
        return out


class Outputs:
    def __init__(self, n_kf, cap):
        self.Tcw = torch.full((n_kf, 12), float("nan"), dtype=torch.float32, device="cuda")
        self.has = torch.full((n_kf,), -7, dtype=torch.int32, device="cuda")
        self.nm = torch.full((n_kf,), -7, dtype=torch.int32, device="cuda")
        self.ni = torch.full((n_kf,), -7, dtype=torch.int32, device="cuda")
        self.row = torch.full((n_kf, cap), -9, dtype=torch.int32, device="cuda")

    def ptrs(self):
        return self.Tcw.data_ptr(), self.has.data_ptr(), self.nm.data_ptr(), self.row.data_ptr(), self.ni.data_ptr()

    def host(self):
        return [x.cpu().numpy() for x in (self.Tcw, self.has, self.nm, self.ni, self.row)]


def check_state(solver, oracles):
    st = solver.state()
    for k, (s, _) in enumerate(oracles):
        assert st["dead"][k] == int(s.dead), k
        if s.dead:
            assert st["N"][k] == 0
            continue
        assert (st["N"][k], st["min_inliers"][k], st["max_its"][k]) == (s.N, s.min_inl, s.max_its), k
        assert (st["iterations"][k], st["best"][k], st["refine_failed"][k]) == (s.iterations, s.best, int(s.refine_failed)), k
        assert st["eps"][k] == s.eps or s.N == 0


def iterate_and_compare(solver, setup, oracles, out, n, active, stream=0):
    before = out.host()
    solver.iterate_device(n, np.asarray(active, np.uint8), *out.ptrs(), stream=stream)
    torch.cuda.synchronize()
    T, hp, nm, ni, row = out.host()
    results = {}
    for k, (s, key) in enumerate(oracles):
        if not active[k]:  # neither run nor written
            assert all(np.array_equal(a[k], b[k], equal_nan=a.dtype.kind == "f") for a, b in zip(out.host(), before)), k
            continue
        res = s.iterate(n)
        results[k] = res
        assert (bool(hp[k]), bool(nm[k]), int(ni[k])) == (res.Tcw is not None, res.no_more, res.n_inliers), (k, n)
        want = np.full(setup.cap, -1, np.int32)
        want[key[res.inliers]] = setup.rows[k][key[res.inliers]]
        assert np.array_equal(row[k], want), k
        if res.Tcw is not None:
            assert np.array_equal(T[k].view(np.uint32), res.Tcw.reshape(12).view(np.uint32)), k
    check_state(solver, oracles)
    return results


def check_hypotheses(solver, k, s, gs):
    """k_pnp_hyp for hypotheses gs (contiguous runs) against the oracle's hypotheses."""
    first, last = min(gs), max(gs)
    got = solver.hypotheses(k, first, last - first + 1)
    for g in gs:
        idx, dbg, mask, cnt = s.hypothesis(g)
        h = g - first
        assert list(got["draws"][h]) == idx, g
        assert np.array_equal(got["R"][h], np.asarray(dbg.R, np.float64), equal_nan=True), g
        assert np.array_equal(got["t"][h], np.asarray(dbg.t, np.float64), equal_nan=True), g
        assert got["counts"][h] == cnt and np.array_equal(got["masks"][h][:s.N], mask), g


def check_refine(s, sc):
    """Refine's kernel path on the best set, every intermediate against compute_pose(tree=True)."""
    sel = np.nonzero(s.best_mask)[0]
    if len(sel) == 0:
        return
    compare_pose(s.p3d[sel], s.p2d[sel], s.max_err[sel], sc.cam)


def compare_pose(p3, p2, err, cam):
    alphas, mask, cnt, d = reloc.compute_pose(p3, p2, err, *cam)
    fu, fv, uc, vc = (float(np.float32(c)) for c in cam)
    o = P.compute_pose(p3.astype(np.float64).tolist(), p2.astype(np.float64).tolist(), fu, fv, uc, vc, tree=True)
    same = lambda a, b: same_bits(np.ravel(a), np.ravel(b))
    assert same(alphas, o.alphas) and same(d.cws, o.cws) and same(d.d, o.d) and same(d.ut, o.ut)
    assert same(d.l_6x10, o.l_6x10) and same(d.rho, o.rho)
    assert same(d.betas, [o.betas[b][i] for b in (1, 2, 3) for i in range(4)]) and same(d.rep_errors, o.rep_errors[1:])
    assert d.best == o.best and same(d.R, o.R) and same(d.t, o.t)
    om, oc = P.check_inliers(o.R, o.t, p3, p2, fu, fv, uc, vc, err)
    assert cnt == oc and np.array_equal(mask, om)
    return o


def run_scene(left, sc, calls=None, n_kf=1, active=None, hyps=(), stream=0, rng_seed=0):
    setup = Setup(left, sc, [sc.kf_id + 7 * k for k in range(n_kf)], rng_seed)
    solver = reloc.PnpSolver(left, n_kf, sc.seed)
    try:
        setup.call(solver, stream)
        oracles = setup.oracles()
        assert np.array_equal(oracles[0][0].p2d, sc.p2d) and np.array_equal(oracles[0][0].p3d, sc.p3d)
        check_state(solver, oracles)
        if hyps:
            check_hypotheses(solver, 0, oracles[0][0], hyps)
        out = Outputs(n_kf, setup.cap)
        act = np.ones(n_kf, bool) if active is None else None
        for i, n in enumerate(sc.calls if calls is None else calls):
            a = act if act is not None else np.asarray(active(i), bool)
            iterate_and_compare(solver, setup, oracles, out, n, a)
        return oracles
    finally:
        solver.close()


def test_the_extractor_tables_are_the_scenes():
    assert np.array_equal(extractor()._s2, S.SIGMA2) and extractor().capacity() == S.capacity()


@pytest.mark.parametrize("name", list(SCENES))
def test_constructed_scene(name):
    sc = SCENES[name]
    left = extractor()
    hyps = sorted(set(sc.targets) | set(range(min(8, P.ransac_parameters(sc.N)[2])))) if 10 <= sc.N <= 600 else ()
    if sc.N < P.ransac_parameters(sc.N)[0]:
        hyps = ()
    oracles = run_scene(left, sc, hyps=tuple(hyps))
    s = oracles[0][0]
    assert sc.paths <= S.paths_reached(sc, s, cap=left.capacity())
    if name.startswith("refine_") or name in ("at_min_fail", "tie_worse_recover", "ok_at_min1"):
        check_refine(s, sc)


def test_draw_swap_remove_lookups():
    """The draws at small N, where the swap-remove reads overwritten positions and moves overwritten back slots."""
    events = set()
    for N in (4, 5, 6, 7, 8, 11, 33):
        got = reloc.draws(S.SEED, 1, S.FRAME, 0, 200, N)
        for g in range(200):
            assert list(got[g]) == P.draws(S.SEED, 1, S.FRAME, g, N), (N, g)
            events |= S.draw_events(S.SEED, 1, S.FRAME, g, N)
    assert events == {"r", "back"}


@pytest.mark.parametrize("kind", ["coincident", "duplicate", "collinear", "coplanar"])
@pytest.mark.parametrize("n", [4, 6, 11])
def test_degenerate_sets_through_refines_path(kind, n):
    """Every intermediate of compute_pose on degenerate sets: coincident points give a zero control-point basis (every singular
    value below the zero threshold) and qr_solve's early return in every Gauss-Newton step."""
    rng = np.random.default_rng(n)
    X = S.world_points(rng, n, np.eye(3), (0, 0, 0))
    if kind == "coincident":
        X[:] = X[0]
    elif kind == "duplicate":
        X[1] = X[0]
    elif kind == "collinear":
        X[:] = (np.array([1.0, -0.5, 12.0]) + np.outer(np.arange(n) * 0.5, [0.5, 0.25, 2.0])).astype(np.float32)
    else:
        X[:, 2] = 20.0
    p2 = S.observe(np.eye(3), (0, 0, 0), X, S.KITTI)
    o = compare_pose(X, p2, np.full(n, 5.991, np.float32), S.KITTI)
    if kind == "coincident":
        assert o.qr_early > 0 and o.alphas[0] == [1.0, 0.0, 0.0, 0.0]


# ---------------------------------------------------------------------------------------------------------- schedule
@pytest.mark.parametrize("n", [-1, 0, 1, 5, 35, 36, 100])
def test_n_iterations(n):
    for name in ("at_min_fail", "no_pose", "tie_worse_recover"):
        run_scene(extractor(), SCENES[name], calls=(n, n, n))


def test_mixed_call_lengths_on_one_handle():
    run_scene(extractor(), SCENES["no_pose"], calls=(1, 0, 36, -1, 5, 100, 2))
    run_scene(extractor(), SCENES["tie_worse_recover"], calls=(2, 1, 3, 0, 40, 5))


# ---------------------------------------------------------------------------------------------------------- handle lifetime
def test_resetup_after_pose_and_no_more_then_no_candidates():
    left = extractor()
    cap = left.capacity()
    solver = reloc.PnpSolver(left, 4, S.SEED)
    try:
        # 4 candidates of the recovering scene until a pose, then 2 of the no-pose scene (a new frame id) until no_more
        for sc, n_kf, rounds in ((SCENES["tie_worse_recover"], 4, 4), (SCENES["no_pose"], 2, 3), (SCENES["ok_on_last"], 3, 3)):
            setup = Setup(left, sc, [sc.kf_id + 7 * k for k in range(n_kf)])
            setup.call(solver)
            oracles = setup.oracles()
            check_state(solver, oracles)
            out = Outputs(n_kf, cap)
            for _ in range(rounds):
                iterate_and_compare(solver, setup, oracles, out, 5, np.ones(n_kf, bool))
        # n_kf = 0: setup enqueues nothing, the iterate has no candidates and writes nothing
        t = Setup(left, SCENES["N_15"], [1]).t
        solver.setup_device(t["kps"].data_ptr(), t["keep"].data_ptr(), t["nk"].data_ptr(), t["match"].data_ptr(), t["nm"].data_ptr(),
                            t["pts"].data_ptr(), 1, [], S.FRAME + 1, *S.KITTI)
        out = Outputs(1, cap)
        before = out.host()
        solver.iterate_device(5, np.zeros(0, np.uint8), *out.ptrs())
        torch.cuda.synchronize()
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(out.host(), before))
        assert solver.state()["N"].size == 0
    finally:
        solver.close()


def test_candidate_inactive_for_a_call_then_resumed():
    pattern = [[1, 0, 1], [0, 1, 1], [1, 1, 0], [1, 1, 1], [1, 0, 1], [1, 1, 1]]
    run_scene(extractor(), SCENES["tie_worse_recover"], calls=(5,) * 6, n_kf=3, active=lambda i: pattern[i])


@pytest.mark.parametrize("n_kf", [64, 256])
def test_many_candidates_with_sparse_active_masks(n_kf):
    rng = np.random.default_rng(n_kf)
    masks = [rng.random(n_kf) < p for p in (0.3, 0.7, 0.5, 1.0)]
    run_scene(extractor(), SCENES["at_min_fail"], calls=(5, 5, 5, 5), n_kf=n_kf, active=lambda i: masks[i])


def test_inputs_overwritten_on_the_stream_right_after_setup():
    """Setup on a user stream; on the same stream, with no host synchronisation, every input buffer is overwritten before the
    iterate calls: the results are the oracle's on the original inputs."""
    left = extractor()
    sc = SCENES["tie_worse_recover"]
    setup = Setup(left, sc, [sc.kf_id, sc.kf_id + 7])
    solver = reloc.PnpSolver(left, 2, sc.seed)
    stream = torch.cuda.Stream()
    try:
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            setup.call(solver, stream.cuda_stream)
            for k, t in setup.t.items():
                if k == "nk" or k == "nm":
                    t.fill_(3)
                elif t.dtype == torch.uint8:
                    t.fill_(0x41)
                else:
                    t.fill_(1)
        oracles = setup.oracles()
        out = Outputs(2, setup.cap)
        for _ in range(4):
            iterate_and_compare(solver, setup, oracles, out, 5, np.ones(2, bool), stream=stream.cuda_stream)
    finally:
        solver.close()


# ---------------------------------------------------------------------------------------------------------- setup edges
@pytest.mark.parametrize("n_keep,n_matches", [(0, None), (-1, None), (-(1 << 40), None), ("cap+", None), (None, (-1, 5, -7))])
def test_counts_outside_the_range(n_keep, n_matches):
    left = extractor()
    sc = SCENES["ok_at_min1"]
    cap = left.capacity()
    nk = cap + 9 if n_keep == "cap+" else n_keep
    n_kf = 3
    setup = Setup(left, sc, [1, 2, 3], n_keep=nk, n_matches=n_matches)
    solver = reloc.PnpSolver(left, n_kf, sc.seed)
    try:
        setup.call(solver)
        oracles = setup.oracles()
        check_state(solver, oracles)
        out = Outputs(n_kf, cap)
        for _ in range(3):
            iterate_and_compare(solver, setup, oracles, out, 5, np.ones(n_kf, bool))
    finally:
        solver.close()


def test_no_points():
    """n_points = 0 with a NULL point array: every match entry is out of range, N = 0."""
    left = extractor()
    sc = SCENES["N_15"]
    setup = Setup(left, sc, [1])
    solver = reloc.PnpSolver(left, 1, sc.seed)
    t = setup.t
    try:
        solver.setup_device(t["kps"].data_ptr(), t["keep"].data_ptr(), t["nk"].data_ptr(), t["match"].data_ptr(), t["nm"].data_ptr(), 0,
                            0, [1], sc.frame_id, *sc.cam)
        st = solver.state()
        assert st["N"][0] == 0 and st["dead"][0] == 0
        out = Outputs(1, setup.cap)
        solver.iterate_device(5, np.ones(1, np.uint8), *out.ptrs())
        T, hp, nm, ni, row = out.host()
        assert hp[0] == 0 and nm[0] == 1 and ni[0] == 0 and (row[0] == -1).all()
    finally:
        solver.close()


def test_four_level_extractor():
    """4 levels at scale 1.5: the sigma2 table and the nlevels rejection (octave 4 among the rejected keys) differ from the
    default.  The scenes are re-octaved (octave % 4), so their thresholds change and the paths they were built for are not
    claimed here: this checks bit equality with the oracle on the 4-level tables, call by call."""
    left = extractor(2000, 1.5, 4)
    assert np.array_equal(left._s2, Tables(ExtractorParams(nfeatures=2000, scale_factor=1.5, nlevels=4)).sigma2)
    for name in ("at_min_fail", "tie_worse_recover", "refine_257", "mask_33"):
        sc = SCENES[name]
        sc4 = S.Scene(name, sc.p2d, sc.p3d, sc.octave % 4, kf_id=sc.kf_id, calls=sc.calls)
        run_scene(left, sc4)


# ---------------------------------------------------------------------------------------------------------- error codes
def test_error_codes():
    lib, left = L.lib(), extractor()
    h = C.c_void_p()
    for m in (0, 257):
        assert lib.sivo_pnp_create(left._h, m, C.c_uint64(1), C.byref(h)) == L.EINVAL
    assert lib.sivo_pnp_create(None, 4, C.c_uint64(1), C.byref(h)) == L.EINVAL
    assert lib.sivo_pnp_create(left._h, 4, C.c_uint64(1), None) == L.EINVAL
    solver = reloc.PnpSolver(left, 2, 1)
    setup = Setup(left, SCENES["N_15"], [1, 2])
    t = setup.t
    p = {k: v.data_ptr() for k, v in t.items()}
    ids = np.array([1, 2], np.uint32)
    vp = C.c_void_p

    def setup_rc(kps=p["kps"], keep=p["keep"], nk=p["nk"], match=p["match"], nm=p["nm"], pts=p["pts"], n_points=8, kf=ids, n_kf=2,
                 cam=S.KITTI, handle=None):
        kfp = kf.ctypes.data_as(vp) if kf is not None else None
        return lib.sivo_pnp_setup_device(solver._h if handle is None else handle, vp(kps), vp(keep), vp(nk), vp(match), vp(nm), vp(pts),
                                         n_points, kfp, n_kf, C.c_uint64(1), *(C.c_float(c) for c in cam), None)
    try:
        assert setup_rc() == L.OK
        for kw in (dict(kps=0), dict(nk=0), dict(match=0), dict(nm=0), dict(pts=0), dict(n_kf=3), dict(n_kf=-1), dict(n_points=-1),
                   dict(kf=None), dict(cam=(np.inf, 1.0, 1.0, 1.0)), dict(cam=(1.0, 1.0, np.nan, 1.0)), dict(handle=vp(0))):
            if "handle" in kw:
                rc = lib.sivo_pnp_setup_device(None, vp(p["kps"]), None, vp(p["nk"]), vp(p["match"]), vp(p["nm"]), vp(p["pts"]), 8,
                                               ids.ctypes.data_as(vp), 2, C.c_uint64(1), *(C.c_float(c) for c in S.KITTI), None)
            else:
                rc = setup_rc(**kw)
            assert rc == L.EINVAL, kw
        assert setup_rc() == L.OK
        out = Outputs(2, setup.cap)
        ptrs = list(out.ptrs())
        act = np.ones(2, np.uint8)
        for i in range(5):
            q = list(ptrs)
            q[i] = 0
            assert lib.sivo_pnp_iterate_device(solver._h, 5, act.ctypes.data_as(vp), *(vp(x) for x in q), None) == L.EINVAL
        assert lib.sivo_pnp_iterate_device(solver._h, 5, None, *(vp(x) for x in ptrs), None) == L.EINVAL
        assert lib.sivo_pnp_iterate_device(None, 5, act.ctypes.data_as(vp), *(vp(x) for x in ptrs), None) == L.EINVAL
        buf = np.zeros(64, np.int64)
        assert lib.sivo_dbg_pnp_state(None, buf.ctypes.data_as(vp), None) == L.EINVAL
        assert lib.sivo_dbg_pnp_state(solver._h, None, None) == L.EINVAL
        d = buf.ctypes.data_as(vp)
        assert lib.sivo_dbg_pnp_hypotheses(solver._h, 2, 0, 1, d, d, d, d) == L.EINVAL  # candidate outside the setup
        assert lib.sivo_dbg_pnp_hypotheses(solver._h, 0, -1, 1, d, d, d, d) == L.EINVAL
        assert lib.sivo_dbg_pnp_hypotheses(solver._h, 0, 0, 0, d, d, d, d) == L.EINVAL
        assert lib.sivo_dbg_pnp_hypotheses(solver._h, 0, 0, 1, None, d, d, d) == L.EINVAL
        assert lib.sivo_dbg_pnp_draws(0, C.c_uint64(1), C.c_uint32(1), C.c_uint64(1), 0, 1, 3, d) == L.EINVAL  # N < 4
        assert lib.sivo_dbg_pnp_draws(0, C.c_uint64(1), C.c_uint32(1), C.c_uint64(1), -1, 1, 8, d) == L.EINVAL
        assert lib.sivo_dbg_pnp_draws(0, C.c_uint64(1), C.c_uint32(1), C.c_uint64(1), 0, 1, 8, None) == L.EINVAL
        f = np.zeros(12, np.float32).ctypes.data_as(vp)
        dbg = reloc.PoseDebug()
        assert lib.sivo_dbg_pnp_compute_pose(0, f, f, f, 0, C.c_float(1), C.c_float(1), C.c_float(0), C.c_float(0), None, None, None,
                                             C.byref(dbg)) == L.EINVAL
        assert lib.sivo_dbg_pnp_compute_pose(0, None, f, f, 4, C.c_float(1), C.c_float(1), C.c_float(0), C.c_float(0), None, None, None,
                                             C.byref(dbg)) == L.EINVAL
        assert lib.sivo_dbg_pnp_compute_pose(0, f, f, f, 4, C.c_float(1), C.c_float(1), C.c_float(0), C.c_float(0), None, None, None,
                                             None) == L.EINVAL
    finally:
        solver.close()


# ---------------------------------------------------------------------------------------------------------- fuzz
@pytest.mark.parametrize("seed", range(200))
def test_fuzz(seed):
    rng = np.random.default_rng(50_000 + seed)
    N = int(rng.choice([10, 11, 12, 14, 15, 20, 22, 31, 32, 33, 60, 150, 300])) if seed % 3 else int(rng.integers(4, 120))
    good = int(rng.integers(0, N + 1))
    near = int(rng.integers(0, good + 1))
    p2, X, oc = S.family(rng, N, good, near, noise=float(rng.uniform(0, 1.0)))
    calls = tuple(int(x) for x in rng.choice([-1, 0, 1, 2, 5, 5, 5, 35, 36], int(rng.integers(2, 6))))
    sc = S.Scene(f"fuzz_{seed}", p2, X, oc, kf_id=int(rng.integers(0, 1 << 32)), frame_id=int(rng.integers(0, 1 << 63)),
                 seed=int(rng.integers(0, 1 << 63)), calls=calls, junk=bool(seed % 2))
    n_kf = int(rng.integers(1, 5))
    masks = [rng.random(n_kf) < 0.8 for _ in calls]
    run_scene(extractor(), sc, n_kf=n_kf, active=lambda i: masks[i], rng_seed=seed)


# ---------------------------------------------------------------------------------------------------------- SearchByBoW's rows
class _Rows:
    def __init__(self, cap, rows):
        self.cap, self.rows = cap, rows


def test_a_row_from_search_by_bow():
    """sivo_search_by_bow_device on an oracle/keymap.py semantic-key map (rejected entries between the keys), then its own keep_idx,
    n_keep, match and n_matches buffers passed unchanged to sivo_pnp_setup_device; the points placed so that most matched
    (key, point) pairs agree with one pose.  Against bow_oracle.search_by_bow followed by pnp_oracle."""
    left = extractor()
    cap = left.capacity()
    f, kfs = BS.search_scene(77, n_frame=600, n_kfs=4, n_nodes=30, angle_spread=10.0)
    n, n_kf = len(f["kps"]), len(kfs)
    for k, kf in enumerate(kfs):  # keyframe k's key i sees point k cap + i: a point is matched by at most one key per call
        kf["point"] = np.where(kf["point"] >= 0, k * cap + np.arange(len(kf["point"])), -1).astype(np.int32)
    rng = np.random.default_rng(5)
    km = keymap(n, cap, rng)
    keep, nk, src = km.keep, km.n_keep, km.src
    key = np.maximum(src, 0)
    slots = np.zeros(cap + SLACK, f["kps"].dtype)
    slots["x"][cap:], slots["y"][cap:] = 600.0, 180.0
    desc = np.zeros((cap + SLACK, 32), np.uint8)
    slots[km.slots], desc[km.slots] = f["kps"], f["desc"]
    node = np.full(cap + SLACK, -1, np.int32)
    node[:nk] = np.where(src >= 0, f["node"][key], f["node"].max())  # a rejected entry carries a live node
    # the oracle's frame, entry by entry: a rejected entry is in no node
    want = [BO.search_by_bow(f["kps"][key], f["desc"][key], np.where(src >= 0, f["node"][key], -1), kf["kps"], kf["desc"], kf["node"],
                             kf["point"], 0.75, True) for kf in kfs]

    def pad(a, fill=0):
        a = np.ascontiguousarray(a)
        out = np.zeros(cap, a.dtype) if a.dtype.names else np.full((cap,) + a.shape[1:], fill, a.dtype)
        out[:len(a)] = a
        return upload(out)
    hold, keys, pts = [], [], []
    for kf in kfs:
        a = [pad(kf["kps"]), pad(kf["desc"]), pad(kf["node"], -1), pad(kf["point"], -1), i64(len(kf["kps"]))]
        hold += a
        keys.append(keyframe_keys(a[0].data_ptr(), a[1].data_ptr(), a[2].data_ptr(), a[4].data_ptr()))
        pts.append(a[3].data_ptr())
    t_kps, t_desc, t_keep, t_node, t_nk = upload(slots), upload(desc), upload(keep), upload(node), i64(nk)
    t_match = sentinel(n_kf * cap + SLACK, -7, torch.int32)
    t_nm = sentinel(n_kf, -7, torch.int64)
    search_by_bow_device(left, t_kps.data_ptr(), t_desc.data_ptr(), t_keep.data_ptr(), t_nk.data_ptr(), t_node.data_ptr(), keys, pts,
                         0.75, True, t_match.data_ptr(), t_nm.data_ptr())
    torch.cuda.synchronize()
    rows = t_match.cpu().numpy()[:n_kf * cap].reshape(n_kf, cap)
    for k, (m, c) in enumerate(want):
        assert np.array_equal(rows[k, :nk], m) and (rows[k, nk:] == -1).all() and int(t_nm[k]) == c, k
    assert sum(c for _, c in want) > 40
    # the points: a matched pair's point on its key's ray at 5 - 40 m under one pose (70 %), elsewhere at random
    R, C = S.rotation((0.2, 1, -0.1), 0.7), np.array([2.0, -0.5, 1.0])
    cam = S.KITTI
    n_points = n_kf * cap
    points = np.zeros((n_points + SLACK, 3), np.float32)
    points[:] = rng.uniform(-30, 30, (len(points), 3)).astype(np.float32)
    for k in range(n_kf):
        for j in np.nonzero(rows[k, :nk] >= 0)[0]:
            if rng.random() < 0.7:
                kp = slots[keep[j]]
                z = rng.uniform(5, 40)
                Pc = np.array([(kp["x"] - cam[2]) * z / cam[0], (kp["y"] - cam[3]) * z / cam[1], z])
                points[rows[k, j]] = (R.T @ Pc + C).astype(np.float32)
    mp_arr = map_points(np.zeros((len(points), 32), np.uint8), points, np.zeros_like(points), 0.0, 1e9)
    t_pts = upload(mp_arr)
    kf_ids = np.arange(n_kf, dtype=np.uint32) * 5 + 3
    solver = reloc.PnpSolver(left, n_kf, S.SEED)
    try:
        solver.setup_device(t_kps.data_ptr(), t_keep.data_ptr(), t_nk.data_ptr(), t_match.data_ptr(), t_nm.data_ptr(), t_pts.data_ptr(),
                            n_points, kf_ids, S.FRAME, *cam)
        oracles = []
        for k in range(n_kf):
            p2, p3, s2, ckey = P.correspondences(slots, rows[k], nk, points[:n_points], left._s2, keep_idx=keep, cap=cap)
            oracles.append((P.Solver(p2, p3, s2, *cam, seed=S.SEED, kf_id=int(kf_ids[k]), frame_id=S.FRAME, log=True), ckey))
        check_state(solver, oracles)
        assert all(s.N >= s.min_inl for s, _ in oracles)
        out = Outputs(n_kf, cap)
        poses = 0
        for _ in range(4):
            res = iterate_and_compare(solver, _Rows(cap, rows), oracles, out, 5, np.ones(n_kf, bool))
            poses += sum(r.Tcw is not None for r in res.values())
        assert poses > 0
    finally:
        solver.close()


# ---------------------------------------------------------------------------------------------------------- 50-digit bounds
def test_device_decompositions_against_50_digits():
    """Refine's kernel path (sivo_dbg_pnp_compute_pose) on noise-free scenes from 5 m to 300 m depth, spread 1 m to 1 cm and
    thickness 1 m to 1 mm: MtM rebuilt in 50 digits from the device's alphas and the float inputs; d, the span of ut rows 8-11
    and the three 6 x K solves (on the device's L_6x10 and rho) within oracle/pnp_bounds.py's bounds.  The pose error against
    the true pose is printed per conditioning."""
    worst = [0.0, 0.0, 0.0]
    for D, s, h in PB.CONDITIONING:
        X, us, R, t = PB.conditioned_scene(D, s, h, n=50, seed=int(D + 100 * s + 1000 * h))
        alphas, _, _, d = reloc.compute_pose(X, us, np.full(len(X), 5.991, np.float32), *S.KITTI)
        r = PB.check_pose_debug(alphas, us, d, S.KITTI)
        worst = [max(a, b) for a, b in zip(worst, r)]
        eR, et = PB.pose_error(list(d.R), list(d.t), R, t)
        print(f"depth {D:5.0f} m spread {s:5.2f} m thickness {h:6.3f} m: pose error R {eR:.1e} t {et:.1e}; ratios "
              f"{[round(x, 2) for x in r]}")
    print("largest ratio to the bound (eigen, span, solve):", [round(x, 2) for x in worst])
    assert max(worst) <= PB.C, worst
