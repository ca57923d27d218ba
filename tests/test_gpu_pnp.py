"""-m gpu: Relocalization's PnP RANSAC (sivo_pnp_*, k_pnp_setup / k_pnp_hyp / k_pnp_decide) and its hooks against
oracle/pnp_oracle.py, bit for bit: the draws, compute_pose's intermediates, and every call's outputs and counters over successive
iterate(5) rounds until no_more."""
import numpy as np
import pytest
import torch

from frame_support import extractor, same_bits
from oracle import pnp_oracle as P
from sivo_b200 import reloc
from sivo_b200.orb import KP_DTYPE
from sivo_b200.track import map_points

pytestmark = pytest.mark.gpu
FX, FY, CX, CY = 718.856, 718.856, 607.1928, 185.2157
SEED, FRAME = 0x5EED5EED1234, 77


@pytest.fixture(scope="module")
def left():
    return extractor()


def test_draws_match_the_oracle():
    for N in (4, 10, 15, 200, 2000, 1 << 20):
        got = reloc.draws(SEED, 5, FRAME, 3, 40, N)
        assert [list(r) for r in got] == [P.draws(SEED, 5, FRAME, 3 + h, N) for h in range(40)]


def pose_scene(n, seed, planar=False):
    r = np.random.default_rng(seed)
    Xw = r.uniform(-5, 5, (n, 3))
    if planar:
        Xw[:, 2] = 1.0
    th = r.normal(size=3) * 0.3
    import cv2
    R, _ = cv2.Rodrigues(th)
    Xc = Xw @ R.T + [0.1, -0.2, 12.0]
    u = np.c_[FX * Xc[:, 0] / Xc[:, 2] + CX, FY * Xc[:, 1] / Xc[:, 2] + CY] + r.normal(size=(n, 2)) * 0.5
    return Xw, u


@pytest.mark.parametrize("n,planar", [(4, False), (4, True), (5, False), (6, False), (50, False), (300, False), (2000, False)])
def test_refine_path_intermediates_match_the_oracle(n, planar):
    """sivo_dbg_pnp_compute_pose runs block_pose, Refine's own device function: every intermediate, the inlier mask and count."""
    for seed in range(3):
        Xw, u = pose_scene(n, seed, planar)
        p3, p2 = Xw.astype(np.float32), u.astype(np.float32)
        err = np.full(n, 5.991, np.float32) * np.float32(1.44)
        alphas, mask, cnt, d = reloc.compute_pose(p3, p2, err, FX, FY, CX, CY)
        fu, fv, uc, vc = (float(np.float32(x)) for x in (FX, FY, CX, CY))
        o = P.compute_pose(p3.astype(np.float64).tolist(), p2.astype(np.float64).tolist(), fu, fv, uc, vc, tree=True)
        assert same_bits(alphas, o.alphas)
        assert same_bits(d.cws, o.cws) and same_bits(d.d, o.d) and same_bits(d.ut, o.ut)
        assert same_bits(d.l_6x10, o.l_6x10) and same_bits(d.rho, o.rho)
        assert same_bits(d.betas, [o.betas[b][i] for b in (1, 2, 3) for i in range(4)])
        assert same_bits(d.rep_errors, o.rep_errors[1:])
        assert same_bits(d.Rs, [x for b in (1, 2, 3) for row in o.Rs[b] for x in row])
        assert same_bits(d.ts, [x for b in (1, 2, 3) for x in o.ts[b]])
        assert d.best == o.best and same_bits(d.R, [x for row in o.R for x in row]) and same_bits(d.t, o.t)
        om, oc = P.check_inliers(o.R, o.t, p3, p2, fu, fv, uc, vc, err)
        assert cnt == oc and np.array_equal(mask, om)
        if planar:
            assert np.isnan(np.array(d.R)).any() and cnt == 0


def batch_scene(left, n_kf, N, outliers, seed, neg=(), has_frac=0.9, planar=False):
    """Frame keys 0..N-1 seen by every candidate; candidate k matches most of them to its own copy of the points, a fraction
    `outliers` of them to wrong positions."""
    cap = left.capacity()
    r = np.random.default_rng(seed)
    import cv2
    R, _ = cv2.Rodrigues(r.normal(size=3) * 0.2)
    t = np.array([0.3, -0.1, 0.5])
    Xw = np.c_[r.uniform(-8, 8, N), r.uniform(-3, 3, N), r.uniform(4, 40, N)]
    if planar:
        Xw[:, 2] = 20.0
    Xc = Xw @ R.T + t
    kps = np.zeros(cap, KP_DTYPE)
    kps["x"][:N] = FX * Xc[:, 0] / Xc[:, 2] + CX + r.normal(size=N) * 0.3
    kps["y"][:N] = FY * Xc[:, 1] / Xc[:, 2] + CY + r.normal(size=N) * 0.3
    kps["octave"][:N] = r.integers(0, left.nlevels, N)
    kps["octave"][N - 1] = left.nlevels  # outside the levels: never a correspondence
    match = np.full((n_kf, cap), -1, np.int32)
    pos = np.zeros((n_kf * N, 3), np.float32)
    for k in range(n_kf):
        has = r.random(N) < has_frac
        wrong = r.random(N) < outliers
        p = Xw + wrong[:, None] * r.normal(size=(N, 3)) * 3.0 * np.array([1.0, 1.0, 0.0 if planar else 1.0])
        pos[k * N:(k + 1) * N] = p
        match[k, :N] = np.where(has, k * N + np.arange(N), -1)
    n_matches = (match >= 0).sum(1).astype(np.int64)
    for k in neg:
        n_matches[k] = -1
    return kps, match, n_matches, pos


def run_and_compare(left, n_kf, N, outliers, seed, neg=(), n_keep=None, active0=None, rounds=4, has_frac=0.9, planar=False,
                    hyps=0):
    cap = left.capacity()
    kps, match, n_matches, pos = batch_scene(left, n_kf, N, outliers, seed, neg, has_frac, planar)
    nk = N if n_keep is None else n_keep
    pts = map_points(np.zeros((len(pos), 32), np.uint8), pos, np.zeros_like(pos), 0.0, 1e9)
    dev = torch.device("cuda")
    t_kps = torch.from_numpy(kps.view(np.uint8).copy()).to(dev)
    t_nk = torch.tensor([nk], dtype=torch.int64, device=dev)
    t_match = torch.from_numpy(match).to(dev)
    t_nm = torch.from_numpy(n_matches).to(dev)
    t_pts = torch.from_numpy(pts.view(np.uint8).copy()).to(dev)
    kf_ids = np.arange(n_kf, dtype=np.uint32) * 3 + 1
    solver = reloc.PnpSolver(left, max(n_kf, 1), SEED)
    solver.setup_device(t_kps.data_ptr(), 0, t_nk.data_ptr(), t_match.data_ptr(), t_nm.data_ptr(), t_pts.data_ptr(), len(pts), kf_ids,
                        FRAME, FX, FY, CX, CY)
    sigma2 = left._s2
    oracles = []
    for k in range(n_kf):
        p2d, p3d, s2, key = P.correspondences(kps, match[k], min(max(nk, 0), cap), pos, sigma2, cap=cap)
        s = P.Solver(p2d, p3d, s2, FX, FY, CX, CY, SEED, int(kf_ids[k]), FRAME, dead=nk < 0 or n_matches[k] < 0)
        oracles.append((s, key))
    st = solver.state()
    for k, (s, _) in enumerate(oracles):
        assert st["dead"][k] == int(s.dead)
        if s.dead:  # a negative count builds no correspondences
            assert st["N"][k] == 0
            continue
        assert (st["N"][k], st["min_inliers"][k], st["max_its"][k]) == (s.N, s.min_inl, s.max_its)
        assert st["eps"][k] == s.eps or s.N == 0
    for k, (s, _) in enumerate(oracles):  # k_pnp_hyp itself, hypothesis by hypothesis
        if hyps == 0 or s.dead or s.N < s.min_inl:
            continue
        got = solver.hypotheses(k, 0, hyps)
        for g in range(hyps):
            idx, dbg, mask, cnt = s.hypothesis(g)
            assert list(got["draws"][g]) == idx
            assert same_bits(got["R"][g], dbg.R) and same_bits(got["t"][g], dbg.t)
            assert got["counts"][g] == cnt and np.array_equal(got["masks"][g][:s.N], mask)
    active = np.ones(n_kf, bool) if active0 is None else np.asarray(active0, bool).copy()
    Tcw = torch.full((n_kf, 12), float("nan"), dtype=torch.float32, device=dev)
    has_pose = torch.full((n_kf,), -7, dtype=torch.int32, device=dev)
    no_more = torch.full((n_kf,), -7, dtype=torch.int32, device=dev)
    n_inl = torch.full((n_kf,), -7, dtype=torch.int32, device=dev)
    inl = torch.full((n_kf, cap), -9, dtype=torch.int32, device=dev)
    seen = {"pose": 0, "no_more": 0}
    for _ in range(rounds):
        if not active.any():
            break
        before = (has_pose.clone(), inl.clone())
        solver.iterate_device(5, active.astype(np.uint8), Tcw.data_ptr(), has_pose.data_ptr(), no_more.data_ptr(), inl.data_ptr(),
                              n_inl.data_ptr())
        torch.cuda.synchronize()
        st = solver.state()
        hp, nm, ni, T, row = (has_pose.cpu().numpy(), no_more.cpu().numpy(), n_inl.cpu().numpy(), Tcw.cpu().numpy(),
                              inl.cpu().numpy())
        for k in range(n_kf):
            if not active[k]:
                assert hp[k] == before[0][k].item() and np.array_equal(row[k], before[1][k].cpu().numpy())
                continue
            s, key = oracles[k]
            res = s.iterate(5)
            assert (bool(hp[k]), bool(nm[k]), int(ni[k])) == (res.Tcw is not None, res.no_more, res.n_inliers), k
            assert (st["iterations"][k], st["best"][k]) == (s.iterations, s.best), k
            want = np.full(cap, -1, np.int32)
            want[key[res.inliers]] = match[k][key[res.inliers]]
            assert np.array_equal(row[k], want), k
            if res.Tcw is not None:
                assert np.array_equal(T[k].view(np.uint32), res.Tcw.reshape(12).view(np.uint32)), k
                seen["pose"] += 1
            if res.no_more:
                active[k] = False
                seen["no_more"] += 1
    solver.close()
    return seen


@pytest.mark.parametrize("n_kf,N,outliers", [(1, 15, 0.0), (8, 200, 0.3), (8, 40, 0.6), (64, 30, 0.3), (2, 2000, 0.3),
                                             (64, 200, 0.6)])
def test_iterate_matches_the_oracle_call_by_call(left, n_kf, N, outliers):
    seen = run_and_compare(left, n_kf, N, outliers, seed=N + n_kf, hyps=8 if n_kf <= 8 else 0)
    assert seen["pose"] + seen["no_more"] > 0


def test_negative_counts_active_mask_and_small_sets(left):
    run_and_compare(left, 6, 120, 0.3, seed=1, neg=(2, 4), active0=[1, 1, 1, 0, 1, 0], hyps=6)
    run_and_compare(left, 3, 120, 0.3, seed=2, n_keep=-1)


def test_N_equal_to_min_inliers(left):
    """11 keys, every one matched, the last one's octave outside the levels: N = 10 = minInliers, maxIts = 1."""
    run_and_compare(left, 4, 11, 0.0, seed=3, has_frac=1.0, hyps=6)
    solver_state = P.ransac_parameters(10)
    assert solver_state[0] == 10 and solver_state[2] == 1


def test_degenerate_minimal_sets_through_the_hypothesis_kernel(left):
    """A planar scene: every minimal set is coplanar, every hypothesis' pose NaN with no inliers, every candidate no_more."""
    seen = run_and_compare(left, 3, 60, 0.0, seed=5, has_frac=1.0, planar=True, hyps=10)
    assert seen["pose"] == 0 and seen["no_more"] == 3


def test_counts_at_the_capacity(left):
    run_and_compare(left, 2, left.capacity(), 0.3, seed=4, n_keep=left.capacity() + 5, rounds=2, hyps=4)


def test_fuzz(left):
    r = np.random.default_rng(99)
    for i in range(200):
        n_kf, N = int(r.integers(1, 7)), int(r.integers(8, 160))
        run_and_compare(left, n_kf, N, float(r.uniform(0, 0.8)), seed=1000 + i, rounds=3, hyps=3 if i % 10 == 0 else 0)
