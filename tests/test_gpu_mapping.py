"""-m gpu: a keyframe's new map points (sivo_create_map_points / _device / sivo_dbg_create_map_points, k_map_create) on constructed
scenes of 2000 keys per keyframe against oracle/mapping_oracle.py, the device form against the host form, and the KeyFrame copy
(sivo_keyframe_gather_device)."""
import numpy as np
import pytest
import torch

from frame_support import KF_FIELDS, extractor, i64, upload
from oracle import mapping_scene as S
from oracle import mapping_oracle as MO
from oracle.keymap import keymap, scatter
from sivo_b200 import _lib as L
from sivo_b200.mapping import HostKeyframe, KeyframeKeys, create_map_points, create_map_points_device, keyframe_gather_device, \
    make_params, set_pose
from sivo_b200.orb import KP_DTYPE

pytestmark = pytest.mark.gpu
TH_CONF, TH_RED, MAX_CLASS = 0.5, 9.5, 8


@pytest.fixture(scope="module")
def left():
    p = S.EXTRACTOR
    return extractor(p.nfeatures, p.scale_factor, p.nlevels)


def host_kf(kf: MO.KeyFrame, count=None) -> HostKeyframe:
    return HostKeyframe(kf.kps, kf.desc, kf.u_right, kf.depth, kf.kp_class, kf.kp_conf, kf.kp_entropy, kf.node, kf.has_point, kf.Rcw,
                        kf.tcw, kf.Ow, count)


def params(th_conf=TH_CONF, th_red=TH_RED):
    return make_params(S.FX, S.FY, S.CX, S.CY, S.MBF, S.sigma_cw(), MAX_CLASS, th_conf, th_red)


def run_host(left, kf1, nbs, debug=True, **kw):
    return create_map_points(left, host_kf(kf1), [host_kf(k) for k in nbs], params(**kw), debug=debug)


@pytest.mark.parametrize("n_nb", [1, 3, 10])
def test_scene_matches_oracle(left, n_nb):
    kf1, nbs = S.make_scene(2000, n_nb, seed=n_nb)
    want = S.oracle_run(kf1, nbs, TH_CONF, TH_RED, MAX_CLASS)
    got = run_host(left, kf1, nbs)
    S.compare(got, want)
    assert want["stage"].max() == MO.CREATED and len(want["created"]) > 100
    # the production path (no per-key search for keys its criteria rule out) creates the same points
    prod = run_host(left, kf1, nbs, debug=False)
    for k in ("created_nb", "created_idx", "created"):
        np.testing.assert_array_equal(prod[k], got[k])
    np.testing.assert_array_equal(prod["world"].view(np.uint32), got["world"].view(np.uint32))


def test_baseline_and_points_on_entry(left):
    kf1, nbs = S.make_scene(800, 3, seed=7)
    nbs[1].Ow = kf1.Ow + np.float32(0.01)  # below mb: skipped
    kf1.has_point[:50] = 1
    want = S.oracle_run(kf1, nbs)
    got = run_host(left, kf1, nbs)
    S.compare(got, want)
    assert (got["stage"][1] == MO.BASELINE).all()
    assert (got["stage"][0, :50] == MO.HAS_POINT).all()
    made0 = np.flatnonzero(got["stage"][0] == MO.CREATED)
    assert len(made0) and (got["stage"][2, made0] == MO.HAS_POINT).all()


def test_thresholds_move_decisions(left):
    kf1, nbs = S.make_scene(600, 2, seed=3)
    for th_conf, th_red in ((0.0, -1e9), (1.5, 0.0), (0.5, float("inf"))):
        want = MO.create_new_map_points(kf1, nbs, S.camera(), S.TABLES.scale, S.TABLES.sigma2, np.float32(1.2), S.sigma_cw(), MAX_CLASS,
                                        th_conf, th_red)
        S.compare(run_host(left, kf1, nbs, th_conf=th_conf, th_red=th_red), want, th_red)


def test_nan_reduction_passes(left):
    kf1, nbs = S.make_scene(600, 1, seed=4)
    kf1.kp_entropy[:] = np.inf  # MI - inf = -inf: rejected; and nan entropy: NaN reduction, which passes
    kf1.kp_entropy[::2] = np.nan
    want = S.oracle_run(kf1, nbs)
    got = run_host(left, kf1, nbs)
    S.compare(got, want)
    made = got["created_nb"] >= 0
    assert made.any() and np.all(np.isnan(kf1.kp_entropy[made]))


def test_empty_and_negative_counts(left):
    kf1, nbs = S.make_scene(300, 2, seed=5)
    r = run_host(left, kf1, [])
    assert r["n_created"] == 0 and (r["created_nb"] == -1).all() and r["stage"].shape == (0, 300)
    e = MO.KeyFrame(kps=kf1.kps[:0], desc=kf1.desc[:0], u_right=kf1.u_right[:0], depth=kf1.depth[:0], kp_class=kf1.kp_class[:0],
                    kp_conf=kf1.kp_conf[:0], kp_entropy=kf1.kp_entropy[:0], node=kf1.node[:0], has_point=kf1.has_point[:0],
                    Rcw=kf1.Rcw, tcw=kf1.tcw)
    assert run_host(left, e, nbs)["n_created"] == 0
    r = run_host(left, kf1, [e] + nbs[1:])
    S.compare(r, S.oracle_run(kf1, [e] + nbs[1:]))
    neg = create_map_points(left, host_kf(kf1), [host_kf(nbs[0], count=-1)], params())
    assert neg["n_created"] == -1


def test_error_codes(left):
    kf1, nbs = S.make_scene(100, 1, seed=6)
    h = host_kf(kf1)
    with pytest.raises(L.SivoError) as e:
        create_map_points(left, h, [h] * 33, params())
    assert e.value.code == L.EINVAL
    bad = host_kf(kf1)
    bad.keys.node = None
    with pytest.raises(L.SivoError) as e:
        create_map_points(left, bad, [h], params())
    assert e.value.code == L.EINVAL


def _device_kf(kf: MO.KeyFrame, cap, keep):
    n = len(kf.kps)
    t = {f: upload(scatter(np.asarray(getattr(kf, f), dt), np.arange(n), cap, 0)) for f, dt in KF_FIELDS.items()}
    t["count"] = i64(n)
    keep.append(t)
    k = KeyframeKeys(*[t[f].data_ptr() for f in ("kps", "desc", "u_right", "depth", "kp_class", "kp_conf", "kp_entropy", "node",
                                                 "has_point", "count")])
    set_pose(k, kf.Rcw, kf.tcw, kf.Ow)
    return k


def test_device_form_equals_host_form(left):
    cap = left.capacity()
    kf1, nbs = S.make_scene(2000, 10, seed=10)
    host = run_host(left, kf1, nbs, debug=False)
    keep = []
    d1 = _device_kf(kf1, cap, keep)
    dn = [_device_kf(k, cap, keep) for k in nbs]
    outs = []
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    for _ in range(2):
        o = dict(nb=torch.full((cap,), -7, dtype=torch.int32, device="cuda"), idx=torch.empty(cap, dtype=torch.int32, device="cuda"),
                 world=torch.empty(cap, 3, dtype=torch.float32, device="cuda"), lst=torch.empty(cap, 2, dtype=torch.int32, device="cuda"),
                 n=torch.empty(1, dtype=torch.int64, device="cuda"))
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            create_map_points_device(left, d1, dn, params(), o["nb"].data_ptr(), o["idx"].data_ptr(), o["world"].data_ptr(),
                                     o["lst"].data_ptr(), o["n"].data_ptr(), stream.cuda_stream)
        stream.synchronize()
        outs.append({k: v.cpu().numpy() for k, v in o.items()})
    n1 = len(kf1.kps)
    for o in outs:
        assert int(o["n"][0]) == host["n_created"]
        np.testing.assert_array_equal(o["nb"][:n1], host["created_nb"])
        np.testing.assert_array_equal(o["idx"][:n1], host["created_idx"])
        np.testing.assert_array_equal(o["world"][:n1].view(np.uint32), host["world"].view(np.uint32))
        np.testing.assert_array_equal(o["lst"][:host["n_created"]], host["created"])
        assert (o["nb"][n1:] == -7).all()
    # a negative count writes only the count
    keep[0]["count"].fill_(-1)
    o = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    create_map_points_device(left, d1, dn, params(), o.data_ptr(), 0, 0, 0, n.data_ptr())
    torch.cuda.synchronize()
    assert int(n[0]) == -1 and (o.cpu() == -7).all()


def test_keyframe_gather(left):
    cap = left.capacity()
    rng = np.random.default_rng(2)
    n = 1500
    kps = np.zeros(cap, KP_DTYPE)
    kps["x"], kps["y"], kps["octave"] = rng.uniform(0, 900, cap), rng.uniform(0, 300, cap), rng.integers(0, 8, cap)
    desc = rng.integers(0, 256, (cap, 32), dtype=np.uint8)
    km = keymap(n, cap, rng, forced=(5,))
    n = km.n_keep
    keep_idx = km.keep[:n]
    ur = rng.uniform(-1, 900, cap).astype(np.float32)
    depth = rng.uniform(-1, 40, cap).astype(np.float32)
    cls = rng.integers(0, 12, cap).astype(np.uint8)
    conf = rng.random(cap)
    ent = rng.random(cap)
    src = [upload(kps), upload(desc), upload(km.keep), i64(n), upload(ur), upload(depth), upload(cls), upload(conf), upload(ent)]
    out = dict(kps=torch.zeros(cap * 28, dtype=torch.uint8, device="cuda"), desc=torch.zeros(cap, 32, dtype=torch.uint8, device="cuda"),
               u_right=torch.zeros(cap, device="cuda"), depth=torch.zeros(cap, device="cuda"),
               kp_class=torch.zeros(cap, dtype=torch.uint8, device="cuda"), kp_conf=torch.zeros(cap, dtype=torch.float64, device="cuda"),
               kp_entropy=torch.zeros(cap, dtype=torch.float64, device="cuda"), count=torch.zeros(1, dtype=torch.int64, device="cuda"))
    torch.cuda.synchronize()
    keyframe_gather_device(left, *[s.data_ptr() for s in src], out)
    torch.cuda.synchronize()
    k = np.clip(keep_idx, 0, cap - 1)
    good = km.src >= 0
    got_kps = out["kps"].cpu().numpy().view(KP_DTYPE)
    assert int(out["count"][0]) == n
    np.testing.assert_array_equal(got_kps[:n][good], kps[k][good])
    assert got_kps[5]["octave"] == -1 and (got_kps[:n][~good]["octave"] == -1).all()
    np.testing.assert_array_equal(out["desc"].cpu().numpy()[:n][good], desc[k][good])
    np.testing.assert_array_equal(out["u_right"].cpu().numpy()[:n], ur[:n])
    np.testing.assert_array_equal(out["depth"].cpu().numpy()[:n], depth[:n])
    np.testing.assert_array_equal(out["kp_class"].cpu().numpy()[:n][good], cls[k][good])
    np.testing.assert_array_equal(out["kp_conf"].cpu().numpy()[:n][good], conf[k][good])
    np.testing.assert_array_equal(out["kp_entropy"].cpu().numpy()[:n][good], ent[k][good])


def _device_outputs(left, d1, dn, prm):
    """The device form on the left extractor's stream, ordered after the output fills and before the reads by device syncs."""
    cap = left.capacity()
    o = dict(nb=torch.full((cap,), -7, dtype=torch.int32, device="cuda"), idx=torch.full((cap,), -7, dtype=torch.int32, device="cuda"),
             world=torch.full((cap, 3), 7.0, dtype=torch.float32, device="cuda"),
             lst=torch.full((cap, 2), -7, dtype=torch.int32, device="cuda"), n=torch.full((1,), -7, dtype=torch.int64, device="cuda"))
    torch.cuda.synchronize()
    create_map_points_device(left, d1, dn, prm, o["nb"].data_ptr(), o["idx"].data_ptr(), o["world"].data_ptr(), o["lst"].data_ptr(),
                             o["n"].data_ptr())
    torch.cuda.synchronize()
    return o


def test_count_equal_to_and_above_the_capacity(left):
    cap = left.capacity()
    kf1, nbs = S.make_scene(cap, 2, seed=12)
    host = run_host(left, kf1, nbs, debug=False)
    assert host["n_created"] > 50
    keep = []
    d1 = _device_kf(kf1, cap, keep)
    dn = [_device_kf(k, cap, keep) for k in nbs]
    torch.cuda.synchronize()
    at = {k: v.cpu().numpy() for k, v in _device_outputs(left, d1, dn, params()).items()}
    torch.cuda.synchronize()
    assert int(at["n"][0]) == host["n_created"]
    np.testing.assert_array_equal(at["nb"], host["created_nb"])
    np.testing.assert_array_equal(at["world"].view(np.uint32), host["world"].view(np.uint32))
    np.testing.assert_array_equal(at["lst"][:host["n_created"]], host["created"])
    # counts above the capacity (current keyframe and a neighbour) are clamped to it: the same result
    keep[0]["count"].fill_(cap + 100)
    keep[2]["count"].fill_(cap + 1)
    torch.cuda.synchronize()
    above = {k: v.cpu().numpy() for k, v in _device_outputs(left, d1, dn, params()).items()}
    for k in at:
        np.testing.assert_array_equal(above[k].view(np.uint8), at[k].view(np.uint8))


def _run_device_dbg_equal(left, kf1, nbs, th_conf=TH_CONF, th_red=TH_RED):
    want = MO.create_new_map_points(kf1, nbs, S.camera(), S.TABLES.scale, S.TABLES.sigma2, np.float32(S.EXTRACTOR.scale_factor),
                                    S.sigma_cw(), MAX_CLASS, th_conf, th_red)
    got = run_host(left, kf1, nbs, th_conf=th_conf, th_red=th_red)
    return got, want


@pytest.mark.parametrize("name", ["dsqr", "reproj1_stereo", "reproj2_stereo", "scale"])
def test_geometric_threshold_at_its_flip(left, name):
    """The varied input steps one float ulp at a time across the flip (pairs 1 and 2): dsqr < 3.84 sigma2, the stereo reprojection
    errors (7.8 sigma2) in both keyframes, the scale ratio."""
    kf1, kf2, reject = BOUNDARY[name]
    got, want = _run_device_dbg_equal(left, kf1, [kf2], 0.5, -1e9)
    st = want["stage"][0]
    assert (st[1] == reject) != (st[2] == reject) and (st[0] == st[1]) and (st[2] == st[3])
    assert S.compare(got, want, -1e9, max_exempt=0) == 0


def test_confidence_at_its_threshold(left):
    th = np.float32(0.7)
    kf1, kf2 = S.pair_scene([S.P0] * 5, o2=3)
    eq = float(th)
    kf1.kp_conf[:] = [np.nextafter(eq, 0), eq, np.nextafter(eq, 1), float(np.nextafter(th, np.float32(0))), float(np.nextafter(th, np.float32(1)))]
    got, want = _run_device_dbg_equal(left, kf1, [kf2], th_conf=float(th), th_red=-1e9)
    assert list(want["stage"][0]) == [MO.SEMANTIC, MO.CREATED, MO.CREATED, MO.SEMANTIC, MO.CREATED]
    assert S.compare(got, want, -1e9, max_exempt=0) == 0


def test_entropy_reduction_at_its_threshold(left):
    kf1, kf2 = S.pair_scene([S.P0] * 7, o2=3)
    mi = S.oracle_run(kf1, [kf2], 0.5, -1e9)["reduction"][0, 0]  # entropy 0: the reduction is the MI
    th = np.float32(mi - 1.0)
    h0 = mi - float(th)
    kf1.kp_entropy[:] = [np.nextafter(np.nextafter(h0, 9), 9), np.nextafter(h0, 9), h0, np.nextafter(h0, -9),
                         np.nextafter(np.nextafter(h0, -9), -9), h0 + 1e-9, h0 - 1e-9]
    got, want = _run_device_dbg_equal(left, kf1, [kf2], th_conf=0.5, th_red=float(th))
    red = want["reduction"][0]
    assert (red < float(th)).any() and (red >= float(th)).any()
    assert want["stage"][0, 5] == MO.SEMANTIC and want["stage"][0, 6] == MO.CREATED
    assert S.compare(got, want, float(th), max_exempt=5) <= 5  # the keys within 1e-12 of the threshold are the log2 exemption


def test_ties_take_the_later_candidate_and_duplicates_match_twice(left):
    kf1, kf2 = S.pair_scene([S.P0] * 4, o2=3)
    kf2.node[:] = 0
    kf1.node[:] = 0
    kf2.desc[0, 0], kf2.desc[1, 0], kf2.desc[2, 0], kf2.desc[3, 0] = 0x1F, 0x07, 0x07, 0x3F  # distances 5, 3, 3, 6
    got, want = _run_device_dbg_equal(left, kf1, [kf2], th_red=-1e9)
    assert (want["match"][0] == 2).all()  # equal distances: the later candidate; every current key matches neighbour key 2
    assert (want["stage"][0] == MO.CREATED).all()
    assert S.compare(got, want, -1e9, max_exempt=0) == 0


def test_epipole_gate_and_the_second_keyframes_stereo_branch(left):
    """Mono-mono pairs near the epipole: the gate is distex^2 + distey^2 < 100 scale[octave], scale not squared; a mono current
    key with a stereo neighbour key takes the `else if (bStereo2)` branch (UnprojectStereo of the neighbour's key)."""
    s3 = float(S.TABLES.scale[3])
    r_gate, r_sq = np.sqrt(100 * s3), np.sqrt(100 * s3 * s3)
    # epipole of the current keyframe's centre in the neighbour's image: the principal point (both on the z axis)
    pts = [(0.0, 0.0, 30.0)] * 3
    kf1, kf2 = S.pair_scene(pts, stereo1=False, stereo2=False, o2=3)
    for i, r in enumerate((0.99 * r_gate, 1.01 * r_gate, 0.99 * r_sq)):
        kf2.kps["x"][i] = np.float32(S.CX + r)
        kf2.kps["y"][i] = np.float32(S.CY)
        kf1.kps["x"][i] = np.float32(S.CX + r)
        kf1.kps["y"][i] = np.float32(S.CY)
    got, want = _run_device_dbg_equal(left, kf1, [kf2], th_red=-1e9)
    assert list(want["match"][0]) == [-1, 1, 2]  # inside the gate; outside it; inside only a squared-scale gate
    assert S.compare(got, want, -1e9, max_exempt=0) == 0
    k1, k2 = S.pair_scene([S.P0] * 2, stereo1=False, stereo2=True, o2=3)
    got, want = _run_device_dbg_equal(left, k1, [k2], th_red=-1e9)
    assert (want["stage"][0] == MO.CREATED).all()
    assert np.array_equal(want["world"][0], MO.unproject(k2, 0, S.camera()))
    assert S.compare(got, want, -1e9, max_exempt=0) == 0


BOUNDARY = {}


@pytest.fixture(scope="module", autouse=True)
def _boundary():
    BOUNDARY.update(S.boundary_cases())
