"""-m gpu: sivo_fuse_device, sivo_fuse and sivo_dbg_fuse held to oracle/fuse_oracle.py bit for bit on SearchInNeighbors' two
phases of constructed and seeded maps, the replay driven by the device's matrices against the literal loop, the target and count
limits and the refused arguments; and the device form on KITTI keyframes gathered through DeviceFrame."""
import ctypes as C

import numpy as np
import pytest
import torch

from frame_support import BOUNDS, CX, CY, FX, MB, MBF, extractors, frame_inputs, seg, upload  # noqa: F401
from fuse_support import camera, host_targets, records, run_device
from oracle import fuse_oracle as FO
from oracle import fuse_scene as S
from oracle import track_oracle as T
from oracle.mapping_scene import rotation
from sivo_b200 import _lib as L
from sivo_b200.frame import DeviceFrame
from sivo_b200.mapping import KeyframeKeys, dbg_fuse, fuse, fuse_device, keyframe_gather_device, set_pose
from sivo_b200.orb import KP_DTYPE, ORBextractor

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def left():
    return ORBextractor(2000, 1.2, 8, 20, 7)


def check_all_forms(left, kfs, cam, points, th, counts=None):
    """Device, host and debug forms against the oracle; returns the oracle's stages."""
    want = FO.decide_all(kfs, points, cam, S.TABLES, th, counts)
    m, d = fuse(left, host_targets(kfs, counts), camera(cam), records(points), th)
    dm, dd, ds = dbg_fuse(left, host_targets(kfs, counts), camera(cam), records(points), th)
    vm, vd = run_device(left, kfs, cam, points, th, counts)
    for got in ((m, d), (dm, dd), (vm, vd)):
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])
    np.testing.assert_array_equal(ds, want[2])
    return want[2]


@pytest.mark.parametrize("prm", S.CONSTRUCTED[:4] + S.CONSTRUCTED[6:9], ids=lambda p: f"seed{p['seed']}")
def test_both_phases_of_constructed_maps(left, prm):
    cur, targets, points = S.make_map(**prm)
    p1 = [mp for mp in cur.points if mp is not None]
    stages = check_all_forms(left, targets, S.CAMERA, p1, 3.0)
    assert (stages == FO.MATCHED).any()
    check_all_forms(left, [cur], S.CAMERA, FO.fuse_candidates(targets), 3.0)


@pytest.mark.parametrize("seed", range(6))
def test_seeded_fuzz(left, seed):
    prm = S.fuzz_params(seed)
    cur, targets, points = S.make_map(**prm)
    th = (3.0, 1.0, 5.5)[seed % 3]
    check_all_forms(left, [cur] + targets, S.CAMERA, points, th)


def device_rows(left, cam, th=3.0):
    return lambda kfs, recs: run_device(left, kfs, cam, recs, th)[0]


@pytest.mark.parametrize("prm", [S.CONSTRUCTED[0], S.CONSTRUCTED[8], S.fuzz_params(3)], ids=lambda p: f"seed{p['seed']}")
def test_replay_with_device_matrices_equals_literal(left, prm):
    cur, targets, points = S.make_map(**prm)
    FO.search_in_neighbors(cur, targets, S.CAMERA, S.TABLES, 3.0)
    want = FO.map_state([cur] + targets, points)
    cur, targets, points = S.make_map(**prm)
    FO.replay(cur, targets, device_rows(left, S.CAMERA))
    assert FO.map_state([cur] + targets, points) == want


def test_target_counts_and_limits(left):
    cap = left.capacity()
    cur, targets, points = S.make_map(**S.CONSTRUCTED[1])
    pts = [mp for mp in points if not mp.bad][:300]
    # 0 targets, 1 target, n_points = 0
    for kfs, pp in (([], pts), (targets[:1], pts), (targets[:3], [])):
        m, d = fuse(left, host_targets(kfs), camera(S.CAMERA), records(pp), 3.0)
        assert m.shape == (len(kfs), len(pp))
        vm, _ = run_device(left, kfs, S.CAMERA, pp, 3.0)
        assert vm.shape == m.shape and np.array_equal(vm, FO.decide_all(kfs, pp, S.CAMERA, S.TABLES, 3.0)[0])
    # 60 targets (the keyframes at jittered poses), one with a negative count
    rng = np.random.default_rng(4)
    many = []
    for k in range(60):
        base = targets[k % len(targets)]
        R = (rotation(*rng.normal(0, 0.004, 3)).astype(np.float32) @ base.Rcw).astype(np.float32)
        t = (base.tcw + rng.normal(0, 0.02, 3)).astype(np.float32)
        many.append(FO.KeyFrame(k + 1, base.kps, base.desc, base.u_right, R, t, T.gemm_neg_t(R, t), S.CAMERA))
    counts = [len(kf.kps) for kf in many]
    counts[17] = -1
    stages = check_all_forms(left, many, S.CAMERA, pts, 3.0, counts)
    assert (stages[17] == FO.NEGATIVE).all() and (stages == FO.MATCHED).sum() > 100
    # a target of exactly the capacity, and a count above it (clamped)
    rng = np.random.default_rng(5)
    kps = np.zeros(cap, KP_DTYPE)
    kps["x"], kps["y"] = rng.uniform(0, 640, cap), rng.uniform(0, 480, cap)
    kps["octave"], kps["angle"] = rng.integers(0, 4, cap), rng.uniform(0, 360, cap)
    full = FO.KeyFrame(1, kps, np.concatenate([targets[0].desc, rng.integers(0, 256, (cap, 32), dtype=np.uint8)])[:cap],
                       np.where(rng.random(cap) < 0.5, rng.uniform(0, 600, cap), -1).astype(np.float32), targets[0].Rcw, targets[0].tcw,
                       targets[0].Ow, S.CAMERA)
    full.kps[:len(targets[0].kps)] = targets[0].kps
    full.u_right[:len(targets[0].kps)] = targets[0].u_right
    full.grid = T.assign_features_to_grid(full.kps, full.geo)
    want = FO.decide_all([full], pts, S.CAMERA, S.TABLES, 3.0)
    assert (want[2] == FO.MATCHED).any()
    for count in (cap, cap + 5):
        vm, vd = run_device(left, [full], S.CAMERA, pts, 3.0, [count])
        np.testing.assert_array_equal(vm, want[0])
        np.testing.assert_array_equal(vd, want[1])


def test_refused_arguments(left):
    cur, targets, points = S.make_map(**S.CONSTRUCTED[0])
    pts = records(points[:10])
    ht = host_targets(targets[:2])
    cam = camera(S.CAMERA)
    for th in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(L.SivoError) as e:
            fuse(left, ht, cam, pts, th)
        assert e.value.code == L.EINVAL
    bad = camera(S.CAMERA)
    bad.max_x = bad.min_x
    with pytest.raises(L.SivoError) as e:
        fuse(left, ht, bad, pts, 3.0)
    assert e.value.code == L.EINVAL
    lib = L.lib()
    m = np.zeros(100, np.int32)
    arr = (type(ht[0].keys) * 2)(ht[0].keys, ht[1].keys)
    assert lib.sivo_fuse(left._h, arr, -1, C.byref(cam), L.ptr(pts), 10, 3.0, L.ptr(m), None) == L.EINVAL
    assert lib.sivo_fuse(left._h, arr, 2, C.byref(cam), L.ptr(pts), -1, 3.0, L.ptr(m), None) == L.EINVAL
    assert lib.sivo_fuse(left._h, arr, 2, None, L.ptr(pts), 10, 3.0, L.ptr(m), None) == L.EINVAL
    assert lib.sivo_fuse(left._h, None, 2, C.byref(cam), L.ptr(pts), 10, 3.0, L.ptr(m), None) == L.EINVAL
    assert lib.sivo_fuse(left._h, arr, 2, C.byref(cam), None, 10, 3.0, L.ptr(m), None) == L.EINVAL
    assert lib.sivo_fuse(None, arr, 2, C.byref(cam), L.ptr(pts), 10, 3.0, L.ptr(m), None) == L.EINVAL
    assert lib.sivo_fuse_device(left._h, arr, 2, C.byref(cam), 16, 1 << 30, 3.0, 16, 0, None) == L.EINVAL  # 2 x 2^30 > INT_MAX
    assert lib.sivo_fuse_device(left._h, arr, 2, C.byref(cam), 16, 10, 3.0, None, 0, None) == L.EINVAL
    # a key angle outside [0, 360]: the host form refuses it
    for a in (-1.0, 360.5, float("nan")):
        k = targets[0].kps.copy()
        k["angle"][3] = a
        t = FO.KeyFrame(1, k, targets[0].desc, targets[0].u_right, targets[0].Rcw, targets[0].tcw, targets[0].Ow, S.CAMERA)
        with pytest.raises(L.SivoError) as e:
            fuse(left, host_targets([t]), cam, pts, 3.0)
        assert e.value.code == L.ERANGE
    # the device form puts such a key in no cell, as the oracle's grid does
    k = targets[0].kps.copy()
    k["angle"][::3] = -5.0
    t = FO.KeyFrame(1, k, targets[0].desc, targets[0].u_right, targets[0].Rcw, targets[0].tcw, targets[0].Ow, S.CAMERA)
    p1 = [mp for mp in cur.points if mp is not None]
    vm, vd = run_device(left, [t], S.CAMERA, p1, 3.0)
    want = FO.decide_all([t], p1, S.CAMERA, S.TABLES, 3.0)
    np.testing.assert_array_equal(vm, want[0])
    np.testing.assert_array_equal(vd, want[1])


def test_chain_on_gathered_keyframes(seg, kitti_bgr):
    """KITTI and synthetic frames through DeviceFrame and sivo_keyframe_gather_device; the gathered buffers (counts on the device)
    fused in place against the host form and the oracle, with points made from the first keyframe's stereo keys."""
    el, er = extractors(2000)
    cap = el.capacity()
    inputs = frame_inputs(kitti_bgr)
    s_t = torch.cuda.Stream()
    s = s_t.cuda_stream
    H, W = inputs[0][1].shape
    kfs, keys = [], []
    for i, inp in enumerate(inputs):
        f = DeviceFrame(el, er, H, W)
        d_in = [upload(x) for x in inp]
        seg.set_frame(700 + i)
        f.extract(seg, *d_in, s)
        f.tail(seg, MB, MBF, s)
        out = dict(kps=torch.zeros(cap * 28, dtype=torch.uint8, device="cuda"), desc=torch.zeros(cap * 32, dtype=torch.uint8, device="cuda"),
                   u_right=torch.zeros(cap, device="cuda"), depth=torch.zeros(cap, device="cuda"),
                   kp_class=torch.zeros(cap, dtype=torch.uint8, device="cuda"), kp_conf=torch.zeros(cap, dtype=torch.float64, device="cuda"),
                   kp_entropy=torch.zeros(cap, dtype=torch.float64, device="cuda"), count=torch.zeros(1, dtype=torch.int64, device="cuda"))
        keyframe_gather_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, f.depth, f.kp_class, f.kp_conf, f.kp_entropy, out, s)
        s_t.synchronize()
        n = int(out["count"][0])
        assert n > 100
        R = rotation(0.0, 0.004 * i, 0.0).astype(np.float32)
        t = (-R.astype(np.float64) @ np.array([0.05 * i, 0.0, 0.1 * i])).astype(np.float32)
        g = {k: v.cpu().numpy() for k, v in out.items()}
        kf = FO.KeyFrame(i, g["kps"].view(KP_DTYPE)[:n].copy(), g["desc"].reshape(cap, 32)[:n].copy(), g["u_right"][:n].copy(), R, t,
                         T.gemm_neg_t(R, t), FO.Camera(FX, FX, CX, CY, MBF, BOUNDS))
        kf.depth = g["depth"][:n].copy()
        kfs.append((kf, out))
    cam = FO.Camera(FX, FX, CX, CY, MBF, BOUNDS)
    kf0 = kfs[0][0]
    pts, idx = T.map_points_from_keys(kf0.kps, kf0.depth, kf0.Rcw.T, kf0.Ow, FX, FX, CX, CY, S.TABLES.scale)
    recs = [{"pos": pts["pos"][i], "normal": pts["normal"][i], "min_distance": pts["min_distance"][i],
             "max_distance": pts["max_distance"][i], "desc": kf0.desc[idx[i]]} for i in range(len(idx))]
    # the device form reads the gathered buffers in place
    kk = []
    for kf, out in kfs:
        k = KeyframeKeys(out["kps"].data_ptr(), out["desc"].data_ptr(), out["u_right"].data_ptr(), None, None, None, None, None, None,
                         out["count"].data_ptr())
        set_pose(k, kf.Rcw, kf.tcw, kf.Ow)
        kk.append(k)
    d_pts = torch.from_numpy(records(recs).view(np.uint8).copy()).cuda()
    match = torch.full((len(kk), len(recs)), -7, dtype=torch.int32, device="cuda")
    dist = torch.full((len(kk), len(recs)), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    fuse_device(el, kk, camera(cam), d_pts.data_ptr(), len(recs), 3.0, match.data_ptr(), dist.data_ptr(), s)
    s_t.synchronize()
    want = FO.decide_all([kf for kf, _ in kfs], recs, cam, S.TABLES, 3.0)
    hm, hd = fuse(el, host_targets([kf for kf, _ in kfs]), camera(cam), records(recs), 3.0)
    np.testing.assert_array_equal(match.cpu().numpy(), want[0])
    np.testing.assert_array_equal(dist.cpu().numpy(), want[1])
    np.testing.assert_array_equal(hm, want[0])
    np.testing.assert_array_equal(hd, want[1])
    assert (want[2][0] == FO.MATCHED).sum() > len(recs) // 2  # the points' own keyframe finds their keys
