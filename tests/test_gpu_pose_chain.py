"""-m gpu: Tracking's per-frame chain on the device, three frames in flight on rotating buffers -- SegNet -> two enqueue_device ->
semantic keys -> stereo -> last-frame search -> gather -> pose -> (the host reads the result) -> local-map search at that pose ->
gather -> pose -> (the host reads the result) -> information selection with its Rwc, Ow and Sigma -- each stage checked against
oracle/track_oracle.py, oracle/pose_oracle.py and oracle/info_oracle.py on the stage's own inputs (the KITTI fixture crop and two
synthetic frames).  The searches and pose calls read the frame's keys, so they run before the next frame's enqueue_device."""
import numpy as np
import pytest
import torch

from frame_support import BOUNDS, CX, CY, FX, MB, MBF, H, W, check_pose, ext, frame_inputs, ptr, seg, upload  # noqa: F401
from oracle import info_oracle as I
from oracle import pose_oracle as P
from oracle import track_oracle as T
from oracle.mapping_scene import rotation
from sivo_b200 import (info_select, info_select_device, make_frame, map_points, pose_gather_device, pose_optimize_device, search_last_frame_device,
                       search_local_points_device)
from sivo_b200.frame import DeviceFrame
from sivo_b200.pose import camera_from_result, frame_from_result, result_from_bytes

pytestmark = pytest.mark.gpu

TH_LAST, TH_LOCAL = 7, 1


def make_map(kps, desc, depth, scale, Rcw, tcw, seed):
    """The map the frame sees: points unprojected from its keys with depth at the true pose (Rcw, tcw), carrying the keys'
    descriptors, octaves and angles; one in eight moved by 0.5-2 m (matches that are geometric outliers).  Even points form the
    last frame's points, odd points the local map."""
    rng = np.random.default_rng(seed)
    Rwc = Rcw.T
    Ow = -Rcw.T @ tcw
    f, idx = T.map_points_from_keys(kps, depth, Rwc, Ow, FX, FX, CX, CY, scale)
    pts = map_points(desc[idx], f["pos"], f["normal"], f["min_distance"], f["max_distance"], 1, kps["octave"][idx], kps["angle"][idx])
    bad = rng.uniform(size=len(pts)) < 0.125
    pts["pos"][bad] += rng.uniform(0.5, 2.0, (bad.sum(), 3)).astype(np.float32) * rng.choice([-1, 1], (bad.sum(), 3))
    return pts[0::2].copy(), pts[1::2].copy()


def test_three_frames_in_flight_through_both_optimisations(seg, ext, kitti_bgr):
    el, er = ext
    inputs = frame_inputs(kitti_bgr)
    d_in = [[upload(x) for x in f] for f in inputs]
    cap = el.capacity()
    scale = el.GetScaleFactors()
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    bufs = []
    for _ in inputs:
        b = {"f": DeviceFrame(el, er, H, W)}
        for k in ("m_last", "m_loc"):
            b[k] = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
        for k in ("n_last", "n_loc", "n_sel"):
            b[k] = torch.full((1,), -7, dtype=torch.int64, device="cuda")
        b["view"] = torch.zeros(4 * cap, dtype=torch.uint8, device="cuda")
        b["xw"] = torch.full((3 * cap,), float("nan"), dtype=torch.float32, device="cuda")
        b["T0"] = torch.zeros(12, dtype=torch.float32, device="cuda")
        for k in ("r1", "r2"):
            b[k] = torch.full((512,), 0x55, dtype=torch.uint8, device="cuda")
        for k in ("o1", "o2", "blocked"):
            b[k] = torch.full((cap,), 7, dtype=torch.uint8, device="cuda")
        b["world"] = torch.full((3 * cap,), 7.0, dtype=torch.float32, device="cuda")
        b["red"] = torch.full((cap,), 7.0, dtype=torch.float64, device="cuda")
        b["sel"] = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
        bufs.append(b)
    torch.cuda.synchronize()

    def front_end(i, b):
        seg.set_frame(400 + i)
        b["f"].extract(seg, *d_in[i], s)  # waits for the previous frame's stereo, searches and optimisations
        b["f"].tail(seg, MB, MBF, s)

    # a first pass of the front end (it captures the network's graph) gives each frame's keys, from which its map is made
    for i, b in enumerate(bufs):
        front_end(i, b)
    stream.synchronize()
    cases = []
    for i, b in enumerate(bufs):
        n_keep, keep, ur, depth = b["f"].host()
        kps_all, desc_all = b["f"].left.host()
        kps, desc = kps_all[keep], desc_all[keep]
        R_true, t_true = rotation(0.01 * i, -0.02, 0.005), np.array([0.1 * i, -0.05, 0.3])
        last_pts, local_pts = make_map(kps, desc, depth, scale, R_true, t_true, 40 + i)
        Tpred = np.concatenate([rotation(0.001, -0.0015, 0.001) @ R_true, (t_true + [0.01, -0.005, 0.01])[:, None]], 1).astype(np.float32)
        cases.append(dict(n_keep=n_keep, keep=keep, kps=kps, desc=desc, ur=ur, depth=depth, last=last_pts, local=local_pts,
                          Tpred=Tpred, ent=b["f"].out["kp_entropy"].cpu().numpy()[keep]))
        b["d_last"], b["d_local"] = upload(last_pts), upload(local_pts)
        b["T0"].copy_(torch.from_numpy(Tpred.reshape(-1)))
        assert len(last_pts) > 40 and len(local_pts) > 40
    torch.cuda.synchronize()

    # the chain: front end, last-frame search, gather, pose for the three frames in flight; each frame's enqueue_device waits for
    # the previous frame's search and optimisation
    for i, b in enumerate(bufs):
        front_end(i, b)
        c, f = cases[i], b["f"]
        frame = make_frame(FX, FX, CX, CY, MBF, BOUNDS, c["Tpred"][:, :3], c["Tpred"][:, 3])
        search_last_frame_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, ptr(b["d_last"]), len(c["last"]), frame, c["Tpred"][:, :3],
                                 c["Tpred"][:, 3], TH_LAST, ptr(b["m_last"]), ptr(b["n_last"]), s)
        pose_gather_device(el, ptr(b["m_last"]), f.n_keep, ptr(b["d_last"]), len(c["last"]), ptr(b["xw"]), s)
        pose_optimize_device(el, f.kps, f.keep, f.n_keep, f.u_right, ptr(b["xw"]), FX, FX, CX, CY, MBF, ptr(b["T0"]), ptr(b["r1"]),
                             ptr(b["o1"]), s)
    stream.synchronize()
    # TrackWithMotionModel discards the outliers; the local-map search then runs at the optimised pose with the kept keys blocked
    r1 = [result_from_bytes(b["r1"].cpu().numpy()) for b in bufs]
    with torch.cuda.stream(stream):
        for i, b in enumerate(bufs):
            c, f = cases[i], b["f"]
            xw = b["xw"].view(-1, 3)
            xw.masked_fill_(b["o1"].bool()[:, None], float("nan"))
            b["blocked"].copy_((~torch.isnan(xw[:, 0])).to(torch.uint8))
            frame = frame_from_result(r1[i], FX, FX, CX, CY, MBF, BOUNDS)
            search_local_points_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, ptr(b["blocked"]), ptr(b["d_local"]), len(c["local"]),
                                       frame, TH_LOCAL, 0.8, ptr(b["view"]), ptr(b["m_loc"]), ptr(b["n_loc"]), s)
            pose_gather_device(el, ptr(b["m_loc"]), f.n_keep, ptr(b["d_local"]), len(c["local"]), ptr(b["xw"]), s)
            pose_optimize_device(el, f.kps, f.keep, f.n_keep, f.u_right, ptr(b["xw"]), FX, FX, CX, CY, MBF, ptr(b["r1"]), ptr(b["r2"]),
                                 ptr(b["o2"]), s)
    stream.synchronize()
    r2 = [result_from_bytes(b["r2"].cpu().numpy()) for b in bufs]
    prior = 1e-4 * np.eye(6)
    cams, thresholds = [], []
    for i, b in enumerate(bufs):
        c = cases[i]
        cam = camera_from_result(r2[i], FX, FX, CX, CY, MB, prior)
        ocam = I.Camera(FX, FX, CX, CY, MB, np.array(r2[i].Rwc, np.float32).reshape(3, 3), np.array(r2[i].Ow, np.float32),
                        r2[i].sigma() if r2[i].sigma_valid else prior)
        _, red, _ = I.select(c["kps"], c["depth"], c["ent"], el.GetScaleSigmaSquares(), ocam, 0.0)
        r = np.unique(red[np.isfinite(red)])
        k = len(r) // 2
        thresholds.append(0.5 * (r[k] + r[k + 1]))
        cams.append((cam, ocam))
        f = b["f"]
        info_select_device(el, f.kps, f.kp_entropy, f.keep, f.n_keep, f.depth, cam, thresholds[i], ptr(b["world"]), ptr(b["red"]),
                           ptr(b["sel"]), ptr(b["n_sel"]), s)
    stream.synchronize()

    n_edges = [0, 0]
    n_bad = [0, 0]
    for i, b in enumerate(bufs):
        c = cases[i]
        n = c["n_keep"]
        # the front end gave the same keys as the first pass
        assert int(b["f"].out["n_keep"].cpu()[0]) == n and np.array_equal(b["f"].out["keep_idx"].cpu().numpy()[:n], c["keep"])
        # last-frame search
        of = T.Frame(FX, FX, CX, CY, MBF, BOUNDS, c["Tpred"][:, :3], c["Tpred"][:, 3])
        om, on = T.search_last_frame(c["kps"], c["desc"], c["ur"], c["last"], of, c["Tpred"][:, :3], c["Tpred"][:, 3], scale, TH_LAST)
        assert np.array_equal(b["m_last"].cpu().numpy()[:n], om) and int(b["n_last"].cpu()[0]) == on and on > 20
        # the first optimisation, from the predicted pose
        x1 = np.full((n, 3), np.nan, np.float32)
        x1[om >= 0] = c["last"]["pos"][om[om >= 0]]
        ref1 = P.pose_optimization(c["kps"], c["ur"], x1, c["Tpred"], el.GetInverseScaleSigmaSquares(), P.Camera(FX, FX, CX, CY, MBF),
                                   order="device")
        o1 = b["o1"].cpu().numpy()[:n].astype(bool)
        check_pose(r1[i], o1, ref1)
        assert ref1.sigma_valid
        n_bad[0] += ref1.n_bad
        # the local-map search at the first result's pose, keys holding a kept last-frame point blocked
        blocked = (om >= 0) & ~o1
        of2 = T.Frame(FX, FX, CX, CY, MBF, BOUNDS, np.array(r1[i].Rcw, np.float32).reshape(3, 3), np.array(r1[i].tcw, np.float32))
        ov, om2, on2 = T.search_local_points(c["kps"], c["desc"], c["ur"], c["local"], of2, scale, TH_LOCAL, 0.8, blocked=blocked)
        assert np.array_equal(b["m_loc"].cpu().numpy()[:n], om2) and int(b["n_loc"].cpu()[0]) == on2 and on2 > 20
        assert np.array_equal(b["view"].cpu().numpy()[:len(c["local"])].astype(bool), ov)
        # the second optimisation, from the first result, over the kept last-frame points and the local-map matches
        x2 = x1.copy()
        x2[o1] = np.nan
        x2[om2 >= 0] = c["local"]["pos"][om2[om2 >= 0]]
        assert np.array_equal(b["xw"].cpu().numpy()[:3 * n].reshape(n, 3), x2, equal_nan=True)
        ref2 = P.pose_optimization(c["kps"], c["ur"], x2, r1[i].pose(), el.GetInverseScaleSigmaSquares(), P.Camera(FX, FX, CX, CY, MBF),
                                   order="device")
        check_pose(r2[i], b["o2"].cpu().numpy()[:n].astype(bool), ref2)
        assert ref2.sigma_valid
        n_bad[1] += ref2.n_bad
        n_edges[0] += ref1.n_initial
        n_edges[1] += ref2.n_initial
        # the information selection with the second result's Rwc, Ow and Sigma
        cam, ocam = cams[i]
        assert np.array_equal(np.array(cam.sigma_cw).reshape(6, 6), r2[i].sigma())
        ow, ored, osel = I.select(c["kps"], c["depth"], c["ent"], el.GetScaleSigmaSquares(), ocam, thresholds[i])
        world = b["world"].cpu().numpy()[:3 * n].reshape(n, 3)
        red = b["red"].cpu().numpy()[:n]
        ns = int(b["n_sel"].cpu()[0])
        sel = b["sel"].cpu().numpy()[:ns]
        # against the oracle as tests/test_gpu_info_select.py holds the selection to it (log2 within an ulp of glibc's) ...
        fin = np.isfinite(ored)
        assert np.array_equal(np.isfinite(red), fin) and np.abs(red[fin] - ored[fin]).max() <= 1e-12
        assert np.array_equal(world[fin], ow[fin])
        close = np.flatnonzero(fin & (np.abs(ored - thresholds[i]) <= 1e-12))
        assert np.array_equal(np.setdiff1d(sel, close), np.setdiff1d(osel, close)) and 0 < ns < n
        # ... and bit for bit against the host form on the same keys and camera
        hw, hr, hs = info_select(el, c["kps"], c["depth"], c["ent"], cam, thresholds[i])
        assert world.tobytes() == hw.tobytes() and red.tobytes() == hr.tobytes() and sel.tobytes() == hs.tobytes()
    print(f"edges: first optimisations {n_edges[0]} ({n_bad[0]} outliers), second {n_edges[1]} ({n_bad[1]} outliers)")
    assert n_bad[0] + n_bad[1] > 0

