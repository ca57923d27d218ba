"""-m gpu: device-form calls that share one left / right extractor pair need no ordering among themselves.  Each call's scratch is
its own, allocated and freed on its stream, so two independent problems issued on two streams that never wait on each other give,
bit for bit, what the same calls give one after the other on one stream."""
import numpy as np
import pytest
import torch

from frame_support import BOUNDS, CX, CY, FX, MB, MBF, H, W, extractors, ptr, synth, upload
from oracle import track_oracle as T
from oracle.mapping_scene import rotation
from sivo_b200 import (info_select_device, make_frame, map_points, pose_gather_device, pose_optimize_device, search_last_frame_device,
                       search_local_points_device, stereo_match, stereo_match_device)
from sivo_b200.frame import FrameKeys
from sivo_b200.info import make_camera
from sivo_b200.pose import result_from_bytes

pytestmark = pytest.mark.gpu


def problem(el, er, kl, dl, kr, dr, keep, angles, seed):
    """A Frame tail over the semantic keys `keep`: its map is unprojected from the keys' host-form depths at a true pose; even
    points form the last frame, odd points the local map.  The pose search and optimisation start from a perturbed pose."""
    rng = np.random.default_rng(seed)
    scale = el.GetScaleFactors()
    R, t = rotation(*angles), rng.uniform(-0.2, 0.2, 3)
    _, depth = stereo_match(el, er, kl[keep], dl[keep], kr, dr, MB, MBF)
    f, idx = T.map_points_from_keys(kl[keep], depth, R.T, -R.T @ t, FX, FX, CX, CY, scale)
    pts = map_points(dl[keep][idx], f["pos"], f["normal"], f["min_distance"], f["max_distance"], 1, kl[keep]["octave"][idx],
                     kl[keep]["angle"][idx])
    Tpred = np.concatenate([rotation(0.001, -0.0015, 0.001) @ R, (t + [0.01, -0.005, 0.01])[:, None]], 1).astype(np.float32)
    cap = el.capacity()
    ent = np.zeros(cap)
    ent[:len(kl)] = rng.uniform(0, 0.5, len(kl))
    p = dict(keep=upload(keep.astype(np.int32)), n=upload(np.array([len(keep)], np.int64)), last=pts[0::2].copy(), local=pts[1::2].copy(),
             Tpred=Tpred, ent=upload(ent), cam=make_camera(FX, FX, CX, CY, MB, R.T, -R.T @ t, 1e-4 * np.eye(6)))
    p["d_last"] = upload(p["last"])
    p["d_local"] = upload(p["local"])
    p["T0"] = upload(Tpred)
    p["frame"] = make_frame(FX, FX, CX, CY, MBF, BOUNDS, Tpred[:, :3], Tpred[:, 3])
    return p


def outputs(cap, n_local):
    o = {"u": torch.full((cap,), 7.0, device="cuda"), "z": torch.full((cap,), 7.0, device="cuda"), "world": torch.full((3 * cap,), 7.0, device="cuda"),
         "red": torch.full((cap,), 7.0, dtype=torch.float64, device="cuda"), "view": torch.full((n_local,), 7, dtype=torch.uint8, device="cuda"),
         "xw": torch.full((3 * cap,), float("nan"), device="cuda"), "res": torch.full((512,), 0x55, dtype=torch.uint8, device="cuda"),
         "outl": torch.full((cap,), 7, dtype=torch.uint8, device="cuda")}
    for k in ("sel", "m_last", "m_loc"):
        o[k] = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
    for k in ("n_sel", "n_last", "n_loc"):
        o[k] = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    return o


def calls(el, er, dkl, dkr, p, o, s):
    """The Frame tail's device calls on one problem, in Tracking's order, each a closure enqueuing on stream `s`."""
    keep, n = ptr(p["keep"]), ptr(p["n"])
    u, z = ptr(o["u"]), ptr(o["z"])
    nl, nloc = len(p["last"]), len(p["local"])
    R, t = p["Tpred"][:, :3], p["Tpred"][:, 3]
    return [
        lambda: stereo_match_device(el, er, ptr(dkl.kps), ptr(dkl.desc), keep, n, ptr(dkr.kps), ptr(dkr.desc), ptr(dkr.count), MB, MBF, u, z,
                                    s),
        lambda: info_select_device(el, ptr(dkl.kps), ptr(p["ent"]), keep, n, z, p["cam"], 0.0, ptr(o["world"]), ptr(o["red"]),
                                   ptr(o["sel"]), ptr(o["n_sel"]), s),
        lambda: search_last_frame_device(el, ptr(dkl.kps), ptr(dkl.desc), keep, n, u, ptr(p["d_last"]), nl, p["frame"], R, t, 7,
                                         ptr(o["m_last"]), ptr(o["n_last"]), s),
        lambda: search_local_points_device(el, ptr(dkl.kps), ptr(dkl.desc), keep, n, u, 0, ptr(p["d_local"]), nloc, p["frame"], 1, 0.8,
                                           ptr(o["view"]), ptr(o["m_loc"]), ptr(o["n_loc"]), s),
        lambda: pose_gather_device(el, ptr(o["m_last"]), n, ptr(p["d_last"]), nl, ptr(o["xw"]), s),
        lambda: pose_optimize_device(el, ptr(dkl.kps), keep, n, u, ptr(o["xw"]), FX, FX, CX, CY, MBF, ptr(p["T0"]), ptr(o["res"]),
                                     ptr(o["outl"]), s),
    ]


def host(o):
    return {k: v.cpu().numpy().tobytes() for k, v in o.items()}


def test_two_problems_on_two_streams_equal_the_calls_in_sequence():
    el, er = extractors(2000)
    _, gl, gr = synth(4)
    dkl, dkr = FrameKeys(el), FrameKeys(er)
    dkl.enqueue(el, upload(gl), H, W, W)
    dkr.enqueue(er, upload(gr), H, W, W)
    torch.cuda.synchronize()
    kl, dl = dkl.host()
    kr, dr = dkr.host()
    cap = el.capacity()
    # two independent problems of different sizes: every key, and every third key with a smaller map
    probs = [problem(el, er, kl, dl, kr, dr, np.arange(len(kl)), (0.01, -0.02, 0.005), 1),
             problem(el, er, kl, dl, kr, dr, np.arange(0, len(kl), 3), (-0.015, 0.01, 0.02), 2)]
    assert len(probs[0]["local"]) > 2 * len(probs[1]["local"]) > 40

    # the reference: every call of both problems one after the other on one stream
    one = torch.cuda.Stream()
    seq = [outputs(cap, len(p["local"])) for p in probs]
    for p, o in zip(probs, seq):
        for c in calls(el, er, dkl, dkr, p, o, one.cuda_stream):
            c()
    one.synchronize()
    for o in seq:
        res = result_from_bytes(o["res"].cpu().numpy())
        assert int(o["n_last"].cpu()[0]) > 20 and int(o["n_loc"].cpu()[0]) > 20 and res.n_initial > 20
        assert np.isfinite(o["red"].cpu().numpy()).sum() > 20
    seq = [host(o) for o in seq]

    # the same calls, each problem on its own stream, issued alternately; neither stream waits on the other
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    par = [outputs(cap, len(p["local"])) for p in probs]
    pending = [calls(el, er, dkl, dkr, p, o, s.cuda_stream) for p, o, s in zip(probs, par, streams)]
    for a, b in zip(*pending):
        a()
        b()
    for s in streams:
        s.synchronize()
    for ref, o in zip(seq, par):
        got = host(o)
        for k in ref:
            assert got[k] == ref[k], k
