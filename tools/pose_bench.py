#!/usr/bin/env python
"""Frame-pose benchmark: Optimizer::PoseOptimization on the device (sivo_pose_optimize_device).  Prints one JSON line
{"metric": "pose optimisation", ...}, timed as DESIGN.md §7 describes.

  python tools/pose_bench.py [--steps 30] [--warmup 5] [--blocks-of 10]

Reports:
  (a) device_call_ms: the device call at 100 / 500 / 1000 / 2000 edges with 0 / 30 % gross outliers, median / p90 over --steps
      calls.  The scenes are synthetic (keys at random pixels and depths seen from a known pose, 0.5 px
      noise times the octave's scale, about 60 % stereo, the initial pose moved by up to 0.01 rad / 5 cm), because a 1024x352 frame
      holds fewer semantic keys with depth than the larger counts;
  (b) host_call_ms: the host form on the same scenes, end to end;
  (c) frames/s of Tracking's device chain SegNet (Basic T=6) + ORB(2000) x2 + semantic keys + stereo + last-frame search +
      local-map search, without and with the two optimisations appended the way Tracking runs them: last-frame search -> gather
      -> pose -> the host reads the 512-byte result -> local-map search at that pose -> gather -> pose.  The host read makes
      every frame of the "with" leg wait for its own first optimisation.  Synthetic 1024x352 frames; each frame's map points are
      its own semantic keys with depth unprojected at a known pose (half as last-frame points, half as the local map, one in eight
      moved by 0.5-2 m), found by a first pass of the front end.  The two legs alternate in blocks.
The g2o host loop the kernel replaces (Eigen + CHOLMOD) is not built here: not measured.  Writes nothing into the source tree."""
import argparse
import json

import numpy as np

from bench_support import (CROP_X, CROP_Y, NET_H, NET_W, add_common_args, alternate, basic_front_end, card, chain_frames,
                           check_device_trees, device_ms, host_ms, require_cuda, stats)
from oracle.mapping_scene import rotation

FX, CX, CY, MBF = 718.856, 607.1928 - CROP_X, 185.2157 - CROP_Y, 386.1448  # KITTI00-02.yaml, principal point in the crop
MB = MBF / FX
EDGES = (100, 500, 1000, 2000)


def synthetic_scene(n, outliers, rng):
    """Keys seen from a true pose, their points, u_right (< 0: mono) and the moved initial pose (3 x 4 float)."""
    from sivo_b200 import KP_DTYPE
    R, t = rotation(*rng.uniform(-0.2, 0.2, 3)), rng.uniform(-2, 2, 3)
    u, v, z = rng.uniform(0, NET_W, n), rng.uniform(0, NET_H, n), rng.uniform(3, 40, n)
    X = ((np.stack([(u - CX) * z / FX, (v - CY) * z / FX, z], 1) - t) @ R).astype(np.float32)
    octave = rng.integers(0, 8, n)
    sc = 1.2 ** octave
    kps = np.zeros(n, KP_DTYPE)
    kps["x"], kps["y"], kps["octave"] = u + 0.5 * sc * rng.standard_normal(n), v + 0.5 * sc * rng.standard_normal(n), octave
    ur = np.where(rng.uniform(size=n) < 0.6, np.maximum(u - MBF / z + 0.5 * sc * rng.standard_normal(n), 0), -1).astype(np.float32)
    bad = rng.permutation(n)[:int(round(outliers * n))]
    X[bad] += rng.uniform(-5, 5, (len(bad), 3)).astype(np.float32)
    Tin = np.concatenate([rotation(*rng.uniform(-0.01, 0.01, 3)) @ R, (t + rng.uniform(-0.05, 0.05, 3))[:, None]], 1)
    return kps, ur, X, Tin.astype(np.float32)


def frame_map(kps, desc, depth, scale, rng):
    """Last-frame points and local-map points made from a frame's keys with depth at the identity pose."""
    from oracle.track_oracle import map_points_from_keys
    from sivo_b200 import map_points
    f, idx = map_points_from_keys(kps, depth, np.eye(3), np.zeros(3), FX, FX, CX, CY, scale)
    pts = map_points(desc[idx], f["pos"], f["normal"], f["min_distance"], f["max_distance"], 1, kps["octave"][idx], kps["angle"][idx])
    bad = rng.uniform(size=len(pts)) < 0.125
    pts["pos"][bad] += (rng.uniform(0.5, 2.0, (bad.sum(), 3)) * rng.choice([-1, 1], (bad.sum(), 3))).astype(np.float32)
    return pts[0::2].copy(), pts[1::2].copy()


def run(args):
    import torch
    from sivo_b200 import (KP_DTYPE, make_frame, pose_gather_device, pose_optimize, pose_optimize_device, search_last_frame_device,
                           search_local_points_device)
    from sivo_b200.frame import DeviceFrame
    from sivo_b200.pose import frame_from_result, result_from_bytes
    T = 6
    seg, el, er = basic_front_end(args.nfeatures, T)
    cap = el.capacity()
    u8, i32, i64, f32 = torch.uint8, torch.int32, torch.int64, torch.float32
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    rng = np.random.default_rng(0)

    # (a) / (b)
    kp_buf = torch.zeros(cap * 28, dtype=u8, device="cuda")
    n_buf = torch.zeros(1, dtype=i64, device="cuda")
    ur_buf = torch.zeros(cap, dtype=f32, device="cuda")
    xw_buf = torch.full((3 * cap,), float("nan"), dtype=f32, device="cuda")
    t_buf = torch.zeros(12, dtype=f32, device="cuda")
    res_buf = torch.zeros(512, dtype=u8, device="cuda")
    out_buf = torch.zeros(cap, dtype=u8, device="cuda")
    calls = {}
    for n in EDGES:
        for frac in (0.0, 0.3):
            kps, ur, X, Tin = synthetic_scene(min(n, cap), frac, rng)
            slots = np.zeros(cap, KP_DTYPE)
            slots[:len(kps)] = kps
            kp_buf.copy_(torch.from_numpy(slots.view(np.uint8).reshape(-1).copy()))
            n_buf.fill_(len(kps))
            ur_buf[:len(kps)].copy_(torch.from_numpy(ur))
            xw_buf[:3 * len(kps)].copy_(torch.from_numpy(X.reshape(-1)))
            t_buf.copy_(torch.from_numpy(Tin.reshape(-1)))
            torch.cuda.synchronize()
            dev_ms = device_ms(lambda: pose_optimize_device(el, kp_buf.data_ptr(), 0, n_buf.data_ptr(), ur_buf.data_ptr(), xw_buf.data_ptr(),
                                                            FX, FX, CX, CY, MBF, t_buf.data_ptr(), res_buf.data_ptr(), out_buf.data_ptr(), s),
                               stream, args.warmup, args.steps)
            host = host_ms(lambda: pose_optimize(el, kps, ur, X, Tin, FX, FX, CX, CY, MBF), args.warmup, args.steps)
            hres, _ = pose_optimize(el, kps, ur, X, Tin, FX, FX, CX, CY, MBF)
            dres = result_from_bytes(res_buf.cpu().numpy())
            calls[f"{n}_edges_{int(frac * 100)}pct_outliers"] = {
                "device_call_ms": stats(dev_ms), "host_call_ms": stats(host), "n_good": int(dres.n_good),
                "device_equals_host": bytes(dres) == bytes(hres)}

    # (c) the chain
    bounds = (0.0, float(NET_W), 0.0, float(NET_H))
    frame0 = make_frame(FX, FX, CX, CY, MBF, bounds, rotation(0.001, -0.0015, 0.001), (0.01, -0.005, 0.01))
    T0 = np.concatenate([np.array(frame0.Rcw, np.float32).reshape(3, 3), np.array(frame0.tcw, np.float32)[:, None]], 1)
    B = [{"in": f, "f": DeviceFrame(el, er, NET_H, NET_W), "m1": torch.empty(cap, dtype=i32, device="cuda"),
          "m2": torch.empty(cap, dtype=i32, device="cuda"), "nm": torch.empty(2, dtype=i64, device="cuda"),
          "view": torch.empty(cap, dtype=u8, device="cuda"), "xw": torch.empty(3 * cap, dtype=f32, device="cuda"),
          "T0": torch.from_numpy(T0.reshape(-1).copy()).cuda(), "r1": torch.empty(512, dtype=u8, device="cuda"),
          "r2": torch.empty(512, dtype=u8, device="cuda"), "o": torch.empty(cap, dtype=u8, device="cuda"),
          "r1_host": torch.empty(512, dtype=u8, pin_memory=True)} for f in chain_frames(6)]
    torch.cuda.synchronize()

    def front(b):
        b["f"].extract(seg, *b["in"], s)  # the extractors first wait for the previous step's searches and optimisations
        b["f"].tail(seg, MB, MBF, s)

    def last_search(b):
        f = b["f"]
        search_last_frame_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, b["last"].data_ptr(), b["n_last"], frame0, T0[:, :3], T0[:, 3],
                                 7.0, b["m1"].data_ptr(), b["nm"][1:].data_ptr(), s)

    def local_search(b, frame):
        f = b["f"]
        search_local_points_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, 0, b["local"].data_ptr(), b["n_local"], frame, 1.0, 0.8,
                                   b["view"].data_ptr(), b["m2"].data_ptr(), b["nm"].data_ptr(), s)

    def pose(b, t_in, res):
        f = b["f"]
        pose_optimize_device(el, f.kps, f.keep, f.n_keep, f.u_right, b["xw"].data_ptr(), FX, FX, CX, CY, MBF, t_in.data_ptr(), res.data_ptr(),
                             b["o"].data_ptr(), s)

    def step(b, with_pose):
        nonlocal last_pose
        front(b)
        last_search(b)
        if with_pose:
            with torch.cuda.stream(stream):
                b["xw"].fill_(float("nan"))
            pose_gather_device(el, b["m1"].data_ptr(), b["f"].n_keep, b["last"].data_ptr(), b["n_last"], b["xw"].data_ptr(), s)
            pose(b, b["T0"], b["r1"])
            with torch.cuda.stream(stream):
                b["r1_host"].copy_(b["r1"], non_blocking=True)
            stream.synchronize()  # Tracking's host read: the local-map search takes the pose as a host struct
            frame = frame_from_result(result_from_bytes(b["r1_host"].numpy()), FX, FX, CX, CY, MBF, bounds)
            local_search(b, frame)
            pose_gather_device(el, b["m2"].data_ptr(), b["f"].n_keep, b["local"].data_ptr(), b["n_local"], b["xw"].data_ptr(), s)
            pose(b, b["r1"], b["r2"])
            last_pose = b
        else:
            local_search(b, frame0)

    last_pose = None
    for b in B:  # first pass: the network's graph is captured, and each frame's keys give its map
        front(b)
        stream.synchronize()
        _, kidx, _, depth = b["f"].host()
        kps, desc = (a[kidx] for a in b["f"].left.host())
        last, local = frame_map(kps, desc, depth, el.GetScaleFactors(), rng)
        b["last"], b["local"] = (torch.from_numpy(p.view(np.uint8).reshape(-1).copy()).cuda() for p in (last, local))
        b["n_last"], b["n_local"] = len(last), len(local)
    torch.cuda.synchronize()
    fps = alternate({"without_pose": lambda i, k: step(B[k], False), "with_two_poses": lambda i, k: step(B[k], True)}, stream, args.steps,
                    args.warmup, args.blocks_of, len(B))
    check_device_trees(el, er)
    r2 = result_from_bytes(last_pose["r2"].cpu().numpy())

    line = {"metric": "pose optimisation", "unit": "ms", "calls": calls, "chain_fps": fps,
            "chain_last_second_optimisation": {"n_initial": int(r2.n_initial), "n_good": int(r2.n_good), "sigma_valid": int(r2.sigma_valid)},
            "g2o_host_loop": "not measured (Eigen + CHOLMOD are not built here)", "calls_timed": args.steps, "warmup": args.warmup, **card(),
            "workload": f"(a, b) synthetic scenes, 60 % stereo; (c) Bayesian SegNet Basic T={T} + ORB({args.nfeatures}) x2 + semantic keys + "
                        "stereo + last-frame search (th 7) + local-map search (th 1), with / without gather + pose after each search, "
                        "synthetic 1024x352 frames"}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    add_common_args(ap, steps=30, warmup=5, chain=True)
    args = ap.parse_args()
    require_cuda("pose_bench.py")
    run(args)


if __name__ == "__main__":
    main()
