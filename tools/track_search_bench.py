#!/usr/bin/env python
"""Projection-search benchmark: the local-map and last-frame searches (ORBmatcher::SearchByProjection) on the Frame tail's device
outputs.  Prints one JSON line {"metric": "track search", ...}.

  python tools/track_search_bench.py [--steps 200] [--warmup 20] [--blocks-of 10]

Reports:
  (a) device_call_ms: sivo_search_local_points_device (th 1) and sivo_search_last_frame_device (th 7) on the KITTI fixture frame's
      crop (ORB(2000); the right image is the left one shifted by 12 px) at 1000, 3000 and 6000 map points, CUDA events around
      the call, median / p90 over --steps calls; local_no_claims is the local search with every point unobserved, so that
      no claim blocks a key and the ordered pass searches no point again;
  (b) host_call_ms: the host forms on the same keys gathered on the host, end to end (host wall time);
  (c) frames/s of the device chain SegNet (Basic T=6) + ORB(2000) x2 + semantic keys + stereo, without and with both searches
      (3000 points) appended, on the headline benchmark's synthetic 1024x352 frames, the two legs alternating in blocks.
The map points are the KITTI frame's semantic keys with depth, unprojected at the identity pose (MapPoint::UpdateNormalAndDepth's
distances and normal), then random points in front of the camera up to the count; the search runs at a small motion.
Writes nothing into the source tree."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import CROP_X, CROP_Y, NET_H, NET_W, frames, model_cache_dir, model_files  # noqa: E402

FX, CX, CY, MBF = 718.856, 607.1928 - CROP_X, 185.2157 - CROP_Y, 386.1448  # KITTI00-02.yaml, principal point in the crop
MB = MBF / FX
COUNTS = (1000, 3000, 6000)


def make_points(kps, desc, depth, scale, n, rng):
    from oracle.track_oracle import map_points_from_keys
    from sivo_b200 import MAP_POINT_DTYPE, map_points
    f, idx = map_points_from_keys(kps, depth, np.eye(3), np.zeros(3), FX, FX, CX, CY, scale)
    base = map_points(desc[idx], f["pos"], f["normal"], f["min_distance"], f["max_distance"], 1, kps["octave"][idx], kps["angle"][idx])
    rnd = np.zeros(max(n - len(base), 0), MAP_POINT_DTYPE)
    z = rng.uniform(3, 60, len(rnd))
    rnd["pos"] = np.c_[(rng.uniform(0, NET_W, len(rnd)) - CX) * z / FX, (rng.uniform(0, NET_H, len(rnd)) - CY) * z / FX, z]
    rnd["normal"] = rnd["pos"] / np.linalg.norm(rnd["pos"], axis=1, keepdims=True)
    d = np.linalg.norm(rnd["pos"], axis=1)
    rnd["max_distance"], rnd["min_distance"] = d * 1.5, d / 3
    rnd["desc"] = rng.integers(0, 256, (len(rnd), 32))
    rnd["octave"] = rng.integers(0, len(scale), len(rnd))
    rnd["observed"] = 1
    pts = np.concatenate([base, rnd])[:n]
    return pts[rng.permutation(len(pts))]


def run(args):
    import gc

    import cv2
    import torch
    from sivo_b200 import (BayesianSegNet, BayesianSegNetParams, ORBextractor, make_frame, search_last_frame, search_last_frame_device,
                           search_local_points, search_local_points_device)
    from sivo_b200.frame import DeviceFrame
    from sivo_b200.synth import bgr_to_gray
    if not torch.cuda.is_available():
        raise SystemExit("track_search_bench.py needs a CUDA device (there is no CPU fallback for the product path)")
    dev = torch.device("cuda", 0)
    T = 6
    _, proto, model, _ = model_files("basic", T, model_cache_dir())
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=T)
    el, er = (ORBextractor(args.nfeatures, 1.2, 8, 20, 7) for _ in range(2))
    c, s_ = np.cos(0.01), np.sin(0.01)
    frame = make_frame(FX, FX, CX, CY, MBF, (0.0, float(NET_W), 0.0, float(NET_H)), [[c, 0, s_], [0, 1, 0], [-s_, 0, c]], (0.02, -0.01, 0.3))
    cap = el.capacity()
    NBUF = 3
    F = [DeviceFrame(el, er, NET_H, NET_W) for _ in range(NBUF)]
    match = [torch.empty(cap, dtype=torch.int32, device=dev) for _ in range(NBUF)]
    n_m = [torch.empty(2, dtype=torch.int64, device=dev) for _ in range(NBUF)]
    in_view = torch.empty(max(COUNTS), dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(dev)
    s = stream.cuda_stream
    ev = [torch.cuda.Event() for _ in range(NBUF)]
    torch.cuda.synchronize(dev)

    def searches(k, pts_dev, n_points, local=True, last=True):
        f = F[k]
        if last:
            search_last_frame_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, pts_dev.data_ptr(), n_points, frame, np.eye(3), np.zeros(3),
                                     7.0, match[k].data_ptr(), n_m[k][1:].data_ptr(), s)
        if local:
            search_local_points_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, 0, pts_dev.data_ptr(), n_points, frame, 1.0, 0.8,
                                       in_view.data_ptr(), match[k].data_ptr(), n_m[k].data_ptr(), s)

    def step(bgr, gl, gr, k, pts_dev=None):
        F[k].extract(seg, bgr, gl, gr, s)  # the extractors first wait for the previous step's tail and searches
        F[k].tail(seg, MB, MBF, s)
        if pts_dev is not None:
            searches(k, pts_dev, pts_dev.numel() // 80)
        ev[k].record(stream)

    # (a) / (b) on the KITTI crop
    img = cv2.imread(os.path.join(ROOT, "tests", "golden", "kitti_000000_1242x375.png"))
    gray = bgr_to_gray(img)[CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W]
    kitti = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in
             (img[CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W], gray, np.roll(gray, -12, axis=1))]
    torch.cuda.synchronize(dev)
    for _ in range(2):  # the first run captures the network's graph
        step(*kitti, 0)
    stream.synchronize()
    m, kidx, h_ur, h_z = F[0].host()
    h_kps, h_desc = (a[kidx] for a in F[0].left.host())
    rng = np.random.default_rng(0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    med = lambda v: float(np.median(v))
    p90 = lambda v: float(np.percentile(v, 90))
    calls = {}
    pts_by_n = {}
    for n in COUNTS:
        pts = make_points(h_kps, h_desc, h_z, el.GetScaleFactors(), n, rng)
        pts_by_n[n] = pts
        pts_dev = torch.from_numpy(pts.view(np.uint8).reshape(-1).copy()).to(dev)
        free = pts.copy()
        free["observed"] = 0
        free_dev = torch.from_numpy(free.view(np.uint8).reshape(-1).copy()).to(dev)
        torch.cuda.synchronize(dev)
        res = {}
        for name, kw, pd in (("local", {"last": False}, pts_dev), ("last_frame", {"local": False}, pts_dev),
                             ("local_no_claims", {"last": False}, free_dev)):
            dev_ms, host_ms = [], []
            gc.collect()
            gc.disable()
            for i in range(args.warmup + args.steps):
                e0.record(stream)
                searches(0, pd, n, **kw)
                e1.record(stream)
                e1.synchronize()
                if name != "local_no_claims":
                    t0 = time.perf_counter()
                    if name == "local":
                        hv, hm, hn = search_local_points(el, h_kps, h_desc, h_ur, pts, frame, 1.0)
                    else:
                        hm, hn = search_last_frame(el, h_kps, h_desc, h_ur, pts, frame, np.eye(3), np.zeros(3), 7.0)
                    t1 = time.perf_counter()
                if i >= args.warmup:
                    dev_ms.append(e0.elapsed_time(e1))
                    if name != "local_no_claims":
                        host_ms.append(1e3 * (t1 - t0))
            gc.enable()
            r = {"device_call_ms": {"median": med(dev_ms), "p90": p90(dev_ms)}}
            if host_ms:
                r["host_call_ms"] = {"median": med(host_ms), "p90": p90(host_ms)}
                got = int(n_m[0][0 if name == "local" else 1].cpu())
                r["matches"] = int(hn)
                r["device_equals_host"] = bool(got == hn and match[0][:m].cpu().numpy().tobytes() == hm.tobytes())
            res[name] = r
        calls[str(n)] = res

    # (c) chain throughput without / with both searches, alternating blocks; bounded run-ahead as in bench.py's device step
    chain_pts = torch.from_numpy(pts_by_n[3000].view(np.uint8).reshape(-1).copy()).to(dev)
    fr = frames(8)
    chain = [[torch.from_numpy(np.ascontiguousarray(f[0][CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W])).to(dev),
              torch.from_numpy(f[1]).to(dev), torch.from_numpy(f[2]).to(dev)] for f in fr]
    torch.cuda.synchronize(dev)
    fps_blocks = {"without_search": [], "with_search": []}
    total = {k: [0, 0.0] for k in fps_blocks}
    n_blocks = max(1, -(-(args.warmup + args.steps) // args.blocks_of))
    i = 0
    gc.collect()
    gc.disable()
    for b in range(n_blocks + 2):
        for name in (("without_search", "with_search") if b % 2 == 0 else ("with_search", "without_search")):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            for _ in range(args.blocks_of):
                step(*chain[i % len(chain)], i % NBUF, chain_pts if name == "with_search" else None)
                if (i & 3) == 3:
                    ev[(i - 1) % NBUF].synchronize()
                i += 1
            torch.cuda.synchronize(dev)
            dt = time.perf_counter() - t0
            if b >= 2:  # the first two blocks of each leg are warm-up
                fps_blocks[name].append(args.blocks_of / dt)
                total[name][0] += args.blocks_of
                total[name][1] += dt
    gc.enable()
    if el.device_status() or er.device_status():
        raise SystemExit("a pyramid level exceeded the device quad tree's capacity: the asynchronous outputs are not valid")

    gpu, power = torch.cuda.get_device_name(dev), None
    try:
        import pynvml
        pynvml.nvmlInit()
        power = pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(0)) / 1e3
    except Exception:
        pass
    line = {"metric": "track search", "unit": "ms", "calls": calls, "semantic_keys": m, "keys_with_depth": int((h_z > 0).sum()),
            "chain_fps": {name: {"overall": total[name][0] / total[name][1], "median_block": med(fps_blocks[name]),
                                 "frames": total[name][0]} for name in fps_blocks},
            "calls_timed": args.steps, "warmup": args.warmup, "gpu": gpu, "power_limit_w": power,
            "workload": f"(a, b) KITTI fixture crop, ORB({args.nfeatures}), local th 1 / last frame th 7, small motion; "
                        f"(c) Bayesian SegNet Basic T={T} + ORB({args.nfeatures}) x2 + semantic keys + stereo (+ both searches, 3000 points), "
                        "synthetic 1024x352 frames"}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed calls / frames per measurement")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--blocks-of", type=int, default=10, help="frames per alternating block of the throughput legs")
    ap.add_argument("--nfeatures", type=int, default=2000)
    args = ap.parse_args()
    if args.steps < 1 or args.blocks_of < 1:
        ap.error("--steps and --blocks-of must be at least 1")
    run(args)


if __name__ == "__main__":
    main()
