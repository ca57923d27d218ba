#!/usr/bin/env python
"""Projection-search benchmark: the local-map and last-frame searches (ORBmatcher::SearchByProjection) on the Frame tail's device
outputs.  Prints one JSON line {"metric": "track search", ...}, timed as DESIGN.md §7 describes.

  python tools/track_search_bench.py [--steps 200] [--warmup 20] [--blocks-of 10]

Reports:
  (a) device_call_ms: sivo_search_local_points_device (th 1) and sivo_search_last_frame_device (th 7) on the KITTI fixture frame's
      crop (ORB(2000); the right image is the left one shifted by 12 px) at 1000, 3000 and 6000 map points, median / p90 over
      --steps calls; local_no_claims is the local search with every point unobserved, so that
      no claim blocks a key and the ordered pass searches no point again;
  (b) host_call_ms: the host forms on the same keys gathered on the host, end to end;
  (c) frames/s of the device chain SegNet (Basic T=6) + ORB(2000) x2 + semantic keys + stereo, without and with both searches
      (3000 points) appended, on the headline benchmark's synthetic 1024x352 frames, the two legs alternating in blocks.
The map points are the KITTI frame's semantic keys with depth, unprojected at the identity pose (MapPoint::UpdateNormalAndDepth's
distances and normal), then random points in front of the camera up to the count; the search runs at a small motion.
Writes nothing into the source tree."""
import argparse
import json

import numpy as np

from bench_support import (CROP_X, CROP_Y, NET_H, NET_W, add_common_args, alternate, basic_front_end, card, chain_frames,
                           check_device_trees, device_ms, host_ms, kitti_frame, require_cuda, stats)

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
    import torch
    from sivo_b200 import make_frame, search_last_frame, search_last_frame_device, search_local_points, search_local_points_device
    from sivo_b200.frame import DeviceFrame
    T = 6
    seg, el, er = basic_front_end(args.nfeatures, T)
    c, s_ = np.cos(0.01), np.sin(0.01)
    frame = make_frame(FX, FX, CX, CY, MBF, (0.0, float(NET_W), 0.0, float(NET_H)), [[c, 0, s_], [0, 1, 0], [-s_, 0, c]], (0.02, -0.01, 0.3))
    cap = el.capacity()
    NBUF = 3
    F = [DeviceFrame(el, er, NET_H, NET_W) for _ in range(NBUF)]
    match = [torch.empty(cap, dtype=torch.int32, device="cuda") for _ in range(NBUF)]
    n_m = [torch.empty(2, dtype=torch.int64, device="cuda") for _ in range(NBUF)]
    in_view = torch.empty(max(COUNTS), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    torch.cuda.synchronize()

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

    # (a) / (b) on the KITTI crop
    kitti = kitti_frame()
    for _ in range(2):  # the first run captures the network's graph
        step(*kitti, 0)
    stream.synchronize()
    m, kidx, h_ur, h_z = F[0].host()
    h_kps, h_desc = (a[kidx] for a in F[0].left.host())
    rng = np.random.default_rng(0)
    calls = {}
    pts_by_n = {}
    for n in COUNTS:
        pts = make_points(h_kps, h_desc, h_z, el.GetScaleFactors(), n, rng)
        pts_by_n[n] = pts
        pts_dev = torch.from_numpy(pts.view(np.uint8).reshape(-1).copy()).cuda()
        free = pts.copy()
        free["observed"] = 0
        free_dev = torch.from_numpy(free.view(np.uint8).reshape(-1).copy()).cuda()
        torch.cuda.synchronize()
        host = {"local": lambda: search_local_points(el, h_kps, h_desc, h_ur, pts, frame, 1.0)[1:],
                "last_frame": lambda: search_last_frame(el, h_kps, h_desc, h_ur, pts, frame, np.eye(3), np.zeros(3), 7.0)}
        res = {}
        for name, kw, pd in (("local", {"last": False}, pts_dev), ("last_frame", {"local": False}, pts_dev),
                             ("local_no_claims", {"last": False}, free_dev)):
            r = {"device_call_ms": stats(device_ms(lambda: searches(0, pd, n, **kw), stream, args.warmup, args.steps))}
            if name in host:
                r["host_call_ms"] = stats(host_ms(host[name], args.warmup, args.steps))
                hm, hn = host[name]()
                got = int(n_m[0][0 if name == "local" else 1].cpu())
                r["matches"] = int(hn)
                r["device_equals_host"] = bool(got == hn and match[0][:m].cpu().numpy().tobytes() == hm.tobytes())
            res[name] = r
        calls[str(n)] = res

    # (c) chain throughput without / with both searches
    chain_pts = torch.from_numpy(pts_by_n[3000].view(np.uint8).reshape(-1).copy()).cuda()
    chain = chain_frames(8)
    fps = alternate({"without_search": lambda i, k: step(*chain[i % len(chain)], k),
                     "with_search": lambda i, k: step(*chain[i % len(chain)], k, chain_pts)}, stream, args.steps, args.warmup, args.blocks_of,
                    NBUF)
    check_device_trees(el, er)

    line = {"metric": "track search", "unit": "ms", "calls": calls, "semantic_keys": m, "keys_with_depth": int((h_z > 0).sum()),
            "chain_fps": fps, "calls_timed": args.steps, "warmup": args.warmup, **card(),
            "workload": f"(a, b) KITTI fixture crop, ORB({args.nfeatures}), local th 1 / last frame th 7, small motion; "
                        f"(c) Bayesian SegNet Basic T={T} + ORB({args.nfeatures}) x2 + semantic keys + stereo (+ both searches, 3000 points), "
                        "synthetic 1024x352 frames"}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    add_common_args(ap, steps=200, warmup=20, chain=True)
    args = ap.parse_args()
    require_cuda("track_search_bench.py")
    run(args)

if __name__ == "__main__":
    main()
