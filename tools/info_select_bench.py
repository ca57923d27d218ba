#!/usr/bin/env python
"""Information-selection benchmark: SIVO's map-point selection (Tracking.cc:470-520 / 953-1000) on the Frame tail's device outputs.
Prints one JSON line {"metric": "info select", ...}, timed as DESIGN.md §7 describes.

  python tools/info_select_bench.py [--steps 200] [--warmup 20] [--blocks-of 10]

Reports:
  (a) device_call_ms: sivo_info_select_device on the KITTI fixture frame's crop (ORB(2000); the right image is the left one shifted by
      12 px), median / p90 over --steps calls;
  (b) host_call_ms: sivo_info_select, the host form on the same keys gathered on the host, end to end;
  (c) frames/s of the device chain SegNet (Basic T=6) + ORB(2000) x2 + semantic keys + stereo, without and with the selection
      appended, on the headline benchmark's synthetic 1024x352 frames, the two legs alternating in blocks of --blocks-of frames.
The camera is the KITTI one (KITTI00-02.yaml) at the identity pose with StereoInitialization's pose covariance (1e-6 I) and
threshold (0).  Writes nothing into the source tree."""
import argparse
import json

import numpy as np

from bench_support import (CROP_X, CROP_Y, NET_H, NET_W, add_common_args, alternate, basic_front_end, card, chain_frames,
                           check_device_trees, device_ms, host_ms, kitti_frame, require_cuda, stats)

FX, CX, CY, MBF = 718.856, 607.1928 - CROP_X, 185.2157 - CROP_Y, 386.1448  # KITTI00-02.yaml, principal point in the crop
MB = MBF / FX
THRESHOLD = 0.0  # Tracking::StereoInitialization's


def run(args):
    import torch
    from sivo_b200 import info_select, info_select_device, make_camera
    from sivo_b200.frame import DeviceFrame
    T = 6
    seg, el, er = basic_front_end(args.nfeatures, T)
    cam = make_camera(FX, FX, CX, CY, MB, np.eye(3), np.zeros(3), 1e-6 * np.eye(6))
    cap = el.capacity()
    NBUF = 3
    F = [DeviceFrame(el, er, NET_H, NET_W) for _ in range(NBUF)]
    world = [torch.empty(cap * 3, dtype=torch.float32, device="cuda") for _ in range(NBUF)]
    red = [torch.empty(cap, dtype=torch.float64, device="cuda") for _ in range(NBUF)]
    sel = [torch.empty(cap, dtype=torch.int32, device="cuda") for _ in range(NBUF)]
    n_sel = [torch.empty(1, dtype=torch.int64, device="cuda") for _ in range(NBUF)]
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    torch.cuda.synchronize()

    def select(k):
        f = F[k]
        info_select_device(el, f.kps, f.kp_entropy, f.keep, f.n_keep, f.depth, cam, THRESHOLD, world[k].data_ptr(), red[k].data_ptr(),
                           sel[k].data_ptr(), n_sel[k].data_ptr(), s)

    def step(bgr, gl, gr, k, with_select):
        """SegNet, both extractors, semantic keys and stereo on the main stream, optionally followed by the selection."""
        F[k].extract(seg, bgr, gl, gr, s)  # the extractors first wait for the previous step's tail and selection
        F[k].tail(seg, MB, MBF, s)
        if with_select:
            select(k)

    # (a) / (b) on the KITTI crop
    kitti = kitti_frame()
    for _ in range(2):  # the first run captures the network's graph
        step(*kitti, 0, True)
    stream.synchronize()
    m, kidx, _, h_z = F[0].host()
    kps = F[0].left.host()[0][kidx]
    h_ent = F[0].out["kp_entropy"].cpu().numpy()[kidx]
    dev_ms = device_ms(lambda: select(0), stream, args.warmup, args.steps)
    hw_, hr, hs = info_select(el, kps, h_z, h_ent, cam, THRESHOLD)
    host = host_ms(lambda: info_select(el, kps, h_z, h_ent, cam, THRESHOLD), args.warmup, args.steps)
    same = (red[0][:m].cpu().numpy().tobytes() == hr.tobytes() and int(n_sel[0].cpu()[0]) == len(hs)
            and sel[0][:len(hs)].cpu().numpy().tobytes() == hs.tobytes())

    # (c) chain throughput without / with the selection
    chain = chain_frames(8)
    fps = alternate({"without_select": lambda i, k: step(*chain[i % len(chain)], k, False),
                     "with_select": lambda i, k: step(*chain[i % len(chain)], k, True)}, stream, args.steps, args.warmup, args.blocks_of, NBUF)
    check_device_trees(el, er)

    line = {"metric": "info select", "unit": "ms", "device_call_ms": stats(dev_ms), "host_call_ms": stats(host),
            "semantic_keys": m, "keys_with_depth": int((h_z > 0).sum()), "selected": len(hs), "device_equals_host": bool(same),
            "chain_fps": fps, "calls_timed": args.steps, "warmup": args.warmup, **card(),
            "workload": f"(a, b) KITTI fixture crop, ORB({args.nfeatures}), Sigma 1e-6 I, identity pose, threshold {THRESHOLD}; "
                        f"(c) Bayesian SegNet Basic T={T} + ORB({args.nfeatures}) x2 + semantic keys + stereo, synthetic 1024x352 frames"}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    add_common_args(ap, steps=200, warmup=20, chain=True)
    args = ap.parse_args()
    require_cuda("info_select_bench.py")
    run(args)

if __name__ == "__main__":
    main()
