#!/usr/bin/env python
"""Information-selection benchmark: SIVO's map-point selection (Tracking.cc:470-520 / 953-1000) on the Frame tail's device outputs.
Prints one JSON line {"metric": "info select", ...}.

  python tools/info_select_bench.py [--steps 200] [--warmup 20] [--blocks-of 10]

Reports:
  (a) device_call_ms: sivo_info_select_device on the KITTI fixture frame's crop (ORB(2000); the right image is the left one shifted by
      12 px), CUDA events around the call, median / p90 over --steps calls;
  (b) host_call_ms: sivo_info_select, the host form on the same keys gathered on the host, end to end (host wall time);
  (c) frames/s of the device chain SegNet (Basic T=6) + ORB(2000) x2 + semantic keys + stereo, without and with the selection
      appended, on the headline benchmark's synthetic 1024x352 frames, the two legs alternating in blocks of --blocks-of frames.
The camera is the KITTI one (KITTI00-02.yaml) at the identity pose with StereoInitialization's pose covariance (1e-6 I) and
threshold (0).  Writes nothing into the source tree."""
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
THRESHOLD = 0.0  # Tracking::StereoInitialization's


def run(args):
    import gc

    import cv2
    import torch
    from sivo_b200 import BayesianSegNet, BayesianSegNetParams, ORBextractor, info_select, info_select_device, make_camera
    from sivo_b200.frame import DeviceFrame
    from sivo_b200.synth import bgr_to_gray
    if not torch.cuda.is_available():
        raise SystemExit("info_select_bench.py needs a CUDA device (there is no CPU fallback for the product path)")
    dev = torch.device("cuda", 0)
    T = 6
    _, proto, model, _ = model_files("basic", T, model_cache_dir())
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=T)
    el, er = (ORBextractor(args.nfeatures, 1.2, 8, 20, 7) for _ in range(2))
    cam = make_camera(FX, FX, CX, CY, MB, np.eye(3), np.zeros(3), 1e-6 * np.eye(6))
    cap = el.capacity()
    NBUF = 3
    F = [DeviceFrame(el, er, NET_H, NET_W) for _ in range(NBUF)]
    world = [torch.empty(cap * 3, dtype=torch.float32, device=dev) for _ in range(NBUF)]
    red = [torch.empty(cap, dtype=torch.float64, device=dev) for _ in range(NBUF)]
    sel = [torch.empty(cap, dtype=torch.int32, device=dev) for _ in range(NBUF)]
    n_sel = [torch.empty(1, dtype=torch.int64, device=dev) for _ in range(NBUF)]
    stream = torch.cuda.Stream(dev)
    s = stream.cuda_stream
    ev = [torch.cuda.Event() for _ in range(NBUF)]
    torch.cuda.synchronize(dev)

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
        ev[k].record(stream)

    # (a) / (b) on the KITTI crop
    img = cv2.imread(os.path.join(ROOT, "tests", "golden", "kitti_000000_1242x375.png"))
    gray = bgr_to_gray(img)[CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W]
    kitti = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in
             (img[CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W], gray, np.roll(gray, -12, axis=1))]
    torch.cuda.synchronize(dev)
    for _ in range(2):  # the first run captures the network's graph
        step(*kitti, 0, True)
    stream.synchronize()
    m, kidx, _, h_z = F[0].host()
    kps = F[0].left.host()[0][kidx]
    h_ent = F[0].out["kp_entropy"].cpu().numpy()[kidx]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ms, host_ms = [], []
    gc.collect()
    gc.disable()
    for i in range(args.warmup + args.steps):
        e0.record(stream)
        select(0)
        e1.record(stream)
        e1.synchronize()
        t0 = time.perf_counter()
        hw_, hr, hs = info_select(el, kps, h_z, h_ent, cam, THRESHOLD)
        t1 = time.perf_counter()
        if i >= args.warmup:
            dev_ms.append(e0.elapsed_time(e1))
            host_ms.append(1e3 * (t1 - t0))
    gc.enable()
    same = (red[0][:m].cpu().numpy().tobytes() == hr.tobytes() and int(n_sel[0].cpu()[0]) == len(hs)
            and sel[0][:len(hs)].cpu().numpy().tobytes() == hs.tobytes())

    # (c) chain throughput without / with the selection, alternating blocks; bounded run-ahead as in bench.py's device step
    fr = frames(8)
    chain = [[torch.from_numpy(np.ascontiguousarray(f[0][CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W])).to(dev),
              torch.from_numpy(f[1]).to(dev), torch.from_numpy(f[2]).to(dev)] for f in fr]
    torch.cuda.synchronize(dev)
    fps_blocks = {"without_select": [], "with_select": []}
    total = {k: [0, 0.0] for k in fps_blocks}
    n_blocks = max(1, -(-(args.warmup + args.steps) // args.blocks_of))
    i = 0
    gc.collect()
    gc.disable()
    for b in range(n_blocks + 2):
        for name in (("without_select", "with_select") if b % 2 == 0 else ("with_select", "without_select")):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            for _ in range(args.blocks_of):
                step(*chain[i % len(chain)], i % NBUF, name == "with_select")
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
    med = lambda v: float(np.median(v))
    p90 = lambda v: float(np.percentile(v, 90))
    line = {"metric": "info select", "unit": "ms",
            "device_call_ms": {"median": med(dev_ms), "p90": p90(dev_ms)},
            "host_call_ms": {"median": med(host_ms), "p90": p90(host_ms)},
            "semantic_keys": m, "keys_with_depth": int((h_z > 0).sum()), "selected": len(hs), "device_equals_host": bool(same),
            "chain_fps": {name: {"overall": total[name][0] / total[name][1], "median_block": med(fps_blocks[name]),
                                 "frames": total[name][0]} for name in fps_blocks},
            "calls_timed": args.steps, "warmup": args.warmup, "gpu": gpu, "power_limit_w": power,
            "workload": f"(a, b) KITTI fixture crop, ORB({args.nfeatures}), Sigma 1e-6 I, identity pose, threshold {THRESHOLD}; "
                        f"(c) Bayesian SegNet Basic T={T} + ORB({args.nfeatures}) x2 + semantic keys + stereo, synthetic 1024x352 frames"}
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
