#!/usr/bin/env python
"""Frame-tail benchmark: the two steps the reference runs on every frame right after the extractors (Frame.cc:131-145),
SelectSemanticKeys and then ComputeStereoMatches over the kept keys, finished from the device pipeline's outputs.  Prints one JSON
line {"metric": "frame tail", ...}.

  python tools/frame_tail_bench.py [--steps 200] [--warmup 20] [--blocks-of 10]

Workload: Bayesian SegNet Basic T=6 + ORB(2000) x2 on synthetic 1024x352 stereo frames resident in HBM (the headline benchmark's
workload helpers and cached calibrated model), KITTI mbf = 386.1448, mb = mbf / 718.856.  Reports, as medians over --steps frames
after --warmup:
  (a) host_tail_ms: today's tail from device outputs -- synchronise, download both keypoint sets and descriptors, the host
      semantic_keys call, host compaction of the kept keys, the host stereo_match call (host wall time per frame);
  (b) device_tail_ms: the same tail through semantic_keys_device + stereo_match_device, ending in one stream synchronisation;
  (c) frames/s of the full device step (SegNet + both extractors) without and with the device tail enqueued after it, the two
      legs alternating in blocks of --blocks-of frames.
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

MBF = 386.1448  # Camera.bf of config/kitti/KITTI00-02.yaml
MB = MBF / 718.856  # bf / fx


def run(args):
    import gc

    import torch
    from sivo_b200 import BayesianSegNet, BayesianSegNetParams, ORBextractor, stereo_match
    from sivo_b200.frame import DeviceFrame
    if not torch.cuda.is_available():
        raise SystemExit("frame_tail_bench.py needs a CUDA device (there is no CPU fallback for the product path)")
    dev = torch.device("cuda", 0)
    T = 6
    _, proto, model, _ = model_files("basic", T, model_cache_dir())
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=T)
    el, er = (ORBextractor(args.nfeatures, 1.2, 8, 20, 7) for _ in range(2))
    if not (el.has_device_tree() and er.has_device_tree()):
        raise SystemExit("frame_tail_bench.py needs the extractors' asynchronous (device quad tree) form")
    n_frames, NBUF = 8, 3
    fr = frames(n_frames)
    d_bgr = [torch.from_numpy(np.ascontiguousarray(f[0][CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W])).to(dev) for f in fr]
    d_gray = [[torch.from_numpy(f[1]).to(dev), torch.from_numpy(f[2]).to(dev)] for f in fr]
    F = [DeviceFrame(el, er, NET_H, NET_W) for _ in range(NBUF)]
    stream = torch.cuda.Stream(dev)  # a real stream: the library's NULL would mean its own
    s = stream.cuda_stream
    ev = [torch.cuda.Event() for _ in range(NBUF)]
    torch.cuda.synchronize(dev)

    def step(i, tail):
        """The device step (SegNet, both extractors joined on the main stream), optionally followed by the device tail."""
        j, k = i % n_frames, i % NBUF
        F[k].extract(seg, d_bgr[j], *d_gray[j], s)  # the extractors first wait for the previous step's tail
        if tail:
            F[k].tail(seg, MB, MBF, s)
        else:
            er.stream_wait(s)
        ev[k].record(stream)

    def host_tail(k):
        kl, dl = F[k].left.host()
        kr, dr = F[k].right.host()
        sel = seg.semantic_keys(kl, 8)[3]
        return stereo_match(el, er, kl[sel], dl[sel], kr, dr, MB, MBF)

    # (a) / (b): per frame, the device step completes, then both tails run on its outputs (alternating which goes first)
    times = {"host": [], "device": []}
    mismatches = 0
    for i in range(NBUF * n_frames):  # graph capture for the stream and first use of every buffer
        step(i, False)
        step(i, True)
    torch.cuda.synchronize(dev)
    gc.collect()
    gc.disable()
    for i in range(args.warmup + args.steps):
        k = i % NBUF
        step(i, False)
        torch.cuda.synchronize(dev)
        res = {}
        for name in (("host", "device") if i % 2 == 0 else ("device", "host")):
            t0 = time.perf_counter()
            if name == "host":
                res[name] = host_tail(k)
            else:
                F[k].tail(seg, MB, MBF, s)
                stream.synchronize()
            if i >= args.warmup:
                times[name].append(1e3 * (time.perf_counter() - t0))
        _, _, u, z = F[k].host()
        mismatches += int(u.tobytes() != res["host"][0].tobytes() or z.tobytes() != res["host"][1].tobytes())
    gc.enable()

    # (c): device-step throughput without / with the tail, alternating blocks; bounded run-ahead as in bench.py's device_step
    fps_blocks = {"without_tail": [], "with_tail": []}
    total = {"without_tail": [0, 0.0], "with_tail": [0, 0.0]}
    n_blocks = max(1, -(-(args.warmup + args.steps) // args.blocks_of))
    i = 0
    gc.collect()
    gc.disable()
    for b in range(n_blocks + 2):
        for name in (("without_tail", "with_tail") if b % 2 == 0 else ("with_tail", "without_tail")):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            for _ in range(args.blocks_of):
                step(i, name == "with_tail")
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
    line = {"metric": "frame tail", "unit": "ms",
            "host_tail_ms": {"median": med(times["host"]), "p90": float(np.percentile(times["host"], 90))},
            "device_tail_ms": {"median": med(times["device"]), "p90": float(np.percentile(times["device"], 90))},
            "tail_speedup_median": med(times["host"]) / med(times["device"]),
            "device_step_fps": {name: {"overall": total[name][0] / total[name][1], "median_block": med(fps_blocks[name]),
                                       "frames": total[name][0]} for name in fps_blocks},
            "tail_result_mismatches": mismatches, "frames_timed": args.steps, "warmup": args.warmup,
            "gpu": gpu, "power_limit_w": power,
            "workload": f"Bayesian SegNet Basic T={T} + ORB({args.nfeatures}) x2, synthetic 1024x352 frames resident in HBM, "
                        f"SelectSemanticKeys (classes <= 8) + ComputeStereoMatches (mbf {MBF}, mb {MB:.6f})"}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed frames per measurement")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--blocks-of", type=int, default=10, help="frames per alternating block of the throughput legs")
    ap.add_argument("--nfeatures", type=int, default=2000)
    args = ap.parse_args()
    if args.steps < 1 or args.blocks_of < 1:
        ap.error("--steps and --blocks-of must be at least 1")
    run(args)


if __name__ == "__main__":
    main()
