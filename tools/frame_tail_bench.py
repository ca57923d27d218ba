#!/usr/bin/env python
"""Frame-tail benchmark: the two steps the reference runs on every frame right after the extractors (Frame.cc:131-145),
SelectSemanticKeys and then ComputeStereoMatches over the kept keys, finished from the device pipeline's outputs.  Prints one JSON
line {"metric": "frame tail", ...}, timed as DESIGN.md §7 describes.

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
import gc
import json
import time

from bench_support import (NET_H, NET_W, add_common_args, alternate, basic_front_end, card, chain_frames, check_device_trees,
                           require_cuda, stats)

MBF = 386.1448  # Camera.bf of config/kitti/KITTI00-02.yaml
MB = MBF / 718.856  # bf / fx


def run(args):
    import torch
    from sivo_b200 import stereo_match
    from sivo_b200.frame import DeviceFrame
    T = 6
    seg, el, er = basic_front_end(args.nfeatures, T)
    n_frames, NBUF = 8, 3
    fr = chain_frames(n_frames)
    F = [DeviceFrame(el, er, NET_H, NET_W) for _ in range(NBUF)]
    stream = torch.cuda.Stream()  # a real stream: the library's NULL would mean its own
    s = stream.cuda_stream

    def step(i, k, tail):
        """The device step (SegNet, both extractors joined on the main stream) into slot k, optionally followed by the device tail."""
        F[k].extract(seg, *fr[i % n_frames], s)  # the extractors first wait for the previous step's tail
        if tail:
            F[k].tail(seg, MB, MBF, s)
        else:
            er.stream_wait(s)

    def host_tail(k):
        kl, dl = F[k].left.host()
        kr, dr = F[k].right.host()
        sel = seg.semantic_keys(kl, 8)[3]
        return stereo_match(el, er, kl[sel], dl[sel], kr, dr, MB, MBF)

    # (a) / (b): per frame, the device step completes, then both tails run on its outputs (alternating which goes first)
    times = {"host": [], "device": []}
    mismatches = 0
    for i in range(NBUF * n_frames):  # graph capture for the stream and first use of every buffer
        step(i, i % NBUF, False)
        step(i, i % NBUF, True)
    torch.cuda.synchronize()
    gc.collect()
    gc.disable()
    for i in range(args.warmup + args.steps):
        k = i % NBUF
        step(i, k, False)
        torch.cuda.synchronize()
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

    # (c): device-step throughput without / with the tail
    fps = alternate({"without_tail": lambda i, k: step(i, k, False), "with_tail": lambda i, k: step(i, k, True)}, stream, args.steps,
                    args.warmup, args.blocks_of, NBUF)
    check_device_trees(el, er)

    host, device = stats(times["host"]), stats(times["device"])
    line = {"metric": "frame tail", "unit": "ms", "host_tail_ms": host, "device_tail_ms": device,
            "tail_speedup_median": host["median"] / device["median"], "device_step_fps": fps,
            "tail_result_mismatches": mismatches, "frames_timed": args.steps, "warmup": args.warmup, **card(),
            "workload": f"Bayesian SegNet Basic T={T} + ORB({args.nfeatures}) x2, synthetic 1024x352 frames resident in HBM, "
                        f"SelectSemanticKeys (classes <= 8) + ComputeStereoMatches (mbf {MBF}, mb {MB:.6f})"}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    add_common_args(ap, steps=200, warmup=20, chain=True)
    args = ap.parse_args()
    require_cuda("frame_tail_bench.py")
    run(args)


if __name__ == "__main__":
    main()
