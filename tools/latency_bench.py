#!/usr/bin/env python
"""Latency-mode benchmark (SURVEY 8e, DESIGN §6/§7): milliseconds per frame when one frame's Monte-Carlo samples are split over
G ranks, against the same frame on one whole-frame handle, frames issued one at a time.  Prints one JSON line
{"metric": "ms per frame, latency mode", ...} on rank 0.

  python -m torch.distributed.run --nproc-per-node=G tools/latency_bench.py [--steps K] [--warmup W] [--model basic|standard]
                                                                            [--T 6] [--precision fp16|fp32]

Uses the headline benchmark's workload helpers (synthetic 1242x375 stereo frames centre-cropped to 1024x352, the calibrated
synthetic models cached in the temporary directory) and writes nothing into the source tree."""
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


def run_latency(args, rank, world, local_rank):
    """Latency mode (SURVEY 8e, DESIGN §6): ms per frame when one frame's T Monte-Carlo samples are split over the ranks
    (sample_ranges(T, world)) -- every rank runs its shard and sums its samples' softmax, one reduce adds the float64 sums on rank 0,
    rank 0 finalises -- against the same frame on ONE whole-frame handle on rank 0 (same T, same inputs).  Both legs include
    ORB(nfeatures) x2 on rank 0's extractor streams, concurrent with the network.  Frames are issued one at a time: every rank is
    synchronised and at a barrier before a frame starts, and a frame is complete on rank 0 before the next is enqueued; the two
    legs alternate frame by frame.  Inputs are resident in HBM.  NCCL with one GPU per rank when world <= device count; otherwise
    gloo with every rank on device 0 (sums staged through host memory) -- a correctness run that claims no speed-up."""
    import gc

    import torch
    import torch.distributed as dist
    from sivo_b200 import BayesianSegNet, BayesianSegNetParams, ORBextractor, sample_ranges
    if not torch.cuda.is_available():
        raise SystemExit("latency_bench.py needs a CUDA device (there is no CPU fallback for the product path)")
    nccl = world <= torch.cuda.device_count()
    dev_index = local_rank if nccl else 0
    torch.cuda.set_device(dev_index)
    dev = torch.device("cuda", dev_index)
    if world > 1:
        if nccl:
            dist.init_process_group("nccl", device_id=dev)
        else:
            dist.init_process_group("gloo")
    T = args.T or (6 if args.model == "basic" else 12)
    cache = model_cache_dir()
    if rank == 0:
        _, proto, model, _ = model_files(args.model, T, cache)
    if world > 1:
        dist.barrier()
    if rank != 0:
        _, proto, model, _ = model_files(args.model, T, cache)
    if world > 1:
        dist.barrier()  # every rank has rewritten the prototxt before anyone parses it
    ranges = sample_ranges(T, world)
    params = BayesianSegNetParams(proto, model)
    shard = BayesianSegNet(params, device=dev_index, seed=1234, T=T, precision=args.precision, engine=args.engine, samples=ranges[rank])
    n_frames = 8
    fr = frames(n_frames)
    hw = NET_H * NET_W
    d_bgr = [torch.from_numpy(np.ascontiguousarray(f[0][CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W])).to(dev) for f in fr]
    d_sum = torch.empty(hw * 16, dtype=torch.float64, device=dev)
    h_sum = torch.empty(hw * 16, dtype=torch.float64).pin_memory() if world > 1 and not nccl else None
    # a real stream as the current one (the default stream's handle, 0, would send the library to its own stream), so that the
    # reduce and the host staging copies are ordered after run_partial
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    if rank == 0:
        full = BayesianSegNet(params, device=dev_index, seed=1234, T=T, precision=args.precision, engine=args.engine)
        orbs = [ORBextractor(args.nfeatures, 1.2, 8, 20, 7, device=dev_index) for _ in range(2)]
        if not all(o.has_device_tree() for o in orbs):
            raise SystemExit("latency_bench.py needs the extractors' asynchronous (device quad tree) form")
        d_gray = [[torch.from_numpy(f[1]).to(dev), torch.from_numpy(f[2]).to(dev)] for f in fr]
        cap = orbs[0].capacity()
        d_kp = [torch.empty(cap * 28, dtype=torch.uint8, device=dev) for _ in range(2)]
        d_desc = [torch.empty(cap * 32, dtype=torch.uint8, device=dev) for _ in range(2)]
        d_cnt = torch.zeros(2, dtype=torch.int64, device=dev)
        maps = {leg: [torch.empty(hw, dtype=torch.uint8, device=dev), torch.empty(hw, dtype=torch.float64, device=dev),
                      torch.empty(hw, dtype=torch.float64, device=dev)] for leg in ("sharded", "unsharded")}

    def orb_start(j):
        for s in range(2):
            orbs[s].enqueue_device(d_gray[j][s].data_ptr(), NET_H, NET_W, NET_W, d_kp[s].data_ptr(), d_desc[s].data_ptr(),
                                   d_cnt[s:].data_ptr())

    def orb_join():
        for o in orbs:
            o.stream_wait(stream.cuda_stream)

    def sharded(i):
        j = i % n_frames
        shard.set_frame(1000 + i)
        if rank == 0:
            orb_start(j)
        shard.run_partial(d_bgr[j].data_ptr(), d_sum.data_ptr(), stream.cuda_stream)
        if world > 1:
            if nccl:
                dist.reduce(d_sum, dst=0)
            else:
                h_sum.copy_(d_sum)
                dist.reduce(h_sum, dst=0)
                if rank == 0:
                    d_sum.copy_(h_sum, non_blocking=True)
        if rank == 0:
            c, f, e = maps["sharded"]
            shard.finalize(d_sum.data_ptr(), c.data_ptr(), f.data_ptr(), e.data_ptr(), 0, 0, stream.cuda_stream)
            orb_join()
        torch.cuda.synchronize(dev)

    def unsharded(i):
        if rank != 0:
            return
        j = i % n_frames
        full.set_frame(1000 + i)
        orb_start(j)
        c, f, e = maps["unsharded"]
        full.run_device_maps(d_bgr[j].data_ptr(), c.data_ptr(), f.data_ptr(), e.data_ptr(), 0, 0, stream.cuda_stream)
        orb_join()
        torch.cuda.synchronize(dev)

    times = {"sharded": [], "unsharded": []}
    legs = {"sharded": sharded, "unsharded": unsharded}
    gc.collect()
    gc.disable()
    for i in range(args.warmup + args.steps):
        for name in (("sharded", "unsharded") if i % 2 == 0 else ("unsharded", "sharded")):  # alternate which leg goes first
            torch.cuda.synchronize(dev)
            if world > 1:
                dist.barrier()
            t0 = time.perf_counter()
            legs[name](i)
            if i >= args.warmup:
                times[name].append(1e3 * (time.perf_counter() - t0))
    gc.enable()
    if rank == 0:
        mism = int((maps["sharded"][0] != maps["unsharded"][0]).sum())  # last frame: both legs ran frame 1000 + i on the same input
        gpu, power = torch.cuda.get_device_name(dev), None
        try:
            import pynvml
            pynvml.nvmlInit()
            power = pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(dev_index)) / 1e3
        except Exception:
            pass
        stat = lambda v: {"median": float(np.median(v)), "p90": float(np.percentile(v, 90))}
        sh, un = stat(times["sharded"]), stat(times["unsharded"])
        measured = world > 1 and nccl
        line = {"metric": "ms per frame, latency mode", "unit": "ms", "higher_is_better": False,
                "sharded": sh, "unsharded": un,
                "speedup_median": un["median"] / sh["median"] if measured else None,
                "kind": ("measurement: one GPU per rank, NCCL reduce" if measured else
                         "correctness run: " + ("one rank, no collective" if world == 1 else "gloo, every rank on device 0, sums staged through host memory")
                         + "; claims no speed-up"),
                "world": world, "backend": "nccl" if nccl and world > 1 else ("gloo" if world > 1 else None), "T": T, "model": args.model,
                "precision": args.precision, "sample_ranges": ranges, "bytes_reduced_per_frame": hw * 16 * 8 if world > 1 else 0,
                "steps": args.steps, "warmup": args.warmup, "gpu": gpu, "power_limit_w": power,
                "class_mismatch_last_frame": mism,
                "workload": f"Bayesian SegNet {args.model.capitalize()} T={T} + ORB({args.nfeatures}) x2 on rank 0's extractor streams, "
                            f"synthetic 1024x352 frames resident in HBM, one frame at a time"}
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed frames per leg")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--model", default="basic", choices=["basic", "standard"])
    ap.add_argument("--T", type=int, default=0, help="MC samples (default 6 basic / 12 standard)")
    ap.add_argument("--nfeatures", type=int, default=2000)
    ap.add_argument("--engine", default="auto", choices=["auto", "simt", "tcgen05"])
    ap.add_argument("--precision", default="fp16", choices=["fp16", "fp32"])
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    run_latency(args, rank, world, local_rank)


if __name__ == "__main__":
    main()
