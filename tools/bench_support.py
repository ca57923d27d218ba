"""The measuring code of the SLAM-call benchmarks (tools/*_bench.py), kept once so that their figures compare (DESIGN.md §7): the
card and power limit read in the measuring process, device calls timed by CUDA events around each call with a synchronise after
it, host calls by the wall clock, median and p90 in ms, and the chain runner that alternates two legs in blocks of frames."""
import argparse
import gc
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import CROP_X, CROP_Y, NET_H, NET_W, frames, model_cache_dir, model_files  # noqa: E402


def card():
    """The name and enforced power limit in W of the GPU the tools measure on (cuda:0), both through NVML (read-only queries);
    None where NVML is unavailable."""
    import torch
    out = {"gpu": None, "power_limit_w": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        try:
            h = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + str(torch.cuda.get_device_properties(0).uuid)).encode())
        except Exception:
            h = pynvml.nvmlDeviceGetHandleByIndex(0)
        name = pynvml.nvmlDeviceGetName(h)
        out["gpu"] = name.decode() if isinstance(name, bytes) else name
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1e3
    except Exception:
        pass
    return out


def require_cuda(tool):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit(f"{tool} needs a CUDA device (there is no CPU fallback for the product path)")


def _timed(fn, warmup, calls, clock):
    for _ in range(warmup):
        fn()
    gc.collect()
    gc.disable()
    try:
        return [clock(fn) for _ in range(calls)]
    finally:
        gc.enable()


def device_ms(fn, stream, warmup, calls):
    """ms of each of `calls` calls of fn after `warmup` untimed ones: CUDA events on `stream` around the call and a synchronise
    after it, so the window holds the call's host enqueue as well as its kernels."""
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def clock(fn):
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b)
    return _timed(fn, warmup, calls, clock)


def host_ms(fn, warmup, calls):
    """ms of each of `calls` calls of a host-form fn after `warmup` untimed ones, by the wall clock (the host forms synchronise)."""
    def clock(fn):
        t0 = time.perf_counter()
        fn()
        return 1e3 * (time.perf_counter() - t0)
    return _timed(fn, warmup, calls, clock)


def stats(ms):
    return {"median": float(np.median(ms)), "p90": float(np.percentile(ms, 90))}


def alternate(legs, stream, steps, warmup, blocks_of, nbuf):
    """Frames/s of each leg of `legs` ({name: step(i, k)}, k = i % nbuf the ring slot the step uses), the legs swapped every block
    of blocks_of frames over about warmup + steps frames each, after two warm-up blocks per leg.  The run-ahead is bounded as in
    bench.py's device step: every fourth frame waits for the step before it.  Returns {name: {"overall", "median_block", "frames"}}."""
    import torch
    ev = [torch.cuda.Event() for _ in range(nbuf)]
    names = list(legs)
    blocks = {name: [] for name in names}
    n_blocks = max(1, -(-(warmup + steps) // blocks_of))
    i = 0
    gc.collect()
    gc.disable()
    for b in range(n_blocks + 2):
        for name in (names if b % 2 == 0 else names[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(blocks_of):
                legs[name](i, i % nbuf)
                ev[i % nbuf].record(stream)
                if (i & 3) == 3:
                    ev[(i - 1) % nbuf].synchronize()
                i += 1
            torch.cuda.synchronize()
            if b >= 2:
                blocks[name].append(time.perf_counter() - t0)
    gc.enable()
    return {name: {"overall": blocks_of * len(dt) / sum(dt), "median_block": float(np.median([blocks_of / t for t in dt])),
                   "frames": blocks_of * len(dt)} for name, dt in blocks.items()}


def basic_front_end(nfeatures, T=6):
    """Bayesian SegNet Basic (bench.py's seeded, calibrated model) and the left and right ORB(nfeatures) extractors, which must
    have the device quad tree: the chains run them asynchronously."""
    from sivo_b200 import BayesianSegNet, BayesianSegNetParams, ORBextractor
    _, proto, model, _ = model_files("basic", T, model_cache_dir())
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=T)
    el, er = (ORBextractor(nfeatures, 1.2, 8, 20, 7) for _ in range(2))
    if not (el.has_device_tree() and er.has_device_tree()):
        raise SystemExit("the chain needs the extractors' asynchronous (device quad tree) form")
    return seg, el, er


def check_device_trees(el, er):
    """After a run: the asynchronous outputs are valid only if no pyramid level overflowed the device quad tree."""
    if el.device_status() or er.device_status():
        raise SystemExit("a pyramid level exceeded the device quad tree's capacity: the asynchronous outputs are not valid")


def chain_frames(n):
    """bench.py's first n synthetic frames as device tensors [bgr crop, left gray, right gray], uploaded before it returns."""
    import torch
    out = [[torch.from_numpy(np.ascontiguousarray(f[0][CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W])).cuda(),
            torch.from_numpy(f[1]).cuda(), torch.from_numpy(f[2]).cuda()] for f in frames(n)]
    torch.cuda.synchronize()
    return out


def kitti_frame():
    """The KITTI fixture frame's crop as device tensors [bgr, left gray, right gray], uploaded before it returns; the right image
    is the left one shifted by 12 px."""
    import cv2
    import torch
    from sivo_b200.synth import bgr_to_gray
    img = cv2.imread(os.path.join(ROOT, "tests", "golden", "kitti_000000_1242x375.png"))
    gray = bgr_to_gray(img)[CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W]
    out = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
           (img[CROP_Y:CROP_Y + NET_H, CROP_X:CROP_X + NET_W], gray, np.roll(gray, -12, axis=1))]
    torch.cuda.synchronize()
    return out


def _at_least_1(s):
    v = int(s)
    if v < 1:
        raise argparse.ArgumentTypeError("must be at least 1")
    return v


def add_common_args(ap, steps, warmup, chain=False):
    """--steps (timed calls or frames) and --warmup with the tool's defaults; with a chain also --blocks-of and --nfeatures."""
    ap.add_argument("--steps", type=_at_least_1, default=steps, help="timed calls / frames per measurement")
    ap.add_argument("--warmup", type=int, default=warmup)
    if chain:
        ap.add_argument("--blocks-of", type=_at_least_1, default=10, help="frames per alternating block of the chain legs")
        ap.add_argument("--nfeatures", type=int, default=2000)
