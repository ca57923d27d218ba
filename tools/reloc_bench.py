"""Times Relocalization's PnP RANSAC on the device: sivo_pnp_setup_device and one sivo_pnp_iterate_device(5) call (the first
round of Tracking::Relocalization's loop) over 1 / 8 / 32 / 64 candidates x 15 / 200 / 2,000 correspondences each, 30 % outliers.
Each repetition re-runs setup, which resets the state, so every timed iterate is a first round.  Three CUDA events
per repetition, around setup and around the iterate, median / p90 in ms over --steps repetitions after --warmup.  Prints one JSON
line per configuration with the card's name and power limit read in the same run (DESIGN.md §7); writes nothing.

    python tools/reloc_bench.py [--steps 30] [--warmup 3]
"""
import argparse
import json

import numpy as np
import torch

from bench_support import add_common_args, card, require_cuda, stats  # puts the repository on sys.path
from sivo_b200 import reloc
from sivo_b200.orb import KP_DTYPE, ORBextractor
from sivo_b200.track import map_points

FX, FY, CX, CY = 718.856, 718.856, 607.1928, 185.2157


def scene(left, n_kf, N, outliers, seed):
    cap = left.capacity()
    r = np.random.default_rng(seed)
    Xw = np.c_[r.uniform(-8, 8, N), r.uniform(-3, 3, N), r.uniform(4, 40, N)]
    kps = np.zeros(cap, KP_DTYPE)
    kps["x"][:N] = FX * Xw[:, 0] / Xw[:, 2] + CX + r.normal(size=N) * 0.3
    kps["y"][:N] = FY * Xw[:, 1] / Xw[:, 2] + CY + r.normal(size=N) * 0.3
    kps["octave"][:N] = r.integers(0, left.nlevels, N)
    match = np.full((n_kf, cap), -1, np.int32)
    pos = np.zeros((n_kf * N, 3), np.float32)
    for k in range(n_kf):
        wrong = r.random(N) < outliers
        pos[k * N:(k + 1) * N] = Xw + wrong[:, None] * r.normal(size=(N, 3)) * 3.0
        match[k, :N] = k * N + np.arange(N)
    return kps, match, np.full(n_kf, N, np.int64), pos


def main():
    ap = argparse.ArgumentParser()
    add_common_args(ap, steps=30, warmup=3)
    args = ap.parse_args()
    require_cuda("reloc_bench.py")
    gpu = card()
    left = ORBextractor(2000, 1.2, 8, 20, 7)
    dev = torch.device("cuda")
    stream = torch.cuda.Stream()
    for n_kf in (1, 8, 32, 64):
        for N in (15, 200, 2000):
            kps, match, nm, pos = scene(left, n_kf, N, 0.3, n_kf * 7 + N)
            pts = map_points(np.zeros((len(pos), 32), np.uint8), pos, np.zeros_like(pos), 0.0, 1e9)
            t = [torch.from_numpy(a).to(dev) for a in (kps.view(np.uint8).copy(), np.array([N], np.int64), match, nm,
                                                       pts.view(np.uint8).copy())]
            cap = left.capacity()
            Tcw = torch.zeros((n_kf, 12), dtype=torch.float32, device=dev)
            outs = [torch.zeros(n_kf, dtype=torch.int32, device=dev) for _ in range(3)]
            inl = torch.zeros((n_kf, cap), dtype=torch.int32, device=dev)
            solver = reloc.PnpSolver(left, n_kf, 1)
            ids = np.arange(n_kf, dtype=np.uint32)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            setup_ms, iter_ms = [], []
            torch.cuda.synchronize()
            for rep in range(args.warmup + args.steps):
                s = stream.cuda_stream
                ev[0].record(stream)
                solver.setup_device(t[0].data_ptr(), 0, t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(), len(pts), ids,
                                    rep, FX, FY, CX, CY, s)
                ev[1].record(stream)
                solver.iterate_device(5, np.ones(n_kf, np.uint8), Tcw.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(), inl.data_ptr(),
                                      outs[2].data_ptr(), s)
                ev[2].record(stream)
                stream.synchronize()
                if rep >= args.warmup:
                    setup_ms.append(ev[0].elapsed_time(ev[1]))
                    iter_ms.append(ev[1].elapsed_time(ev[2]))
            solver.close()
            print(json.dumps({"candidates": n_kf, "correspondences": N, "outliers": 0.3, "unit": "ms", "setup_ms": stats(setup_ms),
                              "iterate5_ms": stats(iter_ms), "poses": int(outs[0].sum().item()), **gpu}), flush=True)


if __name__ == "__main__":
    main()
