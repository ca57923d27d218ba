"""Times Relocalization's PnP RANSAC on the device: sivo_pnp_setup_device and one sivo_pnp_iterate_device(5) call (the first
round of Tracking::Relocalization's loop) over 1 / 8 / 32 / 64 candidates x 15 / 200 / 2,000 correspondences each, 30 % outliers.
Each repetition re-runs setup, which resets the state, so every timed iterate is a first round.  CUDA events around the calls,
median of --reps.  Prints one JSON line per configuration with the card's name and power limit; writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from sivo_b200 import reloc  # noqa: E402
from sivo_b200.orb import KP_DTYPE, ORBextractor  # noqa: E402
from sivo_b200.track import map_points  # noqa: E402

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
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
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
            for rep in range(args.reps + 3):
                s = stream.cuda_stream
                ev[0].record(stream)
                solver.setup_device(t[0].data_ptr(), 0, t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(), len(pts), ids,
                                    rep, FX, FY, CX, CY, s)
                ev[1].record(stream)
                solver.iterate_device(5, np.ones(n_kf, np.uint8), Tcw.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(), inl.data_ptr(),
                                      outs[2].data_ptr(), s)
                ev[2].record(stream)
                stream.synchronize()
                if rep >= 3:
                    setup_ms.append(ev[0].elapsed_time(ev[1]))
                    iter_ms.append(ev[1].elapsed_time(ev[2]))
            solver.close()
            print(json.dumps({"candidates": n_kf, "correspondences": N, "outliers": 0.3, "setup_ms": float(np.median(setup_ms)),
                              "iterate5_ms": float(np.median(iter_ms)), "poses": int(outs[0].sum().item()), "card": card}), flush=True)


if __name__ == "__main__":
    main()
