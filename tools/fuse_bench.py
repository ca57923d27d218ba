"""ORBmatcher::Fuse on the device (sivo_fuse_device) at SearchInNeighbors' sizes: phase 1 at (targets, points) = (1, 2000),
(10, 2000), (25, 2000) and (60, 2000), phase 2 at (1, 50000), and the host form (sivo_fuse) end to end at (10, 2000).  Each
target holds 2000 keys, and about half of the points project near one of a target's keys with a few descriptor bits changed, so the
windows and fold see real candidates.  Prints one JSON line with each call's median / p90 ms, timed as DESIGN.md §7 describes, and
the device form's equality with the host form on every configuration.  The reference's host loop is not built here, so it is not
measured.

    python tools/fuse_bench.py [--steps 200] [--warmup 20]
"""
import argparse
import json

import numpy as np
import torch

from bench_support import add_common_args, card, device_ms, host_ms, require_cuda, stats  # puts the repository on sys.path
from oracle.mapping_scene import rotation
from oracle.track_oracle import gemm_neg_t
from sivo_b200.mapping import FuseTarget, KeyframeKeys, fuse, fuse_device, make_fuse_camera, set_pose
from sivo_b200.orb import KP_DTYPE, ORBextractor
from sivo_b200.track import MAP_POINT_DTYPE

FX, CX, CY, MBF, W, H = 718.856, 607.19, 185.22, 386.14, 1241.0, 376.0
N_KEYS = 2000


def scene(n_targets, n_points, seed):
    """Target 0 at the origin and the others at small offsets from it; points in front of them, half of them near target 0's
    keys with their descriptors a few bits off."""
    rng = np.random.default_rng(seed)
    targets = []
    for k in range(n_targets):
        R = rotation(*rng.normal(0, 0.01, 3)).astype(np.float32)
        t = (-R.astype(np.float64) @ np.array([0.1 * rng.normal(), 0.02 * rng.normal(), 0.2 * rng.normal()])).astype(np.float32)
        if k == 0:  # the points are made from target 0's keys at the identity pose
            R, t = np.eye(3, dtype=np.float32), np.zeros(3, np.float32)
        kps = np.zeros(N_KEYS, KP_DTYPE)
        kps["x"], kps["y"] = rng.uniform(0, W, N_KEYS), rng.uniform(0, H, N_KEYS)
        kps["octave"], kps["angle"], kps["size"] = rng.integers(0, 4, N_KEYS), rng.uniform(0, 360, N_KEYS), 31
        desc = rng.integers(0, 256, (N_KEYS, 32), dtype=np.uint8)
        ur = np.where(rng.random(N_KEYS) < 0.6, kps["x"] - rng.uniform(5, 60, N_KEYS), -1).astype(np.float32)
        targets.append((kps, desc, ur, R, t, gemm_neg_t(R, t)))
    z = rng.uniform(4, 40, n_points)
    kps0, desc0 = targets[0][0], targets[0][1]
    src = rng.integers(0, N_KEYS, n_points)
    near = rng.random(n_points) < 0.5
    u = np.where(near, kps0["x"][src] + rng.normal(0, 0.5, n_points), rng.uniform(0, W, n_points))
    v = np.where(near, kps0["y"][src] + rng.normal(0, 0.5, n_points), rng.uniform(0, H, n_points))
    pos = np.stack([(u - CX) / FX * z, (v - CY) / FX * z, z], 1).astype(np.float32)
    pts = np.zeros(n_points, MAP_POINT_DTYPE)
    pts["pos"] = pos
    pts["normal"] = (pos / np.linalg.norm(pos, axis=1, keepdims=True)).astype(np.float32)
    dist = np.linalg.norm(pos, axis=1).astype(np.float32)
    pts["max_distance"] = dist * np.float32(1.2) ** kps0["octave"][src].astype(np.float32)
    pts["min_distance"] = pts["max_distance"] / np.float32(1.2 ** 7)
    d = np.where(near[:, None], desc0[src], rng.integers(0, 256, (n_points, 32), dtype=np.uint8))
    d[:, 0] ^= rng.integers(0, 256, n_points, dtype=np.uint8) & np.uint8(0x0F)
    pts["desc"] = d
    return targets, pts


def device_targets(targets, cap):
    keep, keys = [], []
    for kps, desc, ur, R, t, Ow in targets:
        b = [torch.zeros(cap * 28, dtype=torch.uint8, device="cuda"), torch.zeros(cap * 32, dtype=torch.uint8, device="cuda"),
             torch.zeros(cap, dtype=torch.float32, device="cuda"), torch.tensor([len(kps)], dtype=torch.int64, device="cuda")]
        b[0][:len(kps) * 28] = torch.from_numpy(kps.view(np.uint8).copy()).cuda()
        b[1][:len(kps) * 32] = torch.from_numpy(desc.reshape(-1)).cuda()
        b[2][:len(kps)] = torch.from_numpy(ur).cuda()
        keep.append(b)
        k = KeyframeKeys(b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), None, None, None, None, None, None, b[3].data_ptr())
        set_pose(k, R, t, Ow)
        keys.append(k)
    return keep, keys


def main():
    ap = argparse.ArgumentParser()
    add_common_args(ap, steps=200, warmup=20)
    a = ap.parse_args()
    require_cuda("fuse_bench.py")
    left = ORBextractor(N_KEYS, 1.2, 8, 20, 7)
    cap = left.capacity()
    cam = make_fuse_camera(FX, FX, CX, CY, MBF, (0.0, W, 0.0, H))
    stream = torch.cuda.Stream()
    out = {"tool": "fuse_bench", "unit": "ms", **card(), "configs": []}
    for nt, npts in ((1, 2000), (10, 2000), (25, 2000), (60, 2000), (1, 50000)):
        targets, pts = scene(nt, npts, seed=nt * 7 + npts)
        keep, keys = device_targets(targets, cap)
        d_pts = torch.from_numpy(pts.view(np.uint8).copy()).cuda()
        match = torch.empty((nt, npts), dtype=torch.int32, device="cuda")
        dist = torch.empty((nt, npts), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        call = lambda: fuse_device(left, keys, cam, d_pts.data_ptr(), npts, 3.0, match.data_ptr(), dist.data_ptr(), stream.cuda_stream)
        ms = device_ms(call, stream, a.warmup, a.steps)
        host = [FuseTarget(kps, desc, ur, R, t, Ow) for kps, desc, ur, R, t, Ow in targets]
        hm, hd = fuse(left, host, cam, pts, 3.0)
        entry = {"targets": nt, "points": npts, "device_call_ms": stats(ms), "equal_to_host_form": bool(
            np.array_equal(match.cpu().numpy(), hm) and np.array_equal(dist.cpu().numpy(), hd)),
            "matched_pairs": int((hm >= 0).sum())}
        if (nt, npts) == (10, 2000):
            entry["host_call_ms"] = stats(host_ms(lambda: fuse(left, host, cam, pts, 3.0), 5, a.steps))
        out["configs"].append(entry)
        del keep
    out["all_equal"] = all(c["equal_to_host_form"] for c in out["configs"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
