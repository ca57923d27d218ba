"""Times the bag of words on the device: sivo_compute_bow_device (Frame::ComputeBoW) and sivo_search_by_bow_device (SearchByBoW,
batches of 1 and 32 keyframes) as CUDA-event medians and p90 over many calls, and the host forms end to end, with the full-shape
seeded vocabulary (oracle/bow_scene.py, 1.08 M nodes) and the ORB(2000) keys of the KITTI fixture crop (tests/golden/orb_kitti_2000.npz).
Prints one JSON line with the card's name and power limit read in the same run.

    python tools/bow_bench.py [--iters 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from oracle import bow_scene as S  # noqa: E402
from sivo_b200 import ORBextractor  # noqa: E402
from sivo_b200.bow import Vocabulary, compute_bow, compute_bow_device, keyframe_keys, search_by_bow, search_by_bow_device  # noqa: E402
from sivo_b200.orb import KP_DTYPE  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def events(fn, iters, stream):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return dict(median_us=round(float(np.median(ts)), 1), p90_us=round(float(np.percentile(ts, 90)), 1))


def wall(fn, iters):
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e6)
    return dict(median_us=round(float(np.median(ts)), 1), p90_us=round(float(np.percentile(ts, 90)), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bow_bench needs a GPU")
    t = S.full_shape_tree(0)
    voc = Vocabulary.from_arrays(t["k"], t["L"], t["scoring"], t["weighting"], t["parent"], t["is_leaf"], t["desc"], t["weight"])
    el = ORBextractor(2000, 1.2, 8, 20, 7)
    cap = el.capacity()
    z = np.load(S.GOLDEN)
    desc = z["descriptors"]
    n = len(desc)
    kps = np.zeros(n, KP_DTYPE)
    kps["x"], kps["y"], kps["angle"], kps["octave"] = z["keypoints"][:, 0], z["keypoints"][:, 1], z["keypoints"][:, 3] % 360.0, 0
    stream = torch.cuda.Stream()
    s = stream.cuda_stream

    def dev(x, dt=None):
        buf = np.zeros((cap,) + np.asarray(x).shape[1:], np.asarray(x).dtype if dt is None else dt)
        buf[:len(x)] = x
        return torch.from_numpy(buf.view(np.uint8).reshape(-1) if buf.dtype.names else buf).cuda()

    d_desc, d_kps = dev(desc), dev(kps)
    d_n = torch.tensor([n], dtype=torch.int64, device="cuda")
    node = torch.full((cap,), -1, dtype=torch.int32, device="cuda")
    bw = torch.zeros(cap, dtype=torch.int32, device="cuda")
    bwt = torch.zeros(cap, dtype=torch.float64, device="cuda")
    ln = torch.zeros(1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()

    def bow():
        compute_bow_device(voc, el, d_desc.data_ptr(), 0, d_n.data_ptr(), 4, node.data_ptr(), 0, bw.data_ptr(), bwt.data_ptr(), ln.data_ptr(), s)

    for _ in range(20):
        bow()
    torch.cuda.synchronize()
    out = {"tool": "bow_bench", "card": card(), "keys": n, "vocabulary_nodes": voc.info()["nodes"]}
    out["compute_bow_device"] = events(bow, a.iters, stream)
    h = compute_bow(voc, desc, 4)
    out["compute_bow_host"] = wall(lambda: compute_bow(voc, desc, 4), max(a.iters // 4, 10))
    out["bow_words"] = len(h["bow_words"])

    # keyframes: the frame's keys with 0-12 bits flipped and their own nodes, two thirds with a point
    rng = np.random.default_rng(0)
    kfs = []
    for k in range(32):
        kd = np.array([S.near(rng, d, int(rng.integers(0, 13))) for d in desc], np.uint8)
        kn = compute_bow(voc, kd, 4)["node"]
        point = np.where(rng.uniform(size=n) < 0.67, np.arange(n), -1).astype(np.int32)
        kfs.append(dict(kps=kps.copy(), desc=kd, node=kn, point=point))
    d_kf = [(dev(kps), dev(kf["desc"]), dev(kf["node"]), dev(kf["point"]), torch.tensor([n], dtype=torch.int64, device="cuda")) for kf in kfs]
    keys = [keyframe_keys(a_[0].data_ptr(), a_[1].data_ptr(), a_[2].data_ptr(), a_[4].data_ptr()) for a_ in d_kf]
    pts = [a_[3].data_ptr() for a_ in d_kf]
    match = torch.zeros((32, cap), dtype=torch.int32, device="cuda")
    nm = torch.zeros(32, dtype=torch.int64, device="cuda")
    bow()
    torch.cuda.synchronize()
    for batch in (1, 32):
        def search():
            search_by_bow_device(el, d_kps.data_ptr(), d_desc.data_ptr(), 0, d_n.data_ptr(), node.data_ptr(), keys[:batch], pts[:batch], 0.7,
                                 True, match.data_ptr(), nm.data_ptr(), s)
        for _ in range(10):
            search()
        torch.cuda.synchronize()
        out[f"search_by_bow_device_batch{batch}"] = events(search, a.iters, stream)
        out[f"matches_batch{batch}_mean"] = round(float(nm[:batch].double().mean().cpu()), 1)
        hn = h["node"]
        out[f"search_by_bow_host_batch{batch}"] = wall(lambda: search_by_bow(el, kps, desc, hn, kfs[:batch], 0.7, True), max(a.iters // 10, 5))
    out["dbow2_host_loop"] = "not measured (needs OpenCV C++)"
    out["tracking_chain_fps"] = "not measured"
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
