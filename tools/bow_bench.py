"""Times the bag of words on the device: sivo_compute_bow_device (Frame::ComputeBoW) and sivo_search_by_bow_device (SearchByBoW,
batches of 1 and 32 keyframes), and the host forms end to end, with the full-shape seeded vocabulary (oracle/bow_scene.py,
1.08 M nodes) and the ORB(2000) keys of the KITTI fixture crop (tests/golden/orb_kitti_2000.npz).  Prints one JSON line, timed
as DESIGN.md §7 describes.

    python tools/bow_bench.py [--steps 200] [--warmup 20]
"""
import argparse
import json

import numpy as np
import torch

from bench_support import add_common_args, card, device_ms, host_ms, require_cuda, stats  # puts the repository on sys.path
from oracle import bow_scene as S
from sivo_b200 import ORBextractor
from sivo_b200.bow import Vocabulary, compute_bow, compute_bow_device, keyframe_keys, search_by_bow, search_by_bow_device
from sivo_b200.orb import KP_DTYPE


def main():
    ap = argparse.ArgumentParser()
    add_common_args(ap, steps=200, warmup=20)
    a = ap.parse_args()
    require_cuda("bow_bench.py")
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

    out = {"tool": "bow_bench", "unit": "ms", **card(), "keys": n, "vocabulary_nodes": voc.info()["nodes"]}
    out["compute_bow_device"] = stats(device_ms(bow, stream, a.warmup, a.steps))
    h = compute_bow(voc, desc, 4)
    out["compute_bow_host"] = stats(host_ms(lambda: compute_bow(voc, desc, 4), 0, max(a.steps // 4, 10)))
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
        out[f"search_by_bow_device_batch{batch}"] = stats(device_ms(search, stream, 10, a.steps))
        out[f"matches_batch{batch}_mean"] = round(float(nm[:batch].double().mean().cpu()), 1)
        hn = h["node"]
        out[f"search_by_bow_host_batch{batch}"] = stats(host_ms(lambda: search_by_bow(el, kps, desc, hn, kfs[:batch], 0.7, True), 0,
                                                                max(a.steps // 10, 5)))
    out["dbow2_host_loop"] = "not measured (needs OpenCV C++)"
    out["tracking_chain_fps"] = "not measured"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
