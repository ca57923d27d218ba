"""Where the end-to-end frame time goes (one GPU): segmentImage alone, the two extractor calls alone, all three
concurrently -- page-locked host buffers, as bench.py's e2e arm.  Prints ms per frame."""
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from sivo_b200 import BayesianSegNet, BayesianSegNetParams, ORBextractor  # noqa: E402

H, W = bench.NET_H, bench.NET_W
net, proto, model, _ = bench.model_files("basic", 6, "/tmp/sivo_b200_models")
seg = BayesianSegNet(BayesianSegNetParams(proto, model), device=0, seed=1234)
orbs = [ORBextractor(2000, 1.2, 8, 20, 7), ORBextractor(2000, 1.2, 8, 20, 7)]
fr = bench.frames(4)


def pin(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    return t, t.numpy()


keep = [[pin(x) for x in f] for f in fr]
out_t = [torch.empty((H, W), dtype=d).pin_memory() for d in (torch.uint8, torch.float64, torch.float64)]
out_np = tuple(t.numpy() for t in out_t)
pyr_t = [[torch.empty(s, dtype=torch.uint8).pin_memory() for s in orbs[0].level_shapes(H, W)] for _ in range(2)]
pyr_np = [[t.numpy() for t in lst] for lst in pyr_t]
pool = ThreadPoolExecutor(max_workers=2)


def seg_only(j):
    seg.segmentImage(keep[j][0][1], out=out_np)


def orb_only(j):
    f = [pool.submit(orbs[k], keep[j][1 + k][1], None, want_pyramid=True, pyramid_buffers=pyr_np[k]) for k in range(2)]
    [x.result() for x in f]


def seg_nocopy(j):
    seg.segment_on_device(keep[j][0][1])


def both(j):
    f = [pool.submit(orbs[k], keep[j][1 + k][1], None, want_pyramid=True, pyramid_buffers=pyr_np[k]) for k in range(2)]
    seg.segmentImage(keep[j][0][1], out=out_np)
    [x.result() for x in f]


for name, fn in (("segmentImage alone", seg_only), ("segmentImage, maps left on the device", seg_nocopy),
                 ("two extractor calls alone", orb_only), ("all three concurrently", both)):
    for i in range(5):
        fn(i % 4)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 40
    for i in range(n):
        fn(i % 4)
    torch.cuda.synchronize()
    print(f"{name:42s} {1e3 * (time.perf_counter() - t0) / n:.3f} ms / frame")
