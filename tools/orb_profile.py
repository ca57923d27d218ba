"""Runs the extractor alone on one frame and times its synchronous calls: a host clock around each call, which returns after the
device has finished.  Prints one JSON line (per-call median / mean / p10 / p90 in ms, the last call's own timing, the GPU).
--nfeatures 5000 takes the host quad tree on every call (a level then asks for more keypoints than the device tree keeps)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sivo_b200 import ORBextractor  # noqa: E402
from sivo_b200.synth import bgr_to_gray, stereo_frame  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--nfeatures", type=int, default=2000)
ap.add_argument("--iters", type=int, default=200)
ap.add_argument("--warmup", type=int, default=20)
a = ap.parse_args()

left, _ = stereo_frame(0)
gray = np.ascontiguousarray(bgr_to_gray(left)[11:11 + 352, 109:109 + 1024])
ext = ORBextractor(a.nfeatures, 1.2, 8, 20, 7)
for _ in range(a.warmup):
    kps, desc = ext(gray, None)
ms = []
for _ in range(a.iters):
    t = time.perf_counter()
    kps, desc = ext(gray, None)
    ms.append((time.perf_counter() - t) * 1e3)
ms = np.array(ms)
import torch  # noqa: E402
print(json.dumps({"nfeatures": a.nfeatures, "device_tree": ext.has_device_tree(), "keypoints": len(kps), "iters": a.iters,
                  "median_ms": round(float(np.median(ms)), 4), "mean_ms": round(float(ms.mean()), 4),
                  "p10_ms": round(float(np.percentile(ms, 10)), 4), "p90_ms": round(float(np.percentile(ms, 90)), 4),
                  "last": ext.last_timing(), "gpu": torch.cuda.get_device_name(0)}))
