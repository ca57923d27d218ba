"""Map-point creation (sivo_create_map_points_device) at 2000 keys x 10 neighbours on a constructed scene: prints one JSON line with
the device call's median / p90 ms (CUDA events, 200 calls after warm-up), the host form's end-to-end ms, and the GPU's name and
power limit read in the same run.  The reference's host loop (LocalMapping::CreateNewMapPoints with OpenCV) is not built here, so it
is not measured."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import mapping_scene as S  # noqa: E402
from sivo_b200.mapping import KeyframeKeys, create_map_points, create_map_points_device, HostKeyframe, make_params, set_pose  # noqa: E402
from sivo_b200.orb import ORBextractor  # noqa: E402


def device_kf(kf, cap, keep):
    n = len(kf.kps)
    pad = lambda a, dt: torch.from_numpy(np.concatenate([np.asarray(a, dt), np.zeros((cap - n,) + np.asarray(a).shape[1:], dt)])).cuda()
    t = [pad(kf.kps.view(np.uint8).reshape(n, 28), np.uint8), pad(kf.desc, np.uint8), pad(kf.u_right, np.float32),
         pad(kf.depth, np.float32), pad(kf.kp_class, np.uint8), pad(kf.kp_conf, np.float64), pad(kf.kp_entropy, np.float64),
         pad(kf.node, np.int32), pad(kf.has_point, np.uint8), torch.tensor([n], dtype=torch.int64, device="cuda")]
    keep.append(t)
    k = KeyframeKeys(*[x.data_ptr() for x in t])
    set_pose(k, kf.Rcw, kf.tcw, kf.Ow)
    return k


def main():
    p = S.EXTRACTOR
    left = ORBextractor(p.nfeatures, p.scale_factor, p.nlevels, 20, 7)
    cap = left.capacity()
    kf1, nbs = S.make_scene(2000, 10, seed=10)
    prm = make_params(S.FX, S.FY, S.CX, S.CY, S.MBF, S.sigma_cw(), 8, 0.5, 9.5)
    keep = []
    d1 = device_kf(kf1, cap, keep)
    dn = [device_kf(k, cap, keep) for k in nbs]
    nb = torch.empty(cap, dtype=torch.int32, device="cuda")
    world = torch.empty(cap, 3, device="cuda")
    lst = torch.empty(cap, 2, dtype=torch.int32, device="cuda")
    n = torch.empty(1, dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    call = lambda: create_map_points_device(left, d1, dn, prm, nb.data_ptr(), 0, world.data_ptr(), lst.data_ptr(), n.data_ptr(), s.cuda_stream)
    for _ in range(20):
        call()
    s.synchronize()
    ms = []
    for _ in range(200):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        call()
        b.record(s)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    hk1 = HostKeyframe(kf1.kps, kf1.desc, kf1.u_right, kf1.depth, kf1.kp_class, kf1.kp_conf, kf1.kp_entropy, kf1.node, kf1.has_point,
                       kf1.Rcw, kf1.tcw, kf1.Ow)
    hn = [HostKeyframe(k.kps, k.desc, k.u_right, k.depth, k.kp_class, k.kp_conf, k.kp_entropy, k.node, k.has_point, k.Rcw, k.tcw, k.Ow)
          for k in nbs]
    create_map_points(left, hk1, hn, prm)
    host = []
    for _ in range(20):
        t0 = time.perf_counter()
        r = create_map_points(left, hk1, hn, prm)
        host.append(1e3 * (time.perf_counter() - t0))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"workload": "create_map_points 2000 keys x 10 neighbours", "device_ms_median": float(np.median(ms)),
                      "device_ms_p90": float(np.percentile(ms, 90)), "host_form_ms_median": float(np.median(host)),
                      "n_created": int(n.item()), "n_created_host": int(r["n_created"]), "gpu": q.stdout.strip().splitlines()[0] if q.stdout else "",
                      "reference_host_loop": "not measured"}))


if __name__ == "__main__":
    main()
