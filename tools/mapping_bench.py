"""Map-point creation (sivo_create_map_points_device) at 2000 keys x 10 neighbours on a constructed scene: prints one JSON line with
the device call's and the host form's median / p90 ms, timed as DESIGN.md §7 describes.  The reference's host loop
(LocalMapping::CreateNewMapPoints with OpenCV) is not built here, so it is not measured.

    python tools/mapping_bench.py [--steps 200] [--warmup 20]
"""
import argparse
import json

import numpy as np
import torch

from bench_support import add_common_args, card, device_ms, host_ms, require_cuda, stats  # puts the repository on sys.path
from oracle import mapping_scene as S
from sivo_b200.mapping import KeyframeKeys, create_map_points, create_map_points_device, HostKeyframe, make_params, set_pose
from sivo_b200.orb import ORBextractor


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
    ap = argparse.ArgumentParser()
    add_common_args(ap, steps=200, warmup=20)
    a = ap.parse_args()
    require_cuda("mapping_bench.py")
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
    ms = device_ms(call, s, a.warmup, a.steps)
    hk1 = HostKeyframe(kf1.kps, kf1.desc, kf1.u_right, kf1.depth, kf1.kp_class, kf1.kp_conf, kf1.kp_entropy, kf1.node, kf1.has_point,
                       kf1.Rcw, kf1.tcw, kf1.Ow)
    hn = [HostKeyframe(k.kps, k.desc, k.u_right, k.depth, k.kp_class, k.kp_conf, k.kp_entropy, k.node, k.has_point, k.Rcw, k.tcw, k.Ow)
          for k in nbs]
    r = create_map_points(left, hk1, hn, prm)
    host = host_ms(lambda: create_map_points(left, hk1, hn, prm), 0, 20)
    print(json.dumps({"workload": "create_map_points 2000 keys x 10 neighbours", "unit": "ms", **card(), "device_call_ms": stats(ms),
                      "host_call_ms": stats(host), "n_created": int(n.item()), "n_created_host": int(r["n_created"]),
                      "reference_host_loop": "not measured"}))


if __name__ == "__main__":
    main()
