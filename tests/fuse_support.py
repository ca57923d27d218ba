"""What the Fuse GPU suites share: the oracle's keyframes and point records as the C ABI takes them, in the host form and in
device buffers of the extractor's capacity.  A plain module the tests import, not a test module."""
import numpy as np
import torch

from oracle import fuse_oracle as FO
from sivo_b200.mapping import FuseTarget, KeyframeKeys, fuse_device, make_fuse_camera, set_pose
from sivo_b200.track import MAP_POINT_DTYPE


def camera(cam: FO.Camera):
    return make_fuse_camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.mbf, (cam.min_x, cam.max_x, cam.min_y, cam.max_y))


def records(points) -> np.ndarray:
    """sivo_map_point records of oracle MapPoints or point dicts."""
    out = np.zeros(len(points), MAP_POINT_DTYPE)
    for i, p in enumerate(points):
        r = FO.point_record(p) if isinstance(p, FO.MapPoint) else p
        out[i]["desc"] = r["desc"]
        out[i]["pos"], out[i]["normal"] = r["pos"], r["normal"]
        out[i]["min_distance"], out[i]["max_distance"] = r["min_distance"], r["max_distance"]
    return out


def host_targets(kfs, counts=None):
    return [FuseTarget(kf.kps, kf.desc, kf.u_right, kf.Rcw, kf.tcw, kf.Ow, None if counts is None else counts[k])
            for k, kf in enumerate(kfs)]


class DeviceTargets:
    """The keyframes' keys in device buffers of `cap` keys each (zeros past the keys), as sivo_keyframe_gather_device leaves them."""

    def __init__(self, kfs, cap, counts=None):
        self.bufs, self.keys = [], []
        for k, kf in enumerate(kfs):
            n = len(kf.kps)
            assert n <= cap
            kps = np.zeros(cap, kf.kps.dtype)
            kps[:n] = kf.kps
            desc = np.zeros((cap, 32), np.uint8)
            desc[:n] = kf.desc
            ur = np.zeros(cap, np.float32)
            ur[:n] = kf.u_right
            b = {"kps": torch.from_numpy(kps.view(np.uint8).copy()).cuda(), "desc": torch.from_numpy(desc).cuda(),
                 "u_right": torch.from_numpy(ur).cuda(),
                 "count": torch.tensor([n if counts is None else counts[k]], dtype=torch.int64).cuda()}
            self.bufs.append(b)
            key = KeyframeKeys(b["kps"].data_ptr(), b["desc"].data_ptr(), b["u_right"].data_ptr(), None, None, None, None, None, None,
                               b["count"].data_ptr())
            set_pose(key, kf.Rcw, kf.tcw, kf.Ow)
            self.keys.append(key)
        torch.cuda.synchronize()


def run_device(left, kfs, cam, points, th, counts=None, targets=None):
    """sivo_fuse_device on device copies; -> (match, dist) numpy (n_targets, n_points).  The outputs start filled with sentinels,
    so a pair the call did not write shows."""
    t = targets or DeviceTargets(kfs, left.capacity(), counts)
    pts = torch.from_numpy(records(points).view(np.uint8).copy()).cuda()
    shape = (len(t.keys), len(points))
    match = torch.full(shape, -7, dtype=torch.int32, device="cuda")
    dist = torch.full(shape, -7, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    fuse_device(left, t.keys, camera(cam), pts.data_ptr(), len(points), th, match.data_ptr(), dist.data_ptr(), s.cuda_stream)
    s.synchronize()
    return match.cpu().numpy(), dist.cpu().numpy()
