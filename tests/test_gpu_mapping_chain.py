"""-m gpu: map-point creation fed by the Frame tail on the KITTI fixture crop and two synthetic frames -- SegNet -> extractors ->
semantic keys -> stereo -> sivo_keyframe_gather_device -> sivo_create_map_points_device of the last keyframe against the earlier
ones -- against oracle/mapping_oracle.py on the gathered buffers, and the same creation on its own stream while the Tracking chain
of another frame runs on the same left extractor."""
import numpy as np
import pytest
import torch

from frame_support import CX, CY, FX, MB, MBF, extractors, frame_inputs, seg, upload  # noqa: F401
from oracle import mapping_oracle as MO
from oracle import mapping_scene as S
from oracle.mapping_scene import rotation
from sivo_b200.frame import DeviceFrame
from sivo_b200.mapping import KeyframeKeys, create_map_points_device, keyframe_gather_device, make_params, set_pose
from sivo_b200.orb import KP_DTYPE

pytestmark = pytest.mark.gpu
TH_CONF, TH_RED, MAX_CLASS = 0.3, -1e9, 8


def test_chain_and_creation_beside_tracking(seg, kitti_bgr):
    el, er = extractors(2000)
    cap = el.capacity()
    inputs = frame_inputs(kitti_bgr)
    d_in = [[upload(x) for x in f] for f in inputs]
    s_track = torch.cuda.Stream()
    s = s_track.cuda_stream
    H, W = inputs[0][1].shape
    bufs = []
    for _ in inputs:
        b = {"f": DeviceFrame(el, er, H, W)}
        b["kf"] = dict(kps=torch.zeros(cap * 28, dtype=torch.uint8, device="cuda"), desc=torch.zeros(cap * 32, dtype=torch.uint8, device="cuda"),
                       u_right=torch.zeros(cap, device="cuda"), depth=torch.zeros(cap, device="cuda"),
                       kp_class=torch.zeros(cap, dtype=torch.uint8, device="cuda"), kp_conf=torch.zeros(cap, dtype=torch.float64, device="cuda"),
                       kp_entropy=torch.zeros(cap, dtype=torch.float64, device="cuda"), count=torch.zeros(1, dtype=torch.int64, device="cuda"))
        bufs.append(b)
    torch.cuda.synchronize()

    def front_end(i, b):
        seg.set_frame(600 + i)
        b["f"].extract(seg, *d_in[i], s)
        b["f"].tail(seg, MB, MBF, s)

    for i, b in enumerate(bufs):
        front_end(i, b)
        f = b["f"]
        keyframe_gather_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, f.depth, f.kp_class, f.kp_conf, f.kp_entropy, b["kf"], s)
    s_track.synchronize()

    # the gather against the Frame tail's layout: keys, descriptors and maps by keep_idx[j], mvRight / mvDepth by j
    kfs = []
    for i, b in enumerate(bufs):
        n, keep, ur, depth = b["f"].host()
        kps_all, desc_all = b["f"].left.host()
        g = {k: v.cpu().numpy() for k, v in b["kf"].items()}
        assert int(g["count"][0]) == n and n > 100
        gk = g["kps"].view(KP_DTYPE)[:n]
        assert np.array_equal(gk.view(np.uint8), kps_all[keep].view(np.uint8))
        assert np.array_equal(g["desc"].reshape(cap, 32)[:n], desc_all[keep])
        assert np.array_equal(g["u_right"][:n].view(np.uint32), ur.view(np.uint32))
        assert np.array_equal(g["depth"][:n].view(np.uint32), depth.view(np.uint32))
        for k in ("kp_class", "kp_conf", "kp_entropy"):
            assert np.array_equal(g[k][:n], b["f"].out[k].cpu().numpy()[keep])
        desc = g["desc"].reshape(cap, 32)[:n]
        node = (desc[:, 0] >> 3).astype(np.int32)  # a stand-in vocabulary: 32 nodes by the first descriptor byte
        b["node"] = torch.from_numpy(np.concatenate([node, np.zeros(cap - n, np.int32)])).cuda()
        hp = (np.arange(n) % 9 == 0).astype(np.uint8)
        b["hp"] = torch.from_numpy(np.concatenate([hp, np.zeros(cap - n, np.uint8)])).cuda()
        R = rotation(0.0, 0.01 * i, 0.0).astype(np.float32)
        t = (-R.astype(np.float64) @ np.array([0.4 * i, 0.0, 0.6 * i])).astype(np.float32)
        kfs.append(MO.KeyFrame(kps=gk.copy(), desc=desc.copy(), u_right=g["u_right"][:n].copy(), depth=g["depth"][:n].copy(),
                               kp_class=g["kp_class"][:n].copy(), kp_conf=g["kp_conf"][:n].copy(), kp_entropy=g["kp_entropy"][:n].copy(),
                               node=node, has_point=hp, Rcw=R, tcw=t))

    def keys(i):
        b = bufs[i]
        k = KeyframeKeys(*[b["kf"][f].data_ptr() for f in ("kps", "desc", "u_right", "depth", "kp_class", "kp_conf", "kp_entropy")],
                         b["node"].data_ptr(), b["hp"].data_ptr(), b["kf"]["count"].data_ptr())
        set_pose(k, kfs[i].Rcw, kfs[i].tcw, kfs[i].Ow)
        return k

    # a third neighbour: the current keyframe's own gathered keys seen from a shifted pose, so that true descriptor matches exist
    shifted = MO.KeyFrame(**{f: getattr(kfs[2], f) for f in ("kps", "desc", "u_right", "depth", "kp_class", "kp_conf", "kp_entropy",
                                                             "node", "has_point")}, Rcw=np.eye(3), tcw=np.array([-0.5, 0.0, -0.3]))

    def shifted_keys():
        k = keys(2)
        set_pose(k, shifted.Rcw, shifted.tcw, shifted.Ow)
        return k

    prm = make_params(FX, FX, CX, CY, MBF, S.sigma_cw(), MAX_CLASS, TH_CONF, TH_RED)
    want = MO.create_new_map_points(kfs[2], kfs[:2] + [shifted], MO.Camera(FX, FX, CX, CY, MBF), el.GetScaleFactors(), el.GetScaleSigmaSquares(),
                                    np.float32(1.2), S.sigma_cw(), MAX_CLASS, TH_CONF, TH_RED)
    n1 = len(kfs[2].kps)
    s_map = torch.cuda.Stream()

    def create():
        o = dict(nb=torch.full((cap,), -7, dtype=torch.int32, device="cuda"), idx=torch.full((cap,), -7, dtype=torch.int32, device="cuda"),
                 world=torch.full((cap, 3), 7.0, device="cuda"), lst=torch.full((cap, 2), -7, dtype=torch.int32, device="cuda"),
                 n=torch.full((1,), -7, dtype=torch.int64, device="cuda"))
        s_map.wait_stream(torch.cuda.current_stream())
        s_map.wait_stream(s_track)
        for _ in range(20):  # long enough to overlap the Tracking chain below
            create_map_points_device(el, keys(2), [keys(0), keys(1), shifted_keys()], prm, o["nb"].data_ptr(), o["idx"].data_ptr(), o["world"].data_ptr(),
                                     o["lst"].data_ptr(), o["n"].data_ptr(), s_map.cuda_stream)
        return o

    serial = create()
    s_map.synchronize()
    # LocalMapping's creation on its own stream while Tracking runs frame 0 again on the same left extractor
    first = {k: bufs[0]["f"].out[k].clone() for k in ("keep_idx", "u_right")}
    torch.cuda.synchronize()
    concurrent = create()
    front_end(0, bufs[0])
    s_map.synchronize()
    s_track.synchronize()
    out = bufs[0]["f"].out
    assert torch.equal(first["keep_idx"], out["keep_idx"]) and torch.equal(first["u_right"].view(torch.int32), out["u_right"].view(torch.int32))
    for o in (serial, concurrent):
        r = {k: v.cpu().numpy() for k, v in o.items()}
        assert int(r["n"][0]) == len(want["created"])
        np.testing.assert_array_equal(r["nb"][:n1], want["created_nb"])
        np.testing.assert_array_equal(r["idx"][:n1], want["created_idx"])
        np.testing.assert_array_equal(r["world"][:n1].view(np.uint32), want["world"].view(np.uint32))
        np.testing.assert_array_equal(r["lst"][:len(want["created"])], want["created"])
    assert (want["match"] >= 0).sum() > 0
