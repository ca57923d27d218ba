"""-m gpu: TrackReferenceKeyFrame's device chain on the KITTI fixture crop and two synthetic frames, three frames in flight on
rotating buffers -- SegNet -> enqueue_device -> semantic keys -> stereo -> BoW(F) -> SearchByBoW(refKF) -> gather -> pose -- with the
reference keyframe gathered from an earlier pass on the Tracking stream and its BoW computed on a second (LocalMapping's) stream
behind one event edge; each stage against oracle/bow_oracle.py and oracle/pose_oracle.py.  A last leg runs BoW(KF) on the
LocalMapping stream while Tracking's chain runs on the same left extractor."""
import numpy as np
import pytest
import torch

from frame_support import CX, CY, FX, MB, MBF, check_pose, extractors, frame_inputs, ptr, seg, upload  # noqa: F401
from oracle import bow_oracle as B
from oracle import bow_scene as S
from oracle import pose_oracle as P
from oracle import track_oracle as T
from oracle.mapping_scene import rotation
from sivo_b200 import map_points, pose_gather_device, pose_optimize_device
from sivo_b200.bow import Vocabulary, compute_bow_device, keyframe_keys, search_by_bow_device
from sivo_b200.frame import DeviceFrame
from sivo_b200.mapping import keyframe_gather_device
from sivo_b200.orb import KP_DTYPE
from sivo_b200.pose import result_from_bytes

pytestmark = pytest.mark.gpu
LEVELSUP = 4


def test_track_reference_keyframe_chain(seg, kitti_bgr):
    t = S.full_shape_tree(0)
    tree = B.Tree(t)
    voc = Vocabulary.from_arrays(t["k"], t["L"], t["scoring"], t["weighting"], t["parent"], t["is_leaf"], t["desc"], t["weight"])
    el, er = extractors(2000)
    cap = el.capacity()
    inputs = frame_inputs(kitti_bgr)
    d_in = [[upload(x) for x in f] for f in inputs]
    s_track, s_map = torch.cuda.Stream(), torch.cuda.Stream()
    s = s_track.cuda_stream
    H, W = inputs[0][1].shape

    def i32(fill=-7, n=cap):
        return torch.full((n,), fill, dtype=torch.int32, device="cuda")

    bufs = []
    for _ in inputs:
        b = {"f": DeviceFrame(el, er, H, W)}
        b["kf"] = dict(kps=torch.zeros(cap * 28, dtype=torch.uint8, device="cuda"), desc=torch.zeros(cap * 32, dtype=torch.uint8, device="cuda"),
                       u_right=torch.zeros(cap, device="cuda"), depth=torch.zeros(cap, device="cuda"),
                       kp_class=torch.zeros(cap, dtype=torch.uint8, device="cuda"), kp_conf=torch.zeros(cap, dtype=torch.float64, device="cuda"),
                       kp_entropy=torch.zeros(cap, dtype=torch.float64, device="cuda"), count=torch.zeros(1, dtype=torch.int64, device="cuda"))
        for k in ("node_f", "word_f", "bw_f", "node_kf", "bw_kf", "match"):
            b[k] = i32()
        b["bwt_f"] = torch.full((cap,), 7.0, dtype=torch.float64, device="cuda")
        for k in ("len_f", "len_kf", "nm"):
            b[k] = torch.full((1,), -7, dtype=torch.int64, device="cuda")
        b["xw"] = torch.full((3 * cap,), float("nan"), dtype=torch.float32, device="cuda")
        b["T0"] = torch.zeros(12, dtype=torch.float32, device="cuda")
        b["r"] = torch.full((512,), 0x55, dtype=torch.uint8, device="cuda")
        b["o"] = torch.full((cap,), 7, dtype=torch.uint8, device="cuda")
        b["ev"] = torch.cuda.Event()
        bufs.append(b)
    torch.cuda.synchronize()

    def front_end(i, b):
        seg.set_frame(700 + i)
        b["f"].extract(seg, *d_in[i], s)
        b["f"].tail(seg, MB, MBF, s)

    def kf_bow(b, stream):
        compute_bow_device(voc, el, ptr(b["kf"]["desc"]), 0, ptr(b["kf"]["count"]), LEVELSUP, ptr(b["node_kf"]), 0, ptr(b["bw_kf"]), 0,
                           ptr(b["len_kf"]), stream.cuda_stream)

    # an earlier pass makes each frame's reference keyframe: the gather on Tracking's stream, its BoW on LocalMapping's stream
    for i, b in enumerate(bufs):
        front_end(i, b)
        f = b["f"]
        keyframe_gather_device(el, f.kps, f.desc, f.keep, f.n_keep, f.u_right, f.depth, f.kp_class, f.kp_conf, f.kp_entropy, b["kf"], s)
        b["ev"].record(s_track)
        s_map.wait_event(b["ev"])
        kf_bow(b, s_map)
    s_track.synchronize()
    s_map.synchronize()

    scale = el.GetScaleFactors()
    cases = []
    for i, b in enumerate(bufs):
        n = int(b["kf"]["count"].cpu()[0])
        g = {k: v.cpu().numpy() for k, v in b["kf"].items()}
        kps, desc, depth = g["kps"].view(KP_DTYPE)[:n].copy(), g["desc"].reshape(cap, 32)[:n].copy(), g["depth"][:n].copy()
        R_true, t_true = rotation(0.01 * i, -0.02, 0.005), np.array([0.1 * i, -0.05, 0.3])
        f, idx = T.map_points_from_keys(kps, depth, R_true.T, -R_true.T @ t_true, FX, FX, CX, CY, scale)
        pts = map_points(desc[idx], f["pos"], f["normal"], f["min_distance"], f["max_distance"], 1, kps["octave"][idx], kps["angle"][idx])
        point = np.full(n, -1, np.int32)
        point[idx] = np.arange(len(idx), dtype=np.int32)
        point[::6] = -1  # GetMapPointMatches() NULL or bad
        Tpred = np.concatenate([rotation(0.001, -0.0015, 0.001) @ R_true, (t_true + [0.01, -0.005, 0.01])[:, None]], 1).astype(np.float32)
        _, _, node_kf, _ = B.transform(tree, desc, LEVELSUP)
        assert np.array_equal(b["node_kf"].cpu().numpy()[:n], node_kf) and n > 100
        b["point"] = torch.from_numpy(np.concatenate([point, np.full(cap - n, -1, np.int32)])).cuda()
        b["pts"] = upload(pts)
        b["T0"].copy_(torch.from_numpy(Tpred.reshape(-1)))
        cases.append(dict(kps=kps, desc=desc, node=node_kf, point=point, pts=pts, Tpred=Tpred))
    torch.cuda.synchronize()

    def track(i, b):
        front_end(i, b)
        f = b["f"]
        compute_bow_device(voc, el, f.desc, f.keep, f.n_keep, LEVELSUP, ptr(b["node_f"]), ptr(b["word_f"]), ptr(b["bw_f"]), ptr(b["bwt_f"]),
                           ptr(b["len_f"]), s)
        ref = keyframe_keys(ptr(b["kf"]["kps"]), ptr(b["kf"]["desc"]), ptr(b["node_kf"]), ptr(b["kf"]["count"]))
        search_by_bow_device(el, f.kps, f.desc, f.keep, f.n_keep, ptr(b["node_f"]), [ref], [ptr(b["point"])], 0.7, True, ptr(b["match"]),
                             ptr(b["nm"]), s)
        b["xw"].fill_(float("nan"))
        pose_gather_device(el, ptr(b["match"]), f.n_keep, ptr(b["pts"]), len(cases[i]["pts"]), ptr(b["xw"]), s)
        pose_optimize_device(el, f.kps, f.keep, f.n_keep, f.u_right, ptr(b["xw"]), FX, FX, CX, CY, MBF, ptr(b["T0"]), ptr(b["r"]),
                             ptr(b["o"]), s)

    with torch.cuda.stream(s_track):
        for i, b in enumerate(bufs):
            track(i, b)
    s_track.synchronize()

    for i, b in enumerate(bufs):
        c = cases[i]
        n, keep, ur, _ = b["f"].host()
        kps_all, desc_all = b["f"].left.host()
        kps, desc = kps_all[keep], desc_all[keep]
        bow, _, node, word = B.transform(tree, desc, LEVELSUP)
        words, vals = B.bow_arrays(bow)
        assert np.array_equal(b["node_f"].cpu().numpy()[:n], node) and np.array_equal(b["word_f"].cpu().numpy()[:n], word)
        assert int(b["len_f"].cpu()[0]) == len(words)
        assert np.array_equal(b["bw_f"].cpu().numpy()[:len(words)], words)
        assert np.array_equal(b["bwt_f"].cpu().numpy()[:len(words)].view(np.uint64), vals.view(np.uint64))
        m, nm = B.search_by_bow(kps, desc, node, c["kps"], c["desc"], c["node"], c["point"], 0.7, True)
        assert np.array_equal(b["match"].cpu().numpy()[:n], m) and int(b["nm"].cpu()[0]) == nm and nm > 20
        x = np.full((n, 3), np.nan, np.float32)
        x[m >= 0] = c["pts"]["pos"][m[m >= 0]]
        ref = P.pose_optimization(kps, ur, x, c["Tpred"], el.GetInverseScaleSigmaSquares(), P.Camera(FX, FX, CX, CY, MBF), order="device")
        check_pose(result_from_bytes(b["r"].cpu().numpy()), b["o"].cpu().numpy()[:n].astype(bool), ref)

    # LocalMapping's BoW(KF) on its own stream while Tracking's chain runs on the same left extractor: the same bits
    before = [(b["node_kf"].clone(), b["bw_kf"].clone(), b["len_kf"].clone()) for b in bufs]
    for b in bufs:
        b["node_kf"].fill_(-7)
        b["bw_kf"].fill_(-7)
    torch.cuda.synchronize()
    for _ in range(5):
        for b in bufs:
            kf_bow(b, s_map)
    with torch.cuda.stream(s_track):
        for i, b in enumerate(bufs):
            track(i, b)
    s_map.synchronize()
    s_track.synchronize()
    for b, (nd, bw, ln) in zip(bufs, before):
        assert torch.equal(b["node_kf"], nd) and torch.equal(b["bw_kf"], bw) and torch.equal(b["len_kf"], ln)
