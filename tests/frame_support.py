"""What the GPU suites of the Frame tail share: the network's crop of a KITTI frame and its camera, synthetic stereo frames, the
extractor pair and one cached extractor per parameter set, the Basic T=2 SegNet fixture, one frame's front end and tail on the
device (Tail), and the device-test helpers (upload, sentinel outputs, int64 counts, bit equality).  A plain module the tests
import, not a test module."""
import os

import numpy as np
import pytest
import torch

from oracle import info_oracle as I
from oracle import pose_oracle as P
from oracle.mapping_scene import rotation
from sivo_b200 import BayesianSegNet, BayesianSegNetParams, KP_DTYPE, ORBextractor, info_select_device, make_camera, stereo_match_device
from sivo_b200.frame import DeviceFrame
from sivo_b200.synth import bgr_to_gray, stereo_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W, Y0, X0 = 352, 1024, 11, 109  # the network's input: the centre crop (109, 11) of a 1242x375 frame
KITTI_MBF = 386.1448  # Camera.bf of config/kitti/KITTI00-02.yaml; mb = bf / fx
BASELINES = {"kitti": (KITTI_MBF / 718.856, KITTI_MBF), "wide": (0.8, 400.0)}
MB, MBF = BASELINES["kitti"]
FX, CX, CY = 718.856, 607.1928 - X0, 185.2157 - Y0  # KITTI00-02.yaml, principal point moved to the network's crop
BOUNDS = (0.0, float(W), 0.0, float(H))  # the crop's image bounds (mnMinX, mnMaxX, mnMinY, mnMaxY)


def seg_paths(model_dir):
    return os.path.join(ROOT, "configs", "bayesian_segnet_basic.prototxt"), os.path.join(str(model_dir), "basic_full.caffemodel")


@pytest.fixture(scope="module")
def seg(model_dir):
    """The shipped Basic topology at T=2 with the calibrated synthetic weights (the file other GPU tests write)."""
    from sivo_b200.caffemodel import shipped_scales, write_synth_model
    from sivo_b200.prototxt import load_net
    proto, model = seg_paths(model_dir)
    if not os.path.exists(model):
        write_synth_model(load_net(open(proto).read(), T=2), model, 0, shipped_scales("basic"))
    return BayesianSegNet(BayesianSegNetParams(proto, model), seed=7, T=2, precision="fp16", engine="auto")


def crop(img):
    return np.ascontiguousarray(img[Y0:Y0 + H, X0:X0 + W])


def synth(seed):
    left, right = stereo_frame(seed)
    return crop(left), crop(bgr_to_gray(left)), crop(bgr_to_gray(right))


def frame_inputs(kitti_bgr):
    """(bgr, left gray, right gray) of the KITTI fixture crop and synthetic frames 1 and 2."""
    gl = crop(bgr_to_gray(kitti_bgr))  # the fixture frame has no right image: the left one shifted by 12 px stands in for it
    out = [(crop(kitti_bgr), gl, np.ascontiguousarray(np.roll(gl, -12, axis=1)))]
    return out + [synth(s) for s in (1, 2)]


def ptr(t):
    return t.data_ptr()


def upload(a):
    """A device copy of the array's bytes (flat uint8), complete before anything else is enqueued (the library's streams do not
    wait for torch's)."""
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    torch.cuda.synchronize()
    return t


def sentinel(n, fill, dtype):
    """n device entries at a sentinel value (one an output that was not written keeps), set before anything else is enqueued."""
    t = torch.full((n,), fill, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    return t


def i64(v):
    """A device count (int64)."""
    return sentinel(1, v, torch.int64)


def same_bits(a, b):
    """The same shape and the same bits, except that a NaN matches any NaN (the device's default NaN is not numpy's); 0.0 and
    -0.0 differ.  Float values compare as float64, which keeps both."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind != "f" and b.dtype.kind != "f":
        return np.array_equal(a, b)
    a, b = a.astype(np.float64), b.astype(np.float64)
    return bool(((a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))).all())


# a keyframe's per-key arrays (sivo_keyframe_keys) and their device layouts
KF_FIELDS = {"kps": KP_DTYPE, "desc": np.uint8, "u_right": np.float32, "depth": np.float32, "kp_class": np.uint8, "kp_conf": np.float64,
             "kp_entropy": np.float64, "node": np.int32, "has_point": np.uint8}


def kp_matrix(kps):
    """Keypoint records as a float32 matrix of their seven fields, the layout of the golden files and the oracle."""
    return np.stack([kps["x"], kps["y"], kps["size"], kps["angle"], kps["response"], kps["octave"].astype(np.float32),
                     kps["class_id"].astype(np.float32)], axis=1)


def extractors(nf, nlevels=8):
    return ORBextractor(nf, 1.2, nlevels, 20, 7), ORBextractor(nf, 1.2, nlevels, 20, 7)


_EXTRACTORS = {}


def extractor(nfeatures=2000, scale_factor=1.2, nlevels=8, right=False):
    """The process's one extractor of these parameters (right: a second one, the right side of a stereo pair)."""
    key = (nfeatures, scale_factor, nlevels, right)
    if key not in _EXTRACTORS:
        _EXTRACTORS[key] = ORBextractor(nfeatures, scale_factor, nlevels, 20, 7)
    return _EXTRACTORS[key]


@pytest.fixture(scope="module")
def ext():
    return extractors(2000)


# ---------------------------------------------------------------------------------------------------------- cameras
def sigmas():
    motion = 1e-6 * np.eye(6)
    for i in range(3):
        motion = I.update_state_covariance_motion(motion, rotation(0.002 * i, 0.01, -0.003), (0.02, -0.01, 0.8 + 0.1 * i))
    a = np.random.default_rng(11).standard_normal((6, 6))
    spd = 1e-3 * (a @ a.T + 0.5 * np.eye(6))
    return {"tiny": 1e-6 * np.eye(6), "motion": motion, "spd": spd}


SIGMAS = sigmas()
POSES = {"identity": (np.eye(3), (0.0, 0.0, 0.0)), "moved": (rotation(0.03, -0.25, 0.08), (3.5, -0.7, 41.0))}


def cameras(sigma, pose):
    """The KITTI camera at a named pose and pose covariance (or a given 6 x 6 one), for the library and for the oracle."""
    R, Ow = POSES[pose]
    S = SIGMAS[sigma] if isinstance(sigma, str) else sigma
    return make_camera(FX, FX, CX, CY, MB, R, Ow, S), I.Camera(FX, FX, CX, CY, MB, R, Ow, S)


def check_pose(res, outl, ref):
    """A device pose result and its outlier flags against the oracle's: rotation and translation within 1e-9, Σ within 1e-8,
    the same flags except on edges whose χ² sits on the threshold."""
    assert np.abs(P.rotation_matrix(np.array(res.q)) - P.rotation_matrix(ref.q)).max() <= 1e-9
    assert np.abs(np.array(res.t) - ref.t).max() <= 1e-9 * (np.abs(ref.t).max() + 1)
    assert res.sigma_valid == ref.sigma_valid and res.n_initial == ref.n_initial and res.rounds_run == ref.rounds_run
    if ref.sigma_valid:
        assert np.linalg.norm(res.sigma() - ref.sigma) <= 1e-8 * np.linalg.norm(ref.sigma)
    near = np.zeros(len(outl), bool)
    with np.errstate(invalid="ignore"):
        near[ref.edges.key] = np.abs(ref.chi2 - float(P.CHI2_STEREO)) <= 1e-6 * float(P.CHI2_STEREO)
    assert np.array_equal(outl[~near], ref.outlier[~near])
    if not near.any():
        assert res.n_good == ref.n_good


# ---------------------------------------------------------------------------------------------------------- one frame's tail
class InfoOut:
    """The information selection's outputs (world points, reductions, selected list and its count) at sentinels."""

    def __init__(self, cap):
        self.world = torch.full((cap * 3,), 7.0, dtype=torch.float32, device="cuda")
        self.red = torch.full((cap,), 7.0, dtype=torch.float64, device="cuda")
        self.sel = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
        self.n = torch.full((1,), -7, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()

    def run(self, el, kps, ent, keep, n_keep, depth, cam, threshold, stream, null=()):
        p = {k: (0 if k in null else ptr(getattr(self, k))) for k in ("world", "red", "sel", "n")}
        info_select_device(el, kps, ent, keep, n_keep, depth, cam, threshold, p["world"], p["red"], p["sel"], p["n"], stream)

    def host(self, n):
        m = int(self.n.cpu()[0])
        return (self.world.cpu().numpy()[:3 * n].reshape(n, 3).copy(), self.red.cpu().numpy()[:n].copy(),
                self.sel.cpu().numpy()[:max(m, 0)].copy(), m)


class Tail:
    """One frame through SegNet -> two enqueue_device -> semantic keys -> stereo on the device (f, a DeviceFrame), a second
    stereo call over every extractor key (keep_idx NULL: u_all, z_all), plus host copies of the selection's inputs
    (mvKeysSemantic, mvDepth, the entropy at each key)."""

    def __init__(self, seg, el, er, bgr, gl, gr):
        seg.set_frame(3)
        stream = torch.cuda.Stream()
        s = stream.cuda_stream
        self.f = f = DeviceFrame(el, er, H, W)
        self.u_all, self.z_all = (torch.full((f.left.cap,), 7.0, dtype=torch.float32, device="cuda") for _ in range(2))
        f.extract(seg, upload(bgr), upload(gl), upload(gr), s)
        f.tail(seg, MB, MBF, s)
        stereo_match_device(el, er, f.kps, f.desc, 0, f.count, ptr(f.right.kps), ptr(f.right.desc), ptr(f.right.count), MB, MBF,
                            ptr(self.u_all), ptr(self.z_all), s)
        stream.synchronize()
        self.kps_all = f.left.host()[0]
        self.n_keep, self.keep, self.ur, self.depth = f.host()
        self.ent_all = f.out["kp_entropy"].cpu().numpy()[:len(self.kps_all)].copy()
        self.kps = self.kps_all[self.keep]
        self.ent = self.ent_all[self.keep]
        self.depth_all = self.z_all.cpu().numpy()[:len(self.kps_all)].copy()


@pytest.fixture(scope="module")
def tails(seg, ext, kitti_bgr):
    """The Tail of the KITTI fixture crop and synthetic frames 0-2, keyed "kitti", 0, 1, 2."""
    out = {}
    for f in ["kitti", 0, 1, 2]:
        if f == "kitti":  # the fixture frame has no right image: the left one shifted by 12 px stands in for it
            gl = crop(bgr_to_gray(kitti_bgr))
            bgr, gr = crop(kitti_bgr), np.ascontiguousarray(np.roll(gl, -12, axis=1))
        else:
            bgr, gl, gr = synth(f)
        out[f] = Tail(seg, ext[0], ext[1], bgr, gl, gr)
        assert out[f].n_keep > 100 and (out[f].depth > 0).sum() > 30, (f, out[f].n_keep)
    return out
