"""-m gpu: the frame pose (sivo_pose_optimize / _device, sivo_pose_gather_device, sivo_dbg_pose_system) against
oracle/pose_oracle.py: one linearisation bit for bit in the kernel's reduction order, whole optimisations to 1e-9, the device
form against the host form, the edge cases and error codes, and three frames in flight through gather -> pose -> gather -> pose."""
import ctypes as C

import numpy as np
import pytest
import torch

from frame_support import extractor
from oracle import pose_oracle as P
from oracle.keymap import keymap
from oracle.pose_scene import CAM, embed, exact_scene, pose34, rotation, scene
from sivo_b200 import _lib as L
from sivo_b200 import PoseResult, map_points, pose_gather_device, pose_optimize, pose_optimize_device
from sivo_b200.orb import KP_DTYPE
from sivo_b200.pose import camera_from_result, frame_from_result, pose_system, result_from_bytes

pytestmark = pytest.mark.gpu

INTR = (CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.mbf)
SCENES = [(seed, n, mode, out) for seed, (n, mode) in enumerate([(120, "mono"), (400, "stereo"), (800, "mixed"), (2000, "mixed")])
          for out in (0.0, 0.1, 0.3)]


@pytest.fixture(scope="module")
def ext():
    return extractor()


def inv_sigma2(ext):
    return ext.GetInverseScaleSigmaSquares()


def pose7(T: P.Pose):
    return np.r_[T.q, T.t]


def check_result(res: PoseResult, outl, ref: P.Result, exact=False):
    if exact:
        assert np.array_equal(res.pose(), ref.Tcw) and np.array_equal(np.array(res.q), ref.q) and np.array_equal(np.array(res.t), ref.t)
    R = P.rotation_matrix(np.array(res.q))
    assert np.abs(R - P.rotation_matrix(ref.q)).max() <= 1e-9
    assert np.abs(np.array(res.t) - ref.t).max() <= 1e-9 * (np.abs(ref.t).max() + 1)
    assert res.sigma_valid == ref.sigma_valid and res.rounds_run == ref.rounds_run and res.n_initial == ref.n_initial
    if ref.sigma_valid:
        assert np.linalg.norm(res.sigma() - ref.sigma) <= 1e-8 * np.linalg.norm(ref.sigma)
    # flags: identical except edges whose oracle chi2 sits within 1e-6 relative of 7.815f
    near = np.zeros(len(outl), bool)
    with np.errstate(invalid="ignore"):
        near[ref.edges.key] = np.abs(ref.chi2 - float(P.CHI2_STEREO)) <= 1e-6 * float(P.CHI2_STEREO)
    assert np.array_equal(outl[~near], ref.outlier[~near])
    if not near.any():
        assert res.n_good == ref.n_good and res.n_bad == ref.n_bad
    return int(near.sum())


# ---------------------------------------------------------------------------------------------------------- one linearisation
@pytest.mark.parametrize("seed,n,mode,out", SCENES)
def test_system_is_bit_identical_to_the_device_order(ext, seed, n, mode, out):
    kps, ur, X, Tin, _ = scene(seed, n=n, mode=mode, outliers=out)
    E = P.make_edges(kps, ur, X, inv_sigma2(ext))
    T = P.to_se3quat(Tin)
    rng = np.random.default_rng(seed)
    level1 = (rng.uniform(size=n) < 0.1).astype(np.uint8)
    for robust_stereo in (True, False):
        robust = ~E.stereo | robust_stereo
        active = level1[E.key] == 0
        g = pose_system(ext, kps, ur, X, pose7(T), *INTR, robust_stereo=robust_stereo, level1=level1)
        d = P.system(E, T, CAM, robust, active, "device")
        ev = d.ev
        k = E.key
        assert np.array_equal(g["err"][k], ev.err) and np.array_equal(g["chi2"][k], ev.chi2, equal_nan=True)
        assert np.array_equal(g["rho"][k], np.c_[ev.rho0, ev.rho1], equal_nan=True)
        assert np.array_equal(g["jac"][k], ev.J)
        assert np.array_equal(g["H"], d.H) and np.array_equal(g["b"], d.b) and g["chi"] == d.chi
        s = P.system(E, T, CAM, robust, active, "sequential")
        assert np.abs(g["H"] - s.H).max() <= 1e-12 * np.abs(s.H).max() and abs(g["chi"] - s.chi) <= 1e-12 * s.chi


# ---------------------------------------------------------------------------------------------------------- whole optimisation
@pytest.mark.parametrize("seed,n,mode,out", SCENES)
def test_optimisation_against_the_oracle(ext, seed, n, mode, out):
    kps, ur, X, Tin, _ = scene(seed, n=n, mode=mode, outliers=out)
    res, outl = pose_optimize(ext, kps, ur, X, Tin, *INTR)
    ref = P.pose_optimization(kps, ur, X, Tin, inv_sigma2(ext), CAM, order="device")
    near = check_result(res, outl, ref)
    print(f"scene {seed}/{mode}/{out}: n_good {res.n_good} (oracle {ref.n_good}), {near} edges within 1e-6 of 7.815f")


@pytest.mark.parametrize("mode", ["mono", "stereo", "mixed"])
def test_noise_free_scene_reaches_the_true_pose(ext, mode):
    cam, kps, ur, X = exact_scene(mode)
    Tin = pose34(rotation(0.01, -0.02, 0.015), (0.05, -0.03, 0.08))
    res, _ = pose_optimize(ext, kps, ur, X, Tin, cam.fx, cam.fy, cam.cx, cam.cy, cam.mbf)
    assert np.abs(P.rotation_matrix(np.array(res.q)) - np.eye(3)).max() <= 1e-9 and np.abs(np.array(res.t)).max() <= 1e-9


# ---------------------------------------------------------------------------------------------------------- device form
class Bufs:
    def __init__(self, cap):
        self.cap = cap
        self.kps = torch.zeros(cap * 28, dtype=torch.uint8, device="cuda")
        self.keep = torch.full((cap,), -1, dtype=torch.int32, device="cuda")
        self.n = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.ur = torch.zeros(cap, dtype=torch.float32, device="cuda")
        self.xw = torch.full((cap * 3,), float("nan"), dtype=torch.float32, device="cuda")
        self.T = torch.zeros(12, dtype=torch.float32, device="cuda")
        self.res = torch.full((512,), 0x55, dtype=torch.uint8, device="cuda")
        self.out = torch.full((cap,), 7, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()

    def load(self, kps, ur, X, Tin, keep=None, n=None):
        """Keys scattered into extractor slots: semantic key j is slot keep[j]."""
        k = len(kps)
        keep = np.arange(k, dtype=np.int32) if keep is None else np.asarray(keep, np.int32)
        slots = np.zeros(self.cap, KP_DTYPE)
        ok = (keep >= 0) & (keep < self.cap)
        slots[keep[ok]] = kps[ok]
        self.kps.copy_(torch.from_numpy(slots.view(np.uint8).reshape(-1).copy()))
        self.keep[:k].copy_(torch.from_numpy(keep))
        self.n.fill_(k if n is None else n)
        self.ur[:k].copy_(torch.from_numpy(np.ascontiguousarray(ur, np.float32)))
        self.xw.fill_(float("nan"))
        self.xw[:3 * k].copy_(torch.from_numpy(np.ascontiguousarray(X, np.float32).reshape(-1)))
        self.T.copy_(torch.from_numpy(np.ascontiguousarray(Tin, np.float32).reshape(-1)))
        torch.cuda.synchronize()

    def run(self, ext, stream=0, keep=True, intr=INTR):
        pose_optimize_device(ext, self.kps.data_ptr(), self.keep.data_ptr() if keep else 0, self.n.data_ptr(), self.ur.data_ptr(),
                             self.xw.data_ptr(), *intr, self.T.data_ptr(), self.res.data_ptr(), self.out.data_ptr(), stream)

    def host(self, k):
        torch.cuda.synchronize()
        return result_from_bytes(self.res.cpu().numpy()), self.out.cpu().numpy()[:max(k, 0)].astype(bool)


def same_result(a: PoseResult, b: PoseResult):
    return bytes(a) == bytes(b)


@pytest.mark.parametrize("seed,n,mode,out", SCENES[::2])
def test_device_form_equals_the_host_form_and_repeats(ext, seed, n, mode, out):
    kps, ur, X, Tin, _ = scene(seed, n=n, mode=mode, outliers=out)
    res, outl = pose_optimize(ext, kps, ur, X, Tin, *INTR)
    b = Bufs(ext.capacity())
    b.load(kps, ur, X, Tin, keep=keymap(n, ext.capacity(), np.random.default_rng(seed), junk=False).keep[:n])
    for _ in range(2):
        b.run(ext)
        r2, o2 = b.host(n)
        assert same_result(res, r2) and np.array_equal(outl, o2)


# ---------------------------------------------------------------------------------------------------------- edge cases
@pytest.mark.parametrize("n_edges", [0, 2, 3, 9])
def test_few_edges(ext, n_edges):
    kps, ur, X, Tin, _ = scene(3, n=30, mode="mixed")
    X = X.copy()
    X[n_edges:] = np.nan
    res, outl = pose_optimize(ext, kps, ur, X, Tin, *INTR)
    ref = P.pose_optimization(kps, ur, X, Tin, inv_sigma2(ext), CAM, order="device")
    check_result(res, outl, ref, exact=n_edges < 3)
    assert res.n_initial == n_edges and (res.rounds_run == (0 if n_edges < 3 else 1))
    if n_edges < 3:
        assert res.n_good == 0 and not res.sigma_valid and not outl.any()


def test_degenerate_scene_has_no_covariance(ext):
    """Every point on the optical axis, observed exactly at the identity: H's omega_z / upsilon_z columns are zero."""
    n = 20
    kps = np.zeros(n, KP_DTYPE)
    kps["x"], kps["y"] = np.float32(CAM.cx), np.float32(CAM.cy)
    X = np.tile(np.array([0, 0, 8], np.float32), (n, 1))
    ur = np.full(n, -1, np.float32)
    Tin = pose34(np.eye(3), np.zeros(3))
    res, outl = pose_optimize(ext, kps, ur, X, Tin, *INTR)
    ref = P.pose_optimization(kps, ur, X, Tin, inv_sigma2(ext), CAM, order="device")
    assert not ref.sigma_valid and res.sigma_valid == 0
    check_result(res, outl, ref, exact=True)


def test_nan_rule_points_behind_and_on_the_camera_plane(ext):
    kps, ur, X, _, Ttrue = scene(6, n=100, mode="mixed", noise=0.3)
    X = X.copy()
    R, t = Ttrue[:, :3].astype(float), Ttrue[:, 3].astype(float)
    X[0] = ((np.array([1.0, 0.5, -10.0]) - t) @ R).astype(np.float32)    # behind the camera
    X[1] = ((np.array([0.0, 0.0, 0.0]) - t) @ R).astype(np.float32)      # at the camera centre
    X[2, 0] = np.nan                                                      # a key without a point
    ur[3] = np.nan                                                        # NaN mvRight: a stereo edge with a NaN error
    res, outl = pose_optimize(ext, kps, ur, X, Ttrue, *INTR)
    ref = P.pose_optimization(kps, ur, X, Ttrue, inv_sigma2(ext), CAM, order="device")
    check_result(res, outl, ref)
    assert outl[3] and not outl[2] and res.n_initial == 99


def test_keep_idx_with_negative_and_out_of_capacity_entries(ext):
    cap = ext.capacity()
    kps, ur, X, Tin, _ = scene(7, n=300, mode="mixed", outliers=0.1)
    km = keymap(300, cap, np.random.default_rng(7))
    b = Bufs(cap)
    b.load(*embed(km, kps, ur, X), Tin, keep=km.keep[:km.n_keep])
    b.run(ext)
    r, o = b.host(km.n_keep)
    ref = P.pose_optimization(kps, ur, X, Tin, inv_sigma2(ext), CAM, order="device")
    check_result(r, o[km.real], ref)
    assert r.n_initial == 300 and not o[km.src < 0].any()


def test_count_equal_to_capacity_and_the_minus_one_count(ext):
    cap = ext.capacity()
    kps, ur, X, Tin, _ = scene(8, n=cap, mode="mixed", outliers=0.1)
    b = Bufs(cap)
    b.load(kps, ur, X, Tin, n=cap + 50)  # clamped to the capacity
    b.run(ext, keep=False)
    r, o = b.host(cap)
    h, ho = pose_optimize(ext, kps, ur, X, Tin, *INTR)
    assert same_result(r, h) and np.array_equal(o, ho)
    b.res.fill_(0x55)
    b.out.fill_(7)
    b.n.fill_(-1)
    torch.cuda.synchronize()
    b.run(ext)
    r, _ = b.host(0)
    raw = b.res.cpu().numpy()
    assert r.n_good == -1 and (b.out.cpu().numpy() == 7).all()
    off = PoseResult.n_good.offset
    assert (np.delete(raw, np.arange(off, off + 4)) == 0x55).all()


def test_error_codes(ext):
    kps, ur, X, Tin, _ = scene(9, n=20)
    for intr in ((0.0, 1, 1, 1, 1), (1, float("nan"), 1, 1, 1), (1, 1, 1, 1, -2.0), (1, 1, float("inf"), 1, 1)):
        with pytest.raises(L.SivoError) as e:
            pose_optimize(ext, kps, ur, X, Tin, *intr)
        assert e.value.code == L.EINVAL
    lib = L.lib()
    res = PoseResult()
    assert lib.sivo_pose_optimize(None, None, None, None, 0, 1, 1, 1, 1, 1, None, C.byref(res), None) == L.EINVAL
    T = np.zeros(12, np.float32)
    assert lib.sivo_pose_optimize(ext._h, None, None, None, -1, 1, 1, 1, 1, 1, T.ctypes.data_as(C.c_void_p), C.byref(res), None) == L.EINVAL
    assert lib.sivo_pose_optimize_device(ext._h, None, None, None, None, None, 1, 1, 1, 1, 1, None, None, None, None) == L.EINVAL
    assert lib.sivo_pose_gather_device(ext._h, None, None, None, 0, None, None) == L.EINVAL
    bad = kps.copy()
    bad["octave"][0] = 8
    with pytest.raises(L.SivoError) as e:
        pose_optimize(ext, bad, ur, X, Tin, *INTR)
    assert e.value.code == L.ERANGE


# ---------------------------------------------------------------------------------------------------------- chain
def test_three_frames_in_flight_gather_pose_gather_pose(ext):
    """Per frame, on rotating buffers and one stream: the last-frame matches gathered into xw, the pose optimised from the
    predicted pose, the outliers dropped, the local-map matches merged into xw by a second gather, the pose optimised again from
    the first result.  The host reads only the small result between the two; the selection's camera is built from the second."""
    cap = ext.capacity()
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    bufs = [Bufs(cap) for _ in range(3)]
    extra = []
    cases = []
    for f in range(3):
        kps, ur, X, Tin, _ = scene(20 + f, n=600, mode="mixed", outliers=0.2)
        pts = map_points(np.zeros((600, 32), np.uint8), X, np.zeros((600, 3)), 0, 1e9)
        pts["pos"][np.isnan(X[:, 0])] = 0
        m_last = np.where(np.arange(600) % 2 == 0, np.arange(600), -1).astype(np.int32)
        m_local = np.where(np.arange(600) % 2 == 1, np.arange(600), -1).astype(np.int32)
        b = bufs[f]
        b.load(kps, ur, np.full_like(X, np.nan), Tin)
        d = dict(pts=torch.from_numpy(pts.view(np.uint8).reshape(-1).copy()).cuda(),
                 m1=torch.from_numpy(m_last).cuda(), m2=torch.from_numpy(m_local).cuda(),
                 res2=torch.zeros(512, dtype=torch.uint8, device="cuda"), out2=torch.zeros(cap, dtype=torch.uint8, device="cuda"))
        torch.cuda.synchronize()
        extra.append(d)
        cases.append((kps, ur, X, Tin, m_last, m_local))
    with torch.cuda.stream(stream):
        for f, (b, d) in enumerate(zip(bufs, extra)):
            pose_gather_device(ext, d["m1"].data_ptr(), b.n.data_ptr(), d["pts"].data_ptr(), 600, b.xw.data_ptr(), s)
            b.run(ext, s)
    firsts = []
    for f, (b, d) in enumerate(zip(bufs, extra)):
        stream.synchronize()
        r1 = result_from_bytes(b.res.cpu().numpy())
        firsts.append(r1)
        frame_from_result(r1, *INTR, (0.0, 1024.0, 0.0, 352.0))  # what the local-map search would take
        with torch.cuda.stream(stream):
            o = b.out[:600].bool().repeat_interleave(3)
            xw = b.xw[:1800]
            xw.masked_fill_(o, float("nan"))
            pose_gather_device(ext, d["m2"].data_ptr(), b.n.data_ptr(), d["pts"].data_ptr(), 600, b.xw.data_ptr(), s)
            pose_optimize_device(ext, b.kps.data_ptr(), b.keep.data_ptr(), b.n.data_ptr(), b.ur.data_ptr(), b.xw.data_ptr(), *INTR,
                                 b.res.data_ptr(), d["res2"].data_ptr(), d["out2"].data_ptr(), s)
    stream.synchronize()
    for f, (b, d) in enumerate(zip(bufs, extra)):
        kps, ur, X, Tin, m1, m2 = cases[f]
        x1 = np.where((m1 >= 0)[:, None], X, np.nan).astype(np.float32)
        r1 = P.pose_optimization(kps, ur, x1, Tin, inv_sigma2(ext), CAM, order="device")
        check_result(firsts[f], b.out.cpu().numpy()[:600].astype(bool), r1)
        x2 = x1.copy()
        x2[r1.outlier] = np.nan
        x2[m2 >= 0] = X[m2 >= 0]
        r2 = P.pose_optimization(kps, ur, x2, firsts[f].pose(), inv_sigma2(ext), CAM, order="device")
        res2 = result_from_bytes(d["res2"].cpu().numpy())
        check_result(res2, d["out2"].cpu().numpy()[:600].astype(bool), r2)
        cam = camera_from_result(res2, CAM.fx, CAM.fy, CAM.cx, CAM.cy, CAM.mbf / CAM.fx, np.eye(6))
        assert np.array_equal(np.array(cam.Rwc, np.float32), np.array(res2.Rwc, np.float32))
