"""-m gpu: the device forms of the Frame tail -- SelectSemanticKeys (sivo_segnet_semantic_keys_device) and ComputeStereoMatches
(sivo_stereo_match_device) -- on the extractors' device outputs, against the host forms, the oracle, and an asynchronous
SegNet -> extractors -> semantic keys -> stereo chain with one host synchronisation."""
import os

import numpy as np
import pytest
import torch

from oracle import orb_oracle as O
from sivo_b200 import KP_DTYPE, BayesianSegNet, BayesianSegNetParams, ORBextractor, stereo_match, stereo_match_device
from sivo_b200 import _lib as L
from sivo_b200.synth import bgr_to_gray, stereo_frame

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W, Y0, X0 = 352, 1024, 11, 109  # the network's input: the centre crop (109, 11) of a 1242x375 frame
KITTI_MBF = 386.1448  # Camera.bf of config/kitti/KITTI00-02.yaml; mb = bf / fx
BASELINES = {"kitti": (KITTI_MBF / 718.856, KITTI_MBF), "wide": (0.8, 400.0)}


@pytest.fixture(scope="module")
def seg(model_dir):
    """The shipped Basic topology at T=2 with the calibrated synthetic weights (the file other GPU tests write)."""
    from sivo_b200.caffemodel import shipped_scales, write_synth_model
    from sivo_b200.prototxt import load_net
    proto = os.path.join(ROOT, "configs", "bayesian_segnet_basic.prototxt")
    model = os.path.join(str(model_dir), "basic_full.caffemodel")
    if not os.path.exists(model):
        write_synth_model(load_net(open(proto).read(), T=2), model, 0, shipped_scales("basic"))
    return BayesianSegNet(BayesianSegNetParams(proto, model), seed=7, T=2, precision="fp16", engine="auto")


def crop(img):
    return np.ascontiguousarray(img[Y0:Y0 + H, X0:X0 + W])


def synth(seed):
    left, right = stereo_frame(seed)
    return crop(left), crop(bgr_to_gray(left)), crop(bgr_to_gray(right))


def ptr(t):
    return t.data_ptr()


def to_dev(a):
    """A device copy that is complete before anything else is enqueued (the library's streams do not wait for torch's)."""
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


class DeviceKeys:
    """The buffers sivo_orb_enqueue_device fills for one extractor: capacity() records, descriptors and an int64 count."""

    def __init__(self, ext):
        self.cap = ext.capacity()
        self.kps = torch.zeros(self.cap * 28, dtype=torch.uint8, device="cuda")
        self.desc = torch.zeros(self.cap * 32, dtype=torch.uint8, device="cuda")
        self.cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()

    def enqueue(self, ext, gray_dev):
        ext.enqueue_device(ptr(gray_dev), H, W, W, ptr(self.kps), ptr(self.desc), ptr(self.cnt))

    def host(self):
        n = int(self.cnt.cpu()[0])
        return self.kps.cpu().numpy()[:n * 28].view(KP_DTYPE).copy(), self.desc.cpu().numpy()[:n * 32].reshape(n, 32).copy()


class SemanticOut:
    def __init__(self, cap):
        self.cls = torch.full((cap,), 77, dtype=torch.uint8, device="cuda")
        self.conf = torch.full((cap,), 7.0, dtype=torch.float64, device="cuda")
        self.ent = torch.full((cap,), 7.0, dtype=torch.float64, device="cuda")
        self.keep = torch.full((cap,), -7, dtype=torch.int32, device="cuda")
        self.n = torch.full((1,), -7, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()

    def run(self, seg, dk, max_static_class, stream, cap=None):
        seg.semantic_keys_device(ptr(dk.kps), ptr(dk.cnt), dk.cap if cap is None else cap, max_static_class, ptr(self.cls),
                                 ptr(self.conf), ptr(self.ent), ptr(self.keep), ptr(self.n), stream)

    def host(self):
        n = int(self.n.cpu()[0])
        return n, self.keep.cpu().numpy()[:max(n, 0)].copy()


class StereoOut:
    def __init__(self, cap):
        self.u = torch.full((cap,), 7.0, dtype=torch.float32, device="cuda")
        self.z = torch.full((cap,), 7.0, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()

    def run(self, el, er, dl_keys, dr_keys, mb, mbf, stream, keep=None, n_left=None):
        stereo_match_device(el, er, ptr(dl_keys.kps), ptr(dl_keys.desc), 0 if keep is None else ptr(keep),
                            ptr(dl_keys.cnt if n_left is None else n_left), ptr(dr_keys.kps), ptr(dr_keys.desc), ptr(dr_keys.cnt), mb, mbf,
                            ptr(self.u), ptr(self.z), stream)

    def host(self, n):
        return self.u.cpu().numpy()[:n].copy(), self.z.cpu().numpy()[:n].copy()


def extractors(nf, nlevels=8):
    return ORBextractor(nf, 1.2, nlevels, 20, 7), ORBextractor(nf, 1.2, nlevels, 20, 7)


# ---------------------------------------------------------------------------------------------------------- semantic keys
@pytest.mark.parametrize("frame", ["kitti", 0, 1, 2])
def test_semantic_keys_device_equals_the_host_form(seg, kitti_bgr, frame):
    bgr, gray = (crop(kitti_bgr), crop(bgr_to_gray(kitti_bgr))) if frame == "kitti" else synth(frame)[:2]
    seg.set_frame(5)
    seg.segment_on_device(bgr)
    ext = ORBextractor(2000, 1.2, 8, 20, 7)
    dk = DeviceKeys(ext)
    stream = torch.cuda.Stream()
    dk.enqueue(ext, to_dev(gray))
    ext.stream_wait(stream.cuda_stream)
    stream.synchronize()
    kps, _ = dk.host()
    assert len(kps) > 500
    for msc in (-1, 8, 14):
        out = SemanticOut(dk.cap)
        out.run(seg, dk, msc, stream.cuda_stream)
        stream.synchronize()
        cls, conf, ent, keep = seg.semantic_keys(kps, msc)
        n = len(kps)
        n_keep, got_keep = out.host()
        assert n_keep == len(keep) and np.array_equal(got_keep, keep), msc
        assert np.array_equal(out.cls.cpu().numpy()[:n], cls)
        assert out.conf.cpu().numpy()[:n].tobytes() == conf.tobytes() and out.ent.cpu().numpy()[:n].tobytes() == ent.tobytes()
        assert (out.keep.cpu().numpy()[n_keep:] == -7).all() and (out.cls.cpu().numpy()[n:] == 77).all()
    assert 0 < len(seg.semantic_keys(kps, 8)[3]) < len(kps)


def test_semantic_keys_device_out_of_map_keys_count_above_cap_and_null_outputs(seg):
    bgr, _, _ = synth(3)
    seg.set_frame(1)
    seg.segment_on_device(bgr)
    rng = np.random.default_rng(3)
    kps = np.zeros(700, KP_DTYPE)
    kps["x"] = rng.uniform(-20, W + 20, len(kps)).astype(np.float32)
    kps["y"] = rng.uniform(-20, H + 20, len(kps)).astype(np.float32)
    kps["x"][:3] = (-0.5, 1e9, W - 0.25)  # -0.5 truncates to column 0, as int(pt.x) does
    cap = 1024
    dk = type("K", (), {})()
    dk.cap = cap
    dk.kps = torch.zeros(cap * 28, dtype=torch.uint8, device="cuda")
    dk.kps[:len(kps) * 28] = torch.from_numpy(kps.view(np.uint8))
    dk.cnt = torch.tensor([len(kps)], dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    out = SemanticOut(cap)
    out.run(seg, dk, 14, stream.cuda_stream)
    stream.synchronize()
    cls, conf, ent, keep = seg.semantic_keys(kps, 14)
    assert (cls == 255).sum() > 10
    assert np.array_equal(out.cls.cpu().numpy()[:len(kps)], cls) and np.array_equal(out.host()[1], keep)
    assert out.conf.cpu().numpy()[:len(kps)].tobytes() == conf.tobytes()
    # only the count and the keep list wanted
    only = SemanticOut(cap)
    L.check(L.lib().sivo_segnet_semantic_keys_device(seg._h, ptr(dk.kps), ptr(dk.cnt), cap, 14, None, None, None, ptr(only.keep),
                                                     ptr(only.n), stream.cuda_stream))
    stream.synchronize()
    assert np.array_equal(only.host()[1], keep) and (only.cls.cpu().numpy() == 77).all()
    # zero keys, and a count above the buffers' capacity: n_keep = -1 and nothing else written
    for count, want in ((0, 0), (cap + 1, -1)):
        dk.cnt.fill_(count)
        torch.cuda.synchronize()
        o = SemanticOut(cap)
        o.run(seg, dk, 14, stream.cuda_stream)
        stream.synchronize()
        assert int(o.n.cpu()[0]) == want
        assert (o.cls.cpu().numpy() == 77).all() and (o.keep.cpu().numpy() == -7).all() and (o.conf.cpu().numpy() == 7.0).all()


def test_semantic_keys_host_form_reads_maps_still_in_flight(seg):
    """The host form runs on the stream of the last run: it reads that run's maps although the host has not waited for them."""
    (bgr_a, _, _), (bgr_b, gray_b, _) = synth(20), synth(21)
    kps, _ = ORBextractor(2000, 1.2, 8, 20, 7)(gray_b, None)
    maps = [torch.empty(H * W, dtype=t, device="cuda") for t in (torch.uint8, torch.float64, torch.float64)]
    d_a, d_b = to_dev(bgr_a), to_dev(bgr_b)
    side = torch.cuda.Stream()

    def run(d_bgr, frame):
        seg.set_frame(frame)
        seg.run_device_maps(ptr(d_bgr), *(ptr(m) for m in maps), 0, 0, side.cuda_stream)

    run(d_b, 41)  # first use of the stream: the network's graph is captured here
    side.synchronize()
    run(d_a, 40)
    side.synchronize()
    maps_a = [m.cpu().numpy().reshape(H, W) for m in maps]
    xy = np.stack([kps["x"], kps["y"]], 1)
    want_a = O.select_semantic_keys(xy, *maps_a)
    # also sizes the call's staging buffers: allocating them in the call below would serialise it behind the side stream
    assert all(np.array_equal(g, w) for g, w in zip(seg.semantic_keys(kps, 8), want_a))
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)  # frame B's maps are written only after this spin
    run(d_b, 41)
    got = seg.semantic_keys(kps, 8)  # no host synchronisation before this call
    side.synchronize()
    want = O.select_semantic_keys(xy, *[m.cpu().numpy().reshape(H, W) for m in maps])
    assert all(np.array_equal(g, w) for g, w in zip(got, want)) and len(want[3]) > 0
    assert not np.array_equal(want_a[1], want[1])  # frame A's maps would show


# ---------------------------------------------------------------------------------------------------------- stereo
@pytest.mark.parametrize("nf", [1000, 2000])
@pytest.mark.parametrize("baseline", sorted(BASELINES))
@pytest.mark.parametrize("with_keep", [False, True])
def test_stereo_device_equals_the_host_form_and_the_oracle(nf, baseline, with_keep):
    mb, mbf = BASELINES[baseline]
    _, gl, gr = synth(1)
    el, er = extractors(nf)
    kl, dl = el(gl, None)  # synchronous runs: the host pyramids for the oracle, the keypoints for the host form
    kr, dr = er(gr, None)
    dkl, dkr = DeviceKeys(el), DeviceKeys(er)
    dkl.enqueue(el, to_dev(gl))
    dkr.enqueue(er, to_dev(gr))
    stream = torch.cuda.Stream()
    out = StereoOut(dkl.cap)
    if with_keep:
        keep = np.sort(np.random.default_rng(nf).choice(len(kl), len(kl) * 2 // 3, replace=False)).astype(np.int32)
        d_keep = torch.from_numpy(keep).cuda()
        d_n = torch.tensor([len(keep)], dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        out.run(el, er, dkl, dkr, mb, mbf, stream.cuda_stream, keep=d_keep, n_left=d_n)
    else:
        keep = np.arange(len(kl), dtype=np.int32)
        out.run(el, er, dkl, dkr, mb, mbf, stream.cuda_stream)
    stream.synchronize()
    assert np.array_equal(dkl.host()[0].view(np.uint8), kl.view(np.uint8))
    u, z = out.host(len(keep))
    hu, hz = stereo_match(el, er, kl[keep], dl[keep], kr, dr, mb, mbf)
    assert u.tobytes() == hu.tobytes() and z.tobytes() == hz.tobytes()
    ru, rz = O.compute_stereo_matches(kl[keep], dl[keep], kr, dr, el._bordered, er._bordered, el.GetScaleFactors(),
                                      el.GetInverseScaleFactors(), mb, mbf)
    assert u.tobytes() == ru.tobytes() and z.tobytes() == rz.tobytes()
    assert (u >= 0).sum() > 50
    assert (out.u.cpu().numpy()[len(keep):] == 7.0).all()


def test_stereo_device_edge_cases():
    mb, mbf = BASELINES["kitti"]
    _, gl, gr = synth(2)
    el, er = extractors(1000)
    kl, dl = el(gl, None)
    kr, dr = er(gr, None)
    dkl, dkr = DeviceKeys(el), DeviceKeys(er)
    dkl.enqueue(el, to_dev(gl))
    dkr.enqueue(er, to_dev(gr))
    torch.cuda.synchronize()  # the copies below read the extractors' outputs on torch's stream
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    zero = torch.zeros(1, dtype=torch.int64, device="cuda")
    keep = torch.arange(dkl.cap, dtype=torch.int32, device="cuda")
    # zero left keypoints, zero kept keys, a negative count (count above capacity upstream): nothing written
    for kw in ({"n_left": zero}, {"keep": keep, "n_left": zero}, {"keep": keep, "n_left": torch.full((1,), -1, dtype=torch.int64, device="cuda")}):
        out = StereoOut(dkl.cap)
        out.run(el, er, dkl, dkr, mb, mbf, s, **kw)
        stream.synchronize()
        assert (out.u.cpu().numpy() == 7.0).all() and (out.z.cpu().numpy() == 7.0).all()
    # zero right keypoints: every left keypoint unmatched
    n = len(kl)
    out = StereoOut(dkl.cap)
    stereo_match_device(el, er, ptr(dkl.kps), ptr(dkl.desc), 0, ptr(dkl.cnt), ptr(dkr.kps), ptr(dkr.desc), ptr(zero), mb, mbf,
                        ptr(out.u), ptr(out.z), s)
    stream.synchronize()
    u, z = out.host(n)
    assert (u == -1).all() and (z == -1).all() and (out.u.cpu().numpy()[n:] == 7.0).all()
    # no match surviving: every right keypoint moved right of every left one, i.e. outside the disparity window [0, mbf / mb)
    moved_kr = kr.copy()
    moved_kr["x"] += np.float32(5000)
    moved = DeviceKeys(er)
    moved.kps[:len(kr) * 28] = torch.from_numpy(moved_kr.view(np.uint8))
    moved.desc.copy_(dkr.desc)
    moved.cnt.copy_(dkr.cnt)
    torch.cuda.synchronize()
    out = StereoOut(dkl.cap)
    out.run(el, er, dkl, moved, mb, mbf, s)
    stream.synchronize()
    u, z = out.host(n)
    hu, hz = stereo_match(el, er, kl, dl, moved_kr, dr, mb, mbf)
    assert (u == -1).all() and (z == -1).all() and np.array_equal(u, hu) and np.array_equal(z, hz)
    # left keypoints with an octave outside [0, nlevels) stay unmatched; the others keep their results
    bad = kl.copy()
    bad["octave"][::3] = 99
    bad_dev = DeviceKeys(el)
    bad_dev.kps[:n * 28] = torch.from_numpy(bad.view(np.uint8))
    bad_dev.desc.copy_(dkl.desc)
    bad_dev.cnt.copy_(dkl.cnt)
    torch.cuda.synchronize()
    out = StereoOut(dkl.cap)
    out.run(el, er, bad_dev, dkr, mb, mbf, s)
    stream.synchronize()
    u, z = out.host(n)
    assert (u[::3] == -1).all() and (z[::3] == -1).all()
    # an unmatched key does not enter the median, so the others get what the host form gives for them alone
    sel = np.setdiff1d(np.arange(n), np.arange(0, n, 3)).astype(np.int32)
    hu, hz = stereo_match(el, er, kl[sel], dl[sel], kr, dr, mb, mbf)
    assert u[sel].tobytes() == hu.tobytes() and z[sel].tobytes() == hz.tobytes() and (hu >= 0).sum() > 20


def test_stereo_host_form_takes_more_left_keys_than_the_capacity():
    """The host form sizes its buffers from the call, not from the left extractor's capacity()."""
    mb, mbf = BASELINES["kitti"]
    _, gl, gr = synth(1)
    el, er = extractors(1000)
    kl, dl = el(gl, None)
    kr, dr = er(gr, None)
    kl2, dl2 = np.concatenate([kl, kl]), np.concatenate([dl, dl])
    assert len(kl2) > el.capacity()
    u, z = stereo_match(el, er, kl2, dl2, kr, dr, mb, mbf)
    ru, rz = O.compute_stereo_matches(kl2, dl2, kr, dr, el._bordered, er._bordered, el.GetScaleFactors(), el.GetInverseScaleFactors(),
                                      mb, mbf)
    assert u.tobytes() == ru.tobytes() and z.tobytes() == rz.tobytes()
    assert (u[len(kl):] >= 0).sum() > 50


def test_error_codes(seg, model_dir):
    lib = L.lib()
    mb, mbf = BASELINES["kitti"]
    el, er = extractors(500)
    dkl, dkr = DeviceKeys(el), DeviceKeys(er)
    out = StereoOut(dkl.cap)
    sem = SemanticOut(dkl.cap)
    args = lambda: [ptr(dkl.kps), ptr(dkl.desc), None, ptr(dkl.cnt), ptr(dkr.kps), ptr(dkr.desc), ptr(dkr.cnt), mb, mbf, ptr(out.u), ptr(out.z), None]
    # extractors that have not run
    assert lib.sivo_stereo_match_device(el._h, er._h, *args()) == L.EINVAL
    _, gl, gr = synth(0)
    dkl.enqueue(el, to_dev(gl))
    assert lib.sivo_stereo_match_device(el._h, er._h, *args()) == L.EINVAL
    dkr.enqueue(er, to_dev(gr))
    assert lib.sivo_stereo_match_device(el._h, er._h, *args()) == L.OK
    # NULL handles and buffers (keep_idx may be NULL)
    assert lib.sivo_stereo_match_device(None, er._h, *args()) == L.EINVAL
    assert lib.sivo_stereo_match_device(el._h, None, *args()) == L.EINVAL
    for i in (0, 1, 3, 4, 5, 6, 9, 10):
        a = args()
        a[i] = None
        assert lib.sivo_stereo_match_device(el._h, er._h, *a) == L.EINVAL, i
    for i, v in ((7, 0.0), (8, -1.0)):
        a = args()
        a[i] = v
        assert lib.sivo_stereo_match_device(el._h, er._h, *a) == L.EINVAL, i
    # extractors with different nlevels
    e4 = ORBextractor(500, 1.2, 4, 20, 7)
    e4(gr, None)
    assert lib.sivo_stereo_match_device(el._h, e4._h, *args()) == L.EINVAL
    assert "differ" in lib.sivo_last_error().decode()
    torch.cuda.synchronize()
    # semantic keys: NULL handle, keypoints or count, negative cap, and a handle that has not run
    sargs = lambda: [ptr(dkl.kps), ptr(dkl.cnt), dkl.cap, 8, ptr(sem.cls), ptr(sem.conf), ptr(sem.ent), ptr(sem.keep), ptr(sem.n), None]
    seg.segment_on_device(synth(0)[0])
    assert lib.sivo_segnet_semantic_keys_device(seg._h, *sargs()) == L.OK
    assert lib.sivo_segnet_semantic_keys_device(None, *sargs()) == L.EINVAL
    for i in (0, 1):
        a = sargs()
        a[i] = None
        assert lib.sivo_segnet_semantic_keys_device(seg._h, *a) == L.EINVAL, i
    a = sargs()
    a[2] = -1
    assert lib.sivo_segnet_semantic_keys_device(seg._h, *a) == L.EINVAL
    fresh = BayesianSegNet(BayesianSegNetParams(seg_paths(model_dir)[0], seg_paths(model_dir)[1]), seed=7, T=2)
    assert lib.sivo_segnet_semantic_keys_device(fresh._h, *sargs()) == L.EINVAL
    torch.cuda.synchronize()


def seg_paths(model_dir):
    return os.path.join(ROOT, "configs", "bayesian_segnet_basic.prototxt"), os.path.join(str(model_dir), "basic_full.caffemodel")


# ---------------------------------------------------------------------------------------------------------- asynchronous chain
def test_stereo_waits_for_the_extractors_itself():
    """Stereo enqueued straight after enqueue_device on another stream, with no manual wait: the call orders itself."""
    mb, mbf = BASELINES["kitti"]
    _, gl, gr = synth(4)
    el, er = extractors(2000)
    kl, dl = el(gl, None)
    kr, dr = er(gr, None)
    hu, hz = stereo_match(el, er, kl, dl, kr, dr, mb, mbf)
    d_gl, d_gr = to_dev(gl), to_dev(gr)
    _, gl2, gr2 = synth(5)  # a different frame first, so that stale pyramids / keypoints would show
    el(gl2, None)
    er(gr2, None)
    dkl, dkr = DeviceKeys(el), DeviceKeys(er)
    stream = torch.cuda.Stream()
    out = StereoOut(dkl.cap)
    dkl.enqueue(el, d_gl)
    dkr.enqueue(er, d_gr)
    out.run(el, er, dkl, dkr, mb, mbf, stream.cuda_stream)
    stream.synchronize()
    u, z = out.host(len(kl))
    assert int(dkl.cnt.cpu()[0]) == len(kl)
    assert u.tobytes() == hu.tobytes() and z.tobytes() == hz.tobytes()


def _chain_frames():
    return [synth(10 + i) for i in range(3)]


def test_three_frames_in_flight_equal_the_host_call_path(seg):
    """SegNet -> two enqueue_device -> semantic keys -> stereo for three frames on rotating buffers, connected only by stream
    and event edges, one host synchronisation at the end; every frame equals the host-call path for that frame."""
    mb, mbf = BASELINES["kitti"]
    frames = _chain_frames()
    el, er = extractors(2000)
    hw = H * W
    d_in = [[torch.from_numpy(x).cuda() for x in f] for f in frames]
    bufs = []
    for _ in frames:
        b = {"cls": torch.empty(hw, dtype=torch.uint8, device="cuda"), "conf": torch.empty(hw, dtype=torch.float64, device="cuda"),
             "ent": torch.empty(hw, dtype=torch.float64, device="cuda"), "kl": DeviceKeys(el), "kr": DeviceKeys(er)}
        b["sem"], b["st"] = SemanticOut(b["kl"].cap), StereoOut(b["kl"].cap)
        bufs.append(b)
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    torch.cuda.synchronize()

    def chain(tail=True):
        for i, b in enumerate(bufs):
            bgr, gl, gr = d_in[i]
            seg.set_frame(100 + i)
            seg.run_device_maps(ptr(bgr), ptr(b["cls"]), ptr(b["conf"]), ptr(b["ent"]), 0, 0, s)
            el.wait_for_stream(s)  # the previous frame's stereo has read the pyramids this enqueue overwrites
            er.wait_for_stream(s)
            b["kl"].enqueue(el, gl)
            b["kr"].enqueue(er, gr)
            el.stream_wait(s)  # semantic keys read the left keypoints
            if tail:
                b["sem"].run(seg, b["kl"], 8, s)
                b["st"].run(el, er, b["kl"], b["kr"], mb, mbf, s, keep=b["sem"].keep, n_left=b["sem"].n)
            else:
                er.stream_wait(s)

    chain()  # first use of the stream: the network's graph is captured here
    stream.synchronize()
    for b in bufs:
        for k in ("cls", "conf", "ent"):
            b[k].fill_(0)
        b["sem"].keep.fill_(-7)
        b["st"].u.fill_(7.0)
    torch.cuda.synchronize()
    chain()
    stream.synchronize()  # the one host synchronisation of the chain
    got = [{"maps": [b[k].cpu().numpy() for k in ("cls", "conf", "ent")], "kl": b["kl"].host(), "kr": b["kr"].host(),
            "sem": b["sem"].host(), "sem_vals": (b["sem"].cls.cpu().numpy(), b["sem"].conf.cpu().numpy()),
            "st": (b["st"].u.cpu().numpy(), b["st"].z.cpu().numpy())} for b in bufs]
    # without the tail the network and extractor outputs are the same bits
    chain(tail=False)
    stream.synchronize()
    for b, g in zip(bufs, got):
        for k, m in zip(("cls", "conf", "ent"), g["maps"]):
            assert b[k].cpu().numpy().tobytes() == m.tobytes()
        for side in ("kl", "kr"):
            kp, de = b[side].host()
            assert kp.tobytes() == g[side][0].tobytes() and np.array_equal(de, g[side][1])
    # the host-call path, frame by frame
    for i, (bgr, gl, gr) in enumerate(frames):
        seg.set_frame(100 + i)
        cls, conf, ent = seg.segmentImage(bgr)
        g = got[i]
        assert g["maps"][0].tobytes() == cls.tobytes() and g["maps"][1].tobytes() == conf.tobytes() and g["maps"][2].tobytes() == ent.tobytes()
        kl, dl = el(gl, None)
        kr, dr = er(gr, None)
        assert g["kl"][0].tobytes() == kl.tobytes() and np.array_equal(g["kl"][1], dl) and g["kr"][0].tobytes() == kr.tobytes()
        kc, kf, _, keep = seg.semantic_keys(kl, 8)
        n_keep, dkeep = g["sem"]
        assert n_keep == len(keep) and np.array_equal(dkeep, keep) and 0 < n_keep < len(kl)
        assert np.array_equal(g["sem_vals"][0][:len(kl)], kc) and g["sem_vals"][1][:len(kl)].tobytes() == kf.tobytes()
        hu, hz = stereo_match(el, er, kl[keep], dl[keep], kr, dr, mb, mbf)
        assert g["st"][0][:n_keep].tobytes() == hu.tobytes() and g["st"][1][:n_keep].tobytes() == hz.tobytes()
        assert (hu >= 0).sum() > 20
