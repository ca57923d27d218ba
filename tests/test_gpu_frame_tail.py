"""-m gpu: the device forms of the Frame tail -- SelectSemanticKeys (sivo_segnet_semantic_keys_device) and ComputeStereoMatches
(sivo_stereo_match_device) -- on the extractors' device outputs, against the host forms, the oracle, and an asynchronous
SegNet -> extractors -> semantic keys -> stereo chain with one host synchronisation."""
import numpy as np
import pytest
import torch

from frame_support import BASELINES, H, W, crop, extractors, ptr, seg, seg_paths, synth, upload  # noqa: F401
from oracle import orb_oracle as O
from sivo_b200 import KP_DTYPE, BayesianSegNet, BayesianSegNetParams, ORBextractor, stereo_match, stereo_match_device
from sivo_b200 import _lib as L
from sivo_b200.frame import DeviceFrame, FrameKeys
from sivo_b200.synth import bgr_to_gray

pytestmark = pytest.mark.gpu


def semantic_keys(seg, f, max_static_class, stream, cap=None):
    """sivo_segnet_semantic_keys_device from f's left keys into f's five outputs."""
    seg.semantic_keys_device(f.kps, f.count, f.left.cap if cap is None else cap, max_static_class, f.kp_class, f.kp_conf, f.kp_entropy,
                             f.keep, f.n_keep, stream)


def stereo(f, mb, mbf, stream, keep=0, n_left=None, right=None):
    """sivo_stereo_match_device from f's left keys (keep_idx `keep`, count `n_left`: all of them by default) against the right
    keys `right` (f's by default) into f's u_right / depth."""
    r = f.right if right is None else right
    stereo_match_device(f.el, f.er, f.kps, f.desc, keep, f.count if n_left is None else n_left, ptr(r.kps), ptr(r.desc), ptr(r.count), mb,
                        mbf, f.u_right, f.depth, stream)


# ---------------------------------------------------------------------------------------------------------- semantic keys
@pytest.mark.parametrize("frame", ["kitti", 0, 1, 2])
def test_semantic_keys_device_equals_the_host_form(seg, kitti_bgr, frame):
    bgr, gray = (crop(kitti_bgr), crop(bgr_to_gray(kitti_bgr))) if frame == "kitti" else synth(frame)[:2]
    seg.set_frame(5)
    seg.segment_on_device(bgr)
    el, er = extractors(2000)
    f = DeviceFrame(el, er, H, W)
    stream = torch.cuda.Stream()
    f.left.enqueue(el, upload(gray), H, W, W)
    el.stream_wait(stream.cuda_stream)
    stream.synchronize()
    kps, _ = f.left.host()
    assert len(kps) > 500
    for msc in (-1, 8, 14):
        f.reset()
        semantic_keys(seg, f, msc, stream.cuda_stream)
        stream.synchronize()
        cls, conf, ent, keep = seg.semantic_keys(kps, msc)
        n = len(kps)
        n_keep, got_keep = f.host()[:2]
        assert n_keep == len(keep) and np.array_equal(got_keep, keep), msc
        assert np.array_equal(f.out["kp_class"].cpu().numpy()[:n], cls)
        assert f.out["kp_conf"].cpu().numpy()[:n].tobytes() == conf.tobytes() and f.out["kp_entropy"].cpu().numpy()[:n].tobytes() == ent.tobytes()
        assert (f.out["keep_idx"].cpu().numpy()[n_keep:] == -7).all() and (f.out["kp_class"].cpu().numpy()[n:] == 77).all()
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
    f = DeviceFrame(*extractors(1000), H, W)  # buffers of at least cap entries
    assert f.left.cap >= cap
    f.left.kps[:len(kps) * 28] = torch.from_numpy(kps.view(np.uint8))
    f.left.count.fill_(len(kps))
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    semantic_keys(seg, f, 14, stream.cuda_stream, cap)
    stream.synchronize()
    cls, conf, ent, keep = seg.semantic_keys(kps, 14)
    assert (cls == 255).sum() > 10
    assert np.array_equal(f.out["kp_class"].cpu().numpy()[:len(kps)], cls) and np.array_equal(f.host()[1], keep)
    assert f.out["kp_conf"].cpu().numpy()[:len(kps)].tobytes() == conf.tobytes()
    # only the count and the keep list wanted
    f.reset()
    L.check(L.lib().sivo_segnet_semantic_keys_device(seg._h, f.kps, f.count, cap, 14, None, None, None, f.keep, f.n_keep,
                                                     stream.cuda_stream))
    stream.synchronize()
    assert np.array_equal(f.host()[1], keep) and (f.out["kp_class"].cpu().numpy() == 77).all()
    # zero keys, and a count above the buffers' capacity: n_keep = -1 and nothing else written
    for count, want in ((0, 0), (cap + 1, -1)):
        f.left.count.fill_(count)
        f.reset()
        semantic_keys(seg, f, 14, stream.cuda_stream, cap)
        stream.synchronize()
        assert int(f.out["n_keep"].cpu()[0]) == want
        assert ((f.out["kp_class"].cpu().numpy() == 77).all() and (f.out["keep_idx"].cpu().numpy() == -7).all()
                and (f.out["kp_conf"].cpu().numpy() == 7.0).all())


def test_semantic_keys_host_form_reads_maps_still_in_flight(seg):
    """The host form runs on the stream of the last run: it reads that run's maps although the host has not waited for them."""
    (bgr_a, _, _), (bgr_b, gray_b, _) = synth(20), synth(21)
    kps, _ = ORBextractor(2000, 1.2, 8, 20, 7)(gray_b, None)
    maps = [torch.empty(H * W, dtype=t, device="cuda") for t in (torch.uint8, torch.float64, torch.float64)]
    d_a, d_b = upload(bgr_a), upload(bgr_b)
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
    f = DeviceFrame(el, er, H, W)
    f.left.enqueue(el, upload(gl), H, W, W)
    f.right.enqueue(er, upload(gr), H, W, W)
    stream = torch.cuda.Stream()
    if with_keep:
        keep = np.sort(np.random.default_rng(nf).choice(len(kl), len(kl) * 2 // 3, replace=False)).astype(np.int32)
        d_keep = torch.from_numpy(keep).cuda()
        d_n = torch.tensor([len(keep)], dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        stereo(f, mb, mbf, stream.cuda_stream, keep=ptr(d_keep), n_left=ptr(d_n))
    else:
        keep = np.arange(len(kl), dtype=np.int32)
        stereo(f, mb, mbf, stream.cuda_stream)
    stream.synchronize()
    assert np.array_equal(f.left.host()[0].view(np.uint8), kl.view(np.uint8))
    u, z = (f.out[k].cpu().numpy()[:len(keep)] for k in ("u_right", "depth"))
    hu, hz = stereo_match(el, er, kl[keep], dl[keep], kr, dr, mb, mbf)
    assert u.tobytes() == hu.tobytes() and z.tobytes() == hz.tobytes()
    ru, rz = O.compute_stereo_matches(kl[keep], dl[keep], kr, dr, el._bordered, er._bordered, el.GetScaleFactors(),
                                      el.GetInverseScaleFactors(), mb, mbf)
    assert u.tobytes() == ru.tobytes() and z.tobytes() == rz.tobytes()
    assert (u >= 0).sum() > 50
    assert (f.out["u_right"].cpu().numpy()[len(keep):] == 7.0).all()


def test_stereo_device_edge_cases():
    mb, mbf = BASELINES["kitti"]
    _, gl, gr = synth(2)
    el, er = extractors(1000)
    kl, dl = el(gl, None)
    kr, dr = er(gr, None)
    f = DeviceFrame(el, er, H, W)
    f.left.enqueue(el, upload(gl), H, W, W)
    f.right.enqueue(er, upload(gr), H, W, W)
    torch.cuda.synchronize()  # the copies below read the extractors' outputs on torch's stream
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    zero = torch.zeros(1, dtype=torch.int64, device="cuda")
    keep = torch.arange(f.left.cap, dtype=torch.int32, device="cuda")
    u_out, z_out = f.out["u_right"], f.out["depth"]
    # zero left keypoints, zero kept keys, a negative count (count above capacity upstream): nothing written
    for kw in ({"n_left": ptr(zero)}, {"keep": ptr(keep), "n_left": ptr(zero)},
               {"keep": ptr(keep), "n_left": ptr(torch.full((1,), -1, dtype=torch.int64, device="cuda"))}):
        f.reset()
        stereo(f, mb, mbf, s, **kw)
        stream.synchronize()
        assert (u_out.cpu().numpy() == 7.0).all() and (z_out.cpu().numpy() == 7.0).all()
    # zero right keypoints: every left keypoint unmatched
    n = len(kl)
    f.reset()
    stereo_match_device(el, er, f.kps, f.desc, 0, f.count, ptr(f.right.kps), ptr(f.right.desc), ptr(zero), mb, mbf, f.u_right, f.depth, s)
    stream.synchronize()
    u, z = u_out.cpu().numpy()[:n], z_out.cpu().numpy()[:n]
    assert (u == -1).all() and (z == -1).all() and (u_out.cpu().numpy()[n:] == 7.0).all()
    # no match surviving: every right keypoint moved right of every left one, i.e. outside the disparity window [0, mbf / mb)
    moved_kr = kr.copy()
    moved_kr["x"] += np.float32(5000)
    moved = FrameKeys(er)
    moved.kps[:len(kr) * 28] = torch.from_numpy(moved_kr.view(np.uint8))
    moved.desc.copy_(f.right.desc)
    moved.count.copy_(f.right.count)
    f.reset()
    stereo(f, mb, mbf, s, right=moved)
    stream.synchronize()
    u, z = u_out.cpu().numpy()[:n], z_out.cpu().numpy()[:n]
    hu, hz = stereo_match(el, er, kl, dl, moved_kr, dr, mb, mbf)
    assert (u == -1).all() and (z == -1).all() and np.array_equal(u, hu) and np.array_equal(z, hz)
    # left keypoints with an octave outside [0, nlevels) stay unmatched; the others keep their results
    bad = kl.copy()
    bad["octave"][::3] = 99
    f.left.kps[:n * 28] = torch.from_numpy(bad.view(np.uint8))
    f.reset()
    stereo(f, mb, mbf, s)
    stream.synchronize()
    u, z = u_out.cpu().numpy()[:n], z_out.cpu().numpy()[:n]
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
    f = DeviceFrame(el, er, H, W)
    args = lambda: [f.kps, f.desc, None, f.count, ptr(f.right.kps), ptr(f.right.desc), ptr(f.right.count), mb, mbf, f.u_right, f.depth, None]
    # extractors that have not run
    assert lib.sivo_stereo_match_device(el._h, er._h, *args()) == L.EINVAL
    _, gl, gr = synth(0)
    f.left.enqueue(el, upload(gl), H, W, W)
    assert lib.sivo_stereo_match_device(el._h, er._h, *args()) == L.EINVAL
    f.right.enqueue(er, upload(gr), H, W, W)
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
    sargs = lambda: [f.kps, f.count, f.left.cap, 8, f.kp_class, f.kp_conf, f.kp_entropy, f.keep, f.n_keep, None]
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


# ---------------------------------------------------------------------------------------------------------- asynchronous chain
def test_stereo_waits_for_the_extractors_itself():
    """Stereo enqueued straight after enqueue_device on another stream, with no manual wait: the call orders itself."""
    mb, mbf = BASELINES["kitti"]
    _, gl, gr = synth(4)
    el, er = extractors(2000)
    kl, dl = el(gl, None)
    kr, dr = er(gr, None)
    hu, hz = stereo_match(el, er, kl, dl, kr, dr, mb, mbf)
    d_gl, d_gr = upload(gl), upload(gr)
    _, gl2, gr2 = synth(5)  # a different frame first, so that stale pyramids / keypoints would show
    el(gl2, None)
    er(gr2, None)
    f = DeviceFrame(el, er, H, W)
    stream = torch.cuda.Stream()
    f.left.enqueue(el, d_gl, H, W, W)
    f.right.enqueue(er, d_gr, H, W, W)
    stereo(f, mb, mbf, stream.cuda_stream)
    stream.synchronize()
    u, z = (f.out[k].cpu().numpy()[:len(kl)] for k in ("u_right", "depth"))
    assert int(f.left.count.cpu()[0]) == len(kl)
    assert u.tobytes() == hu.tobytes() and z.tobytes() == hz.tobytes()


def _chain_frames():
    return [synth(10 + i) for i in range(3)]


def test_three_frames_in_flight_equal_the_host_call_path(seg):
    """SegNet -> two enqueue_device -> semantic keys -> stereo for three frames on rotating buffers, connected only by stream
    and event edges, one host synchronisation at the end; every frame equals the host-call path for that frame."""
    mb, mbf = BASELINES["kitti"]
    frames = _chain_frames()
    el, er = extractors(2000)
    d_in = [[upload(x) for x in f] for f in frames]
    bufs = [DeviceFrame(el, er, H, W) for _ in frames]
    stream = torch.cuda.Stream()
    s = stream.cuda_stream

    def chain(tail=True):
        for i, f in enumerate(bufs):
            seg.set_frame(100 + i)
            f.extract(seg, *d_in[i], s)
            if tail:
                f.tail(seg, mb, mbf, s)
            else:
                er.stream_wait(s)

    chain()  # first use of the stream: the network's graph is captured here
    stream.synchronize()
    for f in bufs:
        for m in f.maps:
            m.fill_(0)
        f.reset()
    chain()
    stream.synchronize()  # the one host synchronisation of the chain
    got = [{"maps": [m.cpu().numpy() for m in f.maps], "kl": f.left.host(), "kr": f.right.host(), "sem": f.host()[:2],
            "sem_vals": (f.out["kp_class"].cpu().numpy(), f.out["kp_conf"].cpu().numpy()),
            "st": (f.out["u_right"].cpu().numpy(), f.out["depth"].cpu().numpy())} for f in bufs]
    # without the tail the network and extractor outputs are the same bits
    chain(tail=False)
    stream.synchronize()
    for f, g in zip(bufs, got):
        for m, want in zip(f.maps, g["maps"]):
            assert m.cpu().numpy().tobytes() == want.tobytes()
        for side, keys in (("kl", f.left), ("kr", f.right)):
            kp, de = keys.host()
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
