"""-m gpu: SIVO's information-based map-point selection (sivo_info_select / _device, k_info_select) on the Frame tail's outputs --
SegNet -> extractors -> semantic keys -> stereo -- against oracle/info_oracle.py, and the device form against the host form."""
import numpy as np
import pytest
import torch

from frame_support import H, MB, MBF, POSES, SIGMAS, W, InfoOut, cameras, ext, i64, ptr, same_bits, seg, synth, tails, upload  # noqa: F401
from oracle import info_oracle as I
from oracle.keymap import keymap
from sivo_b200 import _lib as L
from sivo_b200 import info_select, stereo_match
from sivo_b200.frame import DeviceFrame
from sivo_b200.info import info_terms

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize("pose", sorted(POSES))
@pytest.mark.parametrize("sigma", sorted(SIGMAS))
def test_terms_are_bit_identical_to_the_oracle(tails, ext, sigma, pose):
    el = ext[0]
    cam, ocam = cameras(sigma, pose)
    for f, t in tails.items():
        world, ds, dm, dj = info_terms(el, t.kps, t.depth, cam)
        ow, ods, odm, odj, valid = I.info_terms(t.kps, t.depth, el.GetScaleSigmaSquares(), ocam)
        assert valid.sum() > 30
        assert same_bits(world[valid], ow[valid]) and np.isnan(world[~valid]).all(), f
        for g, o in ((ds, ods), (dm, odm), (dj, odj)):
            assert same_bits(g[valid], o[valid]) and np.isnan(g[~valid]).all(), f


def thresholds(red):
    """0, 4 and the 25 / 50 / 75 percentiles of the oracle's reductions, each placed halfway between two neighbouring values so
    that no key sits on it."""
    r = np.unique(red[np.isfinite(red)])
    out = [0.0, 4.0]
    for q in (0.25, 0.5, 0.75):
        i = min(int(q * len(r)), len(r) - 2)
        out.append(0.5 * (r[i] + r[i + 1]))
    return out


@pytest.mark.parametrize("pose", sorted(POSES))
@pytest.mark.parametrize("sigma", sorted(SIGMAS))
def test_host_form_against_the_oracle(tails, ext, sigma, pose):
    el = ext[0]
    cam, ocam = cameras(sigma, pose)
    near = 0
    for f, t in tails.items():
        _, ored, _ = I.select(t.kps, t.depth, t.ent, el.GetScaleSigmaSquares(), ocam, 0.0)
        fin = np.isfinite(ored)
        for th in thresholds(ored):
            world, red, sel = info_select(el, t.kps, t.depth, t.ent, cam, th)
            ow, _, osel = I.select(t.kps, t.depth, t.ent, el.GetScaleSigmaSquares(), ocam, th)
            assert np.array_equal(np.isfinite(red), fin) and np.abs(red[fin] - ored[fin]).max() <= 1e-12, (f, th)
            assert same_bits(world[fin], ow[fin])
            close = fin & (np.abs(ored - th) <= 1e-12)
            near += int(close.sum())
            assert np.array_equal(np.setdiff1d(sel, np.flatnonzero(close)), np.setdiff1d(osel, np.flatnonzero(close))), (f, th)
            assert (np.diff(sel) > 0).all()
    assert near == 0


# ---------------------------------------------------------------------------------------------------------- device form
@pytest.mark.parametrize("pose", sorted(POSES))
@pytest.mark.parametrize("sigma", sorted(SIGMAS))
def test_device_form_equals_the_host_form(tails, ext, sigma, pose):
    el = ext[0]
    cam, _ = cameras(sigma, pose)
    stream = torch.cuda.Stream()
    for f, t in tails.items():
        th = thresholds(info_select(el, t.kps, t.depth, t.ent, cam, 0.0)[1])[3]  # the median: some keys on either side
        hw, hr, hs = info_select(el, t.kps, t.depth, t.ent, cam, th)
        out = InfoOut(t.f.left.cap)
        out.run(el, t.f.kps, t.f.kp_entropy, t.f.keep, t.f.n_keep, t.f.depth, cam, th, stream.cuda_stream)
        stream.synchronize()
        w, r, s, m = out.host(t.n_keep)
        assert same_bits(w, hw) and same_bits(r, hr) and same_bits(s, hs) and m == len(hs), f
        assert (out.red.cpu().numpy()[t.n_keep:] == 7.0).all() and (out.sel.cpu().numpy()[m:] == -7).all()
        # the same keys through an oracle/keymap.py map: its rejected entries come out unselected
        km = keymap(t.n_keep, t.f.left.cap, np.random.default_rng(t.n_keep))
        keep = km.keep.copy()
        keep[km.real] = t.keep
        depth = np.full(len(keep), 10.0, np.float32)  # a rejected entry has a depth, but no key
        depth[km.real] = t.depth
        d_keep, d_n, d_depth = upload(keep), i64(km.n_keep), upload(depth)
        out = InfoOut(t.f.left.cap)
        out.run(el, t.f.kps, t.f.kp_entropy, ptr(d_keep), ptr(d_n), ptr(d_depth), cam, th, stream.cuda_stream)
        stream.synchronize()
        w, r, s, m = out.host(km.n_keep)
        assert same_bits(w[km.real], hw) and same_bits(r[km.real], hr) and same_bits(s, km.real[hs].astype(np.int32)), f
        assert m == len(hs) and not np.isin(s, np.flatnonzero(km.src < 0)).any()
        # keep_idx NULL: semantic key j is extractor key j (depth from the stereo call without keep_idx)
        n = len(t.kps_all)
        hw, hr, hs = info_select(el, t.kps_all, t.depth_all, t.ent_all, cam, th)
        out = InfoOut(t.f.left.cap)
        out.run(el, t.f.kps, t.f.kp_entropy, 0, t.f.count, ptr(t.z_all), cam, th, stream.cuda_stream)
        stream.synchronize()
        w, r, s, m = out.host(n)
        assert same_bits(w, hw) and same_bits(r, hr) and same_bits(s, hs) and m == len(hs), f
        assert 0 < len(hs) < n


def test_device_form_edge_cases(tails, ext):
    el = ext[0]
    t = tails[1]
    cam, ocam = cameras("motion", "moved")
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    cap = t.f.left.cap

    def dev(kw=None, cam_=cam, th=0.0, null=()):
        kw = kw or {}
        out = InfoOut(cap)
        out.run(el, t.f.kps, t.f.kp_entropy, kw.get("keep", t.f.keep), ptr(kw["n"]) if "n" in kw else t.f.n_keep,
                ptr(kw["depth"]) if "depth" in kw else t.f.depth, cam_, th, s, null)
        stream.synchronize()
        return out

    # a negative count writes only n_selected = -1; a zero count writes only n_selected = 0
    for v in (-1, 0):
        out = dev({"n": i64(v)})
        assert int(out.n.cpu()[0]) == v and (out.red.cpu().numpy() == 7.0).all() and (out.world.cpu().numpy() == 7.0).all()
        assert (out.sel.cpu().numpy() == -7).all()
    # a count above capacity is clamped (keep_idx NULL: key j; all cap keys processed, the ones past the extractor's count are zeros)
    depth = torch.full((cap,), -1.0, dtype=torch.float32, device="cuda")
    depth[:len(t.kps_all)] = torch.from_numpy(t.depth_all).cuda()
    torch.cuda.synchronize()
    out = dev({"keep": 0, "n": i64(cap + 1000), "depth": depth})
    w, r, sl, m = out.host(cap)
    hw, hr, hs = info_select(el, t.f.left.kps.cpu().numpy().view(t.kps_all.dtype)[:cap], depth.cpu().numpy(),
                             t.f.out["kp_entropy"].cpu().numpy()[:cap], cam, 0.0)
    assert same_bits(r, hr) and same_bits(sl, hs) and m == len(hs) and np.isnan(r[len(t.kps_all):]).all()
    # all depths -1: every key invalid, nothing selected
    out = dev({"depth": torch.full((cap,), -1.0, dtype=torch.float32, device="cuda")})
    w, r, sl, m = out.host(t.n_keep)
    assert np.isnan(r).all() and np.isnan(w).all() and m == 0
    # NULL outputs: each alone, and only the count
    full = dev().host(t.n_keep)
    for null in (("world",), ("red",), ("sel",), ("n",), ("world", "red", "sel")):
        out = dev(null=null)
        got = out.host(t.n_keep)
        if "n" in null:  # the list without its count: read as many entries as the full call selected
            assert int(out.n.cpu()[0]) == -7
            got = got[:2] + (out.sel.cpu().numpy()[:full[3]].copy(), full[3])
        for name, a, b in zip(("world", "red", "sel"), got[:3], full[:3]):
            if name not in null:
                assert same_bits(a, b), null
            elif name == "sel":
                assert len(a) == 0 or (a == -7).all()
        assert got[3] == full[3] and full[3] > 0
    # Σ = 0: det S = det M = 0, every reduction NaN, nothing selected
    zero_cam, _ = cameras(np.zeros((6, 6)), "moved")
    w, r, sl, m = dev(cam_=zero_cam, th=-1e300).host(t.n_keep)
    assert np.isnan(r).all() and m == 0 and np.isfinite(w[t.depth > 0]).all()


def test_host_form_edge_cases(tails, ext):
    el = ext[0]
    t = tails[0]
    # a world Z of exactly 0: identity rotation and Ow_z = -z for the keys at depth 5
    z = t.depth.copy()
    z[::2] = 5.0
    cam, ocam = cameras("spd", "identity")
    cam.Ow[2] = -5.0
    ocam.Ow[2] = np.float32(-5.0)
    world, red, sel = info_select(el, t.kps, z, t.ent, cam, -1e300)
    ow, ored, osel = I.select(t.kps, z, t.ent, el.GetScaleSigmaSquares(), ocam, -1e300)
    assert (world[::2, 2] == 0).all() and np.abs(red[::2] + t.ent[::2]).max() <= 1e-12
    fin = np.isfinite(ored)
    assert np.abs(red[fin] - ored[fin]).max() <= 1e-12 and np.array_equal(sel, osel)
    # octaves out of range are invalid
    bad = t.kps.copy()
    bad["octave"][::3] = 99
    bad["octave"][1::3] = -1
    _, red, sel = info_select(el, bad, t.depth, t.ent, cam, -1e300)
    assert np.isnan(red[::3]).all() and np.isnan(red[1::3]).all() and not np.isin(sel, np.r_[0:len(bad):3]).any()
    # zero keys
    world, red, sel = info_select(el, t.kps[:0], t.depth[:0], t.ent[:0], cam, 0.0)
    assert world.shape == (0, 3) and len(red) == 0 and len(sel) == 0


def test_error_codes(tails, ext):
    lib = L.lib()
    el = ext[0]
    t = tails[0]
    cam, _ = cameras("tiny", "identity")
    import ctypes as C
    k, z, h = t.kps, t.depth, t.ent
    n = len(k)
    world, red, sel, ns = np.empty((n, 3), np.float32), np.empty(n), np.empty(n, np.int32), C.c_int()
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    hargs = lambda: [el._h, P(k), P(z), P(h), n, C.byref(cam), 0.0, P(world), P(red), P(sel), C.byref(ns)]
    assert lib.sivo_info_select(*hargs()) == L.OK
    for i, v in ((0, None), (1, None), (2, None), (3, None), (4, -1), (5, None)):
        a = hargs()
        a[i] = v
        assert lib.sivo_info_select(*a) == L.EINVAL, i
    a = hargs()
    a[7:] = [None] * 4
    assert lib.sivo_info_select(*a) == L.OK
    out = InfoOut(t.f.left.cap)
    dargs = lambda: [el._h, t.f.kps, t.f.kp_entropy, t.f.keep, t.f.n_keep, t.f.depth, C.byref(cam), 0.0, ptr(out.world), ptr(out.red),
                     ptr(out.sel), ptr(out.n), None]
    assert lib.sivo_info_select_device(*dargs()) == L.OK
    for i in (0, 1, 2, 4, 5, 6):
        a = dargs()
        a[i] = None
        assert lib.sivo_info_select_device(*a) == L.EINVAL, i
    assert lib.sivo_dbg_info_terms(None, P(k), P(z), n, C.byref(cam), None, None, None, None) == L.EINVAL
    assert lib.sivo_dbg_info_terms(el._h, P(k), P(z), -1, C.byref(cam), None, None, None, None) == L.EINVAL
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- asynchronous chain
def test_three_frames_in_flight_with_the_selection_equal_the_host_call_path(seg, ext):
    """SegNet -> two enqueue_device -> semantic keys -> stereo -> selection for three frames on rotating buffers, one host
    synchronisation; each frame's selection equals the host-call path's."""
    el, er = ext
    frames = [synth(20 + i) for i in range(3)]
    cam, _ = cameras("motion", "moved")
    d_in = [[upload(x) for x in f] for f in frames]
    bufs = [(DeviceFrame(el, er, H, W), InfoOut(el.capacity())) for _ in frames]
    stream = torch.cuda.Stream()
    s = stream.cuda_stream

    def chain():
        for i, (f, info) in enumerate(bufs):
            seg.set_frame(200 + i)
            f.extract(seg, *d_in[i], s)
            f.tail(seg, MB, MBF, s)
            info.run(el, f.kps, f.kp_entropy, f.keep, f.n_keep, f.depth, cam, 4.0, s)

    chain()  # first use of the stream: the network's graph is captured here
    stream.synchronize()
    for _, info in bufs:
        info.sel.fill_(-7)
        info.red.fill_(7.0)
        info.n.fill_(-7)
    torch.cuda.synchronize()
    chain()
    stream.synchronize()  # the one host synchronisation of the chain
    got = [(f.host()[0], info) for f, info in bufs]
    for i, (bgr, gl, gr) in enumerate(frames):
        seg.set_frame(200 + i)
        seg.segmentImage(bgr)
        kl, dl = el(gl, None)
        kr, dr = er(gr, None)
        _, _, ent, keep = seg.semantic_keys(kl, 8)
        _, hz = stereo_match(el, er, kl[keep], dl[keep], kr, dr, MB, MBF)
        hw_, hr, hs = info_select(el, kl[keep], hz, ent[keep], cam, 4.0)
        n_keep, info = got[i]
        w, r, sl, m = info.host(n_keep)
        assert n_keep == len(keep) and same_bits(w, hw_) and same_bits(r, hr) and same_bits(sl, hs) and m == len(hs)
        assert np.isfinite(r).sum() > 20
