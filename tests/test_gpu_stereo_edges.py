"""-m gpu: Frame::ComputeStereoMatches on constructed worst cases (oracle/stereo_scene.py) through the oracle, the host form
(sivo_stereo_match) and the device form (sivo_stereo_match_device, through an oracle/keymap.py map with rejected entries),
bit for bit; the Hamming stage through sivo_stereo_hamming; the median cut alone through sivo_dbg_stereo_median_cut; the rule
for keys outside the domain (also for the semantic keys); the refusals; the rule's inertness on extractor keys; 200 fuzz scenes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from frame_support import extractor, i64, sentinel, upload
from oracle import orb_oracle as O
from oracle import stereo_scene as S
from oracle.keymap import keymap, scatter
from sivo_b200 import KP_DTYPE, ORBextractor, stereo_hamming, stereo_match, stereo_match_device
from sivo_b200 import _lib as L
from sivo_b200.orb import stereo_median_cut
from sivo_b200.synth import bgr_to_gray, stereo_frame

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KITTI_MBF = 386.1448
KITTI_MB = KITTI_MBF / 718.856
f32 = np.float32


def pair(nfeatures, scale_factor, nlevels):
    return extractor(nfeatures, scale_factor, nlevels), extractor(nfeatures, scale_factor, nlevels, right=True)


def device_form(el, er, km, kl, dl, kr, dr, mb, mbf, n_left=None, n_right=None):
    """sivo_stereo_match_device with the left keys at the slots of the map km (oracle/keymap.py) and the right keys in order, in
    capacity-sized device buffers; returns the left buffers as the device reads them and the outputs (7.0 = unwritten)."""
    cap_l, cap_r = el.capacity(), er.capacity()
    assert len(kr) <= cap_r
    none = np.zeros(1, KP_DTYPE)
    sl, sdl = scatter(kl, km.slots, cap_l, none), scatter(dl, km.slots, cap_l, 0)
    right = np.arange(len(kr))
    bufs = [upload(a) for a in (sl, sdl, km.keep, scatter(kr, right, cap_r, none), scatter(dr, right, cap_r, 0))]
    nl, nr = i64(km.n_keep if n_left is None else n_left), i64(len(kr) if n_right is None else n_right)
    u, z = sentinel(cap_l, 7.0, torch.float32), sentinel(cap_l, 7.0, torch.float32)
    stream = torch.cuda.Stream()
    stereo_match_device(el, er, bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), nl.data_ptr(), bufs[3].data_ptr(),
                        bufs[4].data_ptr(), nr.data_ptr(), mb, mbf, u.data_ptr(), z.data_ptr(), stream.cuda_stream)
    stream.synchronize()
    return sl, sdl, u.cpu().numpy(), z.cpu().numpy()


def check_scene(sc, seed=0, device=True):
    el, er = pair(500, sc.scale_factor, sc.nlevels)
    el(sc.left, None)
    er(sc.right, None)
    ru, rz = O.compute_stereo_matches(sc.kl, sc.dl, sc.kr, sc.dr, el._bordered, er._bordered, el.GetScaleFactors(),
                                      el.GetInverseScaleFactors(), sc.mb, sc.mbf)
    hu, hz = stereo_match(el, er, sc.kl, sc.dl, sc.kr, sc.dr, sc.mb, sc.mbf)
    assert hu.tobytes() == ru.tobytes() and hz.tobytes() == rz.tobytes(), (sc.name, np.nonzero((hu != ru) | (hz != rz))[0])
    if device:
        km = keymap(len(sc.kl), el.capacity(), np.random.default_rng(seed))
        _, _, u, z = device_form(el, er, km, sc.kl, sc.dl, sc.kr, sc.dr, sc.mb, sc.mbf)
        bad = np.flatnonzero(km.src < 0)
        assert u[km.real].tobytes() == hu.tobytes() and z[km.real].tobytes() == hz.tobytes(), sc.name
        assert (u[bad] == -1).all() and (z[bad] == -1).all() and (u[km.n_keep:] == 7.0).all()
    # the Hamming stage as sivo_stereo_hamming shows it, at the scene's window and with min_d > 0
    rows = sc.left.shape[0]
    for min_d in (0.0, 3.0):
        max_d = f32(f32(sc.mbf) / f32(sc.mb))
        idx, dist = stereo_hamming(sc.kl, sc.dl, sc.kr, sc.dr, el.GetScaleFactors(), rows, min_d, max_d)
        ri, rd = O.stereo_hamming(sc.kl, sc.dl, sc.kr, sc.dr, el.GetScaleFactors(), rows, min_d, max_d)
        assert np.array_equal(idx, ri) and np.array_equal(dist, rd), (sc.name, min_d)
    return hu, hz


@pytest.mark.parametrize("name", [sc.name for sc in S.constructed_scenes()])
def test_constructed_scene_oracle_host_device_and_hamming_agree(name):
    sc = {s.name: s for s in S.constructed_scenes()}[name]
    trace = []
    el, er = pair(500, sc.scale_factor, sc.nlevels)
    el(sc.left, None)
    er(sc.right, None)
    O.compute_stereo_matches(sc.kl, sc.dl, sc.kr, sc.dr, el._bordered, er._bordered, el.GetScaleFactors(),
                             el.GetInverseScaleFactors(), sc.mb, sc.mbf, trace)
    for il, want in sc.want.items():  # the extractor's pyramid is the oracle's: the scene's stages hold on the device's levels
        assert trace[il]["stage"] in O.STAGE_GROUPS.get(want, (want,)), (il, want, trace[il])
    hu, hz = check_scene(sc)
    if name == "disparity":  # disparity 0: depth mbf / 0.01f and u = (float) (uL - 0.01) in double
        il = next(i for i, t in enumerate(trace) if t["disp"] == 0)
        assert hz[il] == f32(f32(sc.mbf) / f32(0.01)) and hu[il] == f32(float(sc.kl["x"][il]) - 0.01)


def test_hamming_99_and_100_and_the_20_bit_index():
    sc = S.sad_scene()
    rng = np.random.default_rng(9)
    kl = sc.kl[:1].copy()
    dl = sc.dl[:1].copy()
    far = np.zeros((4, 32), np.uint8)
    for nbits, want in ((99, 99), (100, 100)):
        bits = np.unpackbits(dl[0])
        bits[rng.choice(256, nbits, replace=False)] ^= 1
        kr = np.repeat(kl, 1)
        kr["x"] -= 1
        idx, dist = stereo_hamming(kl, dl, kr, np.packbits(bits)[None], np.ones(8, np.float32), 240, 0.0, 40.0)
        assert dist[0] == want and idx[0] == (0 if want < 100 else -1)
    # 2^20 - 1 right keys, the best at the last index: the index fills all 20 bits of the packed search word
    n = (1 << 20) - 1
    el, er = pair(500, sc.scale_factor, sc.nlevels)
    el(sc.left, None)
    er(sc.right, None)
    kr = np.zeros(n, KP_DTYPE)
    kr["x"], kr["y"] = S.COLS - 1, 2
    dr = rng.integers(0, 256, (n, 32)).astype(np.uint8)
    kr[-len(sc.kr):] = sc.kr
    dr[-len(sc.kr):] = sc.dr
    idx, dist = stereo_hamming(sc.kl, sc.dl, kr, dr, el.GetScaleFactors(), 240, 0.0, 40.0)
    ri, rd = O.stereo_hamming(sc.kl, sc.dl, kr, dr, el.GetScaleFactors(), 240, 0.0, 40.0)
    assert np.array_equal(idx, ri) and np.array_equal(dist, rd) and (idx == n - 1).any()
    hu, hz = stereo_match(el, er, sc.kl, sc.dl, kr, dr, sc.mb, sc.mbf)
    ru, rz = O.compute_stereo_matches(sc.kl, sc.dl, kr, dr, el._bordered, er._bordered, el.GetScaleFactors(),
                                      el.GetInverseScaleFactors(), sc.mb, sc.mbf)
    assert hu.tobytes() == ru.tobytes() and hz.tobytes() == rz.tobytes() and (hu >= 0).sum() > 5
    kr2 = np.concatenate([kr, kr[:1]])
    dr2 = np.concatenate([dr, dr[:1]])
    for call in (lambda: stereo_hamming(sc.kl, sc.dl, kr2, dr2, el.GetScaleFactors(), 240, 0.0, 40.0),
                 lambda: stereo_match(el, er, sc.kl, sc.dl, kr2, dr2, sc.mb, sc.mbf)):
        with pytest.raises(L.SivoError) as e:
            call()
        assert e.value.code == L.EINVAL


# ---------------------------------------------------------------------------------------------------------- the median cut
def cut_cases():
    rng = np.random.default_rng(11)
    cases = [np.array(c, np.int64) for c in ([], [-1], [0], [5], [5, 6], [6, 5], [3, 1, 2], [1, 2, 3, 4], [9] * 7, [0] * 10, [0, 0, 5],
                                             [61710, 61710, 0], [61710] * 3)]
    # medians 255 / 256 / 257 / 511 / 512, with rank m / 2 at the first and at the last entry of its high-byte bin
    for med in (255, 256, 257, 511, 512):
        for below, above in ((2, 2), (3, 2), (2, 3)):
            lo = rng.integers(0, (med >> 8) << 8 or 1, below) if (med >> 8) else rng.integers(0, med + 1, below)
            hi = rng.integers(med + 1, 4000, above)
            cases.append(rng.permutation(np.concatenate([lo, [med], hi])))
    cases.append(rng.permutation(np.array([200, 256, 256, 300, 511, 600, 700])))  # rank 3 = 300 inside bin 1
    cases.append(rng.permutation(np.array([100, 255, 256, 511, 512])))
    # threshold equality: medians M whose threshold 1.5f * 1.4f * M is an integer T: SAD T is cut, T - 1 kept
    ms = [m for m in range(1, 29386) if f32(f32(2.0999999) * f32(m)) == round(float(f32(f32(2.0999999) * f32(m))))]
    assert len(ms) > 50
    for m in ms[::max(1, len(ms) // 12)][:12] + [10]:
        t = int(f32(f32(2.0999999) * f32(m)))
        cases.append(rng.permutation(np.array([m, m, m, 0, 1, t - 1, t], np.int64)))
    for n in (1023, 1024, 1025, 2047, 2049, 4095, 4097, 30001):
        s = rng.integers(-1, 61711, n)
        s[rng.random(n) < 0.3] = -1
        cases.append(s)
        cases.append(np.where(rng.random(n) < 0.5, rng.integers(0, 600, n), -1))
    return cases


def test_median_cut_hook_equals_the_oracle():
    for sad in cut_cases():
        n = len(sad)
        u0 = np.arange(n, dtype=np.float32)
        z0 = u0 + f32(0.5)
        u, z = stereo_median_cut(sad, u0, z0)
        cut = O.median_cut(sad)
        want_u = np.where(cut, f32(-1), u0)
        want_z = np.where(cut, f32(-1), z0)
        assert u.tobytes() == want_u.tobytes() and z.tobytes() == want_z.tobytes(), (n, sad[:20])


def test_median_cut_at_the_extractor_capacity():
    el = extractor(500, 1.2, 8)
    for cap in (el.capacity(), 2000 + 4 * 8 + 64, 5000 + 4 * 8 + 64):
        rng = np.random.default_rng(cap)
        sad = np.where(rng.random(cap) < 0.8, rng.integers(0, 61711, cap), -1)
        u, z = stereo_median_cut(sad, np.ones(cap, np.float32), np.ones(cap, np.float32))
        assert np.array_equal(u == -1, O.median_cut(sad)) and np.array_equal(z == -1, O.median_cut(sad))


# ---------------------------------------------------------------------------------------------------------- refusals
def refused_without_writing(el, er, sc, lib_msg):
    lib = L.lib()
    n = len(sc.kl)
    u = np.full(n, 7.0, np.float32)
    z = np.full(n, 7.0, np.float32)
    rc = lib.sivo_stereo_match(el._h, er._h, sc.kl.ctypes.data_as(C.c_void_p), sc.dl.ctypes.data_as(C.c_void_p), n,
                               sc.kr.ctypes.data_as(C.c_void_p), sc.dr.ctypes.data_as(C.c_void_p), len(sc.kr), C.c_float(sc.mb),
                               C.c_float(sc.mbf), u.ctypes.data_as(C.c_void_p), z.ctypes.data_as(C.c_void_p))
    assert rc == L.EINVAL and (u == 7.0).all() and (z == 7.0).all()
    assert lib_msg in lib.sivo_last_error().decode()


def device_refused_without_writing(el, er, sc, lib_msg):
    cap = el.capacity()
    kps, desc = sentinel(cap * 28, 0, torch.uint8), sentinel(cap * 32, 0, torch.uint8)
    rk, rd = sentinel(max(len(sc.kr), 1) * 28, 0, torch.uint8), sentinel(max(len(sc.kr), 1) * 32, 0, torch.uint8)
    n = i64(len(sc.kl))
    u, z = sentinel(cap, 7.0, torch.float32), sentinel(cap, 7.0, torch.float32)
    with pytest.raises(L.SivoError) as e:
        stereo_match_device(el, er, kps.data_ptr(), desc.data_ptr(), 0, n.data_ptr(), rk.data_ptr(), rd.data_ptr(), n.data_ptr(),
                            sc.mb, sc.mbf, u.data_ptr(), z.data_ptr(), 0)
    torch.cuda.synchronize()
    assert e.value.code == L.EINVAL and lib_msg in str(e.value)
    assert (u.cpu().numpy() == 7.0).all() and (z.cpu().numpy() == 7.0).all()


def test_refusals():
    sc = S.sad_scene()
    el, er = pair(500, 1.2, 8)
    el(sc.left, None)
    # a right image 40 rows shorter, and a right extractor with another scale factor: different level tables
    er(np.ascontiguousarray(sc.right[:-40]), None)
    refused_without_writing(el, er, sc, "on the left and")
    device_refused_without_writing(el, er, sc, "on the left and")
    er125 = ORBextractor(500, 1.25, 8, 20, 7)
    er125(sc.right, None)
    refused_without_writing(el, er125, sc, "on the left and")
    device_refused_without_writing(el, er125, sc, "on the left and")
    # a right extractor whose capacity needs more than the 20 index bits of the packed search word (device form)
    big = ORBextractor(1 << 20, 1.2, 8, 20, 7)
    big(sc.right, None)
    assert big.capacity() >= 1 << 20
    device_refused_without_writing(el, big, sc, "20 index bits")
    # the same pair of extractors is accepted once the tables agree again
    er(sc.right, None)
    check_scene(sc, device=False)


# ---------------------------------------------------------------------------------------------------------- the rule
@pytest.fixture(scope="module")
def seg(model_dir):
    from sivo_b200 import BayesianSegNet, BayesianSegNetParams
    from sivo_b200.caffemodel import shipped_scales, write_synth_model
    from sivo_b200.prototxt import load_net
    proto = os.path.join(ROOT, "configs", "bayesian_segnet_basic.prototxt")
    model = os.path.join(str(model_dir), "basic_full.caffemodel")
    if not os.path.exists(model):
        write_synth_model(load_net(open(proto).read(), T=2), model, 0, shipped_scales("basic"))
    return BayesianSegNet(BayesianSegNetParams(proto, model), seed=7, T=2, precision="fp16", engine="auto")


def test_semantic_keys_of_non_finite_keys(seg):
    H, W = 352, 1024
    left, _ = stereo_frame(4)
    bgr = np.ascontiguousarray(left[11:11 + H, 109:109 + W])
    maps = [torch.empty(H * W, dtype=t, device="cuda") for t in (torch.uint8, torch.float64, torch.float64)]
    d_bgr = torch.from_numpy(bgr).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    seg.set_frame(3)
    seg.run_device_maps(d_bgr.data_ptr(), *(m.data_ptr() for m in maps), 0, 0, side.cuda_stream)
    side.synchronize()
    cls_map, conf_map, ent_map = (m.cpu().numpy().reshape(H, W) for m in maps)
    nan, inf = f32(np.nan), f32(np.inf)
    xs = [nan, 5, inf, -inf, 5, 5, nan, 3e9, -3e9, -0.5, W - 0.5, 7, 100.25]
    ys = [5, nan, 5, 5, inf, -inf, nan, 5, 5, 5, H - 0.5, -0.5, 200.75]
    kps = np.zeros(len(xs), KP_DTYPE)
    kps["x"], kps["y"] = xs, ys
    want = O.select_semantic_keys(np.stack([kps["x"], kps["y"]], 1), cls_map, conf_map, ent_map, 14)
    assert (want[0][:9] == 255).all() and (want[0][9:] != 255).all()
    got = seg.semantic_keys(kps, 14)
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    # the device form
    cap = 64
    buf = upload(scatter(kps, np.arange(len(kps)), cap, np.zeros(1, KP_DTYPE)))
    cnt = i64(len(kps))
    cls, conf, ent = sentinel(cap, 77, torch.uint8), sentinel(cap, 7.0, torch.float64), sentinel(cap, 7.0, torch.float64)
    keep, nk = sentinel(cap, -7, torch.int32), i64(0)
    seg.semantic_keys_device(buf.data_ptr(), cnt.data_ptr(), cap, 14, cls.data_ptr(), conf.data_ptr(), ent.data_ptr(), keep.data_ptr(),
                             nk.data_ptr(), side.cuda_stream)
    side.synchronize()
    n = len(kps)
    assert np.array_equal(cls.cpu().numpy()[:n], want[0]) and conf.cpu().numpy()[:n].tobytes() == want[1].tobytes()
    assert ent.cpu().numpy()[:n].tobytes() == want[2].tobytes()
    assert int(nk.cpu()[0]) == len(want[3]) and np.array_equal(keep.cpu().numpy()[:len(want[3])], want[3])


def frame_keys(name, nf, sf, nlevels, kitti_gray_crop):
    if name == "kitti":
        gl = kitti_gray_crop
        gr = np.ascontiguousarray(np.roll(gl, -9, axis=1))  # the fixture is one image: a 9 px disparity everywhere
    else:
        left, right = stereo_frame(name)
        gl = np.ascontiguousarray(bgr_to_gray(left)[11:11 + 352, 109:109 + 1024])
        gr = np.ascontiguousarray(bgr_to_gray(right)[11:11 + 352, 109:109 + 1024])
    el, er = ORBextractor(nf, sf, nlevels, 20, 7), ORBextractor(nf, sf, nlevels, 20, 7)
    kl, dl = el(gl, None)
    kr, dr = er(gr, None)
    return el, er, kl, dl, kr, dr


@pytest.mark.parametrize("frame", ["kitti", 0, 1, 2])
@pytest.mark.parametrize("cfg", [(1000, 1.2, 8), (2000, 1.2, 8), (5000, 1.2, 8), (2000, 1.5, 4)])
def test_the_rule_is_inert_on_extractor_keys(frame, cfg, kitti_gray_crop):
    el, er, kl, dl, kr, dr = frame_keys(frame, *cfg, kitti_gray_crop)
    trace = []
    ru, rz = O.compute_stereo_matches(kl, dl, kr, dr, el._bordered, er._bordered, el.GetScaleFactors(), el.GetInverseScaleFactors(),
                                      KITTI_MB, KITTI_MBF, trace)
    stages = [t["stage"] for t in trace]
    assert not set(stages) & set(O.RULE_STAGES), {s: stages.count(s) for s in set(stages)}
    assert stages.count("matched") > 30
    hu, hz = stereo_match(el, er, kl, dl, kr, dr, KITTI_MB, KITTI_MBF)
    assert hu.tobytes() == ru.tobytes() and hz.tobytes() == rz.tobytes()


# ---------------------------------------------------------------------------------------------------------- fuzz
@pytest.mark.parametrize("block", range(10))
def test_differential_fuzz(block):
    for seed in range(block * 20, block * 20 + 20):
        probe = S.fuzz_scene(seed)
        el, er = pair(200, probe.scale_factor, probe.nlevels)
        ekl, edl = el(probe.left, None)
        ekr, edr = er(probe.right, None)
        rng = np.random.default_rng(seed)
        # planted near-duplicates of extractor descriptors among the right keys
        edr = edr.copy()
        for j in rng.choice(len(edr), min(len(edr), 20), replace=False):
            edr[j] = edl[rng.integers(len(edl))] ^ np.uint8(1 << int(rng.integers(8)))
        sc = S.fuzz_scene(seed, extra=(ekl, edl, ekr, edr))
        ru, rz = O.compute_stereo_matches(sc.kl, sc.dl, sc.kr, sc.dr, el._bordered, er._bordered, el.GetScaleFactors(),
                                          el.GetInverseScaleFactors(), sc.mb, sc.mbf)
        hu, hz = stereo_match(el, er, sc.kl, sc.dl, sc.kr, sc.dr, sc.mb, sc.mbf)
        assert hu.tobytes() == ru.tobytes() and hz.tobytes() == rz.tobytes(), seed
        cap_l, cap_r = el.capacity(), er.capacity()
        nl, nr = min(len(sc.kl), cap_l), min(len(sc.kr), cap_r)
        kind = seed % 5
        km = keymap(nl, cap_l, rng)
        if kind == 0:  # count -1: nothing written
            _, _, u, z = device_form(el, er, km, sc.kl[:nl], sc.dl[:nl], sc.kr[:nr], sc.dr[:nr], sc.mb, sc.mbf, n_left=-1)
            assert (u == 7.0).all() and (z == 7.0).all()
            continue
        kr, dr = sc.kr[:nr], sc.dr[:nr]
        n_right = None
        if kind == 1:  # a right count above the capacity reads the whole buffer
            pad = cap_r - nr
            kr = np.concatenate([kr, np.repeat(sc.kr[:1], pad)]) if pad and nr else kr
            dr = np.concatenate([dr, np.repeat(sc.dr[:1], pad, 0)]) if pad and nr else dr
            n_right = cap_r + 7
        n_left = cap_l + 3 if kind == 2 else None  # clamped: the entries past n_keep are valid slots
        sl, sdl, u, z = device_form(el, er, km, sc.kl[:nl], sc.dl[:nl], kr, dr, sc.mb, sc.mbf, n_left=n_left, n_right=n_right)
        m = min(km.n_keep if n_left is None else n_left, cap_l)
        keep = km.keep[:m]
        good = (keep >= 0) & (keep < cap_l)
        wu, wz = O.compute_stereo_matches(sl[keep[good]], sdl[keep[good]], kr, dr, el._bordered, er._bordered, el.GetScaleFactors(),
                                          el.GetInverseScaleFactors(), sc.mb, sc.mbf)
        assert u[:m][good].tobytes() == wu.tobytes() and z[:m][good].tobytes() == wz.tobytes(), seed
        assert (u[:m][~good] == -1).all() and (u[m:] == 7.0).all()
