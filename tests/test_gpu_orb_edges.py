"""-m gpu: the ORB extractor on dense and extreme frames (oracle/orb_scene.py) against the oracle, bit for bit, in both forms:
the synchronous operator with the device quad tree, the same with the host tree forced, and the asynchronous form, whose records
must equal the synchronous ones whenever its status is 0 and whose count must be -1 otherwise.  Also the size limits of the
pyramid and the 12-bit packing, pitched input, and a frame that overflows the device tree through the device-resident Frame tail."""
import functools

import numpy as np
import pytest
import torch

from frame_support import MB, MBF, InfoOut, cameras, kp_matrix, seg, synth, upload  # noqa: F401
from oracle import orb_oracle as O
from oracle import orb_scene as S
from sivo_b200 import KP_DTYPE, ORBextractor, info_select, stereo_match
from sivo_b200 import _lib as L
from sivo_b200.frame import DeviceFrame
from sivo_b200.synth import bgr_to_gray

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def kitti_gray(kitti_bgr):
    return bgr_to_gray(kitti_bgr)


@pytest.fixture(scope="module")
def case(kitti_gray):
    """name -> (image, parameters, oracle result, oracle level stats), each computed once."""
    @functools.lru_cache(maxsize=None)
    def get(name):
        build, p = S.CASES[name]
        img = build(kitti_gray)
        r = O.extract(img, p)
        return img, p, r, S.level_stats(r, img.shape, p)
    return get


def make(p):
    return ORBextractor(p.nfeatures, p.scale_factor, p.nlevels, p.ini_th, p.min_th)


def run_async(ext, img):
    """sivo_orb_enqueue_device on a device copy of img: (count, records, descriptors, status mask)."""
    rows, cols = img.shape
    cap = ext.capacity()
    d_gray = upload(img)
    d_kps = torch.zeros(cap * 28, dtype=torch.uint8, device="cuda")
    d_desc = torch.zeros(cap * 32, dtype=torch.uint8, device="cuda")
    d_cnt = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ext.enqueue_device(d_gray.data_ptr(), rows, cols, cols, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr())
    ext.stream_wait(torch.cuda.current_stream().cuda_stream)
    status = ext.device_status()
    n = int(d_cnt.cpu()[0])
    m = max(n, 0)
    return n, d_kps.cpu().numpy()[:m * 28].view(KP_DTYPE), d_desc.cpu().numpy()[:m * 32].reshape(m, 32), status


def margins(name, p, stats, status=None):
    """One line per case: per level, candidates / kTreeKeyCap, the densest cell / kCellCap and the initial node count."""
    lv = " | ".join(f"L{l} {s['candidates']}/{S.TREE_KEY_CAP} cell {s['cell_max']}/{S.CELL_CAP} ini {s['n_ini']}"
                    for l, s in enumerate(stats))
    print(f"\n[{name}] nf {p.nfeatures} sf {p.scale_factor} nl {p.nlevels} th {p.ini_th}/{p.min_th} status {status}: {lv}")


def expected_mask(stats):
    """Levels the device tree cannot hold by its key cap or its 16 initial nodes (a level without candidates never reaches either)."""
    return sum(1 << l for l, s in enumerate(stats) if s["candidates"] > S.TREE_KEY_CAP or (s["candidates"] > 0 and s["n_ini"] > 16))


@pytest.mark.parametrize("name", list(S.CASES))
def test_case_bit_exact_in_both_forms(name, case, monkeypatch):
    img, p, r, stats = case(name)
    want_k, want_d = r.keypoints.astype(np.float32), r.descriptors
    bound = p.nfeatures + 3 * p.nlevels  # what the header promises (sivo_orb_run)
    assert all(s["cell_max"] <= S.CELL_CAP for s in stats)

    ext = make(p)
    kps, desc = ext(img, None)
    assert len(kps) <= bound
    assert np.array_equal(kp_matrix(kps), want_k) and np.array_equal(desc, want_d)
    for lvl in range(p.nlevels):
        xs, ys, rs = ext.candidates(lvl)
        assert np.array_equal(xs, r.candidates[lvl][0]) and np.array_equal(ys, r.candidates[lvl][1]), lvl
        assert np.array_equal(rs, r.candidates[lvl][2]), lvl

    status = None
    if ext.has_device_tree():
        n, akps, adesc, status = run_async(ext, img)
        assert status == expected_mask(stats), (status, expected_mask(stats))
        if status == 0:
            assert n == len(kps) and akps.tobytes() == kps.tobytes() and np.array_equal(adesc, desc)
        else:
            assert n == -1
    margins(name, p, stats, status)

    monkeypatch.setenv("SIVO_B200_ORB_DEVICE_TREE", "0")  # read by the constructor
    host = make(p)
    assert not host.has_device_tree()
    hk, hd = host(img, None)
    assert hk.tobytes() == kps.tobytes() and np.array_equal(hd, desc)
    assert host.last_timing()["tree_ms"] > 0.0


@pytest.mark.parametrize("form", ["run", "enqueue_device"])
def test_size_limits_are_refused(kitti_gray, form):
    """The smallest 8-level image is accepted (test_case_bit_exact_in_both_forms); one row less leaves the coarsest level 44 px
    high.  4,058 px wide fits the 12-bit candidate packing with the 19-px borders; 4,059 does not.  Both forms refuse with EINVAL,
    and a refused size leaves nothing of itself behind: the handle's next call, at the size before, gives the same result."""
    crop = S.kitti_crop(kitti_gray)
    small = np.ascontiguousarray(crop[:S.min_rows() - 1])
    wide = np.ascontiguousarray(np.tile(kitti_gray[100:260], (1, 4))[:, :S.MAX_PACKED_WIDTH + 1])
    ext = ORBextractor(2000, 1.2, 8, 20, 7)
    kps, desc = ext(crop, None)
    for img in (small, wide):
        with pytest.raises(L.SivoError) as e:
            if form == "run":
                ext(img, None)
            else:
                run_async(ext, img)
        assert e.value.code == L.EINVAL
        k, d = ext(crop, None)
        assert k.tobytes() == kps.tobytes() and np.array_equal(d, desc)


def test_pitched_input_in_every_form(case):
    """A row pitch wider than the image (stride > cols): host buffer, device buffer, and the asynchronous form."""
    img, p, r, _ = case("ladder_below")
    rows, cols = img.shape
    pitch = cols + 77
    big = np.full((rows, pitch), 255, np.uint8)
    big[:, :cols] = img
    view = big[:, :cols]
    assert view.strides[0] == pitch
    want_k, want_d = r.keypoints.astype(np.float32), r.descriptors
    ext = make(p)
    k, d = ext(view, None)
    assert np.array_equal(kp_matrix(k), want_k) and np.array_equal(d, want_d)
    d_big = upload(big)
    k2, d2 = ext.run_device_input(d_big.data_ptr(), rows, cols, pitch)
    assert k2.tobytes() == k.tobytes() and np.array_equal(d2, d)
    cap = ext.capacity()
    d_kps = torch.zeros(cap * 28, dtype=torch.uint8, device="cuda")
    d_desc = torch.zeros(cap * 32, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ext.enqueue_device(d_big.data_ptr(), rows, cols, pitch, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr())
    ext.stream_wait(torch.cuda.current_stream().cuda_stream)
    assert ext.device_status() == 0
    n = int(d_cnt.cpu()[0])
    assert n == len(k) and d_kps.cpu().numpy()[:n * 28].tobytes() == k.tobytes()
    assert np.array_equal(d_desc.cpu().numpy()[:n * 32].reshape(n, 32), d)


def _chain(seg, el, er, bgr, gl, gr, cam):
    """SegNet -> both extractors' enqueue_device -> semantic keys -> stereo -> information selection, all on the device."""
    seg.set_frame(3)
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    f = DeviceFrame(el, er, *gl.shape)
    info = InfoOut(f.left.cap)
    f.extract(seg, upload(bgr), upload(gl), upload(gr), s)
    f.tail(seg, MB, MBF, s)
    info.run(el, f.kps, f.kp_entropy, f.keep, f.n_keep, f.depth, cam, 0.0, s)
    stream.synchronize()
    return f, info


def test_overflow_propagates_through_the_device_frame_tail(seg):
    """A full-noise frame overflows the device tree on both extractors: the count is -1, the semantic keys and the information
    selection report -1 and stereo writes nothing.  A normal frame through the same handles gives the host forms' results."""
    cam, _ = cameras("motion", "moved")
    el, er = ORBextractor(2000, 1.2, 8, 20, 7), ORBextractor(2000, 1.2, 8, 20, 7)
    gl, gr = S.noise(S.H, S.W, 1), S.noise(S.H, S.W, 2)
    bgr = np.ascontiguousarray(np.repeat(gl[:, :, None], 3, axis=2))
    f, info = _chain(seg, el, er, bgr, gl, gr, cam)
    assert el.device_status() & 0b111 == 0b111 and er.device_status() & 0b111 == 0b111
    assert int(f.left.count.cpu()[0]) == -1
    out = {k: v.cpu().numpy() for k, v in f.out.items()}
    assert int(out["n_keep"][0]) == -1 and (out["keep_idx"] == -7).all() and (out["kp_class"] == 77).all()
    assert (out["u_right"] == 7.0).all() and (out["depth"] == 7.0).all()
    assert int(info.n.cpu()[0]) == -1 and (info.sel.cpu().numpy() == -7).all() and (info.red.cpu().numpy() == 7.0).all()

    bgr, gl, gr = synth(1)
    f, info = _chain(seg, el, er, bgr, gl, gr, cam)
    assert el.device_status() == 0 and er.device_status() == 0
    kl, dl = ORBextractor(2000, 1.2, 8, 20, 7)(gl, None)
    kr, dr = ORBextractor(2000, 1.2, 8, 20, 7)(gr, None)
    kps, _ = f.left.host()
    assert kps.tobytes() == kl.tobytes()
    n_keep, keep, u, z = f.host()
    assert np.array_equal(keep, seg.semantic_keys(kl, 8)[3]) and n_keep > 100
    hu, hz = stereo_match(el, er, kl[keep], dl[keep], kr, dr, MB, MBF)
    assert u.tobytes() == hu.tobytes() and z.tobytes() == hz.tobytes()
    ent = f.out["kp_entropy"].cpu().numpy()[:len(kl)][keep]
    _, _, sel = info_select(el, kl[keep], z, ent, cam, 0.0)
    assert int(info.n.cpu()[0]) == len(sel) > 0 and np.array_equal(info.sel.cpu().numpy()[:len(sel)], sel)
