"""-m gpu: `ORBextractor::operator()` and the stereo Hamming stage through the C-ABI, bit-exact against
the oracle and the committed golden fixtures."""
import os
import threading

import numpy as np
import pytest

from conftest import GOLDEN
from frame_support import kp_matrix
from oracle import orb_oracle as O
from sivo_b200 import ORBextractor, stereo_hamming, KP_DTYPE
from sivo_b200.synth import bgr_to_gray, stereo_frame

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,nf", [("orb_kitti_2000", 2000), ("orb_kitti_1000", 1000)])
def test_kitti_fixture_bit_exact_vs_golden(kitti_gray_crop, name, nf):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    ext = ORBextractor(nf, 1.2, 8, 20, 7)
    kps, desc = ext(kitti_gray_crop, None)
    for lvl in range(8):
        assert len(ext.candidates(lvl)[0]) == g["cand_counts"][lvl]
    assert len(kps) == len(g["keypoints"])
    assert np.array_equal(kp_matrix(kps), g["keypoints"])
    assert np.array_equal(desc, g["descriptors"])


def test_pyramid_and_candidates_vs_oracle(kitti_gray_crop):
    ext = ORBextractor(2000, 1.2, 8, 20, 7)
    ext(kitti_gray_crop, None)
    r = O.extract(kitti_gray_crop)
    for lvl in range(8):
        assert np.array_equal(ext._bordered[lvl], r.pyramid[lvl]), lvl
        xs, ys, rs = ext.candidates(lvl)
        assert np.array_equal(xs, r.candidates[lvl][0]) and np.array_equal(ys, r.candidates[lvl][1])
        assert np.array_equal(rs, r.candidates[lvl][2])
    assert ext.mvImagePyramid[0].shape == (352, 1024) and np.array_equal(ext.mvImagePyramid[0], kitti_gray_crop)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_synthetic_frames_bit_exact_vs_oracle(seed):
    left, right = stereo_frame(seed)
    for img in (left, right):
        gray = np.ascontiguousarray(bgr_to_gray(img)[11:11 + 352, 109:109 + 1024])
        ext = ORBextractor(2000, 1.2, 8, 20, 7)
        kps, desc = ext(gray, None)
        r = O.extract(gray)
        assert np.array_equal(kp_matrix(kps), r.keypoints.astype(np.float32))
        assert np.array_equal(desc, r.descriptors)


def test_edge_cases():
    ext = ORBextractor(500, 1.2, 8, 20, 7)
    k, d = ext(np.zeros((0, 0), np.uint8), None)           # empty image returns silently (:1023-1024)
    assert len(k) == 0 and d.shape == (0, 32)
    flat = np.full((352, 1024), 128, np.uint8)              # no corners -> zero keypoints, descriptors released
    k, d = ext(flat, None)
    assert len(k) == 0 and d.shape == (0, 32)
    rng = np.random.default_rng(0)                          # odd, non-multiple-of-anything size
    img = rng.integers(0, 256, size=(301, 517), dtype=np.uint8)
    k, d = ext(img, None)
    r = O.extract(img, O.ExtractorParams(500))
    assert np.array_equal(kp_matrix(k), r.keypoints.astype(np.float32)) and np.array_equal(d, r.descriptors)
    with pytest.raises(Exception):
        ext(np.zeros((40, 40), np.uint8), None)             # too small for 8 levels


def test_two_extractors_concurrently(kitti_gray_crop):
    # Frame.cc:126-129 runs left and right on two std::threads
    g = np.load(os.path.join(GOLDEN, "orb_kitti_2000.npz"))
    exts = [ORBextractor(2000, 1.2, 8, 20, 7) for _ in range(2)]
    out = [None, None]

    def work(i):
        for _ in range(5):
            out[i] = exts[i](kitti_gray_crop, None)
    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    [t.start() for t in th]
    [t.join() for t in th]
    for kps, desc in out:
        assert np.array_equal(kp_matrix(kps), g["keypoints"]) and np.array_equal(desc, g["descriptors"])


def test_stereo_hamming_vs_brute_force():
    left, right = stereo_frame(0)
    gl = np.ascontiguousarray(bgr_to_gray(left)[11:11 + 352, 109:109 + 1024])
    gr = np.ascontiguousarray(bgr_to_gray(right)[11:11 + 352, 109:109 + 1024])
    el, er = ORBextractor(2000, 1.2, 8, 20, 7), ORBextractor(2000, 1.2, 8, 20, 7)
    kl, dl = el(gl, None)
    kr, dr = er(gr, None)
    sf = el.GetScaleFactors()
    max_d = 100.0
    idx, dist = stereo_hamming(kl, dl, kr, dr, sf, 352, 0.0, max_d)
    # restatement of Frame.cc:452-533 (row table, octave gate, disparity window, first strictly smaller distance)
    rows = [[] for _ in range(352)]
    for i in range(len(kr)):
        r = np.float32(2.0) * sf[kr["octave"][i]]
        lo, hi = int(np.floor(kr["y"][i] - r)), int(np.ceil(kr["y"][i] + r))
        for y in range(lo, hi + 1):
            rows[y].append(i)
    xor = np.unpackbits(dl[:, None, :] ^ dr[None, :, :], axis=2).sum(axis=2) if len(kl) * len(kr) < 6e6 else None
    matched = 0
    for i in range(len(kl)):
        best, bi = 100, -1
        u, v, lv = kl["x"][i], kl["y"][i], kl["octave"][i]
        if u - np.float32(0) >= 0:
            for j in rows[int(v)]:
                if kr["octave"][j] < lv - 1 or kr["octave"][j] > lv + 1:
                    continue
                if np.float32(u - np.float32(max_d)) <= kr["x"][j] <= u:
                    d = int(xor[i, j]) if xor is not None else O.descriptor_distance(dl[i], dr[j])
                    if d < best:
                        best, bi = d, j
        assert dist[i] == best and idx[i] == bi, i
        matched += bi >= 0
    assert matched > 200


def test_stereo_match_full_vs_oracle():
    """The whole ComputeStereoMatches (Hamming + SAD slide + parabola + median cut) on the device pyramids."""
    from sivo_b200 import stereo_match
    left, right = stereo_frame(1)
    gl = np.ascontiguousarray(bgr_to_gray(left)[11:11 + 352, 109:109 + 1024])
    gr = np.ascontiguousarray(bgr_to_gray(right)[11:11 + 352, 109:109 + 1024])
    el, er = ORBextractor(2000, 1.2, 8, 20, 7), ORBextractor(2000, 1.2, 8, 20, 7)
    kl, dl = el(gl, None)
    kr, dr = er(gr, None)
    mbf = 386.1448  # Camera.bf of config/kitti/KITTI00-02.yaml; mb = bf / fx
    mb = mbf / 718.856
    u, z = stereo_match(el, er, kl, dl, kr, dr, mb, mbf)
    ru, rz = O.compute_stereo_matches(kl, dl, kr, dr, el._bordered, er._bordered, el.GetScaleFactors(), el.GetInverseScaleFactors(), mb, mbf)
    assert np.array_equal(u, ru) and np.array_equal(z, rz)
    assert (u >= 0).sum() > 150


def test_hamming_best2_equals_the_sequential_loop():
    """Next row 8(f)-4: best / second-best over candidate lists, ties and empty lists included (bit-exact: integers)."""
    from sivo_b200.orb import hamming_best2
    rng = np.random.default_rng(11)
    nt, nq = 700, 400
    train = rng.integers(0, 256, size=(nt, 32), dtype=np.uint8)
    # queries near some train descriptors (a few bits flipped) so that small distances and exact ties occur
    src = rng.integers(0, nt, nq)
    query = train[src].copy()
    for i in range(nq):
        flips = rng.integers(0, 256, size=rng.integers(0, 40))
        for b in flips:
            query[i, b >> 3] ^= np.uint8(1 << (b & 7))
    train[5] = train[9]  # duplicated descriptors: equal distances inside one list
    train[17] = train[9]
    level = rng.integers(0, 8, nt).astype(np.int32)
    lens = rng.integers(0, 90, nq)
    lens[:5] = 0
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cand = np.concatenate([rng.permutation(nt)[:n] for n in lens] + [np.empty(0, np.int64)]).astype(np.int32)
    for i in range(5, 40):  # make sure the true source and the duplicates are among the candidates of some queries
        if lens[i] >= 3:
            cand[off[i]:off[i] + 3] = (17, 5, 9)
            query[i] = train[9]
    want = O.hamming_best2(query, train, off, cand, level)
    got = hamming_best2(query, train, off, cand, level)
    assert np.array_equal(got, want)
    assert np.array_equal(hamming_best2(query, train, off, cand, None)[:, [0, 1, 3]], want[:, [0, 1, 3]])
    assert (got[:5] == np.array([-1, 256, -1, 256, -1])).all()


def test_hamming_best2_on_a_fresh_thread_small_large_small():
    """The host-call staging is per thread, so a new thread starts with none.  The first call is small; the second needs several
    times what the first left behind, so it gets more device memory while its earlier buffers are in use; the third runs on what
    the second's pieces were merged into.  Each result equals the sequential loop."""
    from sivo_b200.orb import hamming_best2
    rng = np.random.default_rng(12)
    cases = []
    for nq, nt, max_len in ((20, 50, 8), (3000, 40000, 20), (20, 50, 8)):
        train = rng.integers(0, 256, size=(nt, 32), dtype=np.uint8)
        query = train[rng.integers(0, nt, nq)] ^ rng.integers(0, 256, size=(nq, 32), dtype=np.uint8) * (rng.random((nq, 32)) < 0.1)
        level = rng.integers(0, 8, nt).astype(np.int32)
        lens = rng.integers(0, max_len, nq)
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        cand = rng.integers(0, nt, off[-1]).astype(np.int32)
        cases.append((query, train, off, cand, level))
    got = []
    t = threading.Thread(target=lambda: got.extend(hamming_best2(*c) for c in cases))
    t.start()
    t.join()
    assert len(got) == len(cases)
    for c, g in zip(cases, got):
        assert np.array_equal(g, O.hamming_best2(*c))


def gpu_tree(xs, ys, rs, min_x, max_x, min_y, max_y, tgt):
    import ctypes as C
    from sivo_b200 import _lib as L
    n = len(xs)
    cap = 4096
    ox, oy, orr = (np.empty(cap, np.int32) for _ in range(3))
    a = [np.ascontiguousarray(v, np.int32) for v in (xs, ys, rs)]
    rc = L.lib().sivo_dbg_orb_distribute_device(0, a[0].ctypes.data_as(C.c_void_p), a[1].ctypes.data_as(C.c_void_p),
                                                a[2].ctypes.data_as(C.c_void_p), n, min_x, max_x, min_y, max_y, tgt,
                                                ox.ctypes.data_as(C.c_void_p), oy.ctypes.data_as(C.c_void_p),
                                                orr.ctypes.data_as(C.c_void_p), cap)
    L.check(rc)
    return ox[:rc].copy(), oy[:rc].copy(), orr[:rc].copy()


def test_device_quad_tree_equals_the_host_tree_on_random_inputs():
    """DistributeOctTree on the device (orb_tree.cu) against the host restatement shared with the oracle: same kept keys in the
    same ORDER, for inputs that exercise every branch -- a single key, fewer keys than the target, heavy response ties, duplicate
    positions, the regular rounds stopping on 'no change', and the last one-at-a-time phase."""
    from sivo_b200.orb import distribute_octtree
    rng = np.random.default_rng(7)
    cases = 0
    for trial in range(60):
        n = int(rng.integers(1, 6000)) if trial % 5 else int(rng.integers(1, 40))
        w, h = int(rng.integers(100, 1000)), int(rng.integers(60, 330))
        xs = rng.integers(0, w, n)
        ys = rng.integers(0, h, n)
        if trial % 7 == 0:  # duplicate positions: nodes that cannot be separated
            xs[: n // 2] = xs[0]
            ys[: n // 2] = ys[0]
        rs = rng.integers(7, 30 if trial % 3 else 255, n)
        tgt = int(rng.integers(1, 500))
        keep = distribute_octtree(xs.astype(np.float32), ys.astype(np.float32), rs.astype(np.float32), 16, 16 + w, 16, 16 + h, tgt)
        gx, gy, gr = gpu_tree(xs, ys, rs, 16, 16 + w, 16, 16 + h, tgt)
        assert len(gx) == len(keep), (trial, n, tgt, len(gx), len(keep))
        assert np.array_equal(gx, xs[keep]) and np.array_equal(gy, ys[keep]) and np.array_equal(gr, rs[keep]), (trial, n, tgt)
        cases += 1
    assert cases == 60


def test_device_and_host_quad_tree_give_the_same_extraction(monkeypatch, kitti_gray_crop):
    """The whole operator with the tree on the device (default: no host round trip) and on the host (SIVO_B200_ORB_DEVICE_TREE=0)."""
    left, _ = stereo_frame(6)
    imgs = [kitti_gray_crop, np.ascontiguousarray(bgr_to_gray(left)[11:11 + 352, 109:109 + 1024])]
    res = {}
    for flag in ("1", "0"):
        monkeypatch.setenv("SIVO_B200_ORB_DEVICE_TREE", flag)
        for nf in (2000, 500):
            ext = ORBextractor(nf, 1.2, 8, 20, 7)
            res[flag, nf] = [ext(im, None) for im in imgs]
            assert ext.last_timing()["tree_ms"] == 0.0 if flag == "1" else ext.last_timing()["tree_ms"] > 0.0
    for nf in (2000, 500):
        for (ka, da), (kb, db) in zip(res["1", nf], res["0", nf]):
            assert ka.tobytes() == kb.tobytes() and np.array_equal(da, db)


def test_host_tree_level_larger_than_the_device_tree_selection(kitti_gray_crop):
    """nfeatures = 5000 asks for 1086 keypoints at level 0, more than one level of the device tree's selection holds (1024), so
    the host tree takes every call; it keeps 1087 at level 0, which the describe pass reads at a stride wider than the device
    tree's."""
    ext = ORBextractor(5000, 1.2, 8, 20, 7)
    assert not ext.has_device_tree()
    kps, desc = ext(kitti_gray_crop, None)
    r = O.extract(kitti_gray_crop, O.ExtractorParams(5000))
    assert (kps["octave"] == 0).sum() == 1087
    assert np.array_equal(kp_matrix(kps), r.keypoints.astype(np.float32))
    assert np.array_equal(desc, r.descriptors)


def test_asynchronous_device_form_writes_the_same_record(kitti_gray_crop):
    """sivo_orb_enqueue_device: gray image, keypoints, descriptors and count all stay on the device (what the multi-GPU record
    path uses); the results equal the synchronous operator's."""
    import torch
    ext = ORBextractor(2000, 1.2, 8, 20, 7)
    kps, desc = ext(kitti_gray_crop, None)
    cap = ext.capacity()
    d_gray = torch.from_numpy(kitti_gray_crop).cuda()
    d_kps = torch.zeros(cap * 28, dtype=torch.uint8, device="cuda")
    d_desc = torch.zeros(cap * 32, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    for _ in range(2):
        ext.enqueue_device(d_gray.data_ptr(), 352, 1024, 1024, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr())
        ext.stream_wait(torch.cuda.current_stream().cuda_stream)
        n = int(d_cnt.cpu()[0])
        assert ext.device_status() == 0
        assert n == len(kps)
        got = d_kps.cpu().numpy()[: n * 28].view(KP_DTYPE)
        assert got.tobytes() == kps.tobytes()
        assert np.array_equal(d_desc.cpu().numpy()[: n * 32].reshape(n, 32), desc)
