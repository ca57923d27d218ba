"""Pins the ORB oracle (numpy restatement of OpenCV's algorithms) to the operational oracle cv2, bit for
bit, and to the committed golden fixtures.  The reference holds no ORB vectors (SURVEY 4); parity with an
OpenCV-3.x build of it is therefore 'unpinned' and the cv2 version is recorded here."""
import functools
import os

import numpy as np
import pytest

from oracle import orb_oracle as O
from oracle import orb_scene as S

cv2 = pytest.importorskip("cv2")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_cv2_version_recorded():
    print("operational oracle: cv2", cv2.__version__)
    assert int(cv2.__version__.split(".")[0]) >= 3


def test_constructor_tables():
    # SURVEY 8a a12: 2000 -> [434,362,302,251,209,175,145,122]; 1000 -> [217,181,151,126,105,87,73,60]
    assert O.Tables(O.ExtractorParams(2000)).per_level == [434, 362, 302, 251, 209, 175, 145, 122]
    assert O.Tables(O.ExtractorParams(1000)).per_level == [217, 181, 151, 126, 105, 87, 73, 60]
    t = O.Tables(O.ExtractorParams())
    assert t.umax == [15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3]
    assert O.level_sizes(1024, 352, t) == [(1024, 352), (853, 293), (711, 244), (593, 204), (494, 170), (412, 141),
                                           (343, 118), (286, 98)]


def test_resize_blur_border_bit_exact(kitti_gray_crop):
    g = kitti_gray_crop
    for (w, h) in [(853, 293), (711, 244), (286, 98), (1000, 100)]:
        assert np.array_equal(cv2.resize(g, (w, h), interpolation=cv2.INTER_LINEAR), O.resize_linear_u8(g, w, h))
    assert np.array_equal(cv2.GaussianBlur(g, (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101), O.gaussian_blur7(g))
    assert np.array_equal(cv2.copyMakeBorder(g, 19, 19, 19, 19, cv2.BORDER_REFLECT_101), O.reflect101(g, 19))


def test_fast_atan2_bit_exact():
    rng = np.random.default_rng(0)
    y = rng.integers(-200000, 200000, 20000).astype(np.float32)
    x = rng.integers(-200000, 200000, 20000).astype(np.float32)
    y[:10] = 0
    x[5:15] = 0
    ref = np.array([cv2.fastAtan2(float(a), float(b)) for a, b in zip(y, x)], np.float32)
    assert np.array_equal(ref, O.fast_atan2(y, x))


def test_fast_cells_bit_exact(kitti_gray_crop):
    g = kitti_gray_crop
    score = O.fast_score_map(g)
    rng = np.random.default_rng(1)
    total = 0
    for _ in range(150):
        x0, y0 = int(rng.integers(0, 960)), int(rng.integers(0, 300))
        x1, y1 = min(x0 + int(rng.integers(7, 60)), 1024), min(y0 + int(rng.integers(7, 50)), 352)
        for th in (7, 20):
            det = cv2.FastFeatureDetector_create(th, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16)
            ref = [(int(k.pt[0]), int(k.pt[1]), int(k.response)) for k in det.detect(np.ascontiguousarray(g[y0:y1, x0:x1]))]
            xs, ys, rs = O.cell_keypoints(score, x0, y0, x1, y1, th)
            assert ref == list(zip(xs.tolist(), ys.tolist(), rs.tolist()))
            total += len(ref)
    assert total > 1000


def _cv2_pipeline(gray, p=O.ExtractorParams()):
    """ORBextractor::operator() composed from cv2 primitives exactly as the reference composes OpenCV
    (ORBextractor.cc:752-847,1019-1122); the quad tree is the oracle's."""
    t = O.Tables(p)
    pattern = O.load_pattern()
    h, w = gray.shape
    levels = []
    for lvl, (lw, lh) in enumerate(O.level_sizes(w, h, t)):
        cur = gray if lvl == 0 else cv2.resize(levels[-1], (lw, lh), interpolation=cv2.INTER_LINEAR)
        levels.append(cur)
    kps, descs = [], []
    for lvl, im in enumerate(levels):
        lh, lw = im.shape
        cells, (mbx, mby, Mbx, Mby) = O.level_cells(lw, lh)
        cx, cy, cr = [], [], []
        for (x0, y0, x1, y1) in cells:
            sub = np.ascontiguousarray(im[y0:y1, x0:x1])
            k = cv2.FastFeatureDetector_create(p.ini_th, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16).detect(sub)
            if not k:
                k = cv2.FastFeatureDetector_create(p.min_th, True, cv2.FAST_FEATURE_DETECTOR_TYPE_9_16).detect(sub)
            for q in k:
                cx.append(q.pt[0] + x0 - mbx)
                cy.append(q.pt[1] + y0 - mby)
                cr.append(q.response)
        if not cx:
            continue
        sel = O.distribute_octtree(np.array(cx), np.array(cy), np.array(cr, np.float32), mbx, Mbx, mby, Mby, t.per_level[lvl])
        bordered = cv2.copyMakeBorder(im, 19, 19, 19, 19, cv2.BORDER_REFLECT_101)
        blur = cv2.GaussianBlur(im.copy(), (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101)
        for s in sel:
            x, y = int(cx[s]) + mbx, int(cy[s]) + mby
            ang = O.ic_angle(bordered, x, y, t.umax)
            descs.append(O.orb_descriptor(blur, x, y, ang, pattern))
            sc = t.scale[lvl]
            fx, fy = (np.float32(x), np.float32(y)) if lvl == 0 else (np.float32(np.float32(x) * sc), np.float32(np.float32(y) * sc))
            kps.append([fx, fy, np.float32(int(np.float32(31) * sc)), ang, cr[s], lvl, -1])
    return np.array(kps, np.float32).reshape(-1, 7), np.array(descs, np.uint8).reshape(-1, 32)


def test_pipeline_matches_cv2_composition(kitti_gray_crop):
    r = O.extract(kitti_gray_crop)
    kp, desc = _cv2_pipeline(kitti_gray_crop)
    assert np.array_equal(r.keypoints.astype(np.float32), kp)
    assert np.array_equal(r.descriptors, desc)
    assert len(kp) >= 2000


@pytest.fixture(scope="module")
def scene(kitti_bgr):
    """name -> (image, parameters, oracle result, oracle level stats) of oracle/orb_scene.py's cases, each computed once."""
    from sivo_b200.synth import bgr_to_gray
    gray = bgr_to_gray(kitti_bgr)

    @functools.lru_cache(maxsize=None)
    def get(name):
        build, p = S.CASES[name]
        img = build(gray)
        r = O.extract(img, p)
        return img, p, r, S.level_stats(r, img.shape, p)
    return get


# every image at its own parameters, and the parameter sets that change what cv2 computes (thresholds, pyramid) on both images
CV2_CASES = [n for n in S.CASES if not n.startswith(("crop_", "dense_"))] + [
    f"{img}_{k}" for img in ("crop", "dense") for k in ("th12_7", "pyr1.5x5", "pyr1.1x12")]


@pytest.mark.parametrize("name", CV2_CASES)
def test_scene_matches_cv2_composition(scene, name):
    img, p, r, _ = scene(name)
    kp, desc = _cv2_pipeline(img, p)
    assert np.array_equal(r.keypoints.astype(np.float32), kp)
    assert np.array_equal(r.descriptors, desc)
    assert len(kp) > 0


def test_level_without_cells():
    """A level whose FAST region is under 30 px in either direction has no cells (the reference's cell loops run zero times)."""
    assert O.level_cells(61, 200)[0] == [] and O.level_cells(200, 61)[0] == []
    assert len(O.level_cells(62, 62)[0]) == 1


def test_scenes_reach_what_they_were_built_for(scene):
    st = lambda name: scene(name)[3]
    # the density ladder: level 0 on either side of the device tree's key cap, then pure noise with levels 0-2 above it
    over = lambda name: {l for l, s in enumerate(st(name)) if s["candidates"] > S.TREE_KEY_CAP}
    assert over("ladder_below") == set() and over("ladder_above") == {0} and over("ladder_full") == {0, 1, 2}
    below, above = st("ladder_below")[0]["candidates"], st("ladder_above")[0]["candidates"]
    assert S.TREE_KEY_CAP - 200 < below <= S.TREE_KEY_CAP < above < S.TREE_KEY_CAP + 200
    assert sum(s["candidates"] for s in st("ladder_full")) > 70000
    # the densest cell holds the whole 27 x 27 lattice, below kCellCap
    assert st("densest_cell")[0]["cell_max"] == 27 * 27 <= S.CELL_CAP and st("densest_cell")[0]["cells"] == 1
    assert all(s["cell_max"] <= S.CELL_CAP for n in S.CASES for s in st(n))
    # binary noise ties: level 0 holds few distinct responses
    assert len(np.unique(scene("binary")[2].candidates[0][2])) < 20
    ch = st("checkerboard")
    assert ch[0]["candidates"] == 0 and ch[1]["candidates"] > 1000 and ch[2]["candidates"] > 1000
    # the smallest 8-level image: its coarsest level is 45 px high (one row less: 44) and, under 30 px of FAST region, has no cells
    img, p, _, _ = scene("smallest_8_levels")
    t = O.Tables(p)
    assert O.level_sizes(img.shape[1], img.shape[0], t)[-1][1] == 45
    assert O.level_sizes(img.shape[1], img.shape[0] - 1, t)[-1][1] == 44
    assert st("smallest_8_levels")[-1]["cells"] == 0
    img, p, _, _ = scene("narrow_level")
    assert 45 <= O.level_sizes(img.shape[1], img.shape[0], O.Tables(p))[-1][0] < 62 and st("narrow_level")[-1]["cells"] == 0
    img = scene("portrait")[0]
    assert int(np.float32(img.shape[1] - 32) / np.float32(img.shape[0] - 32) + np.float32(0.5)) == 0  # n_ini 0, clamped to 1
    assert scene("wide_4058")[0].shape[1] == S.MAX_PACKED_WIDTH and min(s["n_ini"] for s in st("wide_4058")) > 16
    # the min_th fallback: at level 0 some cells keep iniThFAST corners and more retry at minThFAST
    img, p, _, _ = scene("min_th_fallback")
    score = O.fast_score_map(img)
    cells, _ = O.level_cells(img.shape[1], img.shape[0])
    at_ini = [len(O.cell_keypoints(score, *c, p.ini_th)[0]) > 0 for c in cells]
    at_min = [not a and len(O.cell_keypoints(score, *c, p.min_th)[0]) > 0 for c, a in zip(cells, at_ini)]
    assert sum(at_ini) > 100 and sum(at_min) > 100


@pytest.mark.parametrize("name,nf", [("orb_kitti_2000", 2000), ("orb_kitti_1000", 1000)])
def test_oracle_matches_golden(kitti_gray_crop, name, nf):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    r = O.extract(kitti_gray_crop, O.ExtractorParams(nf))
    assert np.array_equal(r.keypoints.astype(np.float32), g["keypoints"])
    assert np.array_equal(r.descriptors, g["descriptors"])
    assert r.level_counts == g["level_counts"].tolist()


def test_hamming_distance():
    rng = np.random.default_rng(2)
    a, b = rng.integers(0, 256, 32, dtype=np.uint8), rng.integers(0, 256, 32, dtype=np.uint8)
    # the bit-hack of ORBmatcher.cc:1582-1596 on 8 x u32
    d = 0
    for va, vb in zip(a.view("<u4"), b.view("<u4")):
        v = int(va) ^ int(vb)
        v = v - ((v >> 1) & 0x55555555)
        v = (v & 0x33333333) + ((v >> 2) & 0x33333333)
        d += ((((v + (v >> 4)) & 0xF0F0F0F) * 0x1010101) & 0xFFFFFFFF) >> 24
    assert d == O.descriptor_distance(a, b)


def test_select_semantic_keys_is_the_reference_loop():
    """Frame::SelectSemanticKeys (Frame.cc:177-203) as the literal loop: truncate pt to (row, col), keep iff class <= TERRAIN."""
    rng = np.random.default_rng(5)
    classes = rng.integers(0, 14, size=(40, 64)).astype(np.uint8)
    classes[rng.random(classes.shape) < 0.05] = 255  # VOID
    conf = rng.random(classes.shape)
    ent = rng.random(classes.shape)
    xy = np.stack([rng.uniform(0, 63.99, 300), rng.uniform(0, 39.99, 300)], 1).astype(np.float32)
    cls, c, e, keep = O.select_semantic_keys(xy, classes, conf, ent)
    want_keep = []
    for i, (x, y) in enumerate(xy):
        col, row = int(x), int(y)
        assert cls[i] == classes[row, col] and c[i] == conf[row, col] and e[i] == ent[row, col]
        if classes[row, col] <= 8:
            want_keep.append(i)
    assert keep.tolist() == want_keep


def test_hamming_best2_tie_and_demotion_rules():
    """The SearchByProjection candidate loop (ORBmatcher.cc:79-113): strict '<' keeps the first minimum; a later equal distance
    becomes the second best; a beaten best is demoted together with its level."""
    def desc(nbits):
        d = np.zeros(32, np.uint8)
        for b in range(nbits):
            d[b >> 3] |= 1 << (b & 7)
        return d
    q = np.zeros((1, 32), np.uint8)
    train = np.stack([desc(5), desc(3), desc(3), desc(7)])
    level = np.array([10, 11, 12, 13])
    r = O.hamming_best2(q, train, [0, 4], [0, 1, 2, 3], level)[0]
    assert r.tolist() == [1, 3, 11, 3, 12]  # idx 2 ties with the best and becomes second best
    r = O.hamming_best2(q, train, [0, 2], [0, 1], level)[0]
    assert r.tolist() == [1, 3, 11, 5, 10]  # idx 0 was best, then demoted with its level
    r = O.hamming_best2(q, train, [0, 2], [1, 0], level)[0]
    assert r.tolist() == [1, 3, 11, 5, 10]
    assert O.hamming_best2(q, train, [0, 0], [], level)[0].tolist() == [-1, 256, -1, 256, -1]
