"""-m gpu: the bag of words -- sivo_compute_bow[_device] and sivo_search_by_bow[_device] -- bit for bit against
oracle/bow_oracle.py on seeded vocabularies (oracle/bow_scene.py): the full-shape tree, the irregular tree and a small tree per
weighting x scoring pair, the fixture's ORB descriptors and synthetic frames; the search on seeded scenes, constructed worst cases
and a differential fuzz."""
import numpy as np
import pytest
import torch

from frame_support import extractors, upload
from oracle import bow_oracle as B
from oracle import bow_scene as S
from oracle.keymap import keymap
from sivo_b200 import _lib as L
from sivo_b200.bow import Vocabulary, compute_bow, compute_bow_device, keyframe_keys, search_by_bow, search_by_bow_device
from sivo_b200.orb import KP_DTYPE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ext():
    return extractors(2000)


@pytest.fixture(scope="module")
def full():
    t = S.full_shape_tree(0)
    return B.Tree(t), Vocabulary.from_arrays(t["k"], t["L"], t["scoring"], t["weighting"], t["parent"], t["is_leaf"], t["desc"], t["weight"])


@pytest.fixture(scope="module")
def irregular():
    t = S.irregular_tree(1, keys=S.fixture_descriptors(), n_ties=200)
    return B.Tree(t), Vocabulary.from_arrays(t["k"], t["L"], t["scoring"], t["weighting"], t["parent"], t["is_leaf"], t["desc"], t["weight"])


def frames():
    return [("kitti", S.fixture_descriptors())] + [(f"synth{s}", S.synthetic_descriptors(s, 1800)) for s in (1, 2, 3)]


def device_bow(voc, el, desc, levelsup, keep=None, count=None):
    """Runs the device form on a capacity-sized copy; returns the per-key and BowVector outputs on the host."""
    cap = el.capacity()
    n = len(desc)
    buf = np.zeros((cap, 32), np.uint8)
    buf[:min(n, cap)] = desc[:cap]
    d = upload(buf)
    nk = upload(np.array([n if count is None else count], np.int64))
    kp = upload(np.asarray(keep, np.int32)) if keep is not None else None
    out = dict(node=torch.full((cap,), -7, dtype=torch.int32, device="cuda"), word=torch.full((cap,), -7, dtype=torch.int32, device="cuda"),
               bw=torch.full((cap,), -7, dtype=torch.int32, device="cuda"), bwt=torch.full((cap,), 7.0, dtype=torch.float64, device="cuda"),
               len=torch.full((1,), -7, dtype=torch.int64, device="cuda"))
    torch.cuda.synchronize()
    compute_bow_device(voc, el, d.data_ptr(), 0 if kp is None else kp.data_ptr(), nk.data_ptr(), levelsup, out["node"].data_ptr(),
                       out["word"].data_ptr(), out["bw"].data_ptr(), out["bwt"].data_ptr(), out["len"].data_ptr())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def check_three_ways(tree, voc, el, desc, levelsup):
    bow, fv, node, word = B.transform(tree, desc, levelsup)
    words, vals = B.bow_arrays(bow)
    h = compute_bow(voc, desc, levelsup)
    np.testing.assert_array_equal(h["node"], node)
    np.testing.assert_array_equal(h["word"], word)
    np.testing.assert_array_equal(h["bow_words"], words)
    np.testing.assert_array_equal(h["bow_weights"].view(np.uint64), vals.view(np.uint64))
    d = device_bow(voc, el, desc, levelsup)
    n = len(desc)
    assert int(d["len"][0]) == len(words)
    np.testing.assert_array_equal(d["node"][:n], node)
    np.testing.assert_array_equal(d["word"][:n], word)
    np.testing.assert_array_equal(d["bw"][:len(words)], words)
    np.testing.assert_array_equal(d["bwt"][:len(words)].view(np.uint64), vals.view(np.uint64))
    return node, words


@pytest.mark.parametrize("which", ["full", "irregular"])
def test_transform_three_ways(request, ext, which):
    tree, voc = request.getfixturevalue(which)
    el = ext[0]
    info = voc.info()
    assert info["nodes"] == len(tree.children) and info["words"] == tree.n_words and info["L"] == 6
    for name, desc in frames():
        for levelsup in (0, 1, 4, tree.L, tree.L + 1):
            node, words = check_three_ways(tree, voc, el, desc, levelsup)
            assert len(words) > 10
            if which == "full" and levelsup == 4:
                assert 20 <= len(np.unique(node[node >= 0])) <= 100  # keys spread over the level-2 nodes


def test_every_weighting_and_scoring(ext):
    el = ext[0]
    desc = S.synthetic_descriptors(7, 900)
    for sc in range(6):
        for wt in range(4):
            t = S.small_tree(40 + 4 * sc + wt, scoring=sc, weighting=wt)
            voc = Vocabulary.from_arrays(t["k"], t["L"], sc, wt, t["parent"], t["is_leaf"], t["desc"], t["weight"])
            for levelsup in (0, 1, 2):
                check_three_ways(B.Tree(t), voc, el, desc, levelsup)
            voc.close()


def test_transform_edges_and_errors(ext, irregular):
    tree, voc = irregular
    el = ext[0]
    cap = el.capacity()
    desc = S.synthetic_descriptors(11, cap)
    bow, _, node, word = B.transform(tree, desc, 4)
    words, vals = B.bow_arrays(bow)
    full = device_bow(voc, el, desc, 4)  # count = capacity
    np.testing.assert_array_equal(full["node"], node)
    np.testing.assert_array_equal(full["bwt"][:len(words)].view(np.uint64), vals.view(np.uint64))
    again = device_bow(voc, el, desc, 4)  # run to run
    for k in full:
        np.testing.assert_array_equal(full[k].view(np.uint8), again[k].view(np.uint8))
    above = device_bow(voc, el, desc, 4, count=cap + 500)  # clamped
    np.testing.assert_array_equal(above["node"], node)
    zero = device_bow(voc, el, desc, 4, count=0)
    assert int(zero["len"][0]) == 0 and (zero["node"] == -7).all()
    neg = device_bow(voc, el, desc, 4, count=-1)
    assert int(neg["len"][0]) == -1 and (neg["node"] == -7).all() and (neg["bwt"] == 7.0).all()
    # keep_idx: negative and out-of-capacity entries give -1, the rest take the extractor key
    km = keymap(600, cap, np.random.default_rng(3), duplicates=True)
    n = km.n_keep
    keep = km.keep[:n]
    k = device_bow(voc, el, desc, 4, keep=km.keep, count=n)
    valid = km.src >= 0
    b2, _, node2, word2 = B.transform(tree, desc[np.where(valid, keep, 0)], 4)
    np.testing.assert_array_equal(k["node"][:n], np.where(valid, node2, -1))
    np.testing.assert_array_equal(k["word"][:n], np.where(valid, word2, -1))
    sel = [i for i in range(n) if valid[i]]
    bsel, _, _, _ = B.transform(tree, desc[keep[sel]], 4)
    w3, v3 = B.bow_arrays(bsel)
    np.testing.assert_array_equal(k["bw"][:len(w3)], w3)
    np.testing.assert_array_equal(k["bwt"][:len(w3)].view(np.uint64), v3.view(np.uint64))
    h = compute_bow(voc, np.zeros((0, 32), np.uint8), 4)
    assert len(h["bow_words"]) == 0
    with pytest.raises(L.SivoError) as e:
        compute_bow(voc, desc[:10], -1)
    assert e.value.code == L.EINVAL
    with pytest.raises(L.SivoError) as e:
        compute_bow(voc, np.zeros((16385, 32), np.uint8), 4)
    assert e.value.code == L.ERANGE
    with pytest.raises(L.SivoError) as e:
        compute_bow_device(voc, el, 0, 0, 0, 4)
    assert e.value.code == L.EINVAL


# ---------------------------------------------------------------------------------------------------------- SearchByBoW
def oracle_batch(f, kfs, ratio, check):
    out = [B.search_by_bow(f["kps"], f["desc"], f["node"], kf["kps"], kf["desc"], kf["node"], kf["point"], ratio, check) for kf in kfs]
    return np.array([m for m, _ in out], np.int32).reshape(len(kfs), -1), np.array([c for _, c in out], np.int64)


def device_search(el, f, kfs, ratio, check, counts=None):
    """The device form with every array at the extractor's capacity (frame keys gathered: keep_idx NULL)."""
    cap = el.capacity()

    def pad(a, dt, fill=0):
        a = np.ascontiguousarray(a)
        out = np.full((cap,) + a.shape[1:], fill, dt) if a.dtype.names is None else np.zeros(cap, a.dtype)
        out[:len(a)] = a
        return upload(out)

    hold = [pad(f["kps"], KP_DTYPE), pad(f["desc"], np.uint8), pad(f["node"], np.int32, -1), upload(np.array([len(f["kps"])], np.int64))]
    keys, pts = [], []
    for i, kf in enumerate(kfs):
        c = len(kf["kps"]) if counts is None else counts[i]
        a = [pad(kf["kps"], KP_DTYPE), pad(kf["desc"], np.uint8), pad(kf["node"], np.int32, -1), pad(kf["point"], np.int32, -1),
             upload(np.array([c], np.int64))]
        hold += a
        keys.append(keyframe_keys(a[0].data_ptr(), a[1].data_ptr(), a[2].data_ptr(), a[4].data_ptr()))
        pts.append(a[3].data_ptr())
    match = torch.full((max(len(kfs), 1), cap), -7, dtype=torch.int32, device="cuda")
    nm = torch.full((max(len(kfs), 1),), -7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    search_by_bow_device(el, hold[0].data_ptr(), hold[1].data_ptr(), 0, hold[3].data_ptr(), hold[2].data_ptr(), keys, pts, ratio, check,
                         match.data_ptr(), nm.data_ptr())
    torch.cuda.synchronize()
    return match.cpu().numpy()[:len(kfs)], nm.cpu().numpy()[:len(kfs)]


def check_search(el, f, kfs, ratio, check, device=True):
    want_m, want_n = oracle_batch(f, kfs, ratio, check)
    m, nm = search_by_bow(el, f["kps"], f["desc"], f["node"], kfs, ratio, check)
    np.testing.assert_array_equal(m, want_m)
    np.testing.assert_array_equal(nm, want_n)
    if device:
        n = len(f["kps"])
        dm, dn = device_search(el, f, kfs, ratio, check)
        np.testing.assert_array_equal(dm[:, :n], want_m)
        assert (dm[:, n:] == -1).all()
        np.testing.assert_array_equal(dn, want_n)
    return want_n


@pytest.mark.parametrize("ratio", [0.7, 0.75])
@pytest.mark.parametrize("check", [True, False])
@pytest.mark.parametrize("n_kf", [1, 8, 64])
def test_search_batches(ext, ratio, check, n_kf):
    el = ext[0]
    rng = np.random.default_rng(n_kf)
    f, kfs = S.search_scene(n_kf * 10 + int(check), n_frame=1500, n_kfs=n_kf, n_nodes=80,
                            kf_sizes=rng.integers(100, 1500, n_kf) if n_kf > 1 else None, angle_spread=25.0)
    got = check_search(el, f, kfs, ratio, check)
    assert got.sum() > 20 * n_kf


def test_search_crowded_node_and_capacity(ext):
    el = ext[0]
    cap = el.capacity()
    f, kfs = S.crowd_scene(5, 500)
    for ratio in (0.7, 0.75, 0.95):
        for check in (True, False):
            n = check_search(el, f, kfs, ratio, check)
            assert n[0] > 30
    f, kfs = S.search_scene(9, n_frame=cap, n_kfs=2, n_nodes=100, kf_sizes=[cap, cap])  # counts equal to the capacity
    check_search(el, f, kfs, 0.75, True)


def _ties_scene():
    rng = np.random.default_rng(21)
    z = np.zeros(32, np.uint8)
    f_desc = np.array([S.near(rng, z, b) for b in (5, 5, 9, 9, 7, 7, 30, 31)], np.uint8)
    f = dict(kps=S.keys(rng, 8, np.full(8, 100.0, np.float32)), desc=f_desc, node=np.array([3, 3, 3, 3, 4, 4, 5, -1], np.int32))
    kf_desc = np.array([z, z, z, z, z, S.near(rng, z, 1), z], np.uint8)
    kf = dict(kps=S.keys(rng, 7, np.array([100, 100, 101, 100, 250, 100, 100], np.float32)), desc=kf_desc,
              node=np.array([3, 3, 3, 4, 4, 5, -1], np.int32), point=np.array([10, -1, 11, 12, 13, 14, 15], np.int32))
    return f, [kf]


def test_search_constructed_cases(ext):
    el = ext[0]
    f, kfs = _ties_scene()
    for ratio in (0.7, 0.75, 1.0):
        for check in (True, False):
            check_search(el, f, kfs, ratio, check)
    # the 0.1 rule: 10 matches in one bin, 1 in another -> the lone bin is culled (1 < 0.1 * 10 is false: kept); 11 vs 1 culls
    rng = np.random.default_rng(2)
    for big in (10, 11):
        n = big + 1
        f_desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        f = dict(kps=S.keys(rng, n, np.zeros(n, np.float32)), desc=f_desc, node=np.arange(n, dtype=np.int32))
        ang = np.zeros(n, np.float32)
        ang[-1] = 200.0
        kf = dict(kps=S.keys(rng, n, ang), desc=f_desc.copy(), node=np.arange(n, dtype=np.int32), point=np.arange(n, dtype=np.int32))
        got = check_search(el, f, [kf], 0.7, True)
        assert got[0] == (n if big == 10 else big)
    # angle-rule violations: refused by the host form, left out by the device form (the oracle's rule)
    f, kfs = S.search_scene(4, n_frame=300, n_kfs=1, n_nodes=10)
    f["kps"]["angle"][5] = np.nan
    kfs[0]["kps"]["angle"][7] = 361.0
    with pytest.raises(L.SivoError) as e:
        search_by_bow(el, f["kps"], f["desc"], f["node"], kfs, 0.7, True)
    assert e.value.code == L.ERANGE
    want_m, want_n = oracle_batch(f, kfs, 0.7, True)
    dm, dn = device_search(el, f, kfs, 0.7, True)
    np.testing.assert_array_equal(dm[:, :300], want_m)
    np.testing.assert_array_equal(dn, want_n)
    # negative counts: only n_matches = -1 for the affected keyframes
    f, kfs = S.search_scene(6, n_frame=300, n_kfs=3, n_nodes=10)
    dm, dn = device_search(el, f, kfs, 0.7, True, counts=[len(kfs[0]["kps"]), -1, len(kfs[2]["kps"])])
    assert dn[1] == -1 and (dm[1] == -7).all() and dn[0] >= 0 and dn[2] >= 0
    m, nm = search_by_bow(el, f["kps"], f["desc"], f["node"], [dict(kfs[0]), dict(kfs[1], count=-1)], 0.7, True)
    assert nm[1] == -1 and nm[0] == oracle_batch(f, kfs[:1], 0.7, True)[1][0]
    for bad in (float("nan"), float("inf")):
        with pytest.raises(L.SivoError) as e:
            search_by_bow(el, f["kps"], f["desc"], f["node"], kfs, bad, True)
        assert e.value.code == L.EINVAL


def test_search_fuzz(ext):
    el = ext[0]
    rng = np.random.default_rng(77)
    for case in range(200):
        n = int(rng.integers(0, 400))
        f, kfs = S.search_scene(5000 + case, n_frame=n, n_kfs=int(rng.integers(1, 4)), n_nodes=int(rng.integers(1, 30)),
                                angle_spread=float(rng.choice([3.0, 40.0, 180.0])))
        check_search(el, f, kfs, float(rng.choice([0.6, 0.7, 0.75, 0.9])), bool(rng.integers(2)), device=case % 10 == 0)
