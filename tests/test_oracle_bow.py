"""CPU: oracle/bow_oracle.py against independent formulations on seeded cases -- the descent and BowVector as whole-array numpy, and
SearchByBoW as one independent claim chain per common node (the decomposition the device runs) -- plus the parser's blank-line
rule and the decision boundaries of the ratio test, TH_LOW and the rotation bin."""
import math

import numpy as np
import pytest

from oracle import bow_oracle as B
from oracle import bow_scene as S
from oracle.track_oracle import compute_three_maxima


def _descend_all(tree: B.Tree, descs, levelsup):
    """Every feature at once: per level, the argmin over each current node's children (np.argmin keeps the first minimum)."""
    n = len(descs)
    bits = np.unpackbits(descs, axis=1).astype(np.int16)
    cur = np.zeros(n, np.int64)
    nid = np.full(n, -1, np.int64)
    nid_level = tree.L - levelsup
    if nid_level <= 0:
        nid[:] = 0
    done = np.zeros(n, bool)
    level = 0
    while not done.all():
        level += 1
        for i in np.nonzero(~done)[0]:
            ch = tree.children[cur[i]]
            d = np.abs(np.unpackbits(tree.desc[ch], axis=1).astype(np.int16) - bits[i]).sum(axis=1)
            cur[i] = ch[int(np.argmin(d))]
            if level == nid_level:
                nid[i] = cur[i]
            if not tree.children[cur[i]]:
                done[i] = True
    nid[nid < 0] = cur[nid < 0]
    return cur, nid


def _bow_numpy(tree: B.Tree, descs, levelsup):
    leafs, nid = _descend_all(tree, descs, levelsup)
    words = tree.word[leafs]
    w = tree.word_weight[words]
    keep = w > 0
    uw = np.unique(words[keep])
    tf = tree.weighting in (B.TF, B.TF_IDF)
    vals = []
    for u in uw:
        c = int((words[keep] == u).sum())
        x = tree.word_weight[u]
        s = x
        for _ in range(c - 1 if tf else 0):
            s += x
        vals.append(s)
    vals = np.array(vals, np.float64)
    must, norm = B.must_normalize(tree.scoring)
    if tf and len(vals) and not must:
        vals = vals / float(len(vals))
    if must:
        if norm == "L1":
            s = 0.0
            for v in vals:
                s += abs(v)
        else:
            s = 0.0
            for v in vals:
                s += v * v
            s = math.sqrt(s)
        if s > 0:
            vals = vals / s
    node = np.where(keep, nid, -1).astype(np.int32)
    word = np.where(keep, words, -1).astype(np.int32)
    return uw.astype(np.int32), vals, node, word


@pytest.mark.parametrize("seed", range(6))
def test_transform_equals_whole_array_form(seed):
    rng = np.random.default_rng(seed)
    descs = S.synthetic_descriptors(seed, 300)
    for sc in range(6):
        for wt in range(4):
            tree = B.Tree(S.irregular_tree(seed * 31 + sc, keys=descs, n_ties=20, scoring=sc, weighting=wt) if (sc + wt) % 3 == 0
                          else S.small_tree(seed * 7 + sc * 4 + wt, scoring=sc, weighting=wt))
            for levelsup in (0, 1, 4, tree.L, tree.L + 1, int(rng.integers(0, 8))):
                bow, fv, node, word = B.transform(tree, descs, levelsup)
                words, vals = B.bow_arrays(bow)
                uw, v2, node2, word2 = _bow_numpy(tree, descs, levelsup)
                np.testing.assert_array_equal(words, uw)
                np.testing.assert_array_equal(vals.view(np.uint64), v2.view(np.uint64))
                np.testing.assert_array_equal(node, node2)
                np.testing.assert_array_equal(word, word2)
                assert sorted(fv) == sorted(set(node[node >= 0].tolist()))
                for nd, idx in fv.items():
                    assert idx == sorted(np.nonzero(node == nd)[0].tolist())


def test_leaf_above_nid_level_records_the_leaf():
    # root -> (leaf 1, inner 2 -> leaves 3, 4); a key nearest leaf 1 ends at depth 1 < nid_level = 2
    d = np.zeros((5, 32), np.uint8)
    d[2] = 0xFF
    d[3], d[4] = 0xF0, 0xFF
    tree = B.Tree(dict(k=2, L=3, scoring=0, weighting=0, parent=np.array([-1, 0, 0, 2, 2]), is_leaf=np.array([0, 1, 0, 1, 1]), desc=d,
                       weight=np.array([0, 1.0, 0, 2.0, 3.0])))
    assert tree.descend(np.zeros(32, np.uint8), 1) == (0, 1.0, 1)
    assert tree.descend(np.full(32, 0xFF, np.uint8), 2) == (2, 3.0, 2)
    assert tree.descend(np.full(32, 0xFF, np.uint8), 1) == (2, 3.0, 4)
    assert tree.descend(np.full(32, 0xFF, np.uint8), 0) == (2, 3.0, 4)
    assert tree.descend(np.full(32, 0xFF, np.uint8), 3)[2] == 0


def _search_by_node(f, kf, nnratio, check):
    """Independent form: one claim chain per common node, in any node order, then the histogram."""
    fv_f = B.feature_vector(f["node"], f["kps"]["angle"])
    fv_kf = B.feature_vector(kf["node"], kf["kps"]["angle"])
    match = np.full(len(f["kps"]), -1, np.int32)
    bins = {}
    for nd in sorted(set(fv_f) & set(fv_kf), reverse=True):
        cand = fv_f[nd]
        for i in fv_kf[nd]:
            if kf["point"][i] < 0:
                continue
            ds = [(B.descriptor_distance(kf["desc"][i], f["desc"][j]), j) for j in cand if match[j] < 0]
            b1, bi, b2 = 256, -1, 256
            for d, j in ds:
                if d < b1:
                    b2, b1, bi = b1, d, j
                elif d < b2:
                    b2 = d
            if b1 <= B.TH_LOW and np.float32(b1) < np.float32(nnratio) * np.float32(b2):
                match[bi] = kf["point"][i]
                bins[bi] = B.rotation_bin(kf["kps"]["angle"][i], f["kps"]["angle"][bi])
    if check:
        counts = [0] * 30
        for b in bins.values():
            counts[b] += 1
        keep = compute_three_maxima(counts)
        for j, b in bins.items():
            if b not in keep:
                match[j] = -1
    return match, int((match >= 0).sum())


@pytest.mark.parametrize("seed", range(10))
def test_search_by_bow_equals_the_per_node_form(seed):
    rng = np.random.default_rng(100 + seed)
    for case in range(200):
        n = int(rng.integers(0, 60))
        f, kfs = S.search_scene(seed * 1000 + case, n_frame=n, n_kfs=1, n_nodes=int(rng.integers(1, 8)),
                                angle_spread=float(rng.choice([2.0, 60.0])))
        kf = kfs[0]
        if rng.uniform() < 0.2 and len(f["kps"]):
            f["kps"]["angle"][rng.integers(len(f["kps"]))] = np.float32(rng.choice([np.nan, -1.0, 400.0]))
        ratio, check = float(rng.choice([0.6, 0.7, 0.75, 0.9])), bool(rng.integers(2))
        m, nm = B.search_by_bow(f["kps"], f["desc"], f["node"], kf["kps"], kf["desc"], kf["node"], kf["point"], ratio, check)
        m2, nm2 = _search_by_node(f, kf, ratio, check)
        np.testing.assert_array_equal(m, m2)
        assert nm == nm2


def test_blank_line_rule():
    tree = S.small_tree(3)
    body = B.to_text(tree, trailing="")
    want = B.parse_text(body + "\n")
    for tail in ("", "\n", "\n\n", "\n \t\n", "\n\r\n"):
        got = B.parse_text(body + tail)
        assert len(got["parent"]) == len(want["parent"]) == len(tree["parent"])
        np.testing.assert_array_equal(got["desc"], tree["desc"])
        np.testing.assert_array_equal(got["weight"], tree["weight"])
    lines = body.split("\n")
    with pytest.raises(B.FormatError):
        B.parse_text("\n".join(lines[:5] + [""] + lines[5:]) + "\n")


def _one_node(d_kf, d_f, ratio, check=False, kf_angle=0.0, f_angle=0.0):
    f = dict(kps=S.keys(np.random.default_rng(0), len(d_f), np.full(len(d_f), f_angle, np.float32)), desc=np.array(d_f, np.uint8),
             node=np.zeros(len(d_f), np.int32))
    kf = dict(kps=S.keys(np.random.default_rng(1), 1, np.full(1, kf_angle, np.float32)), desc=np.array([d_kf], np.uint8),
              node=np.zeros(1, np.int32), point=np.array([5], np.int32))
    return B.search_by_bow(f["kps"], f["desc"], f["node"], kf["kps"], kf["desc"], kf["node"], kf["point"], ratio, check)


def _at(base, bits):
    m = np.zeros(256, np.uint8)
    m[:bits] = 1
    return base ^ np.packbits(m)


@pytest.mark.parametrize("ratio,d1,d2,accept", [(0.7, 7, 10, False), (0.7, 6, 10, True), (0.7, 7, 11, True), (0.7, 8, 10, False),
                                                (0.75, 15, 20, False), (0.75, 14, 20, True), (0.75, 15, 21, True), (0.75, 16, 20, False)])
def test_ratio_test_in_float_at_exact_equality(ratio, d1, d2, accept):
    assert np.float32(0.7) * np.float32(10) == np.float32(7) and np.float32(0.75) * np.float32(20) == np.float32(15)
    z = np.zeros(32, np.uint8)
    m, nm = _one_node(z, [_at(z, d1), np.bitwise_not(_at(np.full(32, 0xFF, np.uint8), d2))], ratio)
    assert nm == (1 if accept else 0)


@pytest.mark.parametrize("d,accept", [(50, True), (51, False)])
def test_th_low(d, accept):
    z = np.zeros(32, np.uint8)
    m, nm = _one_node(z, [_at(z, d)], 0.9)
    assert nm == (1 if accept else 0) and (m[0] == 5) == accept


def test_rotation_bin_half_rounds_away():
    # 45 / 30 = 1.5 in float: round half away -> 2; 15 / 30 = 0.5 -> 1; 345 / 30 = 11.5 -> 12
    assert B.rotation_bin(np.float32(45), np.float32(0)) == 2
    assert B.rotation_bin(np.float32(15), np.float32(0)) == 1
    assert B.rotation_bin(np.float32(0), np.float32(15)) == 12
    assert B.rotation_bin(np.float32(360), np.float32(0)) == 12


# ---------------------------------------------------------------------------------------------------------- constructed cases
TRANSFORM_CASES = S.transform_cases()
SEARCH_CASES = S.search_cases()


@pytest.mark.parametrize("case", TRANSFORM_CASES, ids=lambda c: c.name)
def test_transform_case_reaches_its_paths(case):
    got = S.transform_paths(case)
    assert case.paths <= got, sorted(case.paths - got)
    assert got <= set(S.PATHS), sorted(got - set(S.PATHS))
    # the trace changes nothing
    tree = B.Tree(case.tree)
    plain = B.transform(tree, case.desc, case.levelsup)
    traced = B.transform(tree, case.desc, case.levelsup, trace=set())
    w0, v0 = B.bow_arrays(plain[0])
    w1, v1 = B.bow_arrays(traced[0])
    np.testing.assert_array_equal(w0, w1)
    np.testing.assert_array_equal(v0.view(np.uint64), v1.view(np.uint64))
    np.testing.assert_array_equal(plain[2], traced[2])


@pytest.mark.parametrize("case", SEARCH_CASES, ids=lambda c: c.name)
def test_search_case_reaches_its_paths(case):
    got = S.search_paths(case)
    assert case.paths <= got, sorted(case.paths - got)
    assert got <= set(S.PATHS), sorted(got - set(S.PATHS))
    f = case.frame
    for kf in S._live(case):
        args = (f["kps"], f["desc"], f["node"], kf["kps"], kf["desc"], kf["node"], kf["point"], case.ratio, case.check)
        m0, n0 = B.search_by_bow(*args)
        m1, n1 = B.search_by_bow(*args, trace=set())
        np.testing.assert_array_equal(m0, m1)
        assert n0 == n1


def test_the_cases_reach_every_path():
    reached = set()
    for c in TRANSFORM_CASES:
        reached |= S.transform_paths(c)
    for c in SEARCH_CASES:
        reached |= S.search_paths(c)
    assert len(set(S.PATHS)) == len(S.PATHS)
    assert set(S.PATHS) - reached == set(S.UNREACHED), sorted(set(S.PATHS) - reached)


def test_the_unreached_bin_needs_an_angle_outside_the_rule():
    # every float rot the rule allows: [0, 360] after the wrap; the largest gives bin 12
    assert B.rotation_bin(np.float32(360), np.float32(0)) == 12
    assert B.rotation_bin(np.float32(0), np.float32(np.nextafter(np.float32(0), np.float32(1)))) == 12
    t = set()
    assert B.rotation_bin(np.float32(900), np.float32(0), t) == 0 and "bin_30_to_0" in t  # 900 breaks the angle rule


def test_the_fuzz_cases_agree_with_the_per_node_form():
    for seed in range(0, 200, 5):
        c = S.fuzz_case(seed)
        for kf in S._live(c):
            m, nm = B.search_by_bow(c.frame["kps"], c.frame["desc"], c.frame["node"], kf["kps"], kf["desc"], kf["node"], kf["point"],
                                    c.ratio, c.check)
            m2, nm2 = _search_by_node(c.frame, kf, c.ratio, c.check)
            np.testing.assert_array_equal(m, m2)
            assert nm == nm2
