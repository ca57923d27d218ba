"""Seeded vocabularies and SearchByBoW scenes for the bag-of-words tests and tools (no vocabulary file is committed).

- full_shape_tree: k = 10, L = 6, about 1.08 M nodes in ORBvoc's layout (each node's children consecutive, parents before
  children).  Level-1 descriptors are drawn from the committed fixture's ORB descriptors (tests/golden/orb_kitti_2000.npz); each
  child is its parent with bits flipped at a per-level rate, so real keys spread over the level-2 nodes.  About 9 % of the words
  have weight 0 (stopped), as in ORBvoc.
- irregular_tree: 2-10 children, leaves at every depth (above nid_level included), nodes in depth-first order (children not
  consecutive), and sibling descriptors at exactly equal distance from chosen keys.
- small_tree: a few hundred nodes for one weighting x scoring pair.
- search_scene: a frame and keyframes whose keys share vocabulary nodes, with crowds, claim chains and ties.
- transform_cases / search_cases: constructed worst cases, each naming the paths it must reach (see below), and fuzz_case.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field

import numpy as np

from oracle import bow_oracle as B
from oracle.track_oracle import angle_ok
from sivo_b200.orb import KP_DTYPE

GOLDEN = os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "orb_kitti_2000.npz")


def fixture_descriptors() -> np.ndarray:
    return np.load(GOLDEN)["descriptors"]


def _flip(rng, desc, and_count):
    """desc with each bit flipped with probability 2^-and_count (the AND of and_count random bytes)."""
    m = rng.integers(0, 256, desc.shape, dtype=np.uint8)
    for _ in range(and_count - 1):
        m &= rng.integers(0, 256, desc.shape, dtype=np.uint8)
    return desc ^ m


def _weights(rng, n, zero_frac=0.09):
    w = rng.uniform(0.5, 9.0, n)
    w[rng.uniform(size=n) < zero_frac] = 0.0
    return w


def full_shape_tree(seed=0, scoring=0, weighting=0) -> dict:
    """Breadth-first: level d's nodes follow level d-1's, each parent's children consecutive.  3 % of the depth-5 nodes are leaves."""
    rng = np.random.default_rng(seed)
    base = fixture_descriptors()
    k, L = 10, 6
    parent, leaf, desc = [np.array([-1], np.int32)], [np.array([0], np.uint8)], [np.zeros((1, 32), np.uint8)]
    level = base[rng.choice(len(base), k, replace=False)].copy()
    parent.append(np.zeros(k, np.int32))
    ids = np.arange(1, k + 1)
    leaf_l = np.zeros(k, np.uint8)
    next_id = k + 1
    rates = {2: 2, 3: 3, 4: 4, 5: 4, 6: 5}
    for depth in range(2, L + 1):
        leaf.append(leaf_l)
        desc.append(level)
        inner = ids[leaf_l == 0]
        inner_desc = level[leaf_l == 0]
        child_desc = _flip(rng, np.repeat(inner_desc, k, axis=0), rates[depth])
        parent.append(np.repeat(inner, k).astype(np.int32))
        ids = np.arange(next_id, next_id + len(child_desc))
        next_id += len(child_desc)
        level = child_desc
        if depth == L:
            leaf_l = np.ones(len(ids), np.uint8)
        elif depth == L - 1:
            leaf_l = (rng.uniform(size=len(ids)) < 0.03).astype(np.uint8)
        else:
            leaf_l = np.zeros(len(ids), np.uint8)
    leaf.append(leaf_l)
    desc.append(level)
    parent = np.concatenate(parent)
    is_leaf = np.concatenate(leaf)
    return dict(k=k, L=L, scoring=scoring, weighting=weighting, parent=parent, is_leaf=is_leaf, desc=np.concatenate(desc),
                weight=np.where(is_leaf == 1, _weights(rng, len(parent)), 0.0))


def _dfs_tree(rng, L, min_children, max_children, leaf_prob, root_desc_pool):
    """Depth-first ids: a node's children are not consecutive when they have subtrees."""
    parent, leaf, desc = [-1], [0], [np.zeros(32, np.uint8)]

    def grow(pid, pdesc, depth):
        nch = int(rng.integers(min_children, max_children + 1))
        for _ in range(nch):
            d = root_desc_pool[rng.integers(len(root_desc_pool))] if depth == 1 else _flip(rng, pdesc, int(rng.integers(2, 5)))
            cid = len(parent)
            parent.append(pid)
            desc.append(d)
            is_leaf = depth >= L or rng.uniform() < leaf_prob(depth)
            leaf.append(1 if is_leaf else 0)
            if not is_leaf:
                grow(cid, d, depth + 1)

    grow(0, None, 1)
    return np.array(parent, np.int32), np.array(leaf, np.uint8), np.array(desc, np.uint8)


def irregular_tree(seed=0, keys=None, n_ties=40, scoring=0, weighting=0) -> dict:
    """L = 6, 2-10 children, leaves at depths 1..6.  For n_ties of `keys`, two siblings on the key's path get descriptors at the same
    (smallest) distance from it, so the descent meets an exact tie there."""
    rng = np.random.default_rng(seed)
    pool = fixture_descriptors() if keys is None else keys
    leaf_prob = lambda depth: {1: 0.1, 2: 0.15, 3: 0.2, 4: 0.3, 5: 0.4}.get(depth, 1.0)  # noqa: E731
    while True:
        parent, is_leaf, desc = _dfs_tree(rng, 6, 2, 5, leaf_prob, pool)
        if 200 < len(parent) < 20000 and is_leaf[1:][parent[1:] == 0].any():
            break
    t = dict(k=10, L=6, scoring=scoring, weighting=weighting, parent=parent, is_leaf=is_leaf, desc=desc,
             weight=np.where(is_leaf == 1, _weights(rng, len(parent)), 0.0))
    if keys is not None:
        children = [[] for _ in range(len(parent))]
        for i in range(1, len(parent)):
            children[parent[i]].append(i)
        for q in keys[rng.choice(len(keys), min(n_ties, len(keys)), replace=False)]:
            node = 0
            for _ in range(int(rng.integers(0, 4))):  # the tie at a random level of the key's path
                ch = [c for c in children[node] if children[c]]
                if not ch:
                    break
                node = ch[int(rng.integers(len(ch)))]
            ch = children[node]
            if len(ch) < 2:
                continue
            a, b = rng.choice(len(ch), 2, replace=False)
            bits = rng.choice(256, 6, replace=False)
            for c, sel in ((ch[a], bits[:3]), (ch[b], bits[3:])):
                m = np.zeros(256, np.uint8)
                m[sel] = 1
                desc[c] = q ^ np.packbits(m)
    return t


def small_tree(seed=0, scoring=0, weighting=0, k=4, L=3) -> dict:
    rng = np.random.default_rng(seed)
    parent, is_leaf, desc = _dfs_tree(rng, L, 2, k, lambda d: 0.15, fixture_descriptors())
    return dict(k=k, L=L, scoring=scoring, weighting=weighting, parent=parent, is_leaf=is_leaf, desc=desc,
                weight=np.where(is_leaf == 1, _weights(rng, len(parent), 0.15), 0.0))


def synthetic_descriptors(seed, n=1500) -> np.ndarray:
    """Frame-like keys: fixture descriptors with 0-24 bits flipped, plus a tenth drawn uniformly."""
    rng = np.random.default_rng(seed)
    base = fixture_descriptors()
    d = base[rng.integers(len(base), size=n)].copy()
    for i in range(n):
        bits = rng.choice(256, int(rng.integers(0, 25)), replace=False)
        m = np.zeros(256, np.uint8)
        m[bits] = 1
        d[i] ^= np.packbits(m)
    rnd = rng.uniform(size=n) < 0.1
    d[rnd] = rng.integers(0, 256, (rnd.sum(), 32), dtype=np.uint8)
    return d


# ------------------------------------------------------------------------------------------------------------------ search scenes
def keys(rng, n, angles=None) -> np.ndarray:
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.uniform(0, 1000, n)
    k["y"] = rng.uniform(0, 370, n)
    k["size"] = 31
    k["angle"] = rng.uniform(0, 360, n) if angles is None else angles
    k["octave"] = rng.integers(0, 8, n)
    return k


def near(rng, d, bits):
    m = np.zeros(256, np.uint8)
    m[rng.choice(256, bits, replace=False)] = 1
    return d ^ np.packbits(m)


def search_scene(seed, n_frame=800, n_kfs=1, n_nodes=60, kf_sizes=None, point_frac=0.7, angle_spread=20.0):
    """A frame and n_kfs keyframes over n_nodes shared nodes.  Keyframe keys are frame keys with 0-40 bits flipped (so the ratio
    test passes and fails), rotated by a common angle plus noise (so the histogram keeps most); some keys have node -1, some
    keyframe keys no point.  Returns (frame dict(kps, desc, node), [keyframe dict(kps, desc, node, point)])."""
    rng = np.random.default_rng(seed)
    node_ids = np.sort(rng.choice(1_000_000, n_nodes, replace=False)).astype(np.int32)
    f_desc = rng.integers(0, 256, (n_frame, 32), dtype=np.uint8)
    f_node = node_ids[rng.integers(n_nodes, size=n_frame)]
    f_node[rng.uniform(size=n_frame) < 0.05] = -1
    f_kps = keys(rng, n_frame)
    kfs = []
    for k in range(n_kfs):
        m = int(kf_sizes[k]) if kf_sizes is not None else int(rng.integers(n_frame // 2, n_frame + 1))
        src = rng.integers(n_frame, size=m)
        d = np.array([near(rng, f_desc[s], int(rng.integers(0, 41))) for s in src], np.uint8).reshape(-1, 32)
        node = f_node[src].copy()
        node[rng.uniform(size=m) < 0.05] = -1
        rot = rng.uniform(0, 360)
        ang = (f_kps["angle"][src] + rot + rng.normal(0, angle_spread, m)) % 360.0
        kk = keys(rng, m, ang.astype(np.float32))
        point = np.where(rng.uniform(size=m) < point_frac, rng.integers(0, 5000, m), -1).astype(np.int32)
        kfs.append(dict(kps=kk, desc=d, node=node, point=point))
    return dict(kps=f_kps, desc=f_desc, node=f_node), kfs


def crowd_scene(seed, n=500):
    """One node holding n frame keys and n keyframe keys, each keyframe key near several frame keys: long claim chains."""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (n // 10 + 1, 32), dtype=np.uint8)
    f_desc = np.array([near(rng, base[i % len(base)], int(rng.integers(0, 12))) for i in range(n)], np.uint8)
    kf_desc = np.array([near(rng, base[rng.integers(len(base))], int(rng.integers(0, 12))) for _ in range(n)], np.uint8)
    f_kps = keys(rng, n, np.full(n, 10.0, np.float32))
    kf_kps = keys(rng, n, np.full(n, 40.0, np.float32))
    node = np.full(n, 77, np.int32)
    return dict(kps=f_kps, desc=f_desc, node=node), [dict(kps=kf_kps, desc=kf_desc, node=node.copy(),
                                                          point=np.arange(n, dtype=np.int32))]


# ------------------------------------------------------------------------------------------------------------------ constructed cases
# Each case names the paths it must reach, and transform_paths / search_paths read them back from the oracle's trace and from the
# case's layout, so a test can check both that a case still reaches what it was built for and that the cases together reach every
# path in PATHS.  Distances are placed by flipping chosen bits of a random descriptor (random descriptors are about 128 bits
# apart, so only the placed ones compete).
MAX_KEYS = 16384          # the block sorts' limit: an extractor with nfeatures 16288 (and 8 levels) has this capacity
INT32_MAX = 2**31 - 1
LAYOUT_PATHS = (
    "children_40",          # a node with 40 children: the descent's lanes take two strides
    "keys_cap",             # 16,384 keys: both block sorts at their shared-memory limit
    "run_at_31",            # a frame node's run starts at sorted position 31
    "run_to_n",             # the last run ends exactly at the frame count (the run-end ballot past n)
    "run_33_late_best",     # a run of 33 keys whose match is its 33rd key
    "run_1000_late_best",   # a run of 1,000 keys whose match is in its last 32
    "node_0", "node_int32_max",  # matches in nodes 0 and 2^31 - 1
    "kf_chunks",            # more than 64 keyframes: later launches (base > 0)
)
PATHS = B.DESCENT_PATHS + B.TRANSFORM_PATHS + B.SEARCH_PATHS + LAYOUT_PATHS
# Paths no input reaches, with the reason; the CPU test checks that they are exactly the paths no case reaches.
UNREACHED = {
    "bin_30_to_0": "with both angles in [0, 360] rot is in [0, 360] after the wrap, and 360 * (1.f / 30) rounds to 12: the "
                   "reference's factor makes bins 0..12 only, so bin 30 needs an angle the angle rule excludes",
}


@dataclass
class TransformCase:
    name: str
    tree: dict
    desc: np.ndarray          # n x 32
    levelsup: int
    paths: set = field(default_factory=set)
    junk: bool = True         # embed rejected keep_idx entries between the keys


@dataclass
class SearchCase:
    name: str
    frame: dict               # kps, desc, node
    kfs: list                 # dicts kps, desc, node, point
    ratio: float
    check: bool
    paths: set = field(default_factory=set)
    counts: list = None       # per-keyframe counts (None: the lengths; negative: that keyframe is affected)
    junk: bool = True


def _bits(d, positions):
    """d with the listed bit positions flipped (np.unpackbits order)."""
    m = np.zeros(256, np.uint8)
    m[list(positions)] = 1
    return np.asarray(d, np.uint8) ^ np.packbits(m)


def _rand(rng, n=None):
    return rng.integers(0, 256, 32 if n is None else (n, 32), dtype=np.uint8)


def _tree(parent, is_leaf, desc, weight, L, scoring=0, weighting=0, k=10) -> dict:
    return dict(k=k, L=L, scoring=scoring, weighting=weighting, parent=np.asarray(parent, np.int32),
                is_leaf=np.asarray(is_leaf, np.uint8), desc=np.asarray(desc, np.uint8).reshape(-1, 32),
                weight=np.asarray(weight, np.float64))


def transform_paths(case: TransformCase) -> set:
    tree = B.Tree(case.tree)
    out = set()
    B.transform(tree, case.desc, case.levelsup, trace=out)
    if max(len(c) for c in tree.children) >= 40:
        out.add("children_40")
    if len(case.desc) == MAX_KEYS:
        out.add("keys_cap")
    return out


def _live(case: SearchCase):
    """The keyframes the search runs (count >= 0) with their arrays cut to the count."""
    out = []
    for i, kf in enumerate(case.kfs):
        c = len(kf["kps"]) if case.counts is None else case.counts[i]
        if c >= 0:
            out.append({k: v[:c] for k, v in kf.items()})
    return out


def search_paths(case: SearchCase) -> set:
    f = case.frame
    out = set()
    n = len(f["kps"])
    valid = [j for j in range(n) if f["node"][j] >= 0 and angle_ok(f["kps"]["angle"][j])]
    order = sorted(valid, key=lambda j: (int(f["node"][j]), j))  # k_sbb_sort's order
    start, runs = 0, []
    while start < len(order):
        e = start
        while e < len(order) and f["node"][order[e]] == f["node"][order[start]]:
            e += 1
        runs.append((start, e))
        start = e
    if any(s == 31 for s, _ in runs):
        out.add("run_at_31")
    if runs and len(valid) == n and runs[-1][1] == n:
        out.add("run_to_n")
    pos = {j: (s, e, p) for s, e in runs for p, j in enumerate(order[s:e])}
    if n == MAX_KEYS:
        out.add("keys_cap")
    if len(case.kfs) > 64:
        out.add("kf_chunks")
    for kf in _live(case):
        m, _ = B.search_by_bow(f["kps"], f["desc"], f["node"], kf["kps"], kf["desc"], kf["node"], kf["point"], case.ratio, case.check,
                               trace=out)
        for j in np.nonzero(m >= 0)[0]:
            s, e, p = pos[int(j)]
            if e - s == 33 and p == 32:
                out.add("run_33_late_best")
            if e - s >= 1000 and p >= e - s - 32:
                out.add("run_1000_late_best")
            if f["node"][j] == 0:
                out.add("node_0")
            if f["node"][j] == INT32_MAX:
                out.add("node_int32_max")
    return out


# ---------------------------------------------------------------------------- transform cases
def wide_tree(seed=0, scoring=0, weighting=0):
    """L = 3: the root has 40 children; the one at position 35 has 40 leaf children of its own and the one at position 3 has 4,
    the rest are leaves (so paths end at depth 1 above nid_level 2).  Returns (tree, queries): queries name keys that tie at
    positions (2, 34) of the root and (3, 35) of the wide inner node, or whose best is at position 37 / 38."""
    rng = np.random.default_rng(seed)
    parent, leaf, desc = [-1], [0], [np.zeros(32, np.uint8)]
    root_ch = _rand(rng, 40)
    q_root = _rand(rng)
    root_ch[2], root_ch[34] = _bits(q_root, [0, 1, 2]), _bits(q_root, [3, 4, 5])
    for p in range(40):
        parent.append(0)
        leaf.append(0 if p in (3, 35) else 1)
        desc.append(root_ch[p])
    wide = 36                                  # id of the root's child at position 35
    q_wide = _bits(root_ch[35], range(10, 15))
    wide_ch = np.array([_bits(root_ch[35], rng.choice(256, 24, replace=False)) for _ in range(40)], np.uint8)
    wide_ch[3], wide_ch[35] = _bits(q_wide, [100, 101, 102]), _bits(q_wide, [103, 104, 105])
    for p in range(40):
        parent.append(wide)
        leaf.append(1)
        desc.append(wide_ch[p])
    for p in range(4):
        parent.append(4)                       # the root's child at position 3
        leaf.append(1)
        desc.append(_bits(root_ch[3], rng.choice(256, 24, replace=False)))
    n = len(parent)
    w = np.where(np.array(leaf) == 1, rng.uniform(0.5, 9.0, n), 0.0)
    queries = dict(tie_root=q_root, tie_wide=q_wide, best_root_37=_bits(root_ch[37], [7, 8]),
                   best_wide_38=_bits(wide_ch[38], [9]), best_root_0=root_ch[0], deep=_bits(desc[-1], [50]))
    return _tree(parent, leaf, desc, w, 3, scoring, weighting), queries


def _star_tree(weights, scoring, weighting, seed=5):
    """L = 2: the root's children are len(weights) leaves (words in order) and one inner node with 3 leaves weighted as the first
    three."""
    rng = np.random.default_rng(seed)
    m = len(weights)
    d = _rand(rng, m + 1)
    parent = [-1] + [0] * (m + 1) + [m + 1] * 3
    leaf = [0] + [1] * m + [0] + [1] * 3
    desc = np.concatenate([np.zeros((1, 32), np.uint8), d, [_bits(d[m], rng.choice(256, 20, replace=False)) for _ in range(3)]])
    weight = [0.0] + list(weights) + [0.0] + list(weights[:3])
    return _tree(parent, leaf, desc, weight, 2, scoring, weighting)


def _keys_on(tree, leaf_ids, rng, bits=2):
    """One descriptor per listed node: the node's descriptor with `bits` random bits flipped."""
    return np.array([_bits(tree["desc"][i], rng.choice(256, bits, replace=False)) for i in leaf_ids], np.uint8).reshape(-1, 32)


def count_tree(seed=3, scoring=0, weighting=0):
    """L = 2: 16 inner nodes x 16 leaves = 256 words; words 5, 77 and 200 stopped (weight 0)."""
    rng = np.random.default_rng(seed)
    top = _rand(rng, 16)
    parent, leaf, desc = [-1], [0], [np.zeros(32, np.uint8)]
    for i in range(16):
        parent.append(0)
        leaf.append(0)
        desc.append(top[i])
    for i in range(16):
        for _ in range(16):
            parent.append(1 + i)
            leaf.append(1)
            desc.append(_bits(top[i], rng.choice(256, 20, replace=False)))
    w = np.zeros(len(parent))
    w[17:] = rng.uniform(0.5, 9.0, 256)
    w[17 + np.array([5, 77, 200])] = 0.0
    return _tree(parent, leaf, desc, w, 2, scoring, weighting)


def count_keys(tree, n, seed, words=None):
    """n keys on count_tree's words (leaf id 17 + word): word 0 and word 255 (next to the sort's sentinel) and the stopped words
    always among them when n allows."""
    rng = np.random.default_rng(seed)
    w = rng.integers(0, 256, n) if words is None else np.resize(np.asarray(words), n)
    if words is None:
        for i, fixed in enumerate((0, 255, 5, 200)):
            if i < n:
                w[(i * 7919) % n] = fixed
    return _keys_on(tree, 17 + w, rng)


KEY_COUNTS = (1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049)


def transform_cases() -> list:
    out = []
    rng = np.random.default_rng(40)
    tree, q = wide_tree(0)
    leaves_d1 = [i for i in range(1, 41) if tree["is_leaf"][i]]
    base = np.array([q["tie_root"], q["tie_wide"], q["best_root_37"], q["best_wide_38"], q["best_root_0"], q["deep"]], np.uint8)
    more = _keys_on(tree, leaves_d1[:20] + list(range(41, 81)), rng)
    desc = np.concatenate([base, more, base[:2]])
    out.append(TransformCase("wide_nid2", tree, desc, 1, {"children_40", "tie_first_child", "tie_across_stride", "best_past_stride",
                                                           "leaf_above_nid", "tf_repeat"}))
    out.append(TransformCase("wide_nid1", tree, desc, 2, {"children_40", "tie_across_stride", "best_past_stride"}))
    out.append(TransformCase("wide_nid_root_at_L", tree, desc, 3, {"children_40", "nid_root", "tie_across_stride"}))
    out.append(TransformCase("wide_nid_root_above_L", tree, desc, 5, {"nid_root"}))
    t2, _ = wide_tree(1, scoring=B.DOT_PRODUCT, weighting=B.TF)
    out.append(TransformCase("wide_dot_tf", t2, desc, 0, {"tf_divide", "tf_repeat", "best_past_stride"}))
    # word weights at the IEEE extremes (words 0..5 of a star tree; keys on each word, two on words 0 and 1)
    tiny = math.ldexp(1.0, -1070)  # subnormal: every square underflows to 0
    extremes = [
        ("weights_subnormal_l2", [tiny, 3 * tiny, 5e-324, tiny, 2 * tiny, tiny], B.L2_NORM, B.TF_IDF, {"norm_zero", "tf_repeat"}),
        ("weights_1e200_l2", [1e200, 2e200, 1.5e200, 1e200, 3e200, 1e200], B.L2_NORM, B.TF, {"norm_inf", "tf_repeat"}),
        ("weights_inf_l1", [math.inf, 2.0, 1.0, 3.0, 0.5, 4.0], B.L1_NORM, B.TF_IDF, {"norm_inf", "tf_repeat"}),
        ("weights_inf_idf", [math.inf, 2.0, 1.0, 3.0, 0.5, 4.0], B.KL, B.IDF, {"norm_inf"}),
        ("weights_inf_dot", [math.inf, 2.0, 1.0, 3.0, 0.5, 4.0], B.DOT_PRODUCT, B.TF, {"tf_divide", "tf_repeat"}),
        ("weights_stopped", [math.nan, -0.0, 0.0, -2.5, -math.inf, 4.0], B.L1_NORM, B.TF_IDF, {"stopped_word"}),
        ("weights_all_stopped", [math.nan, -0.0, 0.0, -2.5, -math.inf, 0.0], B.L2_NORM, B.TF, {"stopped_word",
                                                                                              "empty_vector_with_keys"}),
        ("weights_mixed_binary", [1e-310, 1e200, 0.0, math.nan, 7.0, 1e-300], B.L2_NORM, B.BINARY, {"stopped_word"}),
    ]
    for name, w, sc, wt, paths in extremes:
        t = _star_tree(w, sc, wt)
        ids = [1, 1, 2, 2, 3, 4, 5, 6, 8, 9, 10, 1]
        out.append(TransformCase(name, t, _keys_on(t, ids, rng), 0, paths))
    # key counts across the warp / block / pow2 boundaries of k_bow_vector's sort and fold
    ct = count_tree()
    for n in KEY_COUNTS:
        out.append(TransformCase(f"keys_{n}", ct, count_keys(ct, n, n), 1, {"stopped_word"} if n > 1 else set()))
    out.append(TransformCase("keys_2049_one_word", ct, count_keys(ct, 2049, 1, words=[255]), 1, {"tf_repeat"}))
    out.append(TransformCase("keys_1025_all_stopped", ct, count_keys(ct, 1025, 2, words=[5, 77, 200]), 1,
                             {"stopped_word", "empty_vector_with_keys"}))
    out.append(TransformCase("keys_2048_word_0", ct, count_keys(ct, 2048, 3, words=[0, 0, 5]), 1, {"tf_repeat", "stopped_word"}))
    out.append(TransformCase("keys_cap", ct, count_keys(ct, MAX_KEYS, 4), 1, {"keys_cap", "tf_repeat", "stopped_word"}, junk=False))
    return out


# ---------------------------------------------------------------------------- search cases
class _Scene:
    """Frame keys and one keyframe's keys appended one by one; every keyframe key gets its own point unless told otherwise."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.f = dict(desc=[], node=[], angle=[])
        self.k = dict(desc=[], node=[], angle=[], point=[])

    def fkey(self, desc, node, angle=100.0):
        self.f["desc"].append(np.asarray(desc, np.uint8))
        self.f["node"].append(node)
        self.f["angle"].append(angle)
        return len(self.f["node"]) - 1

    def kkey(self, desc, node, angle=100.0, point=None):
        self.k["desc"].append(np.asarray(desc, np.uint8))
        self.k["node"].append(node)
        self.k["angle"].append(angle)
        self.k["point"].append(1000 + len(self.k["point"]) if point is None else point)

    def at(self, q, d):
        return _bits(q, self.rng.choice(256, d, replace=False))

    def pair(self, node, d=3, kf_angle=100.0, f_angle=100.0):
        """A keyframe key and a frame key d bits from it, alone in their node."""
        q = _rand(self.rng)
        self.fkey(self.at(q, d), node, f_angle)
        self.kkey(q, node, kf_angle)

    def build(self):
        nf, nk = len(self.f["node"]), len(self.k["node"])
        f = dict(kps=keys(self.rng, nf, np.asarray(self.f["angle"], np.float32)), desc=np.array(self.f["desc"], np.uint8).reshape(-1, 32),
                 node=np.asarray(self.f["node"], np.int64).astype(np.int32))
        kf = dict(kps=keys(self.rng, nk, np.asarray(self.k["angle"], np.float32)), desc=np.array(self.k["desc"], np.uint8).reshape(-1, 32),
                  node=np.asarray(self.k["node"], np.int64).astype(np.int32), point=np.asarray(self.k["point"], np.int32))
        return f, [kf]


def _decisions(sc: _Scene, ratio_pair=(7, 10)):
    """Node 10: a key claims the middle of three candidates (7, 2, 7 bits away: a second-best tie), then a second key finds the
    claimed one between two tied ones; a keyframe key without a point.  Node 11 frame only, 12 keyframe only.  Nodes 13 / 14:
    one candidate at 50 / 51 bits.  Node 15: candidates at ratio_pair bits."""
    q = _rand(sc.rng)
    for d in (7, 2, 7):
        sc.fkey(sc.at(q, d), 10)
    sc.kkey(q, 10)
    sc.kkey(q, 10)
    sc.kkey(q, 10, point=-1)
    sc.fkey(_rand(sc.rng), 11)
    sc.kkey(_rand(sc.rng), 12)
    sc.pair(13, 50)
    sc.pair(14, 51)
    q = _rand(sc.rng)
    sc.fkey(sc.at(q, ratio_pair[1]), 15)
    sc.fkey(sc.at(q, ratio_pair[0]), 15)
    sc.kkey(q, 15)


def _rotations(sc: _Scene, bins, node0=100):
    """One single-candidate pair per (kf angle, frame angle, copies) entry, each in its own node."""
    node = node0
    for kf_a, f_a, copies in bins:
        for _ in range(copies):
            sc.pair(node, 3, kf_a, f_a)
            node += 1


def _runs(seed):
    """Frame nodes 0 x 31 keys, 5 x 33, 7 x 1000, 2^31 - 1 x 40 on interleaved indices: sorted runs start at 0, 31, 64 and 1064 and
    the last ends at n.  Keyframe keys near the last key of each run (node 7's twice: the second finds it claimed)."""
    rng = np.random.default_rng(seed)
    layout = [(0, 31), (5, 33), (7, 1000), (INT32_MAX, 40)]
    node = rng.permutation(np.concatenate([np.full(c, v, np.int64) for v, c in layout])).astype(np.int32)
    n = len(node)
    f_desc = _rand(rng, n)
    kf_desc, kf_node = [], []
    for v, c in layout:
        last = np.nonzero(node == v)[0][-1]
        q = _rand(rng)
        f_desc[last] = _bits(q, [1, 2, 3])
        reps = 2 if c == 1000 else 1
        kf_desc += [q] * reps
        kf_node += [v] * reps
    f = dict(kps=keys(rng, n, np.full(n, 100.0, np.float32)), desc=f_desc, node=node)
    m = len(kf_node)
    kf = dict(kps=keys(rng, m, np.full(m, 100.0, np.float32)), desc=np.array(kf_desc, np.uint8), node=np.array(kf_node, np.int32),
              point=np.arange(7, 7 + m, dtype=np.int32))
    return f, [kf]


def _frame_at_capacity(seed, n=MAX_KEYS, n_nodes=512, m=400):
    rng = np.random.default_rng(seed)
    node_ids = np.sort(rng.choice(1_000_000, n_nodes, replace=False)).astype(np.int32)
    f_desc = _rand(rng, n)
    f_node = node_ids[rng.integers(n_nodes, size=n)]
    f_kps = keys(rng, n)
    src = rng.choice(n, m, replace=False)
    kf_desc = np.array([near(rng, f_desc[s], int(rng.integers(0, 30))) for s in src], np.uint8)
    ang = ((f_kps["angle"][src] + 40.0 + rng.normal(0, 15.0, m)) % 360.0).astype(np.float32)
    kf = dict(kps=keys(rng, m, ang), desc=kf_desc, node=f_node[src].copy(), point=np.arange(m, dtype=np.int32))
    return dict(kps=f_kps, desc=f_desc, node=f_node), [kf]


KF_BATCHES = (63, 64, 65, 128, 129, 200)


def keyframe_batch(n_kf, seed=None):
    """n_kf keyframes of 5-40 keys over a 300-key frame; counts -1 on keyframes 0, 63, 64 and the last, 0 on keyframe 1."""
    rng = np.random.default_rng(n_kf if seed is None else seed)
    f, kfs = search_scene(900 + n_kf if seed is None else seed, n_frame=300, n_kfs=n_kf, n_nodes=30, kf_sizes=rng.integers(5, 41, n_kf),
                          angle_spread=10.0)
    counts = [len(kf["kps"]) for kf in kfs]
    for k in (0, 63, 64, n_kf - 1):
        if k < n_kf:
            counts[k] = -1
    counts[1] = 0
    return f, kfs, counts


def search_cases() -> list:
    out = []
    r70, r75 = float(np.float32(0.7)), float(np.float32(0.75))
    ulp70 = float(np.nextafter(np.float32(0.7), np.float32(1)))
    base = {"candidate_claimed", "best_tie", "second_tie", "kf_key_no_point", "node_frame_only", "node_kf_only", "th_low_50_accept",
            "th_low_51_reject", "single_candidate", "no_orientation"}
    sc = _Scene(1)
    _decisions(sc)
    out.append(SearchCase("decisions_070", *sc.build(), r70, False, base | {"ratio_equal_reject"}))
    sc = _Scene(2)
    _decisions(sc)
    out.append(SearchCase("decisions_070_ulp", *sc.build(), ulp70, False, base | {"ratio_ulp_accept"}))
    sc = _Scene(3)
    _decisions(sc, (15, 20))
    out.append(SearchCase("decisions_075", *sc.build(), r75, False, base | {"ratio_equal_reject"}))
    # rotation histograms: bins 9 (wrapped) x 10, 1 (15 / 30 = 0.5) x 1, 5 (135 / 30 = 4.5) x 1, 12 (rot 360) x 1
    sc = _Scene(4)
    _rotations(sc, [(10.0, 100.0, 10), (15.0, 0.0, 1), (135.0, 0.0, 1), (360.0, 0.0, 1)])
    out.append(SearchCase("maxima_3_at_tenth", *sc.build(), r70, True, {"rot_wrap", "bin_half_up", "bin_12", "three_maxima_3",
                                                                          "tenth_rule_equal", "single_candidate"}))
    # bin 12 x 11 and one match at rot 0 exactly (bin 0), culled by the 0.1 rule
    sc = _Scene(5)
    _rotations(sc, [(355.0, 0.0, 11), (100.0, 100.0, 1)])
    out.append(SearchCase("maxima_1_rot_zero_culled", *sc.build(), r70, True, {"rot_zero", "three_maxima_1", "tenth_rule_cull"}))
    # bins 3 x 20, 6 x 2 (= 0.1f * 20: kept), 7 x 1 (culled)
    sc = _Scene(6)
    _rotations(sc, [(90.0, 0.0, 20), (300.0, 120.0, 2), (0.0, 150.0, 1)])
    out.append(SearchCase("maxima_2_at_and_below_tenth", *sc.build(), r75, True, {"three_maxima_2", "tenth_rule_equal",
                                                                                    "tenth_rule_cull", "rot_wrap"}))
    out.append(SearchCase("runs", *_runs(7), r75, True, {"run_at_31", "run_to_n", "run_33_late_best", "run_1000_late_best", "node_0",
                                                          "node_int32_max", "candidate_claimed", "three_maxima_1"}, junk=False))
    out.append(SearchCase("frame_at_capacity", *_frame_at_capacity(8), r75, True, {"keys_cap", "run_to_n"}, junk=False))
    for n_kf in KF_BATCHES:
        f, kfs, counts = keyframe_batch(n_kf)
        out.append(SearchCase(f"keyframes_{n_kf}", f, kfs, r75 if n_kf % 2 else r70, n_kf != 128,
                              {"kf_chunks"} if n_kf > 64 else set(), counts=counts))
    return out


FUZZ_RATIOS = (0.6, float(np.float32(0.7)), float(np.nextafter(np.float32(0.7), np.float32(1))), float(np.float32(0.75)), 0.9)


def fuzz_case(seed) -> SearchCase:
    """A seeded scene mixing the above: 0-400 frame keys, 1-3 keyframes (one in eight: 65-70 small ones with negative and zero
    counts), exact angles 0 / 15 / 135 / 360 on some keys, nodes renamed to 0 and 2^31 - 1."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 400))
    many = rng.uniform() < 0.125
    n_kf = int(rng.integers(65, 71)) if many else int(rng.integers(1, 4))
    f, kfs = search_scene(70000 + seed, n_frame=n, n_kfs=n_kf, n_nodes=int(rng.integers(1, 30)),
                          kf_sizes=rng.integers(0, 30, n_kf) if many else None, angle_spread=float(rng.choice([3.0, 40.0, 180.0])))
    if n and rng.uniform() < 0.5:
        nodes = np.unique(f["node"][f["node"] >= 0])
        if len(nodes):
            ren = {int(nodes[0]): 0, int(nodes[-1]): INT32_MAX}
            for a in [f] + kfs:
                a["node"] = np.array([ren.get(int(v), int(v)) for v in a["node"]], np.int64).astype(np.int32)
    for a in [f] + kfs:
        m = len(a["kps"])
        if m:
            sel = rng.uniform(size=m) < 0.1
            a["kps"]["angle"][sel] = rng.choice(np.array([0.0, 15.0, 135.0, 360.0], np.float32), int(sel.sum()))
    counts = None
    if many or rng.uniform() < 0.2:
        counts = [len(kf["kps"]) for kf in kfs]
        for k in rng.choice(n_kf, min(n_kf, int(rng.integers(1, 4))), replace=False):
            counts[k] = int(rng.choice([-1, 0]))
    return SearchCase(f"fuzz_{seed}", f, kfs, float(rng.choice(FUZZ_RATIOS)), bool(rng.integers(2)), set(), counts=counts)
