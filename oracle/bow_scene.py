"""Seeded vocabularies and SearchByBoW scenes for the bag-of-words tests and tools (no vocabulary file is committed).

- full_shape_tree: k = 10, L = 6, about 1.08 M nodes in ORBvoc's layout (each node's children consecutive, parents before
  children).  Level-1 descriptors are drawn from the committed fixture's ORB descriptors (tests/golden/orb_kitti_2000.npz); each
  child is its parent with bits flipped at a per-level rate, so real keys spread over the level-2 nodes.  About 9 % of the words
  have weight 0 (stopped), as in ORBvoc.
- irregular_tree: 2-10 children, leaves at every depth (above nid_level included), nodes in depth-first order (children not
  consecutive), and sibling descriptors at exactly equal distance from chosen keys.
- small_tree: a few hundred nodes for one weighting x scoring pair.
- search_scene: a frame and keyframes whose keys share vocabulary nodes, with crowds, claim chains and ties.
"""
from __future__ import annotations

import os

import numpy as np

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
