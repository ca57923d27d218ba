"""-m gpu: the bag of words (k_bow_descend / k_bow_vector / k_sbb_sort / k_sbb_init / k_sbb_walk / k_sbb_finish) on the constructed
cases of oracle/bow_scene.py, bit for bit against oracle/bow_oracle.py with no exemption, through the host form and the device form:
descents through nodes of 40 children with ties across the lanes' two strides, word weights at the IEEE extremes (NaN weights
compared by position), key counts across the warp, block and power-of-two boundaries of the BowVector sort and at the 16,384-key
capacity, frame runs at exact sorted positions, nodes 0 and 2^31 - 1, batches of 63-200 keyframes (later launches) with negative,
zero and above-capacity counts, every NULL output combination of sivo_compute_bow_device, the capacity limits and 200 seeded fuzz
scenes.  Every device call passes an oracle/keymap.py semantic-key map holding rejected and duplicate entries, and every
buffer carries slack rows past its bound that a bound one too wide would read or write."""
import zlib

import numpy as np
import pytest
import torch

from frame_support import extractor, i64, same_bits, sentinel, upload
from oracle import bow_oracle as B
from oracle import bow_scene as S
from oracle.keymap import SLACK, keymap, scatter
from sivo_b200 import _lib as L
from sivo_b200.bow import Vocabulary, compute_bow, compute_bow_device, keyframe_keys, search_by_bow, search_by_bow_device
from sivo_b200.orb import KP_DTYPE, ORBextractor

pytestmark = pytest.mark.gpu
FORCED = (0, 31, 32, -1)  # semantic keys whose entry is rejected: the first, both sides of a warp boundary, the last
TRANSFORM = {c.name: c for c in S.transform_cases()}
SEARCH = {c.name: c for c in S.search_cases()}
_VOC = {}


def el_for(n):
    """The 2,000-feature extractor (capacity 2,096) when n keys and the rejected entries fit, else the 16,384-key one."""
    return extractor(2000) if n + 32 <= extractor(2000).capacity() else extractor(16288)


def vocabulary(tree):
    if id(tree) not in _VOC:
        _VOC[id(tree)] = (tree, Vocabulary.from_arrays(tree["k"], tree["L"], tree["scoring"], tree["weighting"], tree["parent"],
                                                       tree["is_leaf"], tree["desc"], tree["weight"]))
    return _VOC[id(tree)][1]


def case_rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def clamp(count, cap):
    return min(count, cap)


def gathered(keep, count, cap):
    """(entries read, valid mask, slot per entry) of the device form for a count."""
    m = max(0, clamp(count, cap))
    k = keep[:m]
    valid = (k >= 0) & (k < cap)
    return m, valid, np.where(valid, k, 0)


# ---------------------------------------------------------------------------------------------------------- transform
def device_bow(voc, el, slot_desc, keep, count, levelsup, want=(True,) * 5):
    """sivo_compute_bow_device with every output at capacity + SLACK (sentinels -7 / 7.0) or NULL where want is False."""
    cap = el.capacity()
    t = [upload(slot_desc), upload(keep), i64(count)]
    out = dict(node=sentinel(cap + SLACK, -7, torch.int32), word=sentinel(cap + SLACK, -7, torch.int32),
               bw=sentinel(cap + SLACK, -7, torch.int32), bwt=sentinel(cap + SLACK, 7.0, torch.float64), len=sentinel(2, -7, torch.int64))
    ptrs = [v.data_ptr() if w else 0 for v, w in zip(out.values(), want)]
    compute_bow_device(voc, el, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), levelsup, *ptrs)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def transform_setup(case_desc, cap, rng, junk):
    km = keymap(len(case_desc), cap, rng, FORCED, duplicates=True, junk=junk)
    slot_desc = scatter(case_desc, km.slots, cap, rng.integers(0, 256, (cap + SLACK, 32), dtype=np.uint8))
    if len(case_desc):
        slot_desc[cap:] = case_desc[0]  # a key a bound one too wide would read
    return slot_desc, km.keep, km.n_keep


def transform_want(tree, slot_desc, keep, count, cap, levelsup, same_as=None):
    """The oracle on what the device reads: node / word per semantic key (-1 for a rejected entry), the BowVector."""
    m, valid, slot = gathered(keep, count, cap)
    if same_as is not None and valid.all() and m == len(same_as[2]) and np.array_equal(slot_desc[slot], same_as[4]):
        bow, _, node_v, word_v, _ = same_as
    else:
        bow, _, node_v, word_v = B.transform(tree, slot_desc[slot[valid]], levelsup)
    node, word = np.full(m, -1, np.int32), np.full(m, -1, np.int32)
    node[valid], word[valid] = node_v, word_v
    words, vals = B.bow_arrays(bow)
    return node, word, words, vals


def check_device_bow(d, want, cap, want_mask=(True,) * 5):
    node, word, words, vals = want
    m, n_bow = len(node), len(words)
    exp = [(node, -7), (word, -7), (words, -7), (vals, 7.0)]
    for (k, (w, sentinel)), on in zip(zip(("node", "word", "bw", "bwt"), exp), want_mask):
        got = d[k]
        if not on:
            assert (got == sentinel).all(), k
            continue
        upto = m if k in ("node", "word") else n_bow
        if k == "bwt":
            assert same_bits(got[:upto], w), k
        else:
            np.testing.assert_array_equal(got[:upto], w, err_msg=k)
        assert (got[upto:] == sentinel).all(), k
    if want_mask[4]:
        assert int(d["len"][0]) == n_bow and int(d["len"][1]) == -7
    else:
        assert (d["len"] == -7).all()


@pytest.mark.parametrize("name", list(TRANSFORM))
def test_transform_case(name):
    case = TRANSFORM[name]
    tree, voc = B.Tree(case.tree), vocabulary(case.tree)
    bow, fv, node, word = B.transform(tree, case.desc, case.levelsup)
    words, vals = B.bow_arrays(bow)
    h = compute_bow(voc, case.desc, case.levelsup)
    np.testing.assert_array_equal(h["node"], node)
    np.testing.assert_array_equal(h["word"], word)
    np.testing.assert_array_equal(h["bow_words"], words)
    assert same_bits(h["bow_weights"], vals)
    el = el_for(len(case.desc))
    cap = el.capacity()
    slot_desc, keep, n_keep = transform_setup(case.desc, cap, case_rng(name), case.junk)
    want = transform_want(tree, slot_desc, keep, n_keep, cap, case.levelsup, same_as=(bow, fv, node, word, case.desc))
    check_device_bow(device_bow(voc, el, slot_desc, keep, n_keep, case.levelsup), want, cap)


def test_transform_counts_and_null_outputs():
    """Counts 0, -1 and above the capacity on the wide tree, then all 32 NULL patterns of the outputs (a NULL word takes the
    stream-scratch path)."""
    case = TRANSFORM["wide_nid2"]
    tree, voc = B.Tree(case.tree), vocabulary(case.tree)
    el = extractor()
    cap = el.capacity()
    slot_desc, keep, n_keep = transform_setup(case.desc, cap, case_rng("counts"), True)
    for count in (0, cap, cap + 1000):
        want = transform_want(tree, slot_desc, keep, count, cap, case.levelsup)
        check_device_bow(device_bow(voc, el, slot_desc, keep, count, case.levelsup), want, cap)
    neg = device_bow(voc, el, slot_desc, keep, -1, case.levelsup)
    assert int(neg["len"][0]) == -1 and int(neg["len"][1]) == -7
    assert all((neg[k] == -7).all() for k in ("node", "word", "bw")) and (neg["bwt"] == 7.0).all()
    want = transform_want(tree, slot_desc, keep, n_keep, cap, case.levelsup)
    for mask in range(32):
        on = tuple(bool(mask >> b & 1) for b in range(5))
        check_device_bow(device_bow(voc, el, slot_desc, keep, n_keep, case.levelsup, on), want, cap, on)


# ---------------------------------------------------------------------------------------------------------- SearchByBoW
class DeviceFrame:
    """A case's frame embedded as sivo_search_by_bow_device reads it: kps / desc at permuted extractor slots, node per semantic
    key.  Rejected entries carry a live node; duplicates sit in node `spare`, which no keyframe has (in a shared node they would tie
    with their key and change what the case was built to reach); entries and slots past every bound hold keys of a live node."""

    def __init__(self, f, cap, rng, junk=True, spare=-1):
        n = len(f["kps"])
        self.cap = cap
        km = keymap(n, cap, rng, FORCED, duplicates=True, junk=junk)
        self.keep, self.n_keep, src, dup = km.keep, km.n_keep, km.src, km.dup
        live = int(f["node"][f["node"] >= 0][0]) if (f["node"] >= 0).any() else 3
        decoy = np.zeros(1, KP_DTYPE)
        decoy["angle"] = 100.0
        self.kps = scatter(f["kps"], km.slots, cap, decoy)
        self.desc = scatter(f["desc"], km.slots, cap, rng.integers(0, 256, (cap + SLACK, 32), dtype=np.uint8))
        if n:
            self.kps[cap:], self.desc[cap:] = f["kps"][0], f["desc"][0]
        self.node = np.full(len(self.keep), live, np.int32)
        self.node[:self.n_keep] = np.where(src >= 0, f["node"][np.maximum(src, 0)] if n else live, live)
        self.node[:self.n_keep][dup] = spare

    def oracle_frame(self, count):
        m, valid, slot = gathered(self.keep, count, self.cap)
        return dict(kps=self.kps[slot], desc=self.desc[slot], node=np.where(valid, self.node[:m], -1).astype(np.int32))


def pad_keyframe(kf, cap):
    """A keyframe's arrays at cap + SLACK: entries past its keys repeat its first key (or a node-3 key) with a point."""
    out = {}
    m = len(kf["kps"])
    for k, fill in (("kps", None), ("desc", None), ("node", 3), ("point", 1)):
        a = kf[k]
        p = np.zeros((cap + SLACK,) + a.shape[1:], a.dtype)
        p[:m] = a
        p[m:] = a[0] if m else (fill if fill is not None else p[m:])
        out[k] = p
    if m == 0:
        out["kps"]["angle"] = 100.0
    out["point"][m:] = np.maximum(out["point"][m:], 0)
    return out


def device_search(el, fr, kfs, counts, ratio, check, frame_count=None):
    """sivo_search_by_bow_device with n_kf rows of cap + SLACK sentinel (-7) entries and n_kf + 1 counts."""
    cap = el.capacity()
    n_kf = len(kfs)
    hold = [upload(fr.kps), upload(fr.desc), upload(fr.keep), i64(fr.n_keep if frame_count is None else frame_count), upload(fr.node)]
    keys, pts = [], []
    for kf, c in zip(kfs, counts):
        a = [upload(kf["kps"]), upload(kf["desc"]), upload(kf["node"]), upload(kf["point"]), i64(c)]
        hold += a
        keys.append(keyframe_keys(a[0].data_ptr(), a[1].data_ptr(), a[2].data_ptr(), a[4].data_ptr()))
        pts.append(a[3].data_ptr())
    match = sentinel(n_kf * cap + SLACK, -7, torch.int32)
    nm = sentinel(n_kf + 1, -7, torch.int64)
    search_by_bow_device(el, hold[0].data_ptr(), hold[1].data_ptr(), hold[2].data_ptr(), hold[3].data_ptr(), hold[4].data_ptr(), keys,
                         pts, ratio, check, match.data_ptr(), nm.data_ptr())
    torch.cuda.synchronize()
    m = match.cpu().numpy()
    return m[:n_kf * cap].reshape(n_kf, cap), m[n_kf * cap:], nm.cpu().numpy()


def oracle(f, kf, ratio, check):
    return B.search_by_bow(f["kps"], f["desc"], f["node"], kf["kps"], kf["desc"], kf["node"], kf["point"], ratio, check)


def check_device_search(el, f, kfs, counts, ratio, check, rng, junk=True, frame_count=None, same_as=None):
    cap = el.capacity()
    used = set(f["node"].tolist()).union(*(kf["node"].tolist() for kf in kfs))
    fr = DeviceFrame(f, cap, rng, junk, spare=min(set(range(len(used) + 1)) - used))
    pk = [pad_keyframe(kf, cap) for kf in kfs]
    rows, slack, nm = device_search(el, fr, pk, counts, ratio, check, frame_count)
    fc = fr.n_keep if frame_count is None else frame_count
    assert (slack == -7).all() and nm[-1] == -7
    of = fr.oracle_frame(fc) if fc >= 0 else None
    reuse = same_as is not None and of is not None and len(of["kps"]) == len(f["kps"]) and np.array_equal(of["desc"], f["desc"]) \
        and np.array_equal(of["node"], f["node"]) and np.array_equal(of["kps"].view(np.uint8), f["kps"].view(np.uint8))
    for k, c in enumerate(counts):
        if fc < 0 or c < 0:  # only n_matches is written
            assert nm[k] == -1 and (rows[k] == -7).all(), k
            continue
        if reuse and c == len(kfs[k]["kps"]):
            m_want, n_want = same_as[k]
        else:
            kf = {key: v[:clamp(c, cap)] for key, v in pk[k].items()}
            m_want, n_want = oracle(of, kf, ratio, check)
        mm = len(m_want)
        np.testing.assert_array_equal(rows[k][:mm], m_want, err_msg=f"keyframe {k}")
        assert (rows[k][mm:] == -1).all(), k
        assert nm[k] == n_want, k


def check_host_search(el, f, kfs, counts, ratio, check):
    want = []
    for kf, c in zip(kfs, counts):
        want.append(oracle(f, {k: v[:c] for k, v in kf.items()}, ratio, check) if c >= 0 else None)
    m, nm = search_by_bow(el, f["kps"], f["desc"], f["node"], [dict(kf, count=c) for kf, c in zip(kfs, counts)], ratio, check)
    for k, w in enumerate(want):
        if w is None:
            assert nm[k] == -1 and (m[k] == -1).all(), k
            continue
        np.testing.assert_array_equal(m[k], w[0], err_msg=f"keyframe {k}")
        assert nm[k] == w[1], k
    return want


def counts_of(case):
    return [len(kf["kps"]) for kf in case.kfs] if case.counts is None else list(case.counts)


@pytest.mark.parametrize("name", list(SEARCH))
def test_search_case(name):
    case = SEARCH[name]
    counts = counts_of(case)
    n = len(case.frame["kps"])
    el = el_for(n)
    want = check_host_search(el, case.frame, case.kfs, counts, case.ratio, case.check)
    check_device_search(el, case.frame, case.kfs, counts, case.ratio, case.check, case_rng(name), case.junk, same_as=want)


@pytest.mark.parametrize("n_kf", [65, 129])
def test_search_counts_out_of_range(n_kf):
    """Frame counts 0, -1 and above the capacity, and a keyframe count above the capacity, with the batch's negative counts."""
    case = SEARCH[f"keyframes_{n_kf}"]
    el = extractor()
    cap = el.capacity()
    counts = counts_of(case)
    counts[2] = cap + 100
    counts[3] = 2**40
    for fc in (None, 0, -1, cap + 100):
        check_device_search(el, case.frame, case.kfs, counts, case.ratio, case.check, case_rng(f"range{n_kf}"), frame_count=fc)


def test_capacity_limits():
    big = extractor(16288)
    assert big.capacity() == S.MAX_KEYS
    f, kfs = S._frame_at_capacity(31, n=S.MAX_KEYS + 1, m=20)
    with pytest.raises(L.SivoError) as e:
        search_by_bow(big, f["kps"], f["desc"], f["node"], kfs, 0.75, True)
    assert e.value.code == L.ERANGE
    with pytest.raises(L.SivoError) as e:
        search_by_bow(big, f["kps"][:10], f["desc"][:10], f["node"][:10], [dict(kfs[0], count=S.MAX_KEYS + 1)], 0.75, True)
    assert e.value.code == L.ERANGE
    over = ORBextractor(16289, 1.2, 8, 20, 7)
    assert over.capacity() == S.MAX_KEYS + 1
    case = TRANSFORM["wide_nid2"]
    voc = vocabulary(case.tree)
    cap = over.capacity()
    slot_desc, keep, n_keep = transform_setup(case.desc, cap, case_rng("over"), True)
    t = [upload(slot_desc), upload(keep), i64(n_keep)]
    outs = [sentinel(cap, -7, torch.int32) for _ in range(3)] + [sentinel(cap, 7.0, torch.float64), sentinel(1, -7, torch.int64)]
    with pytest.raises(L.SivoError) as e:
        compute_bow_device(voc, over, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), case.levelsup, *(o.data_ptr() for o in outs))
    assert e.value.code == L.ERANGE
    torch.cuda.synchronize()
    assert all((o == (7.0 if o.dtype == torch.float64 else -7)).all() for o in outs)
    sc = SEARCH["decisions_070"]
    fr = DeviceFrame(sc.frame, cap, case_rng("over2"))
    hold = [upload(fr.kps), upload(fr.desc), upload(fr.keep), i64(fr.n_keep), upload(fr.node)]
    pk = pad_keyframe(sc.kfs[0], cap)
    a = [upload(pk["kps"]), upload(pk["desc"]), upload(pk["node"]), upload(pk["point"]), i64(len(sc.kfs[0]["kps"]))]
    match, nm = sentinel(cap, -7, torch.int32), sentinel(1, -7, torch.int64)
    with pytest.raises(L.SivoError) as e:
        search_by_bow_device(over, *(h.data_ptr() for h in hold), [keyframe_keys(a[0].data_ptr(), a[1].data_ptr(), a[2].data_ptr(),
                                                                                 a[4].data_ptr())], [a[3].data_ptr()], sc.ratio, sc.check,
                             match.data_ptr(), nm.data_ptr())
    assert e.value.code == L.ERANGE
    torch.cuda.synchronize()
    assert (match == -7).all() and (nm == -7).all()


def test_search_fuzz():
    el = extractor()
    for seed in range(200):
        c = S.fuzz_case(seed)
        counts = counts_of(c)
        want = check_host_search(el, c.frame, c.kfs, counts, c.ratio, c.check)
        if seed % 10 == 0:
            check_device_search(el, c.frame, c.kfs, counts, c.ratio, c.check, np.random.default_rng(seed), same_as=want)
