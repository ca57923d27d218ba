"""Scalar restatement of the DBoW2 vocabulary as ORB-SLAM2 uses it: TemplatedVocabulary::loadFromTextFile
(dependencies/DBoW2/DBoW2/TemplatedVocabulary.h:1338-1420), transform(features, v, fv, levelsup) (:1127-1195) and the per-feature
descent (:1218-1259), BowVector::addWeight / addIfNotExist / normalize (BowVector.cpp:34-84), FeatureVector::addFeature
(FeatureVector.cpp:31-44), the scoring objects' normalisation (ScoringObject.h:69-88), and ORBmatcher::SearchByBoW(KeyFrame*,
Frame&) (src/orbslam/ORBmatcher.cc:161-284).

Reference facts kept:
- Header `k L scoring weighting`, refused where the reference returns false (TemplatedVocabulary.h:1359): k < 0 || k > 20 || L < 1
  || L > 10 || scoring outside [0, 5] || weighting outside [0, 3].  Enums: weighting TF_IDF, TF, IDF, BINARY; scoring L1_NORM,
  L2_NORM, CHI_SQUARE, KL, BHATTACHARYYA, DOT_PRODUCT (BowVector.h:36-53).
- Node id = line number (the root 0 has no line); `parent isLeaf d0 .. d31 weight`; nIsLeaf > 0 is a leaf and gets the next word
  id (:1408-1415); children are pushed in file order (:1392); a descriptor byte is (unsigned char) of its int token
  (FORB.cpp:120-135); the weight is a double.
- isLeaf() is children.empty(): the descent stops at the first node without children (:1254).
- Descent: distances are FORB::distance (integer Hamming) as double, strict `<` over the children in order (:1238-1249), so the
  first child wins ties; nid is the node at current_level == L - levelsup, the root when that is <= 0 (:1226-1252).
- transform: a feature enters v and fv only if w > 0 (:1157, :1185).  TF / TF_IDF: addWeight, the double sum per word in feature
  order; then, if the scoring needs no normalisation, each weight / v.size() (:1164-1170).  IDF / BINARY: addIfNotExist (the
  first feature's weight), never divided.  Then normalize when the scoring says so (:1193).
- Scoring -> normalisation (ScoringObject.h): L1_NORM, CHI_SQUARE, KL, BHATTACHARYYA -> L1; L2_NORM -> L2; DOT_PRODUCT none.
  normalize: L1 = sum of |w| in ascending word order; L2 = sqrt(sum of w * w); divide only if norm > 0 (BowVector.cpp:62-84).
- SearchByBoW: the two FeatureVectors walked with lower_bound (:185-263), so only common nodes, ascending; keyframe keys of the
  node ascending, skipped without a point (NULL or isBad); frame candidates ascending, skipped once matched in this call
  (vpMapPointMatches starts empty, :166); best / second with strict `<` (:219-225); accepted iff bestDist1 <= TH_LOW (50) and
  (float) bestDist1 < mfNNratio * (float) bestDist2 (:228-230); rot = kp.angle - F angle, + 360 if < 0, bin = round(rot * (1 /
  30)) with 30 -> 0 (only bins 0..12: the reference's factor), ComputeThreeMaxima and the culling of every other bin (:265-281).

Rules where the reference is undefined (each stated in include/sivo_b200.h):
- Trailing whitespace-only lines add no node (the reference's `while (!f.eof())` appends a phantom node after the final newline);
  a blank line followed by a further node is refused.  A parent that is not an earlier node, a leaf parent, a short line, a
  missing weight, a non-leaf without children and an empty tree are refused.  Tokens after the weight are ignored.
- A path that reaches a leaf above nid_level records the leaf itself (the reference leaves nid uninitialised).
- Angles: a frame key with an angle outside [0, 360] (or NaN) is in no node, a keyframe key with one is not searched (the angle
  rule of track_oracle); the host form of the library refuses them instead.
"""
from __future__ import annotations

import bisect
import math

import numpy as np

from oracle.orb_oracle import descriptor_distance
from oracle.track_oracle import F32, HISTO_LENGTH, angle_ok, compute_three_maxima, round_half_away

TH_LOW = 50
TF_IDF, TF, IDF, BINARY = range(4)
L1_NORM, L2_NORM, CHI_SQUARE, KL, BHATTACHARYYA, DOT_PRODUCT = range(6)

# The paths the optional `trace` of Tree.descend, transform and search_by_bow records (oracle/bow_scene.py builds cases for each).
DESCENT_PATHS = (
    "tie_first_child",    # a later child at the best distance: the first keeps it
    "tie_across_stride",  # the winner at child position < 32, a tied child at >= 32 (the warp's second lane stride)
    "best_past_stride",   # the winner at child position >= 32
    "leaf_above_nid",     # the path ends at a leaf above nid_level: the leaf is the node
    "nid_root",           # levelsup >= L: the node is the root
)
TRANSFORM_PATHS = (
    "stopped_word",            # w > 0 fails: 0, negative, -0.0 or NaN
    "tf_repeat",               # TF / TF_IDF: a further feature on a word already in the vector
    "tf_divide",               # DOT_PRODUCT with TF / TF_IDF: each weight / the number of words
    "norm_zero",               # a non-empty vector whose norm is 0 (subnormal squares): nothing is divided
    "norm_inf",                # the norm overflows to inf (or sums an inf weight): finite weights become 0, inf / inf NaN
    "empty_vector_with_keys",  # keys, but every one on a stopped word
)
SEARCH_PATHS = (
    "node_frame_only", "node_kf_only",   # a node in one FeatureVector only
    "kf_key_no_point",                   # a keyframe key without a point is not searched
    "candidate_claimed",                 # a frame key matched earlier in the call is skipped
    "best_tie", "second_tie",            # a later candidate at the best / second distance
    "th_low_50_accept", "th_low_51_reject",
    "ratio_equal_reject",                # bestDist == nnratio * bestDist2 in float
    "ratio_ulp_accept",                  # nnratio * bestDist2 one float above bestDist
    "single_candidate",                  # accepted with bestDist2 = 256
    "rot_wrap", "rot_zero",              # rot < 0 then + 360; rot exactly 0 (not wrapped)
    "bin_half_up",                       # rot * (1 / 30) exactly k + 0.5: rounded up
    "bin_12",                            # rot = 360
    "bin_30_to_0",                       # the reference's 30 -> 0 rule
    "three_maxima_0", "three_maxima_1", "three_maxima_2", "three_maxima_3",  # bins kept
    "tenth_rule_equal", "tenth_rule_cull",  # max2 / max3 at exactly 0.1f * max1 (kept) and below it (culled)
    "no_orientation",
)


class FormatError(ValueError):
    pass


# ------------------------------------------------------------------------------------------------------------------ the parser
def _int(tok: str) -> int:
    s = tok[1:] if tok[:1] in "+-" else tok
    if not s or not s.isdigit() or not s.isascii():
        raise FormatError(f"not an integer: {tok!r}")
    v = int(tok)
    if not -2**31 <= v < 2**31:
        raise FormatError(f"integer out of range: {tok!r}")
    return v


def check_tree(k, L, scoring, weighting, parent, is_leaf):
    if k < 0 or k > 20 or L < 1 or L > 10 or not 0 <= scoring <= 5 or not 0 <= weighting <= 3:
        raise FormatError("header out of range")
    n = len(parent)
    if n < 2:
        raise FormatError("empty tree")
    nch = [0] * n
    for i in range(1, n):
        p = int(parent[i])
        if p < 0 or p >= i:
            raise FormatError(f"node {i}: parent {p} is not an earlier node")
        if p > 0 and is_leaf[p]:
            raise FormatError(f"node {i}: parent {p} is a leaf")
        nch[p] += 1
    for i in range(n):
        if (i == 0 or not is_leaf[i]) and nch[i] == 0:
            raise FormatError(f"node {i} is not a leaf and has no children")


def parse_text(text: str) -> dict:
    """The text format -> dict(k, L, scoring, weighting, parent, is_leaf, desc, weight) indexed by node id (root at 0)."""
    lines = text.split("\n")
    if text.endswith("\n"):
        lines.pop()  # a final newline ends the last line
    if not lines or text == "":
        raise FormatError("empty file")
    ws = " \t\r\v\f"
    hdr = [t for t in _split(lines[0], ws)]
    if len(hdr) < 4:
        raise FormatError("the header needs k L scoring weighting")
    k, L, scoring, weighting = (_int(t) for t in hdr[:4])
    parent, leaf, desc, weight = [-1], [0], [bytes(32)], [0.0]
    blank = False
    for line in lines[1:]:
        tok = _split(line, ws)
        if not tok:
            blank = True
            continue
        if blank:
            raise FormatError("blank line before a further node")
        if len(tok) < 34:
            raise FormatError("fewer than 34 integer tokens before the weight")
        v = [_int(t) for t in tok[:34]]
        if len(tok) < 35:
            raise FormatError("no weight")
        try:
            w = float(tok[34])
        except ValueError:
            raise FormatError("weight is not a number") from None
        parent.append(v[0])
        leaf.append(1 if v[1] > 0 else 0)
        desc.append(bytes(x & 0xFF for x in v[2:]))
        weight.append(w)
    check_tree(k, L, scoring, weighting, parent, leaf)
    return dict(k=k, L=L, scoring=scoring, weighting=weighting, parent=np.array(parent, np.int32), is_leaf=np.array(leaf, np.uint8),
                desc=np.frombuffer(b"".join(desc), np.uint8).reshape(-1, 32).copy(), weight=np.array(weight, np.float64))


def _split(line: str, ws: str) -> list:
    out, cur = [], []
    for ch in line:
        if ch in ws:
            if cur:
                out.append("".join(cur))
                cur = []
        else:
            cur.append(ch)
    if cur:
        out.append("".join(cur))
    return out


def to_text(tree: dict, trailing: str = "\n") -> str:
    """The text form of a tree (weights with repr, which round-trips)."""
    out = [f"{tree['k']} {tree['L']}  {tree['scoring']} {tree['weighting']}"]
    for i in range(1, len(tree["parent"])):
        d = " ".join(str(int(x)) for x in tree["desc"][i])
        out.append(f"{int(tree['parent'][i])} {int(tree['is_leaf'][i])} {d} {float(tree['weight'][i])!r}")
    return "\n".join(out) + trailing


# ------------------------------------------------------------------------------------------------------------------ the tree
class Tree:
    """The loaded vocabulary: children lists in id order, word ids in id order of the leaves."""

    def __init__(self, t: dict):
        check_tree(t["k"], t["L"], t["scoring"], t["weighting"], t["parent"], t["is_leaf"])
        self.k, self.L, self.scoring, self.weighting = t["k"], t["L"], t["scoring"], t["weighting"]
        n = len(t["parent"])
        self.desc = np.ascontiguousarray(t["desc"], np.uint8).reshape(n, 32)
        self.children = [[] for _ in range(n)]
        for i in range(1, n):
            self.children[int(t["parent"][i])].append(i)
        self.word = np.full(n, -1, np.int64)
        leaves = [i for i in range(1, n) if t["is_leaf"][i]]
        self.word[leaves] = np.arange(len(leaves))
        self.word_weight = np.asarray(t["weight"], np.float64)[leaves]
        self.n_words = len(leaves)

    def descend(self, d, levelsup, trace=None):
        """transform(feature, word_id, weight, &nid, levelsup) -> (word, weight, nid).  trace: a set that receives the names of
        the descent paths taken (DESCENT_PATHS)."""
        d = np.asarray(d, np.uint8)
        nid_level = self.L - levelsup
        nid = 0 if nid_level <= 0 else None
        if trace is not None and nid_level <= 0:
            trace.add("nid_root")
        final, level = 0, 0
        while True:
            level += 1
            nodes = self.children[final]
            dist = np.unpackbits(np.bitwise_xor(self.desc[nodes], d), axis=1).sum(axis=1)
            final = nodes[0]
            best, pos = float(dist[0]), 0
            for p, (c, dc) in enumerate(zip(nodes[1:], dist[1:]), 1):
                if float(dc) < best:
                    best, final, pos = float(dc), c, p
            if trace is not None:
                tied = [p for p in range(pos + 1, len(nodes)) if float(dist[p]) == best]
                if tied:
                    trace.add("tie_first_child")
                if pos < 32 and any(p >= 32 for p in tied):
                    trace.add("tie_across_stride")
                if pos >= 32:
                    trace.add("best_past_stride")
            if level == nid_level:
                nid = final
            if not self.children[final]:
                break
        if nid is None:
            nid = final  # a leaf above nid_level: the leaf itself
            if trace is not None:
                trace.add("leaf_above_nid")
        w = int(self.word[final])
        return w, float(self.word_weight[w]), int(nid)


def must_normalize(scoring):
    """ScoringObject::mustNormalize -> (must, norm) with norm 'L1' / 'L2'."""
    if scoring == DOT_PRODUCT:
        return False, "L1"
    return True, ("L2" if scoring == L2_NORM else "L1")


def normalize(bow: dict, norm: str, trace=None):
    """BowVector::normalize over a dict walked in ascending word order."""
    s = 0.0
    if norm == "L1":
        for w in sorted(bow):
            s += abs(bow[w])
    else:
        for w in sorted(bow):
            s += bow[w] * bow[w]
        s = math.sqrt(s)
    if trace is not None and bow:
        if s == 0.0:
            trace.add("norm_zero")  # every square underflowed: nothing is divided
        elif s == math.inf:
            trace.add("norm_inf")   # finite weights become 0, an infinite one NaN
    if s > 0.0:
        for w in sorted(bow):
            bow[w] /= s


def transform(tree: Tree, descs, levelsup, trace=None):
    """transform(features, v, fv, levelsup) -> (bow {word: weight}, fv {node: [feature indices]}, node per key, word per key);
    node / word -1 for a key in neither vector.  trace: a set that receives the names of the paths taken (DESCENT_PATHS and
    TRANSFORM_PATHS)."""
    must, norm = must_normalize(tree.scoring)
    bow, fv = {}, {}
    n = len(descs)
    node, word = np.full(n, -1, np.int32), np.full(n, -1, np.int32)
    tf = tree.weighting in (TF, TF_IDF)
    for i in range(n):
        w_id, w, nid = tree.descend(descs[i], levelsup, trace)
        if w > 0:
            if tf:
                if trace is not None and w_id in bow:
                    trace.add("tf_repeat")
                bow[w_id] = bow[w_id] + w if w_id in bow else w
            elif w_id not in bow:
                bow[w_id] = w
            fv.setdefault(nid, []).append(i)
            node[i], word[i] = nid, w_id
        elif trace is not None:
            trace.add("stopped_word")  # w = 0, negative, -0.0 or NaN
    if trace is not None and n and not bow:
        trace.add("empty_vector_with_keys")
    if tf and bow and not must:
        if trace is not None:
            trace.add("tf_divide")
        nd = float(len(bow))
        for w_id in bow:
            bow[w_id] /= nd
    if must:
        normalize(bow, norm, trace)
    return bow, fv, node, word


def bow_arrays(bow: dict):
    words = np.array(sorted(bow), np.int32)
    return words, np.array([bow[w] for w in words], np.float64)


# ------------------------------------------------------------------------------------------------------------------ SearchByBoW
def feature_vector(node, angles) -> dict:
    """{node: [key indices ascending]} of the keys with node >= 0 whose angle obeys the angle rule."""
    fv = {}
    for i, v in enumerate(node):
        if v >= 0 and angle_ok(angles[i]):
            fv.setdefault(int(v), []).append(i)
    return fv


def rotation_bin(kf_angle, f_angle, trace=None) -> int:
    rot = F32(kf_angle) - F32(f_angle)
    if rot < F32(0):
        rot = rot + F32(360)
        if trace is not None:
            trace.add("rot_wrap")
    q = rot * (F32(1) / F32(HISTO_LENGTH))
    b = int(round_half_away(q))
    if trace is not None:
        if rot == F32(0):
            trace.add("rot_zero")
        if q == F32(math.floor(q)) + F32(0.5):
            trace.add("bin_half_up")
        if rot == F32(360):
            trace.add("bin_12")
        if b == HISTO_LENGTH:
            trace.add("bin_30_to_0")
    return 0 if b == HISTO_LENGTH else b


def _trace_accept(trace, best1, best2, nnratio, accept):
    bound = nnratio * F32(best2)
    if best2 == 256 and accept:
        trace.add("single_candidate")
    if best1 == TH_LOW and accept:
        trace.add("th_low_50_accept")
    if best1 == TH_LOW + 1 and F32(best1) < bound:
        trace.add("th_low_51_reject")  # the ratio test alone would accept
    if best1 <= TH_LOW and F32(best1) == bound:
        trace.add("ratio_equal_reject")
    if accept and bound == np.nextafter(F32(best1), F32(np.inf)):
        trace.add("ratio_ulp_accept")


def _trace_maxima(trace, counts, keep):
    top = sorted(counts, reverse=True)[:3]  # ComputeThreeMaxima's max1, max2, max3
    trace.add(f"three_maxima_{sum(i >= 0 for i in keep)}")
    tenth = F32(0.1) * F32(top[0])
    if any(0 < m and F32(m) == tenth for m in top[1:]):
        trace.add("tenth_rule_equal")
    if any(0 < m and F32(m) < tenth for m in top[1:]):
        trace.add("tenth_rule_cull")


def search_by_bow(f_kps, f_desc, f_node, kf_kps, kf_desc, kf_node, kf_point, nnratio, check_orientation, trace=None):
    """SearchByBoW(pKF, F, vpMapPointMatches) as the literal loop -> (match int32 per frame key: the point index or -1, nmatches).
    trace: a set that receives the names of the paths taken (SEARCH_PATHS)."""
    fv_f = feature_vector(f_node, f_kps["angle"])
    fv_kf = feature_vector(kf_node, kf_kps["angle"])
    kf_keys, f_keys = sorted(fv_kf), sorted(fv_f)
    if trace is not None:
        if set(f_keys) - set(kf_keys):
            trace.add("node_frame_only")
        if set(kf_keys) - set(f_keys):
            trace.add("node_kf_only")
        if not check_orientation:
            trace.add("no_orientation")
    n = len(f_kps)
    match = np.full(n, -1, np.int32)
    nnratio = F32(nnratio)
    nmatches = 0
    rot_hist = [[] for _ in range(HISTO_LENGTH)]
    a, b = 0, 0
    while a < len(kf_keys) and b < len(f_keys):
        if kf_keys[a] == f_keys[b]:
            for i_kf in fv_kf[kf_keys[a]]:
                p = int(kf_point[i_kf])
                if p < 0:
                    if trace is not None:
                        trace.add("kf_key_no_point")
                    continue
                best1, best_idx, best2 = 256, -1, 256
                for i_f in fv_f[f_keys[b]]:
                    if match[i_f] >= 0:
                        if trace is not None:
                            trace.add("candidate_claimed")
                        continue
                    d = descriptor_distance(kf_desc[i_kf], f_desc[i_f])
                    if trace is not None and d < 256:
                        if d == best1:
                            trace.add("best_tie")    # the earlier candidate stays best
                        elif d == best2:
                            trace.add("second_tie")  # changes nothing
                    if d < best1:
                        best2, best1, best_idx = best1, d, i_f
                    elif d < best2:
                        best2 = d
                accept = best1 <= TH_LOW and F32(best1) < nnratio * F32(best2)
                if trace is not None:
                    _trace_accept(trace, best1, best2, nnratio, accept)
                if accept:
                    match[best_idx] = p
                    if check_orientation:
                        rot_hist[rotation_bin(kf_kps["angle"][i_kf], f_kps["angle"][best_idx], trace)].append(best_idx)
                    nmatches += 1
            a += 1
            b += 1
        elif kf_keys[a] < f_keys[b]:
            a = bisect.bisect_left(kf_keys, f_keys[b])
        else:
            b = bisect.bisect_left(f_keys, kf_keys[a])
    if check_orientation:
        counts = [len(h) for h in rot_hist]
        keep = compute_three_maxima(counts)
        if trace is not None:
            _trace_maxima(trace, counts, keep)
        for i in range(HISTO_LENGTH):
            if i in keep:
                continue
            for j in rot_hist[i]:
                match[j] = -1
                nmatches -= 1
    return match, nmatches
