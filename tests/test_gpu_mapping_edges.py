"""-m gpu: map-point creation (k_map_create / k_map_list / k_kf_gather) on the constructed scenes of oracle/mapping_scene.py through
the oracle, the debug host form, the production host form and the device form, bit for bit; 32 neighbours; the ordered list at
its warp and chunk boundaries and at the capacity; the device form's negative-count rule and optional outputs; the host form
beyond the capacity; a 4-level 1.5x extractor; sivo_keyframe_gather_device's edges; 200 seeded fuzz scenes."""
import numpy as np
import pytest
import torch

from frame_support import KF_FIELDS, extractor, i64, upload
from oracle import mapping_oracle as MO
from oracle import mapping_scene as S
from oracle.keymap import keymap, scatter
from oracle.orb_oracle import ExtractorParams
from sivo_b200.mapping import HostKeyframe, KeyframeKeys, create_map_points, create_map_points_device, keyframe_gather_device, \
    make_params, set_pose
from sivo_b200.orb import KP_DTYPE

pytestmark = pytest.mark.gpu
SCENES = {sc.name: sc for sc in S.constructed_scenes()}
FOUR = ExtractorParams(nfeatures=2000, scale_factor=1.5, nlevels=4)
def host_kf(kf: MO.KeyFrame) -> HostKeyframe:
    return HostKeyframe(kf.kps, kf.desc, kf.u_right, kf.depth, kf.kp_class, kf.kp_conf, kf.kp_entropy, kf.node, kf.has_point, kf.Rcw,
                        kf.tcw, kf.Ow)


def params(max_class=8, th_conf=0.5, th_red=-1e9):
    return make_params(S.FX, S.FY, S.CX, S.CY, S.MBF, S.sigma_cw(), max_class, th_conf, th_red)


def device_kf(kf: MO.KeyFrame, cap, keep, count=None):
    """The keyframe's keys in capacity-sized device buffers, padded with keys in no node."""
    n = len(kf.kps)
    assert n <= cap
    t = {f: upload(scatter(np.asarray(getattr(kf, f), dt), np.arange(n), cap, -1 if f == "node" else 0)) for f, dt in KF_FIELDS.items()}
    t["count"] = i64(n if count is None else count)
    keep.append(t)
    k = KeyframeKeys(*[t[f].data_ptr() for f in ("kps", "desc", "u_right", "depth", "kp_class", "kp_conf", "kp_entropy", "node",
                                                 "has_point", "count")])
    set_pose(k, kf.Rcw, kf.tcw, kf.Ow)
    return k


def device_call(left, d1, dn, prm, want=("nb", "idx", "world", "lst", "n")):
    """sivo_create_map_points_device on its own stream; outputs not in `want` are NULL.  Every output starts at a sentinel."""
    cap = left.capacity()
    o = dict(nb=torch.full((cap,), -7, dtype=torch.int32, device="cuda"), idx=torch.full((cap,), -7, dtype=torch.int32, device="cuda"),
             world=torch.full((cap, 3), 7.0, dtype=torch.float32, device="cuda"),
             lst=torch.full((cap, 2), -7, dtype=torch.int32, device="cuda"), n=torch.full((1,), -7, dtype=torch.int64, device="cuda"))
    ptr = {k: (v.data_ptr() if k in want else 0) for k, v in o.items()}
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    create_map_points_device(left, d1, dn, prm, ptr["nb"], ptr["idx"], ptr["world"], ptr["lst"], ptr["n"], stream.cuda_stream)
    stream.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def as_result(o, n1):
    n = int(o["n"][0])
    return dict(created_nb=o["nb"][:n1], created_idx=o["idx"][:n1], world=o["world"][:n1], created=o["lst"][:max(n, 0)], n_created=n)


def all_forms(kf1, nbs, max_class=8, th_conf=0.5, th_red=-1e9, ext=S.EXTRACTOR, max_exempt=0, device=True):
    """The oracle, the debug and production host forms and the device form, each compared with mapping_scene.compare.  Returns
    (oracle result, debug result, exempt keys)."""
    left = extractor(ext.nfeatures, ext.scale_factor, ext.nlevels)
    want = S.oracle_run(kf1, nbs, th_conf, th_red, max_class, ext)
    prm = params(max_class, th_conf, th_red)
    hk1, hn = host_kf(kf1), [host_kf(k) for k in nbs]
    dbg = create_map_points(left, hk1, hn, prm, debug=True)
    ex = S.compare(dbg, want, th_red, max_exempt)
    S.compare(create_map_points(left, hk1, hn, prm), want, th_red, max_exempt)
    if device:
        keep = []
        cap = left.capacity()
        dev = device_call(left, device_kf(kf1, cap, keep), [device_kf(k, cap, keep) for k in nbs], prm)
        S.compare(as_result(dev, len(kf1.kps)), want, th_red, max_exempt)
        assert (dev["nb"][len(kf1.kps):] == -7).all() and (dev["lst"][max(int(dev["n"][0]), 0):] == -7).all()
    return want, dbg, ex


@pytest.mark.parametrize("name", list(SCENES))
def test_constructed_scene_every_form_equals_the_oracle(name):
    sc = SCENES[name]
    want, dbg, _ = all_forms(sc.kf1, sc.nbs, sc.max_class, sc.th_conf, sc.th_red, sc.ext)
    for k, st in sc.want.items():
        assert dbg["stage"][k] == st, (k, int(dbg["stage"][k]), st)
    for k, m in sc.match.items():
        assert dbg["match"][k] == m, (k, int(dbg["match"][k]), m)
    if sc.flip is not None:
        st = dbg["stage"][0]
        assert (st[1] == sc.flip) != (st[2] == sc.flip) and st[0] == st[1] and st[2] == st[3]


def _disjoint_32(n=256):
    """32 neighbours, neighbour i able to match only the current keys j with 7 j = i (mod 32): every neighbour creates its own
    interleaved set, so the list's neighbour-major order differs from key order."""
    kf1, kf2 = S.pair_scene([S.P0] * n, o2=3)
    nbs = []
    for i in range(32):
        k = MO.KeyFrame(kps=kf2.kps.copy(), desc=kf2.desc.copy(), u_right=kf2.u_right.copy(), depth=kf2.depth.copy(),
                        kp_class=kf2.kp_class.copy(), kp_conf=kf2.kp_conf.copy(), kp_entropy=kf2.kp_entropy.copy(),
                        node=np.where((7 * np.arange(n)) % 32 == i, np.arange(n), -1).astype(np.int32), has_point=kf2.has_point.copy(),
                        Rcw=kf2.Rcw, tcw=kf2.tcw)
        nbs.append(k)
    return kf1, nbs


def test_32_neighbours_disjoint_sets_in_neighbour_major_order():
    kf1, nbs = _disjoint_32()
    want, _, _ = all_forms(kf1, nbs)
    assert len(want["created"]) == 256 and set(want["created"][:, 0]) == set(range(32))
    assert list(want["created"][:, 0]) == sorted(want["created"][:, 0]) and list(want["created"][:, 1]) != sorted(want["created"][:, 1])


def test_32_neighbours_with_empty_and_larger_keyframes():
    cap = extractor().capacity()
    kf1, nbs = S.make_scene(500, 32, seed=30)
    big = S.make_scene(cap, 1, seed=31)[1][0]
    nbs[3] = S.make_scene(0, 1, seed=32)[1][0]
    nbs[17] = S.make_scene(1200, 1, seed=33)[1][0]
    nbs[31] = big
    want, _, _ = all_forms(kf1, nbs, th_red=9.5, max_exempt=5)
    assert len(want["created"]) > 20 and len(np.unique(want["created"][:, 0])) >= 3
    # the device form with the capacity-sized neighbour's count above the capacity: clamped, the same result
    left = extractor()
    keep = []
    d1 = device_kf(kf1, cap, keep)
    dn = [device_kf(k, cap, keep) for k in nbs]
    prm = params(th_red=9.5)
    full = device_call(left, d1, dn, prm)
    keep[-1]["count"].fill_(cap + 5)
    above = device_call(left, d1, dn, prm)
    for k in full:
        assert full[k].tobytes() == above[k].tobytes(), k


def test_device_form_negative_count_and_optional_outputs():
    left = extractor()
    cap = left.capacity()
    kf1, nbs = _disjoint_32()
    keep = []
    d1 = device_kf(kf1, cap, keep)
    dn = [device_kf(k, cap, keep) for k in nbs]
    prm = params()
    full = device_call(left, d1, dn, prm)
    assert int(full["n"][0]) == 256
    # one neighbour's count -1, the first or the last of 32: only n_created = -1, every other output untouched
    for i in (0, 31):
        keep[1 + i]["count"].fill_(-1)
        neg = device_call(left, d1, dn, prm)
        keep[1 + i]["count"].fill_(len(nbs[i].kps))
        assert int(neg["n"][0]) == -1
        assert (neg["nb"] == -7).all() and (neg["idx"] == -7).all() and (neg["world"] == 7.0).all() and (neg["lst"] == -7).all()
    # every optional output NULL but n_created; created_nb NULL with the others given (the call's own scratch)
    only_n = device_call(left, d1, dn, prm, want=("n",))
    assert int(only_n["n"][0]) == 256 and (only_n["nb"] == -7).all() and (only_n["lst"] == -7).all()
    no_nb = device_call(left, d1, dn, prm, want=("idx", "world", "lst", "n"))
    assert (no_nb["nb"] == -7).all()
    for k in ("idx", "world", "lst", "n"):
        assert no_nb[k].tobytes() == full[k].tobytes(), k


def _list_scene(n, made):
    """n pairs at P0, only the current keys in `made` searchable (the others have no node)."""
    kf1, kf2 = S.pair_scene([S.P0] * n, o2=3)
    keep = np.zeros(n, bool)
    keep[list(made)] = True
    kf1.node[~keep] = -1
    return kf1, kf2


@pytest.mark.parametrize("made", ["boundaries", "all", "none"])
def test_ordered_list_at_warp_chunk_and_capacity_boundaries(made):
    """k_map_list (one 1024-thread block walking neighbours x chunks) with created points at j = 0, 31, 32, 1023, 1024, 2047,
    2048 and the capacity - 1; every key up to the capacity created; none created."""
    cap = extractor().capacity()
    sel = {"boundaries": [0, 31, 32, 1023, 1024, 2047, 2048, cap - 1], "all": range(cap), "none": []}[made]
    kf1, kf2 = _list_scene(cap, sel)
    want, _, _ = all_forms(kf1, [kf2])
    assert list(want["created"][:, 1]) == list(sel) and (want["created"][:, 0] == 0).all()


def test_host_form_beyond_the_capacity():
    """The host form does not clamp: three times the capacity against 10 neighbours equals the oracle."""
    cap = extractor().capacity()
    kf1, nbs = S.make_scene(3 * cap, 10, seed=40)
    left = extractor()
    want = S.oracle_run(kf1, nbs)
    prm = params(th_red=9.5)
    dbg = create_map_points(left, host_kf(kf1), [host_kf(k) for k in nbs], prm, debug=True)
    S.compare(dbg, want, 9.5, max_exempt=10)
    S.compare(create_map_points(left, host_kf(kf1), [host_kf(k) for k in nbs], prm), want, 9.5, max_exempt=10)
    assert len(want["created"]) > 500 and want["created"][:, 1].max() >= 2 * cap


def test_four_level_extractor_scene():
    """A 4-level 1.5x extractor's own tables and ratioFactor 2.25, keys drawn at octaves 0-4 (4 is outside its levels)."""
    kf1, nbs = S.make_scene(1500, 4, seed=41)
    rng = np.random.default_rng(41)
    for kf in [kf1] + nbs:
        kf.kps["octave"] = rng.integers(0, 5, len(kf.kps))
    want, _, _ = all_forms(kf1, nbs, th_red=9.5, ext=FOUR, max_exempt=5)
    assert len(want["created"]) > 50


def test_keyframe_gather_edges():
    left = extractor()
    cap = left.capacity()
    rng = np.random.default_rng(42)
    kps = np.zeros(cap, KP_DTYPE)
    kps["x"], kps["y"], kps["octave"] = rng.uniform(0, 900, cap), rng.uniform(0, 300, cap), rng.integers(0, 8, cap)
    desc = rng.integers(0, 256, (cap, 32), dtype=np.uint8)
    ur, depth = rng.uniform(-1, 900, cap).astype(np.float32), rng.uniform(-1, 40, cap).astype(np.float32)
    cls, conf, ent = rng.integers(0, 12, cap).astype(np.uint8), rng.random(cap), rng.random(cap)

    def run(keep_idx, n_keep):
        src = [upload(kps), upload(desc), upload(keep_idx) if keep_idx is not None else None, i64(n_keep), upload(ur), upload(depth),
               upload(cls), upload(conf), upload(ent)]
        out = dict(kps=torch.full((cap * 28,), 0xAB, dtype=torch.uint8, device="cuda"),
                   desc=torch.full((cap, 32), 0xAB, dtype=torch.uint8, device="cuda"), u_right=torch.full((cap,), 7.0, device="cuda"),
                   depth=torch.full((cap,), 7.0, device="cuda"), kp_class=torch.full((cap,), 0xAB, dtype=torch.uint8, device="cuda"),
                   kp_conf=torch.full((cap,), 7.0, dtype=torch.float64, device="cuda"),
                   kp_entropy=torch.full((cap,), 7.0, dtype=torch.float64, device="cuda"),
                   count=torch.full((1,), -7, dtype=torch.int64, device="cuda"))
        torch.cuda.synchronize()
        keyframe_gather_device(left, *[s.data_ptr() if s is not None else 0 for s in src], out)
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in out.items()}

    def check(o, keep_idx, n):
        assert int(o["count"][0]) == n
        k = np.arange(n) if keep_idx is None else np.asarray(keep_idx[:n])
        good = (k >= 0) & (k < cap)
        kc = np.clip(k, 0, cap - 1)
        got = o["kps"].view(KP_DTYPE)
        assert got[:n][good].tobytes() == kps[kc][good].tobytes()
        assert (got[:n][~good]["octave"] == -1).all() and (o["kp_class"][:n][~good] == 255).all()
        assert (o["desc"][:n][~good] == 0).all() and (o["desc"][:n][good] == desc[kc][good]).all()
        assert (o["u_right"][:n] == ur[:n]).all() and (o["depth"][:n] == depth[:n]).all()
        assert (o["kp_class"][:n][good] == cls[kc][good]).all() and (o["kp_conf"][:n][good] == conf[kc][good]).all()
        assert (o["kp_entropy"][:n][good] == ent[kc][good]).all() and (o["kp_conf"][:n][~good] == 0).all()
        assert (o["kp_class"][n:] == 0xAB).all() and (o["u_right"][n:] == 7.0).all()

    check(run(None, 1000), None, 1000)  # keep_idx NULL: the identity
    km = keymap(1000, cap, rng, forced=(0, 5, 999))
    keep_idx = km.keep
    check(run(keep_idx, km.n_keep), keep_idx, km.n_keep)  # rejected entries
    check(run(keep_idx, cap + 50), keep_idx, cap)  # a count above the capacity: clamped
    o = run(keep_idx, -1)  # a negative count writes only the count
    assert int(o["count"][0]) == -1 and (o["kps"] == 0xAB).all() and (o["u_right"] == 7.0).all() and (o["kp_conf"] == 7.0).all()


def _fuzz_scene(seed):
    rng = np.random.default_rng(1000 + seed)
    ext = S.EXTRACTOR if rng.random() < 0.6 else FOUR
    cap = 2000 + 4 * ext.nlevels + 64
    n1 = int(min(cap, np.floor(np.exp(rng.uniform(0, np.log(cap + 1))))))
    n1 = 0 if rng.random() < 0.03 else n1
    nn = int(rng.integers(0, 33))
    # few nodes crowd the candidate lists; the node count grows with the scene so that the oracle's work stays bounded
    n_nodes = max(int(rng.choice([3, 20, 300])), n1 * nn // 400)
    kf1, nbs = S.make_scene(max(n1, 1), nn, seed=seed, n_nodes=n_nodes)
    nl = ext.nlevels
    for kf in [kf1] + nbs:
        n = len(kf.kps)
        kf.kps["octave"] = np.where(rng.random(n) < 0.05, rng.choice([-1, nl], n), rng.integers(0, nl, n))
        kf.depth[rng.random(n) < 0.03] = np.nan
        kf.kp_conf[rng.random(n) < 0.03] = np.nan
        kf.u_right[rng.random(n) < 0.01] = np.nan
    if n1 == 0:
        kf1 = MO.KeyFrame(kps=kf1.kps[:0], desc=kf1.desc[:0], u_right=kf1.u_right[:0], depth=kf1.depth[:0], kp_class=kf1.kp_class[:0],
                          kp_conf=kf1.kp_conf[:0], kp_entropy=kf1.kp_entropy[:0], node=kf1.node[:0], has_point=kf1.has_point[:0],
                          Rcw=kf1.Rcw, tcw=kf1.tcw)
    # neighbour key counts: 0 to the capacity (a neighbour's keys truncated)
    for i, kf in enumerate(nbs):
        m = int(rng.integers(0, len(kf.kps) + 1))
        nbs[i] = MO.KeyFrame(kps=kf.kps[:m], desc=kf.desc[:m], u_right=kf.u_right[:m], depth=kf.depth[:m], kp_class=kf.kp_class[:m],
                             kp_conf=kf.kp_conf[:m], kp_entropy=kf.kp_entropy[:m], node=kf.node[:m], has_point=kf.has_point[:m],
                             Rcw=kf.Rcw, tcw=kf.tcw, Ow=kf.Ow)
    th_conf = float(rng.choice([0.0, rng.uniform(0.2, 1.0), np.nan]))
    th_red = float(rng.choice([-1e9, rng.uniform(6.0, 12.0), np.nan]))
    max_class = int(rng.choice([-1, 2, 8, 254, 255]))
    return kf1, nbs, ext, th_conf, th_red, max_class


def test_fuzz_200_scenes():
    exempt = 0
    for seed in range(200):
        kf1, nbs, ext, th_conf, th_red, max_class = _fuzz_scene(seed)
        try:
            _, _, ex = all_forms(kf1, nbs, max_class, th_conf, th_red, ext, max_exempt=5)
        except AssertionError as e:
            raise AssertionError(f"fuzz scene {seed}") from e
        exempt += ex
    assert exempt <= 30, exempt
