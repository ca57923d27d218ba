"""CPU: the per-element float64 interval checker (oracle/conv_bounds.py) checks itself.  It must accept the correctly rounded
result and an fp32 result summed in another order, and reject each of a list of realistic kernel bugs applied to the
reference -- otherwise the GPU walk in test_gpu_layer_bounds.py would prove nothing."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import conv_bounds as B
from oracle import philox

N, CIN, COUT, H, W, K = 2, 64, 64, 10, 160, 7  # 160 px: two 128-pixel strips


def _h(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


@pytest.fixture(scope="module")
def layer():
    rng = np.random.default_rng(11)
    x = np.maximum(_h(rng.normal(0, 1, size=(N, CIN, H, W))), 0)  # ReLU'd half activations, a quarter of them 0
    x = np.where(rng.random(x.shape) < 0.3, 0, x).astype(np.float32)
    w = _h(rng.normal(0, 1, size=(COUT, CIN, K, K)) / np.sqrt(CIN * K * K))
    b = rng.normal(0, 0.1, size=COUT).astype(np.float32)
    sc = (1 + rng.normal(0, 0.1, size=COUT)).astype(np.float32)
    sc[3] = -0.7  # a negative BN scale: f decreasing
    sh = rng.normal(0, 0.1, size=COUT).astype(np.float32)
    cb = B.ConvBound(x, w, K // 2, B.gamma_tc(K, CIN), b, sc, sh, relu=True)
    return x, w, b, sc, sh, cb


def _epi(acc, b, sc, sh, relu=True):
    t = acc + b.reshape(1, -1, 1, 1)
    if sc is not None:
        t = t * sc.reshape(1, -1, 1, 1) + sh.reshape(1, -1, 1, 1)
    return np.maximum(t, 0) if relu else t


def _rejected(out, cb):
    lo, hi = cb.half_interval()
    return int(B.outside(out, lo, hi).sum())


def test_accepts_the_rounded_reference(layer):
    *_, cb = layer
    assert _rejected(B.half_rn(cb.center()), cb) == 0
    lo, hi = cb.float_interval()
    assert not B.outside(cb.center(), lo, hi).any()


def test_accepts_fp32_in_another_summation_order(layer):
    x, w, b, sc, sh, cb = layer
    acc = F.conv2d(torch.from_numpy(x), torch.from_numpy(w), padding=K // 2).numpy()     # float32, torch's order
    acc_t = F.conv2d(torch.from_numpy(x).transpose(2, 3).contiguous(), torch.from_numpy(w).transpose(2, 3).contiguous(),
                     padding=K // 2).transpose(2, 3).numpy()                                 # other tap order
    for a in (acc, acc_t):
        out = B.half_rn(_epi(a.astype(np.float32), b, sc, sh).astype(np.float32))
        assert _rejected(out, cb) == 0
    ratio, frac = cb.stats(B.half_rn(_epi(acc, b, sc, sh)))
    assert ratio <= 1 and frac < 0.05


def test_rejects_mirrored_kw_taps_of_one_channel(layer):
    x, w, b, sc, sh, cb = layer
    wm = w.copy()
    wm[5] = wm[5][:, :, ::-1]
    out = B.half_rn(_epi(B.conv64(x, wm, K // 2), b, sc, sh))
    assert _rejected(out, cb) > 0


def test_rejects_a_dropped_bias(layer):
    x, w, b, sc, sh, cb = layer
    bm = b.copy()
    bm[9] = 0
    assert _rejected(B.half_rn(_epi(cb.r, bm, sc, sh)), cb) > 0


def test_rejects_bn_applied_as_acc_plus_bias_plus_shift_times_scale(layer):
    x, w, b, sc, sh, cb = layer
    t = (cb.r + b.reshape(1, -1, 1, 1) + sh.reshape(1, -1, 1, 1)) * sc.reshape(1, -1, 1, 1)
    assert _rejected(B.half_rn(np.maximum(t, 0)), cb) > 0


def test_rejects_input_shifted_across_the_strip_boundary(layer):
    x, w, b, sc, sh, cb = layer
    xm = x.copy()
    xm[:, :, :, 128:-1] = x[:, :, :, 129:]  # the second strip reads its halo one pixel off
    out = B.half_rn(_epi(B.conv64(xm, w, K // 2), b, sc, sh))
    bad = B.outside(out, *cb.half_interval())
    assert bad.any() and not bad[..., :125].any()


def test_rejects_keep_bits_of_the_next_sample(layer):
    *_, cb = layer
    lo, hi = cb.half_interval()
    v = B.half_rn(cb.center())
    keep = philox.dropout_keep(1234, 3, 2, N + 1, COUT, H, W)
    right = v * 2 * keep[:N]
    wrong = v * 2 * keep[1:]
    assert not B.check_dropped(right, keep[:N], lo, hi).any()
    assert B.check_dropped(wrong, keep[:N], lo, hi).any()


def _pool(v, last=False):
    n, c, h, w = v.shape
    win = B._windows(v)
    code = np.argmax(win[..., ::-1], axis=-1) if last else np.argmax(win, axis=-1)
    if last:
        code = 3 - code
    val = np.take_along_axis(win, code[..., None], -1)[..., 0]
    yy = np.arange(h // 2).reshape(1, 1, -1, 1)
    xx = np.arange(w // 2).reshape(1, 1, 1, -1)
    return val, (2 * yy + code // 2) * w + 2 * xx + code % 2


def test_pool_first_max_accepted_and_last_of_ties_rejected(layer):
    *_, cb = layer
    lo, hi = cb.half_interval()
    v = B.half_rn(cb.center())
    val, mask = _pool(v)
    assert not B.check_pool(val, mask, lo, hi).any()
    assert (np.all(B._windows(hi) == 0, axis=-1)).any()  # all-zero windows occur
    val2, mask2 = _pool(v, last=True)
    assert B.check_pool(val2, mask2, lo, hi).any()
    assert B.check_mask_only(mask2, lo, hi).any() and not B.check_mask_only(mask, lo, hi).any()
    neg = val.copy()
    neg[val == 0] = -0.0  # a ReLU that leaves -0: the all-zero windows must pool to +0
    assert B.check_pool(neg, mask, lo, hi).any()


def test_unpooled_parts_round_trip(layer):
    *_, cb = layer
    v = B.half_rn(cb.center())
    val, mask = _pool(v)
    up = torch.zeros(v.shape, dtype=torch.float64).view(N, COUT, -1)
    up.scatter_(2, torch.from_numpy(mask.reshape(N, COUT, -1)), torch.from_numpy(val.reshape(N, COUT, -1)))
    sel, others = B.unpooled_parts(up.view(v.shape).numpy(), mask)
    assert np.array_equal(sel, val) and others.all()
    up2 = up.view(v.shape).numpy().copy()
    up2[0, 0, 0, 0] = up2[0, 0, 0, 1] = 1.0
    assert not B.unpooled_parts(up2, mask)[1].all()


def test_composed_classifier_bound_and_the_half_w_mutation():
    """The composed weights built from half(W) instead of the raw float W.  With these weights the mutation is caught only
    at the margin of the bound: a fraction of a percent of the logits fall outside, by up to about 1.3x the bound, while
    most lie well inside gamma * S.  The test asserts that it is caught here and prints how much; a composition error of
    this size can sit wholly inside the bound for other weights, and the checker is not loosened to catch it."""
    rng = np.random.default_rng(12)
    x = np.maximum(_h(rng.normal(0, 1, size=(1, 64, 12, 40))), 0)
    Wd = (rng.normal(0, 1, size=(64, 64, 7, 7)) / np.sqrt(64 * 49)).astype(np.float32)
    bd = rng.normal(0, 0.1, size=64).astype(np.float32)
    wc = (rng.normal(0, 1, size=(15, 64)) / 8).astype(np.float32)
    bc = rng.normal(0, 0.1, size=15).astype(np.float32)
    wh, bias, _, _ = B.compose_classifier(Wd, bd, wc, bc)
    cb = B.ConvBound(x, wh, 3, B.gamma_tc(7, 64), bias)
    lo, hi = cb.float_interval()
    assert not B.outside(cb.center().astype(np.float32), lo, hi).any()
    wm, _, _, _ = B.compose_classifier(_h(Wd), bd, wc, bc)
    mutated = _epi(B.conv64(x, wm, 3), bias.astype(np.float32), None, None, relu=False)
    out = B.outside(mutated, lo, hi)
    print(f"half(W) composition: {out.mean():.2%} of the logits outside, largest |out - f(r)| / bound "
          f"{float((np.abs(mutated - cb.center()) / cb.e).max()):.2f}")
    assert out.any()


def test_map_bounds_hold_for_float32_softmax():
    rng = np.random.default_rng(13)
    logits = rng.normal(0, 3, size=(5, 15, 6, 7)).astype(np.float32)
    logits[:, :, 0, 0] = 0
    logits[:, 2, 0, 1] = -80
    cls, conf, ent, conf_b, ent_b, margin = B.map_bounds(logits)
    lt = torch.from_numpy(logits)
    p = torch.softmax(lt, dim=1).double().mean(0).numpy()
    with np.errstate(divide="ignore", invalid="ignore"):
        e = -np.where(p > 0, p * np.log2(p.astype(np.float32).astype(np.float64)), 0).sum(0)
    assert (np.abs(p.max(0) - conf) <= conf_b).all() and (np.abs(e - ent) <= ent_b).all()
    print(f"map bounds: confidence {conf_b.max():.2e}, entropy {ent_b.max():.2e}")
    assert conf_b.max() < 2e-6 and ent_b.max() < 2e-5
    assert cls[0, 0] == 0
