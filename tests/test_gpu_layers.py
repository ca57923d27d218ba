"""-m gpu: every SegNet layer kernel of the product, called through the C-ABI test hooks, against the
oracle and the reference's known-answer vectors."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import conv_bounds as B
from oracle import philox, segnet_oracle as S
from sivo_b200 import _lib as L

pytestmark = pytest.mark.gpu


def interval_violations(x, wt, b, sc, sh, out, gamma, relu=True, half=True, abs_per_input=0.0):
    """Outputs outside the float64 interval of oracle/conv_bounds.py, over the whole output tensor."""
    k = wt.shape[-1]
    extra = abs_per_input * B.conv_abs(np.ones_like(x), wt, k // 2) if abs_per_input else None
    cb = B.ConvBound(x, wt, k // 2, gamma, b, sc, sh, relu=relu, extra=extra)
    lo, hi = cb.half_interval() if half else cb.float_interval()
    bad = B.outside(out, lo, hi)
    ratio, frac = cb.stats(out, half)
    print(f"interval: {int(bad.sum())} of {bad.size} outside, max |out - f(r)| / bound {ratio:.3f}"
          + (f", {frac:.2e} != half_rn(f(r))" if half else ""))
    return int(bad.sum())


def gpu_pool(x):
    n, c, h, w = x.shape
    out = np.empty((n, c, h // 2, w // 2), np.float32)
    mask = np.empty((n, c, h // 2, w // 2), np.int32)
    L.check(L.lib().sivo_dbg_pool(0, L.ptr(x), n, c, h, w, L.ptr(out), L.ptr(mask)))
    return out, mask


def test_pool_first_max_wins_and_mask_index():
    rng = np.random.default_rng(0)
    x = rng.integers(0, 4, size=(2, 8, 6, 10)).astype(np.float32)  # ties everywhere
    out, mask = gpu_pool(x)
    v, m = S.pool_with_mask(torch.from_numpy(x))
    assert np.array_equal(out, v.numpy())
    assert np.array_equal(mask, m.numpy())


def test_upsample_kat_and_round_trip():
    x = np.zeros((1, 8, 2, 2), np.float32)
    m = np.zeros((1, 8, 2, 2), np.int32)
    x[0, :] = [[1, 2], [3, 4]]
    m[0, :] = [[0, 3], [8, 15]]   # one index per 2x2 block (test_upsample_layer.cpp:58-105 uses [2 5 / 12 14])
    m[0, 0] = [[1, 2], [12, 14]]
    out = np.empty((1, 8, 4, 4), np.float32)
    L.check(L.lib().sivo_dbg_unpool(0, L.ptr(x), L.ptr(m), 1, 8, 2, 2, L.ptr(out)))
    ref = S.unpool(torch.from_numpy(x), torch.from_numpy(m.astype(np.int64))).numpy()
    assert np.array_equal(out, ref)
    rng = np.random.default_rng(1)
    y = rng.normal(size=(2, 8, 8, 12)).astype(np.float32)
    v, mk = gpu_pool(y)
    up = np.empty_like(y)
    L.check(L.lib().sivo_dbg_unpool(0, L.ptr(v), L.ptr(mk), 2, 8, 4, 6, L.ptr(up)))
    nz = up != 0
    assert nz.sum() == v.size and np.array_equal(up[nz], y[nz])


def test_lrn_matches_oracle():
    rng = np.random.default_rng(2)
    x = rng.uniform(0, 255, size=(1, 3, 16, 24)).astype(np.float32)
    out = np.empty_like(x)
    L.check(L.lib().sivo_dbg_lrn(0, L.ptr(x), 1, 3, 16, 24, 5, C.c_float(9.99999974738e-05), C.c_float(0.75), C.c_float(1.0),
                                 L.ptr(out)))
    ref = S.lrn_across(torch.from_numpy(x), 5, 9.99999974738e-05, 0.75, 1.0).numpy()
    assert np.allclose(out, ref, rtol=2e-6, atol=1e-5)  # test_lrn_layer.cpp uses 1e-5


def test_dropout_bits_equal_oracle():
    T, Cc, H, W = 3, 192, 5, 7
    keep = np.empty((T, Cc, H, W), np.uint8)
    L.check(L.lib().sivo_dbg_dropout_mask(0, C.c_uint64(0xDEADBEEF12345678), C.c_uint64(41), 5, T, Cc, H, W, L.ptr(keep)))
    ref = philox.dropout_keep(0xDEADBEEF12345678, 41, 5, T, Cc, H, W)
    assert np.array_equal(keep.astype(bool), ref)


def test_mc_reduce_matches_oracle_and_first_max():
    rng = np.random.default_rng(3)
    T, H, W = 6, 9, 33
    logits = rng.normal(0, 3, size=(T, 15, H, W)).astype(np.float32)
    logits[:, :, 0, 0] = 0.0           # exact 15-way tie -> class 0
    logits[:, 3, 0, 1] = 200.0         # saturated softmax -> p = 0 elsewhere -> 0 log 0 := 0
    cls = np.empty((H, W), np.uint8)
    conf = np.empty((H, W), np.float64)
    ent = np.empty((H, W), np.float64)
    L.check(L.lib().sivo_dbg_mc_reduce(0, L.ptr(logits), T, 15, H, W, L.ptr(cls), L.ptr(conf), L.ptr(ent)))
    rc, rf, re = S.mc_reduce(S.softmax_channels(torch.from_numpy(logits)).numpy())
    assert np.array_equal(cls, rc)
    assert cls[0, 0] == 0 and cls[0, 1] == 3 and ent[0, 1] == 0.0
    assert np.abs(conf - rf).max() < 1e-6 and np.abs(ent - re).max() < 1e-5
    assert abs(ent[0, 0] - np.log2(15)) < 1e-6


# T across the 6-sample load batches of k_mc_reduce_quad; C up to 16 on the quad kernel, 17 and 21 on k_mc_reduce_generic
@pytest.mark.parametrize("T", [2, 3, 6, 7, 12, 13, 24])
@pytest.mark.parametrize("Cn", [1, 4, 5, 11, 15, 16, 17, 21])
def test_mc_reduce_sweep_within_float64_bounds(T, Cn):
    rng = np.random.default_rng(100 * T + Cn)
    H, W = 5, 13  # hw = 65: not a multiple of 8
    logits = rng.normal(0, 3, size=(T, Cn, H, W)).astype(np.float32)
    logits[:, :, 0, 2] = rng.uniform(-80, 0, size=(T, Cn)).astype(np.float32)   # spread down to -80 below the max
    logits[:, :, 0, 2][:, 0] = 0.0
    if Cn > 12:  # classes 3 and 12 in different lanes of the quad kernel, identical and on top: 3 wins
        logits[:, :, 0, 0] = -5.0
        logits[:, 3, 0, 0] = logits[:, 12, 0, 0] = 4.0
    if Cn > 5:  # classes 4 and 5 in the same lane
        logits[:, :, 0, 1] = -5.0
        logits[:, 4, 0, 1] = logits[:, 5, 0, 1] = 4.0
    cls = np.empty((H, W), np.uint8)
    conf = np.empty((H, W), np.float64)
    ent = np.empty((H, W), np.float64)
    L.check(L.lib().sivo_dbg_mc_reduce(0, L.ptr(logits), T, Cn, H, W, L.ptr(cls), L.ptr(conf), L.ptr(ent)))
    rc, rf, re = S.mc_reduce(S.softmax_channels(torch.from_numpy(logits)).numpy())
    bc, bconf, bent, conf_b, ent_b, margin = B.map_bounds(logits)
    print(f"mc reduce T={T} C={Cn}: |d conf| {np.abs(conf - bconf).max():.2e} (bound {conf_b.max():.2e}), "
          f"|d entropy| {np.abs(ent - bent).max():.2e} (bound {ent_b.max():.2e})")
    if Cn > 12:
        assert cls[0, 0] == 3
    if Cn > 5:
        assert cls[0, 1] == 4
    sure = margin > 2 * conf_b
    assert np.array_equal(cls[sure], bc[sure])
    assert (np.abs(conf - bconf) <= conf_b).all() and (np.abs(ent - bent) <= ent_b).all()
    assert np.abs(conf - rf).max() < 1e-6 and np.abs(ent - re).max() < 1e-5


@pytest.mark.parametrize("k,cin,cout,prec", [(7, 3, 64, "fp32"), (7, 64, 64, "fp32"), (3, 64, 128, "fp32"), (1, 64, 15, "fp32"),
                                             (3, 3, 64, "fp16"), (7, 64, 64, "fp16"), (3, 128, 64, "fp16"), (3, 64, 15, "fp16")])
def test_conv_simt_matches_oracle(k, cin, cout, prec):
    import torch.nn.functional as F
    rng = np.random.default_rng(4)
    n, h, w = 2, 20, 36
    x = rng.normal(0, 1, size=(n, cin, h, w)).astype(np.float32)
    wt = (rng.normal(0, 1, size=(cout, cin, k, k)) / np.sqrt(cin * k * k)).astype(np.float32)
    b = rng.normal(0, 0.1, size=cout).astype(np.float32)
    sc = (1 + rng.normal(0, 0.1, size=cout)).astype(np.float32)
    sh = rng.normal(0, 0.1, size=cout).astype(np.float32)
    out = np.empty((n, cout, h, w), np.float32)
    L.check(L.lib().sivo_dbg_conv(0, L.ENGINE_SIMT, L.PRECISION_FP32 if prec == "fp32" else L.PRECISION_FP16, L.ptr(x), n, cin, h, w,
                                  L.ptr(wt), L.ptr(b), L.ptr(sc), L.ptr(sh), cout, k, (k - 1) // 2, 1, L.ptr(out)))
    xt, wtt = torch.from_numpy(x), torch.from_numpy(wt)
    if prec == "fp16":
        xt, wtt = xt.half().float(), wtt.half().float()
    ref = F.conv2d(xt, wtt, None, padding=(k - 1) // 2) + torch.from_numpy(b).view(1, -1, 1, 1)
    ref = torch.relu(ref * torch.from_numpy(sc).view(1, -1, 1, 1) + torch.from_numpy(sh).view(1, -1, 1, 1))
    if prec == "fp16" and cout % 8 == 0:
        ref = ref.half().float()
    tol = 1e-4 if prec == "fp32" else 2e-3   # caffe's conv test: 1e-4 vs the naive loop; half storage: 1 ulp = 2^-11 rel
    assert np.abs(out - ref.numpy()).max() < tol * max(1.0, float(ref.abs().max()))
    xs, ws = (x, wt) if prec == "fp32" else (xt.numpy(), wtt.numpy())
    assert interval_violations(xs, ws, b, sc, sh, out, B.gamma_simt(k, cin), half=prec == "fp16" and cout % 8 == 0) == 0


@pytest.mark.parametrize("k,cin,cout,n,h,w", [(7, 64, 64, 1, 8, 128), (7, 64, 64, 2, 22, 200), (3, 64, 64, 1, 16, 128),
                                              (3, 64, 128, 2, 11, 96), (7, 64, 64, 3, 44, 128), (3, 64, 64, 1, 64, 300),
                                              (1, 64, 15, 2, 10, 140), (3, 64, 15, 1, 12, 128), (3, 128, 128, 2, 11, 96),
                                              (3, 256, 64, 1, 22, 64), (3, 512, 512, 2, 11, 32), (1, 128, 64, 1, 6, 130),
                                              # full-size layers: many row blocks per CTA
                                              (7, 64, 64, 2, 176, 512), (7, 64, 64, 1, 352, 300), (3, 64, 64, 1, 160, 512),
                                              (3, 64, 64, 2, 90, 520),
                                              # at most 64 pixels wide, Cin > 64: two images per M tile, kw shift by TMA (PK2)
                                              (3, 128, 128, 3, 22, 64), (3, 512, 512, 12, 22, 64), (3, 256, 256, 2, 11, 33), (3, 128, 64, 5, 6, 20)])
def test_conv_tcgen05_matches_oracle(k, cin, cout, n, h, w):
    """The tensor-core convolution against torch fp32 on identical half-rounded operands; sizes cover partial
    strips (W not a multiple of 128), an odd height, several images, the 16 / 64 / 128-wide wgmma N tiles, and the
    full-size shapes the nets run."""
    import torch.nn.functional as F
    rng = np.random.default_rng(5)
    x = rng.normal(0, 1, size=(n, cin, h, w)).astype(np.float32)
    wt = (rng.normal(0, 1, size=(cout, cin, k, k)) / np.sqrt(cin * k * k)).astype(np.float32)
    b = rng.normal(0, 0.1, size=cout).astype(np.float32)
    sc = (1 + rng.normal(0, 0.1, size=cout)).astype(np.float32)
    sh = rng.normal(0, 0.1, size=cout).astype(np.float32)
    out = np.empty((n, cout, h, w), np.float32)
    L.check(L.lib().sivo_dbg_conv(0, L.ENGINE_TCGEN05, L.PRECISION_FP16, L.ptr(x), n, cin, h, w, L.ptr(wt), L.ptr(b), L.ptr(sc),
                                  L.ptr(sh), cout, k, (k - 1) // 2, 1, L.ptr(out)))
    xt, wtt = torch.from_numpy(x).half().float(), torch.from_numpy(wt).half().float()
    ref = F.conv2d(xt, wtt, None, padding=(k - 1) // 2) + torch.from_numpy(b).view(1, -1, 1, 1)
    ref = torch.relu(ref * torch.from_numpy(sc).view(1, -1, 1, 1) + torch.from_numpy(sh).view(1, -1, 1, 1))
    ref = (ref.half().float() if cout % 8 == 0 else ref).numpy()  # the 15-channel logits layer stays float
    err = np.abs(out - ref)
    assert err.max() < 2e-3 * max(1.0, float(np.abs(ref).max())), float(err.max())
    assert interval_violations(xt.numpy(), wtt.numpy(), b, sc, sh, out, B.gamma_tc(k, cin), half=cout % 8 == 0) == 0


@pytest.mark.parametrize("k,cin,cout,n,h,w", [(7, 64, 64, 2, 22, 200), (3, 64, 64, 1, 16, 128), (3, 64, 128, 2, 11, 96),
                                              (1, 64, 15, 2, 10, 140), (3, 64, 15, 1, 12, 128), (3, 128, 128, 2, 11, 96),
                                              (3, 256, 64, 1, 22, 64), (3, 512, 512, 2, 11, 32), (7, 64, 64, 1, 60, 300)])
def test_conv_tcgen05_split_operand_mode_is_fp32_grade(k, cin, cout, n, h, w):
    """precision fp32 on the tensor-core engine: x = hi + lo, w = hi + lo in half, x*w ~ hi*hi + hi*lo + lo*hi accumulated in fp32
    (registers).  Compared with a float64 convolution of the same fp32 inputs; the bar is caffe's own conv tolerance (1e-4,
    test_convolution_layer.cpp) with two orders of margin, and torch's fp32 convolution is measured next to it."""
    import torch.nn.functional as F
    rng = np.random.default_rng(6)
    x = rng.normal(0, 1, size=(n, cin, h, w)).astype(np.float32)
    wt = (rng.normal(0, 1, size=(cout, cin, k, k)) / np.sqrt(cin * k * k)).astype(np.float32)
    b = rng.normal(0, 0.1, size=cout).astype(np.float32)
    sc = (1 + rng.normal(0, 0.1, size=cout)).astype(np.float32)
    sh = rng.normal(0, 0.1, size=cout).astype(np.float32)
    out = np.empty((n, cout, h, w), np.float32)
    L.check(L.lib().sivo_dbg_conv(0, L.ENGINE_TCGEN05, L.PRECISION_FP32, L.ptr(x), n, cin, h, w, L.ptr(wt), L.ptr(b), L.ptr(sc),
                                  L.ptr(sh), cout, k, (k - 1) // 2, 1, L.ptr(out)))
    xd, wd = torch.from_numpy(x).double(), torch.from_numpy(wt).double()
    ref = F.conv2d(xd, wd, None, padding=(k - 1) // 2) + torch.from_numpy(b).double().view(1, -1, 1, 1)
    ref = torch.relu(ref * torch.from_numpy(sc).double().view(1, -1, 1, 1) + torch.from_numpy(sh).double().view(1, -1, 1, 1)).numpy()
    r32 = F.conv2d(torch.from_numpy(x), torch.from_numpy(wt), None, padding=(k - 1) // 2) + torch.from_numpy(b).view(1, -1, 1, 1)
    r32 = torch.relu(r32 * torch.from_numpy(sc).view(1, -1, 1, 1) + torch.from_numpy(sh).view(1, -1, 1, 1)).numpy()
    scale = max(1.0, float(np.abs(ref).max()))
    err, err32 = float(np.abs(out - ref).max()) / scale, float(np.abs(r32 - ref).max()) / scale
    print(f"split conv k={k} {cin}->{cout}: max err {err:.2e} of scale (torch fp32: {err32:.2e})")
    assert err < 1e-5, err
    assert interval_violations(x, wt, b, sc, sh, out, B.gamma_split(k, cin), half=False, abs_per_input=B.SPLIT_ABS) == 0
