"""TEST INFRASTRUCTURE -- per-element float64 bounds for the device convolutions and the exact layers fused around them.
Never imported by the product path.

A convolution on the device cannot be compared bit for bit with a host reference: the host and the tensor core sum in
different orders, and the tensor core's accumulator add truncates (DESIGN §4.3).  What can be promised is an interval per
output element, derived from the kernel's arithmetic and not from a measurement.

Reference.  For the exact operands the device used (its half-rounded activations and weights; in the split-operand mode
the fp32 values), `r` = the float64 convolution and `S` = sum |x| |w| over the same taps (float32, scaled by 1 + 1e-3: it
is only a bound).  The device accumulator then satisfies |acc - r| <= gamma * S with gamma from the longest chain of fp32
accumulator adds per output element:

  * k_conv_tc / k_conv_stack (fp16 operands, fp32 accumulators).  Half x half products are exact in fp32.  One wgmma
    K step adds 16 products to the accumulator; the tensor core aligns the addends to the largest exponent and truncates
    (DESIGN §4.3), so one step loses less than one fp32 ulp of the largest addend to the alignment and less than one to
    the final truncation: <= 2 * 2^-23 * (|acc| + sum |p|) per step, and |acc| <= S.  The chain is K^2 taps x
    ceil(Cin / 16) steps (k_conv_stack adds in the same order, DESIGN §4.1; the window-folded first layer has K tap rows of
    64 folded channels, K x 4 steps):  gamma = 2^-22 * steps * (1 + 1e-3).
  * Split-operand fp32 mode (DESIGN §4.3): x = x_hi + x_lo and w 2^s = w_hi + w_lo in half; x_lo and w_lo are rounded to
    half (relative 2^-11 of a remainder that is itself <= 2^-11 of the value: 2^-22 each), the term x_lo w_lo (<= 2^-22
    |x w|) is dropped.  That is 3 * 2^-22 per product, plus, where x_lo falls into half's subnormal range, an absolute
    2^-25 per input (the weights are pre-scaled out of it), charged as SPLIT_ABS * sum |w|.  Accumulation: segments of at most
    m steps with the truncating add (2^-22 per step as above), each scaled by 1 + 0.216 * 2^-23 * m (< 2^-23 * m) and
    summed with round-to-nearest FMAs (2^-24 per segment, 2 Cin/64 * K segments):
    gamma = 3 * 2^-22 + (2.216 * m + segments / 2 + 1) * 2^-23, with m = 2 * 4 * K (the hi chunk meets two weight tiles).
  * k_conv_simt (fp32 FMA engine): one round-to-nearest FMA chain of Cin * K^2 terms, gamma = 2^-24 * terms * (1 + 1e-3).

Input uncertainty.  Where the device's own input to a layer is not stored (the LRN output inside k_input_lrn_pad8), the
input is an interval [lo, hi] of adjacent halves only where the float64 value lies within the device's float error of a
half rounding boundary; the convolution uses the midpoint and adds sum |w| (hi - lo) / 2 over those inputs only.

Epilogue.  bias -> BN (mul, then add) -> ReLU in float, possibly contracted (conv_tc.cu is not built with -fmad=false):
the interval [r - e, r + e] is carried through each operation in float64 and widened by 2 fp32 ulps of every
intermediate; a negative BN scale swaps the ends.  Half outputs: half_rn(lo) <= out <= half_rn(hi) -- half rounding is
monotone, so this is exact.  Float outputs (logits): lo <= out <= hi.

Pool, unpool and dropout move half values exactly, so they are checked bit for bit against that interval model
(`check_pool`, `check_unpooled`): first maximum in scan order (0,0), (0,1), (1,0), (1,1) with a strict '>', an all-zero
window gives +0 and code 0 (Caffe's first-max rule on ReLU zeros), non-selected positions are +0, dropped ones 0, kept
ones exactly 2 x the half value.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

U23 = 2.0 ** -23  # fp32 ulp of 1
SPLIT_ABS = 2.0 ** -25  # split mode: absolute error per input of a subnormal x_lo
_BAND_BYTES = 1 << 28  # float64 im2col budget of one band of output rows


def gamma_tc(k, cin, folded=False):
    steps = (k if folded else k * k) * math.ceil(cin / 16)
    return 2.0 * U23 * steps * (1 + 1e-3)


def gamma_split(k, cin):
    m = 2 * 4 * k
    segments = 2 * (cin // 64) * k
    return (3 * 2.0 ** -22 + (2.216 * m + segments / 2 + 1) * U23) * (1 + 1e-3)


def gamma_simt(k, cin):
    return 0.5 * U23 * cin * k * k * (1 + 1e-3)


def half_rn(x):
    """IEEE half, round to nearest even, of float64 values (numpy converts double -> half directly, one rounding)."""
    return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def conv64(x, w, pad):
    """float64 convolution of x [N, Cin, H, W] with w [Cout, Cin, K, K], 'same' zero padding, in bands of output rows so
    that torch's im2col stays within a few hundred MB at full size."""
    x = torch.as_tensor(np.asarray(x, np.float64))
    wt = torch.as_tensor(np.asarray(w, np.float64))
    n, cin, h, wd = x.shape
    k = wt.shape[-1]
    xp = F.pad(x, (pad, pad, pad, pad))
    band = max(1, _BAND_BYTES // (8 * cin * k * k * (wd + 2 * pad)))
    out = torch.empty((n, wt.shape[0], h, wd), dtype=torch.float64)
    with torch.no_grad():
        for i in range(n):
            for y0 in range(0, h, band):
                y1 = min(h, y0 + band)
                out[i:i + 1, :, y0:y1] = F.conv2d(xp[i:i + 1, :, y0:y1 + 2 * pad], wt)
    return out.numpy()


def conv_abs(x, w, pad):
    """S = sum |x| |w| over the taps, float32, scaled by 1 + 1e-3 (an upper bound, not a value)."""
    with torch.no_grad():
        s = F.conv2d(torch.as_tensor(np.abs(np.asarray(x, np.float32))), torch.as_tensor(np.abs(np.asarray(w, np.float32))),
                     padding=pad)
    return s.numpy().astype(np.float64) * (1 + 1e-3)


class ConvBound:
    """One convolution's float64 reference r, accumulator bound e and epilogue (bias, BN scale / shift, ReLU)."""

    def __init__(self, x, w, pad, gamma, bias=None, scale=None, shift=None, relu=False, x_radius=None, extra=None):
        self.r = conv64(x, w, pad)
        self.e = gamma * conv_abs(x, w, pad)
        if x_radius is not None:  # inputs known only to within +-x_radius (0 where exact)
            self.e += conv_abs(x_radius, w, pad) / (1 + 1e-3)
        if extra is not None:
            self.e += extra
        cout = self.r.shape[1]
        self.bias = np.zeros(cout) if bias is None else np.asarray(bias, np.float32).astype(np.float64)
        self.scale = None if scale is None else np.asarray(scale, np.float32).astype(np.float64)
        self.shift = None if shift is None else np.asarray(shift, np.float32).astype(np.float64)
        self.relu = relu

    def _f(self, lo, hi, ulps):
        def ch(v):
            return v.reshape(1, -1, 1, 1)

        def widen(a, b):
            s = ulps * ulp32(np.maximum(np.abs(a), np.abs(b)))
            return a - s, b + s

        lo, hi = widen(lo + ch(self.bias), hi + ch(self.bias))
        if self.scale is not None:
            a, b = lo * ch(self.scale), hi * ch(self.scale)
            lo, hi = widen(np.minimum(a, b), np.maximum(a, b))
            lo, hi = widen(lo + ch(self.shift), hi + ch(self.shift))
        if self.relu:
            lo, hi = np.maximum(lo, 0.0), np.maximum(hi, 0.0)
        return lo, hi

    def center(self):
        """f(r) in float64, no rounding."""
        return self._f(self.r, self.r, 0)[0]

    def float_interval(self):
        return self._f(self.r - self.e, self.r + self.e, 2)

    def half_interval(self):
        lo, hi = self.float_interval()
        return half_rn(lo), half_rn(hi)

    def stats(self, out, half=True):
        """(largest |out - f(r)| relative to the room the output interval leaves on that side of f(r) -- <= 1 inside the
        bound; fraction of half outputs != half_rn(f(r))) -- numbers to compare kernels by."""
        lo, hi = self.half_interval() if half else self.float_interval()
        return interval_stats(out, self.center(), lo, hi, half)


def interval_stats(out, c, lo, hi, half=True):
    """(largest |out - c| relative to the room [lo, hi] leaves on that side of c, fraction of outputs != half_rn(c))."""
    d = np.asarray(out, np.float64) - c
    room = np.where(d >= 0, hi - c, c - lo)
    ratio = float(np.where(d == 0, 0.0, np.where(room > 0, np.abs(d) / np.where(room > 0, room, 1), np.inf)).max())
    return ratio, (float((np.asarray(out) != half_rn(c)).mean()) if half else float("nan"))


def at_mask(a, mask):
    """The entries [N, C, h, w] of a full-resolution tensor [N, C, 2h, 2w] that Caffe plane indices `mask` name."""
    h, w = mask.shape[2], mask.shape[3]
    k = np.clip(mask_codes(mask, 2 * w), 0, 3)[..., None]
    return np.take_along_axis(_windows(np.asarray(a)[:, :, :2 * h, :2 * w]), k, -1)[..., 0]


def outside(out, lo, hi):
    """Boolean mask of the outputs outside [lo, hi] (NaN counts as outside)."""
    out = np.asarray(out, np.float64)
    return ~((out >= lo) & (out <= hi))


def is_pos_zero(v):
    return (np.asarray(v) == 0) & ~np.signbit(v)


def mask_codes(mask, w_full):
    """Caffe's plane index of a 2x2 window's argmax -> scan-order code 2 dy + dx (-1 where it is not in the window)."""
    mask = np.asarray(mask).astype(np.int64)
    n, c, h, w = mask.shape
    yy = np.arange(h).reshape(1, 1, -1, 1)
    xx = np.arange(w).reshape(1, 1, 1, -1)
    dy, dx = mask // w_full - 2 * yy, mask % w_full - 2 * xx
    code = 2 * dy + dx
    return np.where((dy >= 0) & (dy <= 1) & (dx >= 0) & (dx <= 1), code, -1)


def _windows(a):
    """[N, C, 2h, 2w] -> [N, C, h, w, 4] in scan order (0,0), (0,1), (1,0), (1,1)."""
    return np.stack([a[:, :, 0::2, 0::2], a[:, :, 0::2, 1::2], a[:, :, 1::2, 0::2], a[:, :, 1::2, 1::2]], axis=-1)


def check_pool(v, mask, lo, hi, valid=None):
    """Boolean mask [N, C, h, w] of pooled outputs that the interval model rejects.  v: pooled half values, mask: Caffe plane
    indices, lo / hi: the half interval of the full-resolution input [N, C, 2h, 2w] (odd trailing rows / columns ignored).
    `valid` restricts the value checks (e.g. to the elements dropout kept); the mask is checked everywhere it can be."""
    h, w = v.shape[2], v.shape[3]
    lo, hi = lo[:, :, :2 * h, :2 * w], hi[:, :, :2 * h, :2 * w]
    code = mask_codes(mask, 2 * w)
    bad = code < 0
    k = np.clip(code, 0, 3)[..., None]
    L, H = _windows(lo), _windows(hi)
    v4 = np.asarray(v, np.float64)[..., None]
    sel_lo = np.take_along_axis(L, k, -1)[..., 0]
    sel_hi = np.take_along_axis(H, k, -1)[..., 0]
    vv = v4[..., 0]
    bad_val = ~((vv >= sel_lo) & (vv <= sel_hi))
    idx = np.arange(4)
    before = idx < k
    after = idx > k
    bad_val |= np.any(before & ~(L < v4), axis=-1)     # an earlier entry that could not have lost to it
    bad_val |= np.any(after & ~(L <= v4), axis=-1)     # a later entry that must have beaten it
    zero = np.all(H == 0, axis=-1)
    bad_val |= zero & ~(is_pos_zero(v) & (code == 0))
    if valid is not None:
        bad_val &= valid
        bad |= zero & (code != 0)
    return bad | bad_val


def check_mask_only(mask, lo, hi):
    """Pooling decisions whose value was not kept (dropped by dropout): the named entry must be able to be the first
    maximum, i.e. some v in its interval beats every earlier entry strictly and no later one."""
    h, w = mask.shape[2], mask.shape[3]
    lo, hi = lo[:, :, :2 * h, :2 * w], hi[:, :, :2 * h, :2 * w]
    code = mask_codes(mask, 2 * w)
    k = np.clip(code, 0, 3)[..., None]
    L, H = _windows(lo), _windows(hi)
    top = np.take_along_axis(H, k, -1)  # the largest value the named entry can have
    idx = np.arange(4)
    bad = np.any((idx < k) & ~(L < top), axis=-1) | np.any((idx > k) & ~(L <= top), axis=-1)
    zero = np.all(H == 0, axis=-1)
    return (code < 0) | bad | (zero & (code != 0))


def unpooled_parts(up, mask):
    """Splits an unpooled tensor [N, C, 2h, 2w] by its mask [N or 1, C, h, w]: (the value at each mask position [N, C, h, w],
    boolean [N, C, h, w]: every other position of the window is +0 bit for bit)."""
    n = up.shape[0]
    mask = np.asarray(mask)
    if mask.shape[0] != n:
        mask = np.broadcast_to(mask[:1], (n,) + mask.shape[1:])
    h, w = mask.shape[2], mask.shape[3]
    code = mask_codes(mask, up.shape[3])
    W4 = _windows(np.asarray(up)[:, :, :2 * h, :2 * w])
    k = np.clip(code, 0, 3)[..., None]
    sel = np.take_along_axis(W4, k, -1)[..., 0]
    others = np.all(np.where(np.arange(4) == k, True, is_pos_zero(W4)), axis=-1) & (code >= 0)
    return sel, others


def check_dropped(sel, keep, lo, hi, half=True):
    """Values after dropout (x keep x 2): boolean mask of the rejected elements.  A dropped element must be 0 (-0 where
    the value was negative: IEEE x * 0), a kept one 2 x a value within [lo, hi] (a half value when `half`)."""
    half_v = np.asarray(sel, np.float64) / 2
    kept_bad = outside(half_v, lo, hi)
    if half:
        kept_bad |= half_rn(half_v) != half_v
    return np.where(keep, kept_bad, np.asarray(sel) != 0)


def lrn_interval(x_bgr_planar, size, alpha, beta, k, rel=2e-6):
    """Half interval of Caffe's cross-channel LRN of [N, 3, H, W] u8-valued input as the device rounds it once to half from
    float arithmetic (powf: a few ulps): returns (mid, radius) with radius 0 where both ends round to the same half."""
    x = np.asarray(x_bgr_planar, np.float64)
    c = x.shape[1]
    pre = (size - 1) // 2
    sq = np.pad(x * x, ((0, 0), (pre, size - 1 - pre), (0, 0), (0, 0)))
    acc = sum(sq[:, i:i + c] for i in range(size))
    v = x * (k + acc * (alpha / size)) ** (-beta)
    lo, hi = half_rn(v * (1 - rel)), half_rn(v * (1 + rel))
    return (lo + hi) / 2, (hi - lo) / 2


def compose_classifier(W, b, wc, bc):
    """Basic's conv_decode1 x classifier as the library composes it: W'[o] = sum_c wc[o, c] W[c] in double (c ascending),
    rounded to float, then to half; bias Wc b + bc in double (from bc, c ascending), rounded to float.  Also returns the
    exact float64 composition, for the two-layer check."""
    W = np.asarray(W, np.float32).astype(np.float64)
    wc = np.asarray(wc, np.float32).astype(np.float64).reshape(wc.shape[0], -1)
    acc = np.zeros((wc.shape[0],) + W.shape[1:])
    bacc = np.asarray(bc, np.float32).astype(np.float64).copy()
    for c in range(W.shape[0]):
        acc += wc[:, c, None, None, None] * W[c]
        bacc += wc[:, c] * float(np.float32(b[c]))
    wh = acc.astype(np.float32).astype(np.float16).astype(np.float64)
    return wh, bacc.astype(np.float32).astype(np.float64), acc, bacc


def map_bounds(logits):
    """Float64 maps of the device's logits [T, C, H, W] and per-pixel bounds on the device's confidence and entropy.
    Per sample the device computes e_k = exp(x_k - m) with __expf (2 + 1.173 |x_k - m| ulps, CUDA's documented bound,
    which also covers expf's 2 ulps; the float subtraction moves the argument by <= 2^-24 |x_k - m|): a relative error
    d_k = 2^-24 * 3.35 |x_k - m| + 2^-22.  The float sum of positive terms is then off by at most sum_k p_k d_k relative,
    plus (C + 2) rounded adds; one reciprocal and one product (or one division) add 2 * 2^-24.  So each probability is
    within p_c * delta_c, delta_c = d_c + sum_k p_k d_k + 2^-24 (C + 4).  The mean over T is in double.  The entropy term
    -p log2 p moves by |dp| (|log2 p| + 1 / ln 2), and log2f of the float-rounded mean adds p (2^-24 / ln 2 + 2^-23 |log2 p|).
    The |x - m| part of __expf's error is what makes these bounds larger than a plain few-ulp estimate: classes some units
    below the maximum carry tens of ulps."""
    x = np.asarray(logits, np.float64)
    T, C = x.shape[:2]
    m = x.max(axis=1, keepdims=True)
    e = np.exp(x - m)
    p = e / e.sum(axis=1, keepdims=True)
    d = 2.0 ** -24 * 3.35 * np.abs(x - m) + 2.0 ** -22
    delta = d + (p * d).sum(axis=1, keepdims=True) + 2.0 ** -24 * (C + 4)
    dp = (p * delta).sum(axis=0) / T * (1 + 1e-6) + 1e-300
    pm = p.mean(axis=0)
    with np.errstate(divide="ignore", invalid="ignore"):
        lg = np.where(pm > 0, np.log2(pm), 0.0)
    ent = -(pm * lg).sum(axis=0)
    ent_b = (dp * (np.abs(lg) + 1 / math.log(2))).sum(axis=0) + (pm * (2.0 ** -24 / math.log(2) + 2.0 ** -23 * np.abs(lg))).sum(axis=0)
    cls = np.argmax(pm, axis=0)
    srt = np.sort(pm, axis=0)
    margin = srt[-1] - srt[-2] if C > 1 else np.full(pm.shape[1:], np.inf)
    conf_b = dp.max(axis=0)
    return cls, pm.max(axis=0), ent, conf_b, ent_b + 1e-15, margin
