"""-m gpu: every launch of the default (fused, benchmarked) Basic fp16 build held to the per-element float64 interval of
oracle/conv_bounds.py, launch by launch.  Each launch is checked from the device's own input blobs, so no error carries
over from one layer to the next; the dropout keep bits come from oracle/philox.py.  Pool, unpool and dropout are checked
bit for bit against the interval model.  Every check prints the largest |out - f(r)| relative to its bound and the
fraction of half outputs that differ from half_rn(f(r)), for later kernel changes to compare against."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import make_model
from oracle import conv_bounds as B
from oracle import philox
from oracle import segnet_oracle as S
from sivo_b200 import BayesianSegNet, BayesianSegNetParams
from sivo_b200 import _lib as L
from sivo_b200.synth import stereo_frame

pytestmark = pytest.mark.gpu

SEED, FRAME = 1234, 3


def _h(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def _report(name, bad, cb=None, out=None, half=True):
    msg = f"{name}: {int(np.sum(bad))} of {np.size(bad)} outside"
    if cb is not None:
        ratio, frac = cb.stats(out, half)
        msg += f", max |out - f(r)| / bound {ratio:.3f}" + (f", {frac:.2e} != half_rn(f(r))" if half else "")
    print(msg)
    assert not np.any(bad), msg


def _unpool(v, mask):
    v = torch.from_numpy(np.ascontiguousarray(v))
    m = torch.from_numpy(np.asarray(mask).astype(np.int64))
    if m.shape[0] != v.shape[0]:
        m = m.expand(v.shape[0], -1, -1, -1)
    return S.unpool(v, m).numpy()


def _conv(weights, name, x, relu=True, gamma=None, **kw):
    w, b = weights[name][0], weights[name][1]
    return B.ConvBound(x, _h(w), w.shape[-1] // 2, gamma or B.gamma_tc(w.shape[-1], w.shape[1]), b, relu=relu, **kw)


def _pool_stats(name, bad, cb, v, mask, keep=None):
    """_report for a pooled launch: the stats of the pooled values against the conv interval of the entries they name."""
    lo, hi = cb.half_interval()
    c, lo, hi = (B.at_mask(np.broadcast_to(a, (mask.shape[0],) + a.shape[1:]), mask) for a in (cb.center(), lo, hi))
    sel = np.ones(v.shape, bool) if keep is None else keep
    ratio, frac = B.interval_stats(v[sel], c[sel], lo[sel], hi[sel])
    msg = f"{name}: {int(np.sum(bad))} of {np.size(bad)} outside, max |out - f(r)| / bound {ratio:.3f}, {frac:.2e} != half_rn(f(r))"
    print(msg)
    assert not np.any(bad), msg


def _keep(layer, T, shape):
    return philox.dropout_keep(SEED, FRAME, layer, T, *shape[1:])


def _bcast(a, T):
    return np.broadcast_to(a, (T,) + a.shape[1:]) if a.shape[0] != T else a


def walk_basic(model_dir, H, W, T, only_tail=False):
    net, weights, proto, model = make_model(model_dir, "basic", T=T, H=H, W=W, seed=0)
    left, _ = stereo_frame(0)
    img = S.center_crop(left, W, H)
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=SEED, T=T, precision="fp16")
    seg.set_frame(FRAME)
    cls, conf, ent = seg.segmentImage(img)
    names = [n for n, _, _ in seg.op_timings()]
    for want in ("input+norm+conv1/pad8", "conv1+pool1"):
        assert want in names, names
    assert any(n.endswith("+decdrop4+upsample3") for n in names), names
    assert "upsample1+conv_decode1*dense_softmax_inner_prod" in names, names
    blob = seg.blob
    tag = f"basic {H}x{W} T={T}"

    if not only_tail:
        # k_input_lrn_pad8 -> window-folded conv1 -> pool1: from the u8 image; the LRN output is not stored, so the
        # inputs within the device's float error of a half rounding boundary carry their interval into the bound
        norm = net.layers[0]
        x0 = np.ascontiguousarray(img.transpose(2, 0, 1))[None].astype(np.float64)
        mid, rad = B.lrn_interval(x0, norm.local_size, norm.alpha, norm.beta, norm.k)
        cb = _conv(weights, "conv1", mid, gamma=B.gamma_tc(7, 64, folded=True), x_radius=rad)
        lo, hi = cb.half_interval()
        p1, m1 = blob("pool1"), blob("pool1_mask")
        _pool_stats(f"{tag} conv1+pool1", B.check_pool(p1, m1, lo, hi), cb, p1, m1)

        # conv2 -> pool2
        cb = _conv(weights, "conv2", p1)
        lo, hi = cb.half_interval()
        p2, m2 = blob("pool2"), blob("pool2_mask")
        _pool_stats(f"{tag} conv2+pool2", B.check_pool(p2, m2, lo, hi), cb, p2, m2)

        # conv3 -> pool3 -> encdrop3 (in place: blob('pool3') is the dropped tensor, batch T; the mask batch 1)
        cb = _conv(weights, "conv3", p2)
        lo, hi = (_bcast(a, T) for a in cb.half_interval())
        p3, m3 = blob("pool3"), blob("pool3_mask")
        k3 = _keep(0, T, p3.shape)
        bad = B.check_pool(p3 / 2, _bcast(m3, T), lo, hi, valid=k3)
        bad |= np.where(k3, B.half_rn(p3 / 2) != p3 / 2, ~B.is_pos_zero(p3))
        _pool_stats(f"{tag} conv3+pool3, encdrop3", bad | B.check_mask_only(_bcast(m3, T), lo, hi), cb, p3 / 2, _bcast(m3, T), k3)

        # conv4 -> pool4, then encdrop4 + upsample4 (k_dropout_h8): pool4 itself is not stored
        cb = _conv(weights, "conv4", p3)
        lo, hi = cb.half_interval()
        u4, m4 = blob("upsample4"), blob("pool4_mask")
        sel, others = B.unpooled_parts(u4, m4)
        k4 = _keep(1, T, m4.shape)
        bad = B.check_pool(sel / 2, m4, lo, hi, valid=k4) | ~others
        bad |= np.where(k4, B.half_rn(sel / 2) != sel / 2, ~B.is_pos_zero(sel))
        _pool_stats(f"{tag} conv4+pool4, encdrop4+upsample4", bad | B.check_mask_only(m4, lo, hi), cb, sel / 2, m4, k4)

        # conv_decode4 + decdrop4 + upsample3, conv_decode3 + decdrop3 + upsample2: the deferred epilogue
        x = u4
        for conv, layer, up, mask in (("conv_decode4", 2, "upsample3", m3), ("conv_decode3", 3, "upsample2", m2)):
            cb = _conv(weights, conv, x, relu=False)  # the decoder convolutions have no ReLU
            lo, hi = cb.half_interval()
            u = blob(up)
            sel, others = B.unpooled_parts(u, mask)
            keep = _keep(layer, T, sel.shape)
            _report(f"{tag} {conv}+dropout+{up}", B.check_dropped(sel, keep, lo, hi) | ~others, cb, np.where(keep, sel / 2, B.half_rn(cb.center())))
            x = u
        u2 = x
    else:
        u2 = blob("upsample2")

    # conv_decode2: the dense pooled-resolution store
    cb = _conv(weights, "conv_decode2", u2, relu=False)
    d2 = blob("conv_decode2")
    _report(f"{tag} conv_decode2", B.outside(d2, *cb.half_interval()), cb, d2)
    del cb

    # upsample1 + conv_decode1 x classifier, composed as the library composes it, read from conv_decode2 and pool1_mask
    up1 = _unpool(d2, blob("pool1_mask"))
    wc, bc = weights["dense_softmax_inner_prod"]
    wd, bd = weights["conv_decode1"]
    wh, bias, w64, b64 = B.compose_classifier(wd, bd, wc, bc)
    cb = B.ConvBound(up1, wh, 3, B.gamma_tc(7, 64), bias)
    logits = blob("dense_softmax_inner_prod")
    lo, hi = cb.float_interval()
    _report(f"{tag} upsample1+conv_decode1*classifier", B.outside(logits, lo, hi), cb, logits, half=False)
    # the same launch against the un-composed two-layer float64 math, the composed weights' half rounding in the bound
    dw = w64 - wh
    with torch.no_grad():
        shift = torch.nn.functional.conv2d(torch.from_numpy(up1.astype(np.float32)), torch.from_numpy(dw.astype(np.float32)),
                                           padding=3).numpy().astype(np.float64)
    e2 = cb.e + B.conv_abs(up1, dw, 3) * 1.01 + np.abs(bias - b64).reshape(1, -1, 1, 1)
    r2 = cb.r + shift + b64.reshape(1, -1, 1, 1)
    e2 = e2 + 2 * B.ulp32(np.abs(r2) + e2)
    _report(f"{tag} classifier vs two-layer float64", ~(np.abs(logits - r2) <= e2))
    del cb

    # the maps from the device logits
    rc, rconf, rent, conf_b, ent_b, margin = B.map_bounds(logits)
    sure = margin > 2 * conf_b
    print(f"{tag} maps: |d conf| max {np.abs(conf - rconf).max():.2e} (bound {conf_b.max():.2e}), |d entropy| max "
          f"{np.abs(ent - rent).max():.2e} (bound {ent_b.max():.2e}), {int((~sure).sum())} near-tie pixels")
    assert np.array_equal(cls[sure], rc[sure])
    assert (np.abs(conf - rconf) <= conf_b).all() and (np.abs(ent - rent) <= ent_b).all()


# 48 x 272 / 80 x 320, T = 3: odd T, partial strips at every level, odd numbers of row blocks; 352 x 1024, T = 2: full size
@pytest.mark.parametrize("H,W,T", [(48, 272, 3), (80, 320, 3), (352, 1024, 2)])
def test_basic_default_build_within_float64_bounds(model_dir, H, W, T):
    walk_basic(model_dir, H, W, T)


def test_basic_T6_full_size_decoder_tail_within_float64_bounds(model_dir):
    """The benchmarked configuration (1024 x 352, T = 6): conv_decode2 and the composed classifier, whose rows-per-CTA
    pieces depend on T and cross strips and images, checked from the device's upsample2 and conv_decode2, then the maps."""
    walk_basic(model_dir, 352, 1024, 6, only_tail=True)


def walk_exposed(model_dir, kind, H, W, T, precision):
    """Every convolution of a build whose convolution inputs are all stored (Standard's fp16 build, the strict fp32
    builds), each from the device's own input blob.  The output is checked where it is stored, through the pool, dropout
    and unpool that follow it where those are fused (or run as their own kernels), and the logits through the maps."""
    net, weights, proto, model = make_model(model_dir, kind, T=T, H=H, W=W, seed=0)
    left, _ = stereo_frame(0)
    img = S.center_crop(left, W, H)
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=SEED, T=T, precision=precision)
    seg.set_frame(FRAME)
    cls, conf, ent = seg.segmentImage(img)
    half = precision == "fp16"
    tag = f"{kind} {precision} {H}x{W} T={T}"
    layers = net.layers
    drop_ord = {ly.name: i for i, ly in enumerate([ly for ly in layers if ly.type == "Dropout"])}

    def read(name):
        try:
            return seg.blob(name)
        except Exception:  # consumed in registers by a fused kernel
            return None

    def follows(j, top, kind_, inplace=None):
        if j >= len(layers) or layers[j].type != kind_ or layers[j].bottoms[0] != top:
            return False
        return inplace is None or (layers[j].tops[0] == top) == inplace

    def report(name, bad, out=None, c=None, lo=None, hi=None):
        msg = f"{tag} {name}: {int(np.sum(bad))} of {np.size(bad)} outside"
        if out is not None:
            ratio, frac = B.interval_stats(out, c, lo, hi, half)
            msg += f", max |out - f(r)| / bound {ratio:.3f}" + (f", {frac:.2e} != half_rn(f(r))" if half else "")
        print(msg)
        assert not np.any(bad), msg

    checked = 0
    for i, ly in enumerate(layers):
        if ly.type != "Convolution":
            continue
        top, j, relu, bn = ly.tops[0], i + 1, False, None
        while j < len(layers) and layers[j].type in ("BN", "ReLU") and follows(j, top, layers[j].type, True):
            if layers[j].type == "BN":
                bn = weights[layers[j].name]
            else:
                relu = True
            j += 1
        x = read(ly.bottoms[0])
        assert x is not None, (tag, ly.name, ly.bottoms[0])
        w, b = weights[ly.name][0], weights[ly.name][1]
        k, cin = w.shape[-1], w.shape[1]
        extra = None
        if half:
            w = _h(w)
            gamma = B.gamma_tc(k, 64, folded=True) if cin == 3 else B.gamma_tc(k, cin)
        elif cin % 64 == 0:  # split operands on the tensor core, or the FMA engine where that does not take the shape
            gamma = max(B.gamma_split(k, cin), B.gamma_simt(k, cin))
            extra = B.SPLIT_ABS * B.conv_abs(np.ones_like(x), w, k // 2)
        else:
            gamma = B.gamma_simt(k, cin)
        cb = B.ConvBound(x, w, k // 2, gamma, b, bn[0] if bn else None, bn[1] if bn else None, relu=relu, extra=extra)
        lo, hi = cb.half_interval() if half else cb.float_interval()
        c = cb.center()
        fill = B.half_rn(c) if half else c  # what a dropped element is compared as in the printed stats
        name = ly.name
        if j < len(layers) and layers[j].type == "Softmax":  # the logits, then the maps
            lo, hi = cb.float_interval()
            out = read(top)
            report(f"{name} (logits)", B.outside(out, lo, hi), out, c, lo, hi)
            rc, rconf, rent, conf_b, ent_b, margin = B.map_bounds(out)
            sure = margin > 2 * conf_b
            print(f"{tag} maps: |d conf| max {np.abs(conf - rconf).max():.2e} (bound {conf_b.max():.2e}), |d entropy| max "
                  f"{np.abs(ent - rent).max():.2e} (bound {ent_b.max():.2e}), {int((~sure).sum())} near-tie pixels")
            assert np.array_equal(cls[sure], rc[sure])
            assert (np.abs(conf - rconf) <= conf_b).all() and (np.abs(ent - rent) <= ent_b).all()
            checked += 1
            continue
        keep = None
        if follows(j, top, "Dropout", True):  # in place after the convolution (fused into its epilogue in fp16)
            keep = _keep(drop_ord[layers[j].name], T, (T,) + cb.r.shape[1:])
            name += "+" + layers[j].name
            j += 1
        lo, hi, c, fill = (_bcast(a, keep.shape[0]) if keep is not None else a for a in (lo, hi, c, fill))
        out = read(top)
        if out is not None:
            bad = B.check_dropped(out, keep, lo, hi, half) if keep is not None else B.outside(out, lo, hi)
            report(name, bad, np.where(keep, out / 2, fill) if keep is not None else out, c, lo, hi)
        if follows(j, top, "Pooling"):
            pool = layers[j]
            mask = read(pool.tops[1])
            ptop, pname, pkeep = pool.tops[0], name + "+" + pool.name, None
            j += 1
            if follows(j, ptop, "Dropout", True):
                pkeep = _keep(drop_ord[layers[j].name], T, (T,) + mask.shape[1:])
                pname += "+" + layers[j].name
                j += 1
            v = read(ptop)
            up = follows(j, ptop, "Upsample") and layers[j]
            n = pkeep.shape[0] if pkeep is not None else mask.shape[0]
            lo_, hi_, c_ = (_bcast(a, n) for a in (lo, hi, c))
            mask_ = _bcast(mask, n)
            bad = B.check_mask_only(mask_, lo_, hi_)
            if up:
                u = read(up.tops[0])
                sel, others = B.unpooled_parts(u, mask_)
                bad |= ~others
                if v is not None:
                    bad |= sel != v
                v, pname = sel, pname + "+" + up.name
            if pkeep is not None:
                bad |= B.check_pool(v / 2, mask_, lo_, hi_, valid=pkeep)
                bad |= np.where(pkeep, (B.half_rn(v / 2) != v / 2) if half else False, v != 0)
                vv = np.where(pkeep, v / 2, B.at_mask(_bcast(fill, n), mask_))
            else:
                bad |= B.check_pool(v, mask_, lo_, hi_)
                vv = v
            report(pname, bad, vv, B.at_mask(c_, mask_), B.at_mask(lo_, mask_), B.at_mask(hi_, mask_))
        elif follows(j, top, "Upsample"):
            up = layers[j]
            mask = read(up.bottoms[1])
            sel, others = B.unpooled_parts(read(up.tops[0]), mask)
            n = sel.shape[0]
            lo, hi, c = (_bcast(a, n) for a in (lo, hi, c))
            bad = ~others
            if keep is not None:
                bad |= B.check_dropped(sel, keep, lo, hi, half)
                shown = np.where(keep, sel / 2, _bcast(fill, n))
            else:
                bad |= B.outside(sel, lo, hi)
                shown = sel
            if out is not None:
                bad |= sel != out
            report(name + "+" + up.name, bad, shown, c, lo, hi)
        else:
            assert out is not None, (tag, name, "neither stored nor pooled / unpooled")
        checked += 1
    assert checked == sum(ly.type == "Convolution" for ly in layers)


def test_standard_fp16_within_float64_bounds(model_dir):
    """Standard's real widths at 128 x 384, T = 2: BN epilogues, 128-wide tiles (immediate epilogue), chunked Cin > 64,
    image-pair (PK2) conv5 tiles, fused dropout + unpool, k_conv_stack<3> for conv1_1_D."""
    walk_exposed(model_dir, "standard", 128, 384, 2, "fp16")


@pytest.mark.parametrize("kind,H,W", [("basic", 80, 320), ("standard", 128, 384)])
def test_strict_mode_within_float64_bounds(model_dir, kind, H, W):
    """Split-operand fp32 convolutions (the FMA engine for 3-channel inputs), every output stored, unfused pool /
    dropout / unpool in fp32."""
    walk_exposed(model_dir, kind, H, W, 2, "fp32")


def test_relu_of_a_negative_input_is_positive_zero():
    """Caffe's ReLU gives max(t, 0) + slope * min(t, 0) = +0 for t < 0; slope * t alone is -0, which pools, drops and
    unpools as -0 and would break the all-zero-window rule (value +0, mask code 0) of every pooled blob."""
    rng = np.random.default_rng(21)
    x = rng.normal(0, 1, size=(1, 64, 6, 130)).astype(np.float32)
    w = (rng.normal(0, 1, size=(64, 64, 3, 3)) / 24).astype(np.float32)
    b = np.full(64, -50.0, np.float32)  # every pre-activation negative
    for engine in (L.ENGINE_TCGEN05, L.ENGINE_SIMT):
        out = np.empty((1, 64, 6, 130), np.float32)
        L.check(L.lib().sivo_dbg_conv(0, engine, L.PRECISION_FP16, x.ctypes.data_as(C.c_void_p), 1, 64, 6, 130,
                                      w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), None, None, 64, 3, 1, 1,
                                      out.ctypes.data_as(C.c_void_p)))
        assert B.is_pos_zero(out).all(), (engine, int(np.signbit(out).sum()))
