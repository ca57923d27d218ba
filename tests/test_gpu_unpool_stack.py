"""-m gpu: the 7x7 float-logits convolution that max-unpools its input as it loads it (k_conv_stack<7, true>: Basic's
upsample1 -> conv_decode1 x classifier).  The unpool is an exact select and the accumulation order is that of the plain
kernel, so it must equal the unpool kernel followed by the convolution bit for bit, and the default network build, which
runs it, must expose the same conv_decode2 and upsample1 blobs as the unfused keep_blobs build."""
import numpy as np
import pytest

import torch

from conftest import make_model
from oracle import conv_bounds as B
from oracle import segnet_oracle as S
from test_gpu_layers import interval_violations
from sivo_b200 import BayesianSegNet, BayesianSegNetParams
from sivo_b200 import _lib as L
from sivo_b200.synth import stereo_frame

pytestmark = pytest.mark.gpu


def _case(n, mask_n, h, w, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1, size=(n, 64, h, w)).astype(np.float32)
    code = rng.integers(0, 4, size=(mask_n, 64, h, w))
    # every third pooled row: all channels of a pixel name the same position (whole pixels of the halo row zero or not)
    code[:, :, ::3, :] = rng.integers(0, 4, size=(mask_n, 1, h, w))[:, :, ::3, :]
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    mask = ((2 * yy + (code >> 1)) * (2 * w) + 2 * xx + (code & 1)).astype(np.int32)  # Caffe's flat argmax index
    wt = (rng.normal(0, 1, size=(15, 64, 7, 7)) / np.sqrt(64 * 49)).astype(np.float32)
    b = rng.normal(0, 0.1, size=15).astype(np.float32)
    sc = (1 + rng.normal(0, 0.1, size=15)).astype(np.float32)
    sh = rng.normal(0, 0.1, size=15).astype(np.float32)
    return x, mask, wt, b, sc, sh


def _fused(x, mask, wt, b, sc, sh):
    n, _, h, w = x.shape
    out = np.empty((n, 15, 2 * h, 2 * w), np.float32)
    L.check(L.lib().sivo_dbg_conv_unpooled(0, L.ptr(np.ascontiguousarray(x)), L.ptr(np.ascontiguousarray(mask)), n, mask.shape[0], h,
                                           w, L.ptr(wt), L.ptr(b), L.ptr(sc), L.ptr(sh), 15, 7, L.ptr(out)))
    return out


def _two_kernels(x, mask, wt, b, sc, sh):
    n, _, h, w = x.shape
    full_mask = np.ascontiguousarray(mask[np.arange(n) % mask.shape[0]])
    up = np.empty((n, 64, 2 * h, 2 * w), np.float32)
    L.check(L.lib().sivo_dbg_unpool(0, L.ptr(np.ascontiguousarray(x)), L.ptr(full_mask), n, 64, h, w, L.ptr(up)))
    out = np.empty((n, 15, 2 * h, 2 * w), np.float32)
    L.check(L.lib().sivo_dbg_conv(0, L.ENGINE_TCGEN05, L.PRECISION_FP16, L.ptr(up), n, 64, 2 * h, 2 * w, L.ptr(wt), L.ptr(b),
                                  L.ptr(sc), L.ptr(sh), 15, 7, 3, 0, L.ptr(out)))
    return out


# pooled n x 64 x h x w: H < K with a partial strip; an odd pooled width, whose last strip ends inside a pooled pixel's
# window; full size (Basic's upsample1 at 352 x 1024), where a CTA's rows cross strips and images
@pytest.mark.parametrize("n,h,w", [(3, 3, 100), (2, 19, 65), (2, 176, 512)])
@pytest.mark.parametrize("shared_mask", [True, False])
def test_unpool_on_load_equals_unpool_then_conv(n, h, w, shared_mask):
    args = _case(n, 1 if shared_mask else n, h, w, seed=h * 1000 + w)
    got, want = _fused(*args), _two_kernels(*args)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), float(np.abs(got - want).max())
    x, mask, wt, b, sc, sh = args
    n_, _, h_, w_ = x.shape
    up = S.unpool(torch.from_numpy(x).half().float(), torch.from_numpy(mask.astype(np.int64)).expand(n_, -1, -1, -1)).numpy()
    assert interval_violations(up, B.half_rn(wt).astype(np.float32), b, sc, sh, got, B.gamma_tc(7, 64), relu=False, half=False) == 0


def test_unpool_on_load_does_not_depend_on_the_row_split():
    x, mask, wt, b, sc, sh = _case(2, 2, 176, 512, seed=5)
    both = _fused(x, mask, wt, b, sc, sh)
    for i in range(2):
        alone = _fused(x[i:i + 1], mask[i:i + 1], wt, b, sc, sh)
        assert np.array_equal(both[i:i + 1].view(np.uint32), alone.view(np.uint32))


def _image(H, W):
    left, _ = stereo_frame(0)
    return np.ascontiguousarray(left[20:20 + H, 40:40 + W])


@pytest.mark.parametrize("H,W", [(80, 320), (352, 464)])
def test_default_build_unpools_on_load(model_dir, H, W):
    _, _, proto, model = make_model(model_dir, "basic", T=2, H=H, W=W, seed=0)
    img = _image(H, W)
    blobs, maps = [], []
    for keep in (True, False):
        seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=2, precision="fp16", engine="auto", keep_blobs=keep)
        seg.set_frame(3)
        maps.append(seg.segmentImage(img))
        blobs.append({n: seg.blob(n) for n in ("conv_decode2", "upsample1")})
        if not keep:
            names = [name for name, _, _ in seg.op_timings()]
            assert "conv_decode2" in names and any(n.startswith("upsample1+conv_decode1*") for n in names), names
            with pytest.raises(Exception):
                seg.blob("conv_decode1")
            seg.set_frame(3)
            again = seg.segmentImage(img)
            for a, b in zip(maps[-1], again):
                assert np.array_equal(a, b)
    for n in blobs[0]:
        assert np.array_equal(blobs[0][n], blobs[1][n]), n
