"""-m gpu: the tensor-core convolution's deferred epilogue (the N = 64 store / dropout / max-unpool stores of a row block
issued under the next block's MMAs, flushed after a CTA's last block).  The fused build scatters the unpooled tensors from
that epilogue; keep_blobs runs the same convolutions with the plain store epilogue followed by the unpool kernel.  Both are
the same arithmetic, so every blob both builds expose must be the same bits, at sizes that exercise the deferred path's
edges: partial 128-pixel strips, odd numbers of row blocks, CTAs that walk one row block and CTAs that walk many."""
import numpy as np
import pytest

from conftest import make_model
from sivo_b200 import BayesianSegNet, BayesianSegNetParams
from sivo_b200.synth import stereo_frame

pytestmark = pytest.mark.gpu


def _image(H, W):
    left, _ = stereo_frame(0)
    return np.ascontiguousarray(left[20:20 + H, 40:40 + W])


def _run(proto, model, img, keep, T):
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=T, precision="fp16", engine="auto", keep_blobs=keep)
    seg.set_frame(3)
    maps = seg.segmentImage(img)
    return seg, maps


def _exposed(seg, names):
    out = {}
    for n in names:
        try:
            out[n] = seg.blob(n)
        except Exception:  # consumed in registers by a fused kernel
            pass
    return out


def _check_fused_equals_unfused(net, proto, model, img, T, must_have="", composed=False):
    names = sorted({t for ly in net.layers for t in ly.tops})
    seg_u, (c0, f0, e0) = _run(proto, model, img, True, T)
    unfused = _exposed(seg_u, names)
    seg_f, (c1, f1, e1) = _run(proto, model, img, False, T)
    fused = _exposed(seg_f, names)
    logits = {b for ly in net.layers if ly.type == "Softmax" for b in ly.bottoms}  # the classifier's output: compared with the maps
    common = [n for n in fused if n in unfused and n not in logits]
    assert any(n.startswith(must_have) for n in common), common
    for n in common:
        assert fused[n].shape == unfused[n].shape, n
        assert np.array_equal(fused[n], unfused[n]), (n, float(np.abs(fused[n] - unfused[n]).max()))
    if composed:
        # the composed classifier never rounds the 64-channel activation to half (its composed weights are), so its maps
        # differ from the two layers' at the half-rounding level
        assert not np.array_equal(e0, e1), "the composed kernel did not engage"
        assert (c0 != c1).mean() < 2e-3
        assert np.abs(e0 - e1).max() < 2e-2 and np.median(np.abs(e0 - e1)) < 1e-3
        assert np.abs(f0 - f1).max() < 1e-2
    else:
        assert (c0 != c1).mean() < 1e-3
        assert np.abs(e0 - e1).max() < 1e-4 and np.abs(f0 - f1).max() < 1e-4


# (H, W): 48 x 272 -- partial strips at every level (272, 136, 68, 34 px) and 3 row blocks at H / 8; 80 x 320 -- 5 row
# blocks at H / 8, a 32-px last strip at H / 2; 352 x 464 -- tall layers, whose CTAs walk many row blocks (and the last
# CTA of a column fewer), with a partial strip everywhere
@pytest.mark.parametrize("H,W", [(48, 272), (80, 320), (352, 464)])
def test_basic_composed_build_blobs_equal_unfused(model_dir, H, W):
    # the default build composes conv_decode1 and the classifier, and its composed kernel unpools conv_decode2's output on
    # load: conv_decode2 and the derived upsample1 are compared bit for bit too
    net, _, proto, model = make_model(model_dir, "basic", T=2, H=H, W=W, seed=0)
    _check_fused_equals_unfused(net, proto, model, _image(H, W), 2, must_have="upsample", composed=True)


def test_standard_fused_blobs_equal_unfused(model_dir):
    # Standard's widths: 128-wide tiles (N = 128, immediate epilogue), chunked Cin > 64 layers and image-pair tiles (conv5 at
    # 4 x 8) next to the 64-wide deferred ones
    net, _, proto, model = make_model(model_dir, "standard", T=2, H=64, W=128, seed=0)
    _check_fused_equals_unfused(net, proto, model, _image(64, 128), 2)


def test_default_build_is_deterministic(model_dir):
    H, W = 80, 320
    _, _, proto, model = make_model(model_dir, "basic", T=2, H=H, W=W, seed=0)
    img = _image(H, W)
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=2, precision="fp16")
    runs = []
    for _ in range(2):
        seg.set_frame(3)
        runs.append(seg.segmentImage(img))
    for a, b in zip(*runs):
        assert np.array_equal(a, b)
