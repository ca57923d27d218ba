"""-m gpu: the 64-wide 7x7 half convolution that max-unpools its input as it loads it (k_conv_tn<7, 7, true>: Basic's
upsample4 -> conv_decode4, upsample3 -> conv_decode3 and upsample2 -> conv_decode2).  The unpool is an exact select and the
consumers are those of the plain kernel, so it must equal the unpool kernel followed by the convolution bit for bit, with
and without the dropout its epilogue applies before the dense store; and the default network build, which runs it, must
expose the same decoder blobs as the unfused keep_blobs build."""
import numpy as np
import pytest

from conftest import make_model
from sivo_b200 import BayesianSegNet, BayesianSegNetParams
from sivo_b200 import _lib as L
from sivo_b200.synth import stereo_frame

pytestmark = pytest.mark.gpu

SEED, FRAME = 1234, 7


def _case(n, mask_n, h, w, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1, size=(n, 64, h, w)).astype(np.float32)
    code = rng.integers(0, 4, size=(mask_n, 64, h, w))
    # every third pooled row: all channels of a pixel name the same position (whole pixels of the halo row zero or not)
    code[:, :, ::3, :] = rng.integers(0, 4, size=(mask_n, 1, h, w))[:, :, ::3, :]
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    mask = ((2 * yy + (code >> 1)) * (2 * w) + 2 * xx + (code & 1)).astype(np.int32)  # Caffe's flat argmax index
    wt = (rng.normal(0, 1, size=(64, 64, 7, 7)) / np.sqrt(64 * 49)).astype(np.float32)
    b = rng.normal(0, 0.1, size=64).astype(np.float32)
    return x, mask, wt, b


def _conv(x, mask, wt, b, drop_layer, on_load):
    n, _, h, w = x.shape
    out = np.empty((n, 64, 2 * h, 2 * w), np.float32)
    L.check(L.lib().sivo_dbg_conv64_unpooled(0, L.ptr(np.ascontiguousarray(x)), L.ptr(np.ascontiguousarray(mask)), n, mask.shape[0],
                                             h, w, L.ptr(wt), L.ptr(b), drop_layer, SEED, FRAME, int(on_load), L.ptr(out)))
    return out


def _keep(layer, n, h, w):
    keep = np.empty((n, 64, h, w), np.uint8)
    L.check(L.lib().sivo_dbg_dropout_mask(0, SEED, FRAME, layer, n, 64, h, w, L.ptr(keep)))
    return keep.astype(bool)


# pooled n x 64 x h x w: an unpooled width below one 128-pixel strip and fewer rows than the filter; an odd pooled width,
# whose last strip ends inside a pooled pixel's window; Basic's upsample3 and upsample2 at 352 x 1024, T = 6, with the batch-1
# masks of the deduplicated encoder and the per-sample mask of upsample4
@pytest.mark.parametrize("n,mask_n,h,w", [(2, 2, 2, 50), (3, 1, 19, 97), (6, 6, 22, 64), (6, 1, 44, 128), (6, 1, 88, 256)])
@pytest.mark.parametrize("drop_layer", [-1, 3])
def test_unpool_on_load_equals_unpool_then_conv(n, mask_n, h, w, drop_layer):
    args = _case(n, mask_n, h, w, seed=h * 1000 + w)
    got, want = _conv(*args, drop_layer, True), _conv(*args, drop_layer, False)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), float(np.abs(got - want).max())
    if drop_layer >= 0:
        # dropout + dense store: the kept values doubled (exact in half), the others zero
        plain = _conv(*args, -1, True)
        keep = _keep(drop_layer, n, 2 * h, 2 * w)
        assert keep.any() and not keep.all()
        assert np.array_equal(got, np.where(keep, 2 * plain, 0))


def test_unpool_on_load_does_not_depend_on_the_batch():
    x, mask, wt, b = _case(2, 2, 44, 128, seed=5)
    both = _conv(x, mask, wt, b, -1, True)
    for i in range(2):
        alone = _conv(x[i:i + 1], mask[i:i + 1], wt, b, -1, True)
        assert np.array_equal(both[i:i + 1].view(np.uint32), alone.view(np.uint32))


def _image(H, W):
    left, _ = stereo_frame(0)
    return np.ascontiguousarray(left[20:20 + H, 40:40 + W])


# 48 x 272: partial strips at every level and an odd number of row blocks; 352 x 1024 at T = 6: the benchmarked shape
@pytest.mark.parametrize("H,W,T", [(48, 272, 3), (352, 1024, 6)])
def test_default_build_unpools_decoder_inputs_on_load(model_dir, H, W, T):
    _, _, proto, model = make_model(model_dir, "basic", T=T, H=H, W=W, seed=0)
    img = _image(H, W)
    names = ("upsample4", "conv_decode4", "upsample3", "conv_decode3", "upsample2", "conv_decode2")
    blobs = []
    for keep in (True, False):
        seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=SEED, T=T, precision="fp16", engine="auto", keep_blobs=keep)
        seg.set_frame(3)
        seg.segmentImage(img)
        blobs.append({n: seg.blob(n) for n in names})
        if not keep:
            ops = [name for name, _, _ in seg.op_timings()]
            # no unpool runs as its own launch, and none is scattered by a 64-wide 7x7 convolution's epilogue
            assert not any(o.startswith("upsample") and "conv" not in o for o in ops), ops
            assert "encdrop4+upsample4" in ops, ops
    for n in names:
        assert np.array_equal(blobs[0][n], blobs[1][n]), n
