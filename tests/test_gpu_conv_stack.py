"""-m gpu: the tap-row-stacked float-logits convolution (k_conv_stack: Cin = 64 -> at most 16 float channels, 3x3 / 7x7),
called through the C-ABI test hook, against torch fp32 on identical half-rounded operands."""
import numpy as np
import pytest
import torch

from oracle import conv_bounds as B
from sivo_b200 import _lib as L
from test_gpu_layers import interval_violations

pytestmark = pytest.mark.gpu


def _layer(k, n, h, w, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1, size=(n, 64, h, w)).astype(np.float32)
    wt = (rng.normal(0, 1, size=(15, 64, k, k)) / np.sqrt(64 * k * k)).astype(np.float32)
    b = rng.normal(0, 0.1, size=15).astype(np.float32)
    sc = (1 + rng.normal(0, 0.1, size=15)).astype(np.float32)
    sh = rng.normal(0, 0.1, size=15).astype(np.float32)
    return x, wt, b, sc, sh


def _run(k, x, wt, b, sc, sh):
    n, _, h, w = x.shape
    out = np.empty((n, 15, h, w), np.float32)
    L.check(L.lib().sivo_dbg_conv(0, L.ENGINE_TCGEN05, L.PRECISION_FP16, L.ptr(np.ascontiguousarray(x)), n, 64, h, w, L.ptr(wt),
                                  L.ptr(b), L.ptr(sc), L.ptr(sh), 15, k, (k - 1) // 2, 1, L.ptr(out)))
    return out


@pytest.mark.parametrize("k,n,h,w", [
    # partial strip (W not a multiple of 128), H < K, odd heights, several images
    (7, 3, 5, 200), (7, 2, 37, 130), (3, 3, 1, 130), (3, 2, 37, 200),
    # full size: a CTA's rows run from one strip (or image) into the next
    (7, 2, 352, 1024), (3, 2, 352, 1024)])
def test_stacked_logits_conv_matches_oracle(k, n, h, w):
    import torch.nn.functional as F
    x, wt, b, sc, sh = _layer(k, n, h, w, seed=7)
    out = _run(k, x, wt, b, sc, sh)
    xt, wtt = torch.from_numpy(x).half().float(), torch.from_numpy(wt).half().float()
    ref = F.conv2d(xt, wtt, None, padding=(k - 1) // 2) + torch.from_numpy(b).view(1, -1, 1, 1)
    ref = torch.relu(ref * torch.from_numpy(sc).view(1, -1, 1, 1) + torch.from_numpy(sh).view(1, -1, 1, 1)).numpy()
    err = np.abs(out - ref)
    assert err.max() < 2e-3 * max(1.0, float(np.abs(ref).max())), float(err.max())
    assert interval_violations(xt.numpy(), wtt.numpy(), b, sc, sh, out, B.gamma_tc(k, 64), half=False) == 0


@pytest.mark.parametrize("k", [3, 7])
def test_stacked_logits_conv_does_not_depend_on_the_row_split(k):
    """A batch of two images and each image alone are cut into different pieces of rows per CTA (other run starts, other
    warm-up rows); every pixel's sum runs in the same order, so the logits are the same bits."""
    x, wt, b, sc, sh = _layer(k, 2, 352, 1024, seed=8)
    both = _run(k, x, wt, b, sc, sh)
    for i in range(2):
        alone = _run(k, x[i:i + 1], wt, b, sc, sh)
        assert np.array_equal(both[i:i + 1].view(np.uint32), alone.view(np.uint32))
