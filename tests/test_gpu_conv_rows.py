"""-m gpu: the Cin = 64 -> 64-wide tensor-core convolution at row and strip shapes the other convolution tests do not reach:
a single output row, an odd height (the second row of the last row block lies outside the image) with a last 128-pixel
strip one pixel wide, images narrower than half a strip, and more than one 64-channel cout tile.  Every output is held to
the per-element float64 interval of oracle/conv_bounds.py."""
import numpy as np
import pytest

from oracle import conv_bounds as B
from sivo_b200 import _lib as L

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k,cout,n,h,w", [
    (7, 64, 1, 1, 128), (3, 64, 2, 1, 200),    # H = 1
    (7, 64, 2, 7, 129), (3, 64, 1, 9, 129),    # H odd, last strip one pixel wide
    (7, 64, 1, 5, 40), (3, 64, 3, 6, 17),      # W < 64
    (3, 192, 1, 3, 129),                       # three cout tiles
])
def test_conv_rows_within_float64_bounds(k, cout, n, h, w):
    rng = np.random.default_rng(1000 * k + h * w)
    cin = 64
    x = rng.normal(0, 1, size=(n, cin, h, w)).astype(np.float16).astype(np.float32)
    wt = (rng.normal(0, 1, size=(cout, cin, k, k)) / np.sqrt(cin * k * k)).astype(np.float16).astype(np.float32)
    b = rng.normal(0, 0.1, size=cout).astype(np.float32)
    sc = (1 + rng.normal(0, 0.1, size=cout)).astype(np.float32)
    sh = rng.normal(0, 0.1, size=cout).astype(np.float32)
    out = np.full((n, cout, h, w), np.nan, np.float32)
    L.check(L.lib().sivo_dbg_conv(0, L.ENGINE_TCGEN05, L.PRECISION_FP16, L.ptr(x), n, cin, h, w, L.ptr(wt), L.ptr(b), L.ptr(sc),
                                  L.ptr(sh), cout, k, (k - 1) // 2, 1, L.ptr(out)))
    cb = B.ConvBound(x, wt, k // 2, B.gamma_tc(k, cin), b, sc, sh, relu=True)
    lo, hi = cb.half_interval()
    bad = B.outside(out, lo, hi)
    ratio, frac = cb.stats(out, True)
    print(f"k={k} cout={cout} {n}x{h}x{w}: {int(bad.sum())} of {bad.size} outside, max |out - f(r)| / bound {ratio:.3f}, "
          f"{frac:.2e} != half_rn(f(r))")
    assert not np.isnan(out).any()
    assert int(bad.sum()) == 0
