"""-m gpu: floating-point parity of `BayesianSegNet::segmentImage` at the configurations that are benchmarked, against the
fp32 oracle (the arithmetic the reference performs: fp32 cuDNN / BLAS convolutions, double MC reduction,
src/bayesian_segnet/bayesian_segnet.cpp:278-318), on the calibrated synthetic nets (tools/calibrate_synth.py: O(1)
activations, logits std ~2.5, entropy spread over [0, log2 15] -- no saturated `0 == 0` comparisons).

north_star bar: classes bit-exact given the dropout seed, confidence / entropy within 1e-4.  Two modes are held to it:

  strict  precision fp32 on the tensor-core engine: split-operand mode (x = hi + lo, w = hi + lo in half, three MMAs per tap,
          fp32 accumulation in registers, fp32 bias / BN / ReLU / pool / unpool / dropout) -- MUST meet 1e-4, and every class
          mismatch must be a tie (top-2 margin of the oracle's mean softmax below 1e-5).
  fast    precision fp16 (the default, benchmarked mode): half operands and half activation storage.  It cannot meet 1e-4
          (half rounding alone is 2^-11 per stored value); the test states its measured gap and bounds it.

Protocol (SURVEY 7 option i, DESIGN.md 2): max-pool argmax is the one discontinuous step; the device's pooling masks are
handed to the oracle so that everything downstream is compared tightly, and separately every mask that differs from the
oracle's own choice is checked to be a tie.  A free-running comparison (no hand-over) is printed as well.
Each test prints one PARITY line; bench / docs quote them."""
import os

import numpy as np
import pytest
import torch

from conftest import make_model
from oracle import segnet_oracle as S
from sivo_b200 import BayesianSegNet, BayesianSegNetParams
from sivo_b200.synth import stereo_frame
from test_gpu_segnet import _full_model, check_masks_are_ties, device_masks

pytestmark = pytest.mark.gpu

MODES = {"strict": dict(precision="fp32", engine="tcgen05"), "fast": dict(precision="fp16", engine="auto"),
         "simt32": dict(precision="fp32", engine="simt")}
_FREE = {}  # (net id, T, frame) -> free-running fp32 oracle result


def report(tag, cls, conf, ent, prob):
    """Compares the operator's maps with the oracle's reduction of `prob` (float32 [T,C,H,W]); returns the figures."""
    rc, rf, re = S.mc_reduce(prob)
    mean = prob.astype(np.float64).mean(axis=0)
    top2 = np.sort(mean, axis=0)[-2:]
    margin = top2[1] - top2[0]
    mm = cls != rc
    r = {"px": int(cls.size), "class_mismatch_px": int(mm.sum()), "max_margin_of_mismatch": float(margin[mm].max()) if mm.any() else 0.0,
         "conf_max": float(np.abs(conf - rf).max()), "ent_max": float(np.abs(ent - re).max()),
         "ent_q99": float(np.quantile(np.abs(ent - re), 0.99)), "ent_median": float(np.median(np.abs(ent - re))),
         "oracle_entropy_median": float(np.median(re)), "oracle_entropy_q01_q99": [float(np.quantile(re, 0.01)), float(np.quantile(re, 0.99))]}
    print(f"PARITY {tag}: " + ", ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}" for k, v in r.items()))
    return r


def run_mode(mode, proto, model, T, img, frame, keep_blobs=False):
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=T, keep_blobs=keep_blobs, **MODES[mode])
    seg.set_frame(frame)
    return seg, seg.segmentImage(img)


def check(mode, r_hand, flip_rate):
    if mode == "fast":
        # expected: entropy max ~3e-3 (Basic) .. ~1e-2 (Standard), class mismatches ~1e-3 of the pixels, all near-ties.  Pooling flips: two window entries that round to the same half tie on the device and
        # not in the fp32 oracle, ~1 % of the windows (each checked to be such a tie by check_masks_are_ties)
        assert r_hand["ent_max"] < 3e-2 and r_hand["conf_max"] < 1e-2 and r_hand["ent_q99"] < 1e-2
        assert r_hand["class_mismatch_px"] < 5e-3 * r_hand["px"] and r_hand["max_margin_of_mismatch"] < 1e-2
        assert flip_rate < 3e-2
    else:
        assert r_hand["ent_max"] <= 1e-4 and r_hand["conf_max"] <= 1e-4, r_hand           # north_star tolerance
        assert r_hand["max_margin_of_mismatch"] < 1e-5, r_hand                              # mismatching pixels are ties
        assert r_hand["class_mismatch_px"] <= 1e-4 * r_hand["px"], r_hand
        assert flip_rate < 1e-4


def parity_case(tag, mode, net, w, proto, model, T, img, frame):
    seg, (cls, conf, ent) = run_mode(mode, proto, model, T, img, frame)
    masks = device_masks(seg, net)  # pooling masks exist in the fused (benchmarked) build too
    prob, blobs = S.forward(net, w, img, seed=1234, frame=frame, precision="fp32", T=T, return_blobs=True, masks=masks)
    flip_rate = check_masks_are_ties(net, blobs, masks, "fp16" if mode == "fast" else "fp32")
    r_hand = report(f"{tag} mode={mode} masks=device flip_rate={flip_rate:.2e}", cls, conf, ent, prob)
    key = (tag, T, frame)
    if key not in _FREE:
        _FREE[key] = S.forward(net, w, img, seed=1234, frame=frame, precision="fp32", T=T)
    report(f"{tag} mode={mode} free-running", cls, conf, ent, _FREE[key])
    check(mode, r_hand, flip_rate)
    # the entropy map really is spread out (not the saturated one-hot softmax of uncalibrated weights)
    assert r_hand["oracle_entropy_median"] > 0.5


@pytest.mark.parametrize("mode", ["strict", "fast", "simt32"])
def test_basic_T6_full_size(model_dir, mode):
    """BASELINE.json configs[1]: Basic, T=6, 1024x352 (the benchmarked configuration)."""
    net, w, proto, model = _full_model(model_dir, "basic", T=6)
    left, _ = stereo_frame(0)
    parity_case("basic_T6_1024x352", mode, net, w, proto, model, 6, left, 3)


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_standard_T12_reduced_size(model_dir, mode):
    """BASELINE.json configs[2] topology (Standard, real 64/128/256/512/512 widths, T=12) at 128x384 so that the CPU oracle
    finishes in seconds."""
    net, w, proto, model = make_model(model_dir, "standard", T=12, H=128, W=384)
    left, _ = stereo_frame(1)
    img = np.ascontiguousarray(left[100:228, 300:684])
    parity_case("standard_T12_128x384", mode, net, w, proto, model, 12, img, 5)


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_standard_T2_full_size(model_dir, mode):
    """Standard at the full 1024x352 geometry (the kernels and grid shapes the bench runs), T=2."""
    net, w, proto, model = _full_model(model_dir, "standard", T=2)
    left, _ = stereo_frame(2)
    parity_case("standard_T2_1024x352", mode, net, w, proto, model, 2, left, 7)
