import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def kitti_bgr():
    """The reference's own fixture frame (tests/data/test_image.png there), 1242x375x3."""
    import cv2
    img = cv2.imread(os.path.join(GOLDEN, "kitti_000000_1242x375.png"))
    assert img is not None and img.shape == (375, 1242, 3)
    return img


@pytest.fixture(scope="session")
def kitti_gray_crop(kitti_bgr):
    from sivo_b200.synth import bgr_to_gray
    return np.ascontiguousarray(bgr_to_gray(kitti_bgr)[11:11 + 352, 109:109 + 1024])


_SCALE_CACHE = {}


def calibrated_scales(kind, net, seed, key):
    """Per-layer LSUV factors (tools/calibrate_synth.py) for a test-sized net: the shipped factors when the topology is one of
    the two shipped ones (they hold at any input size), else computed once per session with the oracle on the net itself."""
    import calibrate_synth
    from sivo_b200.caffemodel import shipped_scales, synth_weights
    shipped = shipped_scales(kind)
    want = {ly.name: ly.num_output for ly in net.layers if ly.type == "Convolution"}
    full_width = max(want.values()) == (64 if kind == "basic" else 512) and min(want.values()) == 15
    if seed == 0 and set(want) == set(shipped) and full_width:
        return shipped
    if key not in _SCALE_CACHE:
        _, _, H, W = net.input_dims
        w = synth_weights(net, seed)
        _SCALE_CACHE[key] = calibrate_synth.lsuv_scales(net, w, calibrate_synth.calibration_image(H, W), T=2)
    return _SCALE_CACHE[key]


def make_model(tmp, kind="basic", T=3, H=32, W=64, seed=0, calibrated=True, **kw):
    """Writes <tmp>/<kind>.prototxt + .caffemodel with seeded synthetic weights, calibrated so that activations stay O(1) and
    the softmax is not saturated (tools/calibrate_synth.py); returns (net, weights, paths)."""
    import gen_prototxt
    from sivo_b200.caffemodel import write_synth_model
    from sivo_b200.prototxt import load_net
    text = getattr(gen_prototxt, kind)(T=T, H=H, W=W, **kw)
    tag = f"{kind}_{T}_{H}x{W}" + ("" if calibrated else "_raw") + "".join(f"_{k}{v}" for k, v in sorted(kw.items())).replace(" ", "")
    tag = tag.replace("(", "").replace(")", "").replace(",", "-")
    proto = os.path.join(str(tmp), tag + ".prototxt")
    model = os.path.join(str(tmp), tag + ".caffemodel")
    open(proto, "w").write(text)
    net = load_net(text)
    scales = calibrated_scales(kind, net, seed, (kind, H, W, seed, tuple(sorted(kw.items())))) if calibrated else None
    weights = write_synth_model(net, model, seed, scales)
    return net, weights, proto, model


@pytest.fixture(scope="session")
def model_dir(tmp_path_factory):
    return tmp_path_factory.mktemp("models")
