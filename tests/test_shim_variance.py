"""SIVO::BayesianSegNet::computeVariance and generateVarianceImage through the C++ shim class of integration/ (compiled with g++
against integration/stubs as tests/shim_build.py does): the map bit-identical to the Python mirror of the same C-ABI, the image equal to
cv2.normalize(..., NORM_MINMAX)."""
import os
import subprocess

import numpy as np
import pytest

from conftest import make_model
from shim_build import BUILD_DIR
from test_shim import write_bin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(BUILD_DIR, "test_shim_variance")  # outside the tree, as tests/shim_build.py builds
SOURCES = [os.path.join(ROOT, "integration", "src", "bayesian_segnet.cpp"), os.path.join(ROOT, "tests", "cpp", "test_shim_variance.cpp")]


def build():
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    lib_dir = os.path.join(ROOT, "sivo_b200")
    cmd = ["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "integration", "stubs"),
           "-I" + os.path.join(ROOT, "integration", "include"), "-I" + os.path.join(ROOT, "include"), *SOURCES,
           "-L" + lib_dir, "-lsivo_b200", "-Wl,-rpath," + lib_dir, "-o", BIN]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("shim build failed:\n" + r.stderr[-4000:])
    return BIN


def test_shim_with_compute_variance_compiles():
    """The shim with the public computeVariance and the driver that calls it build with -Wall -Werror.  Needs no GPU."""
    assert os.path.exists(build())


@pytest.mark.gpu
def test_shim_compute_variance_equals_the_python_mirror(tmp_path, kitti_bgr):
    import cv2
    from sivo_b200 import BayesianSegNet, BayesianSegNetParams
    exe = build()
    H, W, T = 96, 256, 3
    _, _, proto, model = make_model(tmp_path, "basic", T=T, H=H, W=W)
    img = np.ascontiguousarray(kitti_bgr[60:60 + H + 20, 200:200 + W + 30])
    write_bin(tmp_path / "bgr.bin", img)
    out = tmp_path / "out"
    out.mkdir()
    env = dict(os.environ, SIVO_B200_SEED="1234")
    r = subprocess.run([exe, proto, model, str(tmp_path / "bgr.bin"), str(out)], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and "SHIM VARIANCE OK" in r.stdout, r.stdout + r.stderr
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234)
    seg.set_frame(0)
    cls, _, _ = seg.segmentImage(img)
    assert np.array_equal(np.fromfile(out / "classes.bin", np.uint8).reshape(H, W), cls)
    want = seg.computeVariance(cls)
    got = np.fromfile(out / "variance.bin", np.float64).reshape(H, W)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)) and want.max() > 0
    img_v = np.fromfile(out / "variance_image.bin", np.float64).reshape(H, W)
    assert np.allclose(img_v, cv2.normalize(want, None, 0.0, 1.0, cv2.NORM_MINMAX, cv2.CV_64FC1), atol=1e-12)
