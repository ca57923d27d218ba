"""-m gpu: the Monte-Carlo variance map (computeVariance, bayesian_segnet.cpp:205-260) on the device.

Kernel level: the product kernels on host logits (sivo_dbg_mc_variance) against the variance oracle of the float32 softmax of
the same logits, on the quad path (C = 15) and the generic path (C = 21).  End to end: the operator's variance after
segmentImage against the fp32 oracle's samples, with the device's pooling masks handed to the oracle as in test_gpu_parity.py
and the device's own class map fed to both sides.  Then the forms agree with each other bit for bit, the variance does not
disturb the frames around it, and the latency-mode moments combine across shards."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import make_model
from oracle import segnet_oracle as S
from oracle.variance_oracle import mc_variance
from sivo_b200 import BayesianSegNet, BayesianSegNetParams, sample_ranges
from sivo_b200 import _lib as L
from sivo_b200.synth import stereo_frame
from test_gpu_parity import MODES
from test_gpu_segnet import _full_model, device_masks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _random_classes(rng, C, H, W):
    cls = rng.integers(0, C, (H, W)).astype(np.uint8)
    bad = rng.random((H, W)) < 0.1
    cls[bad] = rng.choice(np.array([255, C, C + 1, 254], np.uint8), int(bad.sum()))
    return cls


@pytest.mark.parametrize("C_", [15, 21])
@pytest.mark.parametrize("T", [2, 6, 12])
def test_kernel_against_the_oracle(C_, T):
    H, W = 19, 53  # pixel count not a multiple of the 64-pixel block
    rng = np.random.default_rng(T * 100 + C_)
    logits = (rng.standard_normal((T, C_, H, W)) * 2.5).astype(np.float32)
    cls = _random_classes(rng, C_, H, W)
    var = np.empty((H, W), np.float64)
    L.check(L.lib().sivo_dbg_mc_variance(0, logits.ctypes.data_as(C.c_void_p), T, C_, H, W, cls.ctypes.data_as(C.c_void_p),
                                         var.ctypes.data_as(C.c_void_p)))
    want = mc_variance(S.softmax_channels(torch.from_numpy(logits)).numpy(), cls)
    assert np.abs(var - want).max() <= 1e-5
    assert not var[cls >= C_].any() and (var[cls < C_] > 0).all()
    # identical samples: no variance; one sample: no sample variance
    one = np.repeat(logits[:1], T, axis=0)
    L.check(L.lib().sivo_dbg_mc_variance(0, one.ctypes.data_as(C.c_void_p), T, C_, H, W, cls.ctypes.data_as(C.c_void_p),
                                         var.ctypes.data_as(C.c_void_p)))
    assert var.max() < 1e-30
    assert L.lib().sivo_dbg_mc_variance(0, logits.ctypes.data_as(C.c_void_p), 1, C_, H, W, cls.ctypes.data_as(C.c_void_p),
                                        var.ctypes.data_as(C.c_void_p)) == L.EINVAL


def _end_to_end(tag, mode, net, w, proto, model, T, img, frame):
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=T, **MODES[mode])
    seg.set_frame(frame)
    cls, conf, _ = seg.segmentImage(img)
    var = seg.computeVariance(cls)
    masks = device_masks(seg, net)
    prob = S.forward(net, w, img, seed=1234, frame=frame, precision="fp32", T=T, masks=masks)
    want = mc_variance(prob, cls)
    gap = np.abs(var - want)
    print(f"PARITY {tag} mode={mode} variance: max={gap.max():.3g}, q99={np.quantile(gap, 0.99):.3g}, "
          f"median={np.median(gap):.3g}, oracle variance median={np.median(want):.3g} max={want.max():.3g}")
    assert (var >= 0).all() and np.median(want) > 1e-6  # the dropout samples really differ
    if mode == "fast":
        assert gap.max() < 1e-2  # as test_gpu_parity.check() bounds confidence in the fast mode
    else:
        assert gap.max() <= 1e-4


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_basic_T6_full_size(model_dir, mode):
    net, w, proto, model = _full_model(model_dir, "basic", T=6)
    left, _ = stereo_frame(0)
    _end_to_end("basic_T6_1024x352", mode, net, w, proto, model, 6, left, 3)


@pytest.mark.parametrize("mode", ["strict", "fast"])
def test_standard_T12_reduced_size(model_dir, mode):
    net, w, proto, model = make_model(model_dir, "standard", T=12, H=128, W=384)
    left, _ = stereo_frame(1)
    img = np.ascontiguousarray(left[100:228, 300:684])
    _end_to_end("standard_T12_128x384", mode, net, w, proto, model, 12, img, 5)


@pytest.fixture(scope="module")
def small(model_dir):
    T = 6
    _, _, proto, model = make_model(model_dir, "basic", T=T, H=64, W=128)
    left, _ = stereo_frame(2)
    img = np.ascontiguousarray(left[100:164, 300:428])
    return dict(T=T, proto=proto, model=model, img=img, H=64, W=128, bgr=torch.from_numpy(img).cuda())


def _seg(small, **kw):
    return BayesianSegNet(BayesianSegNetParams(small["proto"], small["model"]), seed=1234, T=small["T"], **kw)


def test_host_and_device_forms_are_bit_identical(small):
    hw = small["H"] * small["W"]
    a = _seg(small)
    a.set_frame(9)
    cls, _, _ = a.segmentImage(small["img"])
    want = a.computeVariance(cls)
    b = _seg(small)
    stream = torch.cuda.Stream()
    d_cls = torch.empty(hw, dtype=torch.uint8, device="cuda")
    d_conf = torch.empty(hw, dtype=torch.float64, device="cuda")
    d_ent = torch.empty(hw, dtype=torch.float64, device="cuda")
    d_var = torch.full((hw,), -1.0, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    b.set_frame(9)
    b.run_device(small["bgr"].data_ptr(), d_cls.data_ptr(), d_conf.data_ptr(), d_ent.data_ptr(), stream.cuda_stream)
    b.variance_device(d_cls.data_ptr(), d_var.data_ptr(), stream.cuda_stream)  # the device's own map, same stream
    stream.synchronize()
    assert np.array_equal(d_cls.cpu().numpy().reshape(cls.shape), cls)
    got = d_var.cpu().numpy().reshape(want.shape)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    # segment_on_device leaves the same samples; a pinned (page-locked) output buffer takes the direct copy
    a.set_frame(9)
    a.segment_on_device(small["img"])
    pinned = torch.empty((small["H"], small["W"]), dtype=torch.float64).pin_memory()
    L.check(L.lib().sivo_segnet_variance(a._h, cls.ctypes.data_as(C.c_void_p), C.c_void_p(pinned.data_ptr())))
    assert np.array_equal(pinned.numpy().view(np.uint64), want.view(np.uint64))


def test_variance_calls_do_not_change_the_frames_around_them(small):
    hw = small["H"] * small["W"]

    def frames(with_variance):
        seg = _seg(small)
        seg.set_frame(3)
        outs = []
        var = torch.empty(hw, dtype=torch.float64, device="cuda")
        for _ in range(3):
            m = [torch.empty(hw, dtype=torch.uint8, device="cuda")] + [torch.empty(hw, dtype=dt, device="cuda") for dt in
                                                                        (torch.float64, torch.float64, torch.float32, torch.float32)]
            torch.cuda.synchronize()
            seg.run_device_maps(small["bgr"].data_ptr(), *[t.data_ptr() for t in m])
            torch.cuda.synchronize()
            if with_variance:
                seg.variance_device(m[0].data_ptr(), var.data_ptr())
                seg.computeVariance(m[0].cpu().numpy().reshape(small["H"], small["W"]))
            torch.cuda.synchronize()
            outs.append([t.cpu().numpy().view(np.uint8) for t in m])
        return outs

    a, b = frames(False), frames(True)
    assert all(np.array_equal(x, y) for fa, fb in zip(a, b) for x, y in zip(fa, fb))
    assert not np.array_equal(a[0][2], a[1][2])  # the frame counter advanced between the frames


def _moments(seg, d_cls, hw):
    m = torch.empty(hw * 2, dtype=torch.float64, device="cuda")
    seg.variance_partial(d_cls.data_ptr(), m.data_ptr())
    torch.cuda.synchronize()
    return m


def test_latency_mode_moments_combine_to_the_whole_frame_variance(small):
    T, hw = small["T"], small["H"] * small["W"]
    full = _seg(small)
    full.set_frame(4)
    cls, _, _ = full.segmentImage(small["img"])
    cls[::7, ::5] = 255
    want = full.computeVariance(cls)
    d_cls = torch.from_numpy(cls.reshape(-1)).cuda()
    d_var = torch.empty(hw, dtype=torch.float64, device="cuda")
    for split in ([(0, T)], sample_ranges(T, 3)):
        total = None
        for b, n in split:
            shard = _seg(small, samples=(b, n))
            s = torch.empty(hw * 16, dtype=torch.float64, device="cuda")
            shard.set_frame(4)
            shard.run_partial(small["bgr"].data_ptr(), s.data_ptr())
            torch.cuda.synchronize()
            m = _moments(shard, d_cls, hw).cpu()
            total = m if total is None else total + m  # summed on the host in rank order
        shard.variance_finalize(total.cuda().data_ptr(), d_var.data_ptr())
        torch.cuda.synchronize()
        got = d_var.cpu().numpy().reshape(want.shape)
        print(f"split {split}: |d variance| max {np.abs(got - want).max():.2e}")
        assert np.abs(got - want).max() <= 1e-12 and not got[::7, ::5].any()


def test_bad_arguments_get_the_right_error_codes(small, model_dir):
    T, hw = small["T"], small["H"] * small["W"]
    lib = L.lib()
    cls = np.zeros((small["H"], small["W"]), np.uint8)
    var = np.empty((small["H"], small["W"]), np.float64)
    d_cls = torch.zeros(hw, dtype=torch.uint8, device="cuda")
    d_buf = torch.zeros(hw * 2, dtype=torch.float64, device="cuda")
    p = lambda a: C.c_void_p(a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr())
    fresh = _seg(small)
    h = fresh._h
    # null handle / buffers
    assert lib.sivo_segnet_variance(None, p(cls), p(var)) == L.EINVAL
    assert lib.sivo_segnet_variance_device(None, p(d_cls), p(d_buf), None) == L.EINVAL
    assert lib.sivo_segnet_variance_partial_device(None, p(d_cls), p(d_buf), None) == L.EINVAL
    assert lib.sivo_segnet_variance_finalize_device(None, p(d_buf), p(d_buf), None) == L.EINVAL
    assert lib.sivo_segnet_variance(h, None, p(var)) == L.EINVAL
    assert lib.sivo_segnet_variance(h, p(cls), None) == L.EINVAL
    assert lib.sivo_segnet_variance_device(h, None, p(d_buf), None) == L.EINVAL
    assert lib.sivo_segnet_variance_device(h, p(d_cls), None, None) == L.EINVAL
    assert lib.sivo_segnet_variance_partial_device(h, None, p(d_buf), None) == L.EINVAL
    assert lib.sivo_segnet_variance_partial_device(h, p(d_cls), None, None) == L.EINVAL
    assert lib.sivo_segnet_variance_finalize_device(h, None, p(d_buf), None) == L.EINVAL
    assert lib.sivo_segnet_variance_finalize_device(h, p(d_buf), None, None) == L.EINVAL
    # no frame run yet
    for call in (lambda: fresh.computeVariance(cls), lambda: fresh.variance_device(d_cls.data_ptr(), d_buf.data_ptr()),
                 lambda: fresh.variance_partial(d_cls.data_ptr(), d_buf.data_ptr())):
        with pytest.raises(L.SivoError) as e:
            call()
        assert e.value.code == L.EINVAL and "not run a frame" in str(e.value)
    with pytest.raises(ValueError):
        fresh.computeVariance(np.zeros((3, 3), np.uint8))
    # the whole-frame forms on a shard owning fewer than T samples point to the partial / finalise pair
    shard = _seg(small, samples=(2, 2))
    s = torch.empty(hw * 16, dtype=torch.float64, device="cuda")
    shard.run_partial(small["bgr"].data_ptr(), s.data_ptr())
    torch.cuda.synchronize()
    for call in (lambda: shard.computeVariance(cls), lambda: shard.variance_device(d_cls.data_ptr(), d_buf.data_ptr())):
        with pytest.raises(L.SivoError) as e:
            call()
        assert e.value.code == L.EINVAL and "run_partial_device" in str(e.value) and "finalize_device" in str(e.value)
    shard.variance_partial(d_cls.data_ptr(), d_buf.data_ptr())
    torch.cuda.synchronize()
    # more than 16 classes: the whole-frame form runs the generic kernel, the moments are refused as run_partial is
    _, _, proto21, model21 = make_model(model_dir, "basic", T=T, H=32, W=64, classes=21, calibrated=False)
    seg21 = BayesianSegNet(BayesianSegNetParams(proto21, model21), seed=1, T=T)
    img = np.ascontiguousarray(small["img"][:32, :64])
    c21, _, _ = seg21.segmentImage(img)
    v21 = seg21.computeVariance(c21)
    assert np.isfinite(v21).all() and (v21 >= 0).all()
    d21 = torch.from_numpy(c21.reshape(-1)).cuda()
    with pytest.raises(L.SivoError) as e:
        seg21.variance_partial(d21.data_ptr(), d_buf.data_ptr())
    assert e.value.code == L.EFORMAT


def test_latency_check_two_ranks_with_variance():
    """tools/latency_check.py --variance: every rank's moments reduced to rank 0 and finalised, against a whole-frame handle."""
    n = torch.cuda.device_count()
    world = min(n, 4) if n >= 2 else 2
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
                        "127.0.0.1", "--master-port", "29617", os.path.join(ROOT, "tools", "latency_check.py"), "--variance"],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "LATENCY OK" in r.stdout and "VARIANCE OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
