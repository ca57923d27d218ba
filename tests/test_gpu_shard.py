"""-m gpu: latency mode (SURVEY 8e, DESIGN §6) on one device -- shard handles that run part of a frame's Monte-Carlo samples,
their partial softmax sums and the finalise step, against a whole-frame handle on the same frame.

Basic T=6 at the full 1024x352 geometry and Standard at a reduced size, in the fast (fp16) and strict (fp32) precisions.  What
is expected to be exact is exact: a shard's sample n draws the masks of global sample begin + n and every pixel's accumulation
order is fixed by the convolution's tap / chunk loop (not by how rows spread over CTAs), so its logits are the whole-frame
handle's bit for bit; the shard [0, T) followed by finalize is the one-pass reduction bit for bit.  Sums of several shards added
in float64 differ from the one-pass sum only by reassociation."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import make_model
from sivo_b200 import BayesianSegNet, BayesianSegNetParams, sample_ranges
from sivo_b200 import _lib as L
from sivo_b200.prototxt import load_net
from sivo_b200.synth import stereo_frame

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 6
SPLITS = [[(0, 3), (3, 3)], [(0, 2), (2, 2), (4, 1), (5, 1)], [(n, 1) for n in range(T)]]
FRAME = 5


def _basic_full(model_dir):
    from sivo_b200.caffemodel import shipped_scales, write_synth_model
    proto = os.path.join(ROOT, "configs", "bayesian_segnet_basic.prototxt")
    net = load_net(open(proto).read(), T=T)
    model = os.path.join(str(model_dir), "basic_full_shard.caffemodel")
    if not os.path.exists(model):
        write_synth_model(net, model, 0, shipped_scales("basic"))
    return proto, model


@pytest.fixture(scope="module", params=["basic_full", "standard_small"])
def case(request, model_dir):
    if request.param == "basic_full":
        proto, model = _basic_full(model_dir)
        H, W = 352, 1024
    else:
        _, _, proto, model = make_model(model_dir, "standard", T=T, H=64, W=128, widths=(64, 64, 64, 64, 64))
        H, W = 64, 128
    left, _ = stereo_frame(2)
    y0, x0 = (left.shape[0] - H) // 2, (left.shape[1] - W) // 2
    d_bgr = torch.from_numpy(np.ascontiguousarray(left[y0:y0 + H, x0:x0 + W])).cuda()
    net = load_net(open(proto).read(), T=T)
    return dict(name=request.param, proto=proto, model=model, H=H, W=W, bgr=d_bgr, logits=net.layers[-1].bottoms[0])


def _seg(case, prec, samples=None, keep_blobs=False):
    return BayesianSegNet(BayesianSegNetParams(case["proto"], case["model"]), seed=1234, T=T, precision=prec, keep_blobs=keep_blobs,
                          samples=samples)


def _maps(hw):
    return dict(cls=torch.empty(hw, dtype=torch.uint8, device="cuda"), c64=torch.empty(hw, dtype=torch.float64, device="cuda"),
                e64=torch.empty(hw, dtype=torch.float64, device="cuda"), c32=torch.empty(hw, dtype=torch.float32, device="cuda"),
                e32=torch.empty(hw, dtype=torch.float32, device="cuda"))


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _run_full(seg, case, frame=FRAME):
    m = _maps(case["H"] * case["W"])
    if frame is not None:
        seg.set_frame(frame)
    seg.run_device_maps(case["bgr"].data_ptr(), m["cls"].data_ptr(), m["c64"].data_ptr(), m["e64"].data_ptr(), m["c32"].data_ptr(),
                        m["e32"].data_ptr(), _stream())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in m.items()}


def _partial(seg, case, frame=FRAME):
    s = torch.empty(case["H"] * case["W"] * 16, dtype=torch.float64, device="cuda")
    if frame is not None:
        seg.set_frame(frame)
    seg.run_partial(case["bgr"].data_ptr(), s.data_ptr(), _stream())
    torch.cuda.synchronize()  # the default stream's handle is 0, i.e. the library's own stream: order the sum before torch reads it
    return s


def _finalize(seg, case, total):
    m = _maps(case["H"] * case["W"])
    seg.finalize(total.data_ptr(), m["cls"].data_ptr(), m["c64"].data_ptr(), m["e64"].data_ptr(), m["c32"].data_ptr(), m["e32"].data_ptr(),
                 _stream())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in m.items()}


def _same(a, b):
    return all(np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)) for k in a)


@pytest.mark.parametrize("prec", ["fp16", "fp32"])
def test_whole_frame_shard_then_finalize_is_bit_identical_to_run_device_maps(case, prec):
    full = _seg(case, prec)
    shard = _seg(case, prec, samples=(0, T))
    assert (shard.sample_begin, shard.sample_count, shard.T) == (0, T, T)
    want = _run_full(full, case)
    got = _finalize(shard, case, _partial(shard, case))
    assert _same(got, want), case["name"]
    # second frame without set_frame: run_partial advances the frame counter exactly as run_device does (graph replay)
    want2 = _run_full(full, case, frame=None)
    got2 = _finalize(shard, case, _partial(shard, case, frame=None))
    assert _same(got2, want2) and not np.array_equal(want2["e64"], want["e64"])
    # the partial sum's padding channels are zero and each pixel's sum is T (each sample's softmax sums to ~1)
    s = _partial(shard, case).view(-1, 16).cpu().numpy()
    assert not s[:, 15:].any() if case["name"] == "basic_full" else True
    assert np.abs(s.sum(axis=1) - T).max() < 1e-4


@pytest.mark.parametrize("keep_blobs", [False, True])
@pytest.mark.parametrize("prec", ["fp16", "fp32"])
def test_shards_draw_the_whole_frames_samples_and_their_sums_combine(case, prec, keep_blobs):
    """Default build: dropout in the convolution epilogue and the dropout + unpool kernel; keep_blobs: the standalone dropout
    kernels.  Between them all four dropout sites run with a sample offset."""
    full = _seg(case, prec, keep_blobs=keep_blobs)
    want = _run_full(full, case)
    full_logits = full.blob(case["logits"])
    del full
    for split in SPLITS:
        total, fin = None, None
        for b, n in split:
            seg = _seg(case, prec, samples=(b, n), keep_blobs=keep_blobs)
            s = _partial(seg, case)
            torch.cuda.synchronize()
            got = seg.blob(case["logits"])
            assert got.shape[0] == n
            assert np.array_equal(got.view(np.uint32), full_logits[b:b + n].view(np.uint32)), (case["name"], prec, keep_blobs, b, n)
            total = s if total is None else total + s  # float64 adds in rank order: what a reduce over ranks computes
            if fin is None:
                fin = seg
            else:
                del seg
        got = _finalize(fin, case, total)
        del fin
        mean = (total.view(-1, 16) / T).cpu().numpy()
        top2 = np.sort(mean, axis=1)[:, -2:]
        tie = (top2[:, 1] - top2[:, 0]) < 1e-12
        diff = got["cls"] != want["cls"]
        print(f"{case['name']}/{prec}/keep={keep_blobs} split {split}: class mismatches {int(diff.sum())} "
              f"(near-tie pixels {int(tie.sum())}), |d conf| {np.abs(got['c64'] - want['c64']).max():.1e}, "
              f"|d entropy| {np.abs(got['e64'] - want['e64']).max():.1e}")
        assert not (diff & ~tie).any()
        assert np.abs(got["c64"] - want["c64"]).max() <= 1e-12
        assert np.abs(got["e64"] - want["e64"]).max() <= 1e-6
        assert np.abs(got["c32"] - want["c32"]).max() <= 1e-6 and np.abs(got["e32"] - want["e32"]).max() <= 1e-6


def _keypoints(H, W, n=3000, seed=0):
    from sivo_b200.orb import KP_DTYPE
    rng = np.random.default_rng(seed)
    kps = np.zeros(n, KP_DTYPE)
    kps["x"] = rng.uniform(-3, W + 3, n).astype(np.float32)  # a few outside the maps
    kps["y"] = rng.uniform(-3, H + 3, n).astype(np.float32)
    return kps


def test_semantic_keys_after_finalize_equal_those_after_run_device(case):
    full = _seg(case, "fp16")
    shard = _seg(case, "fp16", samples=(0, T))
    kps = _keypoints(case["H"], case["W"])
    _run_full(full, case)
    want = full.semantic_keys(kps)
    _finalize(shard, case, _partial(shard, case))
    got = shard.semantic_keys(kps)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert len(want[3]) > 0
    # a whole-frame handle finalises a sum too, and its keypoint reads then follow the finalised maps
    _finalize(full, case, _partial(shard, case))
    assert all(np.array_equal(a, b) for a, b in zip(full.semantic_keys(kps), want))


def test_bad_sample_ranges_and_refused_calls(model_dir):
    _, _, proto, model = make_model(model_dir, "basic", T=T, H=64, W=128)
    params = BayesianSegNetParams(proto, model)
    for bad in [(-1, 2), (0, 0), (2, -1), (5, 2), (0, T + 1), (T, 1)]:
        with pytest.raises(ValueError):
            BayesianSegNet(params, T=T, samples=bad)
    with pytest.raises(ValueError):  # T <= 1 keeps the reference's constructor error
        BayesianSegNet(params, T=1, samples=(0, 1))
    lib = L.lib()
    opt = L.SegnetOptions(device=0, T=T, seed=1, precision=0, engine=0, keep_blobs=0, reserved=0)
    assert lib.sivo_segnet_create_shard(proto.encode(), model.encode(), C.byref(opt), 0, 1, None) == L.EINVAL
    shard = BayesianSegNet(params, T=T, samples=(4, 2))
    assert (shard.sample_begin, shard.sample_count, shard.T) == (4, 2, T)
    hw = shard.width * shard.height
    bgr = torch.zeros(hw * 3, dtype=torch.uint8, device="cuda")
    s = torch.zeros(hw * 16, dtype=torch.float64, device="cuda")
    out = torch.empty(hw, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    h = shard._h
    assert lib.sivo_segnet_run_partial_device(h, None, C.c_void_p(s.data_ptr()), None) == L.EINVAL
    assert lib.sivo_segnet_run_partial_device(h, C.c_void_p(bgr.data_ptr()), None, None) == L.EINVAL
    assert lib.sivo_segnet_finalize_device(h, None, None, C.c_void_p(out.data_ptr()), None, None, None, None) == L.EINVAL
    assert lib.sivo_segnet_run_partial_device(None, C.c_void_p(bgr.data_ptr()), C.c_void_p(s.data_ptr()), None) == L.EINVAL
    # the whole-frame operator on a partial shard: refused, and the message names the partial / finalise pair
    for call in (lambda: shard.run_device(bgr.data_ptr(), 0, out.data_ptr(), 0),
                 lambda: shard.run_device_maps(bgr.data_ptr(), 0, out.data_ptr(), 0, 0, 0),
                 lambda: shard.segmentImage(np.zeros((64, 128, 3), np.uint8))):
        with pytest.raises(L.SivoError) as e:
            call()
        assert e.value.code == L.EINVAL and "run_partial_device" in str(e.value) and "finalize_device" in str(e.value)
    # ... while the partial / finalise pair runs
    shard.run_partial(bgr.data_ptr(), s.data_ptr())
    shard.finalize(s.data_ptr(), 0, out.data_ptr(), 0)
    torch.cuda.synchronize()
    # counters: prefix once + sample_count x the per-sample part; profiling covers the partial op list
    fl = {n: BayesianSegNet(params, T=T, samples=(0, n)).flops() for n in (1, 2, 3)}
    whole = BayesianSegNet(params, T=T).flops()
    per = fl[2]["dedup"] - fl[1]["dedup"]
    assert per > 0 and abs(fl[3]["dedup"] - fl[1]["dedup"] - 2 * per) < 1e-6 * whole["dedup"]
    assert abs(whole["dedup"] - fl[1]["dedup"] - (T - 1) * per) < 1e-6 * whole["dedup"]
    assert abs(fl[3]["naive"] * T / 3 - whole["naive"]) < 1e-6 * whole["naive"]
    shard.set_profiling(True)
    shard.run_partial(bgr.data_ptr(), s.data_ptr())
    t = shard.last_timing()
    assert t["launches"] == len(shard.op_timings()) and t["total_ms"] > 0 and t["reduce_ms"] > 0


def test_latency_check_two_ranks():
    """tools/latency_check.py under torch.distributed.run: NCCL with one GPU per rank (up to 4 ranks, so T=6 splits unevenly)
    where there are enough devices, else gloo with both ranks on device 0 and the sums staged through host memory."""
    n = torch.cuda.device_count()
    world = min(n, 4) if n >= 2 else 2
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
                        "127.0.0.1", "--master-port", "29613", os.path.join(ROOT, "tools", "latency_check.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "LATENCY OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
