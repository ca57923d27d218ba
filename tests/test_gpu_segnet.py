"""-m gpu: `BayesianSegNet::segmentImage` through the C-ABI against the oracle -- blob by blob on small
nets (identical weights and dropout masks), against the committed golden fixtures, and at the full
1024x352 geometry.

Max-pool argmax positions are the one discontinuous step of the net: two window entries that differ by
<= 1 ulp can swap order between two fp32 summation orders (the same happens between the reference's own CPU
and cuDNN paths), and one swapped position moves a whole activation under the next filter.  The tests
therefore (1) check that every device mask either equals the oracle's or picks a value within 2 ulp of the
oracle's maximum, and (2) hand the device's masks to the oracle (`masks=`) and require everything else --
every blob, the classes, confidence and entropy -- to agree tightly."""
import os

import numpy as np
import pytest
import torch

from conftest import make_model, GOLDEN
from oracle import segnet_oracle as S
from sivo_b200 import BayesianSegNet, BayesianSegNetParams
from sivo_b200.synth import stereo_frame

pytestmark = pytest.mark.gpu

ENGINES = ["simt", "auto"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _crop(kitti_bgr, h, w):
    return np.ascontiguousarray(kitti_bgr[100:100 + h, 300:300 + w])


def device_masks(seg, net):
    return {ly.tops[1]: seg.blob(ly.tops[1]).astype(np.int64) for ly in net.layers if ly.type == "Pooling"}


def check_masks_are_ties(net, blobs, masks, prec):
    """Where a device mask differs from the oracle's own argmax, both must point at (nearly) the same value."""
    flips = total = 0
    for ly in net.layers:
        if ly.type != "Pooling":
            continue
        x = blobs[ly.bottoms[0]]
        _, own = S.pool_with_mask(x)
        m = torch.from_numpy(masks[ly.tops[1]])[:x.shape[0]]
        flat = x.reshape(x.shape[0], x.shape[1], -1)
        v_dev = torch.gather(flat, 2, m.reshape(m.shape[0], m.shape[1], -1))
        v_own = torch.gather(flat, 2, own.reshape(own.shape[0], own.shape[1], -1))
        diff = (m != own).reshape(m.shape[0], m.shape[1], -1)
        # 2 ulp of the stored precision, plus the input-rounding noise of the producing convolution: each output sums
        # hundreds of stored inputs, ~0.2 % of which sit one ulp apart between two fp32 summation orders, so outputs
        # carry absolute noise of order 1e-4..1e-3 of the blob's scale whatever their own magnitude (fp32 engine: 1e-6)
        rel = 2.0 ** -9 if prec == "fp16" else 2.0 ** -20
        ok = (v_own - v_dev).abs() <= rel * v_own.abs() + (1e-3 if prec == "fp16" else 2e-6) * float(x.abs().max())
        assert bool(ok[diff].all()), (ly.name, float((v_own - v_dev).abs()[diff].max()), float(x.abs().max()))
        flips += int(diff.sum())
        total += diff.numel()
    return flips / max(total, 1)


@pytest.mark.parametrize("kind,kw", [("basic", dict(T=3, H=64, W=128)),
                                     ("standard", dict(T=2, H=64, W=128, widths=(64, 64, 64, 64, 64)))])
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("engine", ENGINES)
def test_blobs_match_oracle(model_dir, kitti_bgr, kind, kw, prec, engine):
    # fp32 + auto = split-operand tensor-core convolutions wherever Cin is a multiple of 64, the SIMT kernel for the 3-channel first layer
    net, w, proto, model = make_model(model_dir, kind, seed=0, **kw)
    img = _crop(kitti_bgr, kw["H"], kw["W"])
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, precision=prec, engine=engine, keep_blobs=True)
    seg.set_frame(0)
    cls, conf, ent = seg.segmentImage(img)
    masks = device_masks(seg, net)
    prob, blobs = S.forward(net, w, img, seed=1234, frame=0, precision=prec, return_blobs=True, masks=masks)
    flip_rate = check_masks_are_ties(net, blobs, masks, prec)
    assert flip_rate < 2e-3
    tol = 1e-4 if prec == "fp32" else 2e-3  # of the blob's scale; a half ulp is 4.9e-4 relative
    if prec == "fp32" and engine != "simt":
        tol = 2e-5  # split-operand tensor-core mode: fp32-grade, far inside caffe's own 1e-4 convolution tolerance
    for ly in net.layers:
        if ly.type in ("Softmax",):
            continue
        top = ly.tops[0]
        ref = blobs[top].numpy()
        got = seg.blob(top)
        if ref.shape[0] == 1 and got.shape[0] > 1:
            ref = np.repeat(ref, got.shape[0], axis=0)
        assert got.shape == ref.shape, top
        scale = max(1.0, float(np.abs(ref).max()))
        err = np.abs(got - ref)
        assert err.max() < 4 * tol * scale, (top, float(err.max()), scale)
        assert (err > tol * scale).mean() < 1e-3, (top, float(err.max()), scale)
    rc, rf, re = S.mc_reduce(prob)
    assert (cls != rc).mean() < 2e-3
    ok = cls == rc
    # Same-precision comparison (the oracle emulates the half rounding of operands and stored activations), calibrated
    # weights: what is left is fp32 summation order (and, on tensor cores, the accumulator's truncation) plus the occasional
    # 1-ulp difference of a stored half.  The fp32 modes are held to the reference's 1e-4.
    split = prec == "fp32" and engine != "simt"
    d_conf, d_ent = np.abs(conf - rf), np.abs(ent - re)
    print(f"blobs {kind}/{prec}/{engine}: class mismatch {(cls != rc).mean():.2e}, |d conf| max {d_conf.max():.2e}, "
          f"|d entropy| max {d_ent.max():.2e} q99 {np.quantile(d_ent, 0.99):.2e} median {np.median(d_ent):.2e}")
    assert d_conf[ok].max() < (1e-4 if prec == "fp32" else 5e-3)
    assert d_ent.max() < (1e-4 if prec == "fp32" else 2e-2)
    assert np.quantile(d_ent, 0.99) < (1e-4 if prec == "fp32" else 5e-3)
    assert np.median(d_ent) < ((2e-5 if split else 1e-6) if prec == "fp32" else 1e-3)


@pytest.mark.parametrize("kind", ["basic", "standard"])
@pytest.mark.parametrize("engine", ENGINES)
def test_matches_golden(model_dir, kitti_bgr, kind, engine):
    """Free-running comparison with the committed oracle outputs (no mask hand-over): statistical agreement."""
    g = np.load(os.path.join(GOLDEN, "segnet_small.npz"))
    kw = dict(T=3, H=64, W=128) if kind == "basic" else dict(T=2, H=64, W=128, widths=(64, 64, 64, 64, 64))
    _, _, proto, model = make_model(model_dir, kind, seed=0, **kw)
    img = _crop(kitti_bgr, 64, 128)
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, precision="fp16", engine=engine)
    seg.set_frame(0)
    cls, conf, ent = seg.segmentImage(img)
    # no mask hand-over here: a handful of swapped pooling positions perturb whole neighbourhoods of this untrained,
    # high-gain net, so the bar is statistical (a wrong kernel scores ~93 % class mismatch and O(1) entropy error)
    m16 = float((cls != g[f"{kind}_fp16_classes"]).mean())
    m32 = float((cls != g[f"{kind}_fp32_classes"]).mean())
    e16 = float(np.median(np.abs(ent - g[f"{kind}_fp16_entropy"])))
    c16 = float(np.median(np.abs(conf - g[f"{kind}_fp16_confidence"])))
    print(f"golden {kind}/{engine}: class mismatch fp16 {m16:.4f} fp32 {m32:.4f}, median |d entropy| {e16:.2e}, |d conf| {c16:.2e}")
    assert m16 < 0.15 and m32 < 0.25, (m16, m32)
    assert e16 < 5e-2 and c16 < 5e-2, (e16, c16)


def _full_model(model_dir, kind="basic", T=2):
    from sivo_b200.caffemodel import read_caffemodel, shipped_scales, write_synth_model
    from sivo_b200.prototxt import load_net
    name = "bayesian_segnet_basic.prototxt" if kind == "basic" else "bayesian_segnet.prototxt"
    proto = os.path.join(ROOT, "configs", name)
    net = load_net(open(proto).read(), T=T)
    model = os.path.join(str(model_dir), f"{kind}_full.caffemodel")
    if os.path.exists(model):
        return net, read_caffemodel(model), proto, model
    w = write_synth_model(net, model, 0, shipped_scales(kind))
    return net, w, proto, model


def test_output_sizes_and_crop_like_the_reference(model_dir, kitti_bgr):
    # tests/test_bayesian_segnet.cpp:152-168 (sizes == H*W) + resizeImage's centre crop of the 1242x375 frame
    net, w, proto, model = _full_model(model_dir)
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=2)
    assert seg.getInputGeometry() == (1024, 352)
    seg.set_frame(7)
    cls, conf, ent = seg.segmentImage(kitti_bgr)
    assert cls.size == conf.size == ent.size == 352 * 1024
    seg.set_frame(7)
    cls2, conf2, ent2 = seg.segmentImage(np.ascontiguousarray(kitti_bgr[11:11 + 352, 109:109 + 1024]))
    assert np.array_equal(cls, cls2) and np.array_equal(conf, conf2) and np.array_equal(ent, ent2)  # deterministic + crop origin (109, 11)
    # properties that hold at any size: probabilities, entropy bounds, argmax consistency
    assert conf.min() >= 1.0 / 15 - 1e-9 and conf.max() <= 1.0 + 1e-9
    assert ent.min() >= 0 and ent.max() <= np.log2(15) + 1e-9
    assert cls.max() < 15
    # a different frame index draws different masks
    cls3, _, ent3 = seg.segmentImage(kitti_bgr)
    assert not np.array_equal(ent, ent3)
    with pytest.raises(Exception):
        seg.segmentImage(np.zeros((100, 100, 3), np.uint8))


@pytest.mark.parametrize("engine", ENGINES)
def test_full_size_basic_against_oracle(model_dir, engine):
    """Config C1 geometry (Basic, T=2, 1024x352) on a synthetic frame: the whole operator vs the oracle."""
    net, w, proto, model = _full_model(model_dir)
    left, _ = stereo_frame(0)
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=2, precision="fp16", engine=engine, keep_blobs=True)
    seg.set_frame(3)
    cls, conf, ent = seg.segmentImage(left)
    masks = device_masks(seg, net)
    prob, blobs = S.forward(net, w, left, seed=1234, frame=3, precision="fp16", T=2, return_blobs=True, masks=masks)
    assert check_masks_are_ties(net, blobs, masks, "fp16") < 2e-3
    rc, rf, re = S.mc_reduce(prob)
    mism = float((cls != rc).mean())
    med, q99 = float(np.median(np.abs(ent - re))), float(np.quantile(np.abs(ent - re), 0.99))
    print(f"full-size basic/{engine}: class mismatch {mism:.2e}, |d entropy| median {med:.2e} q99 {q99:.2e}")
    assert mism < 5e-3, mism
    assert med < 1e-3 and q99 < 0.1, (med, q99)


def test_tcgen05_conv_equals_simt_conv_on_device(model_dir):
    """Both engines on the same frame: only the convolution engine differs, so every stored half must agree
    to within summation-order noise."""
    net, w, proto, model = _full_model(model_dir)
    left, _ = stereo_frame(1)
    outs = []
    for engine in ("simt", "tcgen05"):
        try:
            seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=2, precision="fp16", engine=engine, keep_blobs=True)
        except Exception as e:  # engine not available for this shape
            pytest.skip(str(e))
        seg.set_frame(0)
        seg.segmentImage(left)
        outs.append({n: seg.blob(n) for n in ("conv2",)})  # conv1 is SIMT in both, so conv2 sees identical inputs
    for n in outs[0]:
        a, b = outs[0][n], outs[1][n]
        scale = max(1.0, float(np.abs(a).max()))
        assert (np.abs(a - b) > 2e-3 * scale).mean() < 1e-3, n


def test_run_device_maps_writes_rounded_single_precision_copies(model_dir):
    """sivo_segnet_run_device_maps: the f32 maps of the packed multi-GPU record are the operator's double maps rounded to
    nearest, and the classes / double maps are those of segmentImage on the same frame."""
    import torch
    net, w, proto, model = _full_model(model_dir)
    left, _ = stereo_frame(2)
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=2)
    seg.set_frame(5)
    cls, conf, ent = (np.array(a) for a in seg.segmentImage(left))
    h, w_ = cls.shape
    y0, x0 = (left.shape[0] - h) // 2, (left.shape[1] - w_) // 2
    d_bgr = torch.from_numpy(np.ascontiguousarray(left[y0:y0 + h, x0:x0 + w_])).cuda()
    d_cls = torch.empty(h * w_, dtype=torch.uint8, device="cuda")
    d_c64, d_e64 = (torch.empty(h * w_, dtype=torch.float64, device="cuda") for _ in range(2))
    d_c32, d_e32 = (torch.empty(h * w_, dtype=torch.float32, device="cuda") for _ in range(2))
    seg.set_frame(5)
    seg.run_device_maps(d_bgr.data_ptr(), d_cls.data_ptr(), d_c64.data_ptr(), d_e64.data_ptr(), d_c32.data_ptr(), d_e32.data_ptr(),
                        torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_cls.cpu().numpy().reshape(h, w_), cls)
    assert np.array_equal(d_c64.cpu().numpy().reshape(h, w_), conf) and np.array_equal(d_e64.cpu().numpy().reshape(h, w_), ent)
    assert np.array_equal(d_c32.cpu().numpy(), conf.reshape(-1).astype(np.float32))
    assert np.array_equal(d_e32.cpu().numpy(), ent.reshape(-1).astype(np.float32))
    # segmentImage with record outputs set leaves the same three device-resident copies
    d_cls.zero_(), d_c32.zero_(), d_e32.zero_()
    seg.set_record_outputs(d_cls.data_ptr(), d_c32.data_ptr(), d_e32.data_ptr())
    seg.set_frame(5)
    cls_b, conf_b, ent_b = (np.array(a) for a in seg.segmentImage(left))
    seg.set_record_outputs()
    assert np.array_equal(cls_b, cls) and np.array_equal(conf_b, conf) and np.array_equal(ent_b, ent)
    assert np.array_equal(d_cls.cpu().numpy().reshape(h, w_), cls)
    assert np.array_equal(d_c32.cpu().numpy(), conf.reshape(-1).astype(np.float32))
    assert np.array_equal(d_e32.cpu().numpy(), ent.reshape(-1).astype(np.float32))
    # the f32 maps alone (double outputs NULL)
    d_c32.zero_()
    seg.set_frame(5)
    seg.run_device_maps(d_bgr.data_ptr(), d_cls.data_ptr(), 0, 0, d_c32.data_ptr(), 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_c32.cpu().numpy(), conf.reshape(-1).astype(np.float32))


def test_fused_epilogues_equal_the_unfused_ops(model_dir):
    """keep_blobs keeps max-unpool and the 1x1 classifier as their own kernels; the default build scatters from the
    tensor-core convolution's epilogue and composes conv_decode1 and the classifier into one 64 -> 16 convolution.  Unpool
    is the same arithmetic.  The composed convolution never rounds the 64-channel activation to half (the composed weights
    are), so its maps differ from the two layers' at the half-rounding level."""
    net, w, proto, model = _full_model(model_dir)
    left, _ = stereo_frame(2)
    res, pooled = [], []
    for keep in (True, False):
        seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=1234, T=2, precision="fp16", engine="auto", keep_blobs=keep)
        seg.set_frame(5)
        res.append(seg.segmentImage(left))
        # pooled activations, argmax masks and unpooled tensors exist in both builds; fused or not they are the same arithmetic
        pooled.append({n: seg.blob(n) for n in ("pool1", "pool1_mask", "pool2", "pool2_mask", "pool3_mask", "pool4_mask",
                                                "upsample4", "upsample3", "upsample1")})
        if not keep:  # blobs a fused kernel consumes in registers are refused, not returned stale
            for elided in ("conv1", "conv_decode1", "norm"):
                with pytest.raises(Exception):
                    seg.blob(elided)
    for n in pooled[0]:
        assert np.array_equal(pooled[0][n], pooled[1][n]), n
    (c0, f0, e0), (c1, f1, e1) = res
    assert not np.array_equal(e0, e1), "the composed kernel did not engage"
    assert (c0 != c1).mean() < 2e-3
    assert np.abs(e0 - e1).max() < 2e-2 and np.median(np.abs(e0 - e1)) < 1e-3
    assert np.abs(f0 - f1).max() < 1e-2


def test_semantic_keys_match_the_oracle_on_device_resident_maps(model_dir):
    """Next-row 8(f)-2: SelectSemanticKeys + per-keypoint map reads evaluated on the device (bit-exact: pure indexing),
    both after a normal segmentImage and after the no-read-back call."""
    from oracle import orb_oracle as O
    from sivo_b200 import ORBextractor
    net, w, proto, model = _full_model(model_dir)
    from sivo_b200.synth import bgr_to_gray
    left, _ = stereo_frame(3)
    seg = BayesianSegNet(BayesianSegNetParams(proto, model), seed=7, T=2, precision="fp16", engine="auto")
    seg.set_frame(9)
    classes, conf, ent = seg.segmentImage(left)
    # the extractor sees the same crop the network does (resizeImage, bayesian_segnet.cpp:142-162)
    y0, x0 = left.shape[0] // 2 - seg.height // 2, left.shape[1] // 2 - seg.width // 2
    g = np.ascontiguousarray(bgr_to_gray(left)[y0:y0 + seg.height, x0:x0 + seg.width])
    kps, _ = ORBextractor(1000, 1.2, 8, 20, 7)(g, None)
    assert len(kps) > 500
    xy = np.stack([kps["x"], kps["y"]], 1)
    want = O.select_semantic_keys(xy, classes, conf, ent)
    for attempt in range(2):
        got = seg.semantic_keys(kps)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
        assert np.array_equal(got[3], want[3])
        seg.set_frame(9)
        seg.segment_on_device(left)  # same frame counter -> same dropout masks -> same maps, left on the device
    # out-of-map keypoints: class 255, never kept; an empty list is fine
    bad = kps[:3].copy()
    bad["x"][0] = -5.0
    bad["y"][1] = 1e6
    c, _, _, keep = seg.semantic_keys(bad)
    assert c[0] == 255 and c[1] == 255 and 0 not in keep and 1 not in keep
    assert len(seg.semantic_keys(kps[:0])[3]) == 0


def test_bn_absorbed_model_runs_and_agrees(tmp_path):
    """8(f)-3: the model BN-absorber.py would write (BN folded into the convolutions, BN layers dropped) goes through the same
    tensor-core path and gives the same segmentation as the BN form up to the half rounding of W * gamma."""
    from sivo_b200 import bn_absorb
    from sivo_b200.caffemodel import write_caffemodel
    from sivo_b200.prototxt import load_net
    net, w, proto, model = make_model(tmp_path, "standard", T=3, H=64, W=128, widths=(64, 64, 64, 64, 64))
    new_text, new_w = bn_absorb.absorb(open(proto).read(), w)
    p2, m2 = str(tmp_path / "merged.prototxt"), str(tmp_path / "merged.caffemodel")
    open(p2, "w").write(new_text)
    types = {l.name: l.type for l in net.layers}
    write_caffemodel(m2, net.name, new_w, {k: types[k] for k in new_w})
    left, _ = stereo_frame(4, w=128, h=64)
    outs, first = [], []
    for pr, mo in ((proto, model), (p2, m2)):
        seg = BayesianSegNet(BayesianSegNetParams(pr, mo), seed=11, precision="fp16", engine="auto", keep_blobs=True)
        seg.set_frame(2)
        outs.append(seg.segmentImage(left))
        first.append({n: seg.blob(n) for n in ("conv1_1", "conv1_2")})
    # upstream of the first pooling decision the two forms differ only by the half rounding of W * gamma vs gamma * (W x)
    for n in first[0]:
        a, b = first[0][n], first[1][n]
        assert np.abs(a - b).max() < 4e-3 * max(1.0, float(np.abs(a).max())), n
    (c0, f0, e0), (c1, f1, e1) = outs
    # downstream, a handful of swapped pooling positions move whole neighbourhoods of this untrained net (see the module
    # docstring), so the final maps agree statistically
    mism, de, df = float((c0 != c1).mean()), float(np.median(np.abs(e0 - e1))), float(np.median(np.abs(f0 - f1)))
    print(f"bn-absorbed vs bn form: class mismatch {mism:.3f}, median |d entropy| {de:.2e}, median |d conf| {df:.2e}")
    assert mism < 0.3 and de < 0.1 and df < 0.05
