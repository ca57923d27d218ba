"""Emits the two Bayesian SegNet topologies as Caffe prototxt text from a compact description, so the
bench and tests have model files without the reference tree.  The layer names,
blob names and hyper-parameters are the ones `Net::CopyTrainedLayersFrom` matches weights against
(config/bayesian_segnet/{basic,standard}/kitti/*.prototxt in the reference); tests/test_host.py checks that these parse to
the reference's layer list (stored in tests/golden/reference_topology.json.gz).

usage: python tools/gen_prototxt.py   -> configs/bayesian_segnet_basic.prototxt, configs/bayesian_segnet.prototxt
"""
import os
import sys


def conv(name, bottom, top, cout, k, filler, pad=None):
    pad = (k - 1) // 2 if pad is None else pad
    pad_line = f"    pad: {pad}\n" if pad else ""
    return (f'layer {{\n  name: "{name}"\n  type: "Convolution"\n  bottom: "{bottom}"\n  top: "{top}"\n'
            f'  param {{ lr_mult: 1 decay_mult: 1 }}\n  param {{ lr_mult: 2 decay_mult: 0 }}\n'
            f'  convolution_param {{\n    num_output: {cout}\n{pad_line}    kernel_size: {k}\n'
            f'    weight_filler {{ type: "{filler}" }}\n    bias_filler {{ type: "constant" }}\n  }}\n}}\n')


def relu(name, blob):
    return f'layer {{\n  name: "{name}"\n  type: "ReLU"\n  bottom: "{blob}"\n  top: "{blob}"\n}}\n'


def bn(name, blob):
    return (f'layer {{\n  name: "{name}"\n  type: "BN"\n  bottom: "{blob}"\n  top: "{blob}"\n'
            f'  bn_param {{\n    bn_mode: INFERENCE\n    scale_filler {{ type: "constant" value: 1 }}\n'
            f'    shift_filler {{ type: "constant" value: 0 }}\n  }}\n}}\n')


def pool(name, bottom):
    return (f'layer {{\n  name: "{name}"\n  type: "Pooling"\n  bottom: "{bottom}"\n  top: "{name}"\n  top: "{name}_mask"\n'
            f'  pooling_param {{ pool: MAX kernel_size: 2 stride: 2 }}\n}}\n')


def drop(name, blob):
    return (f'layer {{\n  name: "{name}"\n  type: "Dropout"\n  bottom: "{blob}"\n  top: "{blob}"\n'
            f'  dropout_param {{ dropout_ratio: 0.5 sample_weights_test: true }}\n}}\n')


def upsample(name, bottom, mask, top):
    return (f'layer {{\n  name: "{name}"\n  type: "Upsample"\n  bottom: "{bottom}"\n  bottom: "{mask}"\n  top: "{top}"\n'
            f'  upsample_param {{ scale: 2 }}\n}}\n')


def softmax(bottom):
    return f'layer {{\n  name: "prob"\n  type: "Softmax"\n  bottom: "{bottom}"\n  top: "prob"\n  softmax_param {{ engine: CAFFE }}\n}}\n'


def header(name, T, H, W):
    return f'name: "{name}"\ninput: "data"\ninput_dim: {T}\ninput_dim: 3\ninput_dim: {H}\ninput_dim: {W}\n'


def basic(T=6, H=352, W=1024, width=64, classes=15):
    s = header("bayesian_segnet_basic", T, H, W)
    s += ('layer {\n  name: "norm"\n  type: "LRN"\n  bottom: "data"\n  top: "norm"\n'
          '  lrn_param { local_size: 5 alpha: 9.99999974738e-05 beta: 0.75 }\n}\n')
    prev = "norm"
    for i in (1, 2, 3, 4):
        s += conv(f"conv{i}", prev, f"conv{i}", width, 7, "msra") + relu(f"relu{i}", f"conv{i}") + pool(f"pool{i}", f"conv{i}")
        prev = f"pool{i}"
        if i >= 3:
            s += drop(f"encdrop{i}", prev)
    for i in (4, 3, 2, 1):
        s += upsample(f"upsample{i}", prev, f"pool{i}_mask", f"upsample{i}")
        s += conv(f"conv_decode{i}", f"upsample{i}", f"conv_decode{i}", width, 7, "msra")
        prev = f"conv_decode{i}"
        if i >= 3:
            s += drop(f"decdrop{i}", prev)
    s += conv("dense_softmax_inner_prod", prev, "dense_softmax_inner_prod", classes, 1, "msra")
    s += softmax("dense_softmax_inner_prod")
    return s


def standard(T=12, H=352, W=1024, widths=(64, 128, 256, 512, 512), classes=15):
    s = header("bayesian_segnet", T, H, W)
    depth = (2, 2, 3, 3, 3)
    prev = "data"
    for b in range(5):
        for j in range(depth[b]):
            n = f"conv{b + 1}_{j + 1}"
            s += conv(n, prev, n, widths[b], 3, "xavier") + bn(n + "_bn", n) + relu(f"relu{b + 1}_{j + 1}", n)
            prev = n
        s += pool(f"pool{b + 1}", prev)
        prev = f"pool{b + 1}"
        if b >= 2:
            s += drop(f"pool{b + 1}_drop", prev)
    for b in (4, 3, 2, 1, 0):
        top = f"pool{b + 1}_D"
        s += upsample(f"upsample{b + 1}", prev, f"pool{b + 1}_mask", top)
        prev = top
        for j in range(depth[b], 0, -1):
            n = f"conv{b + 1}_{j}_D"
            last = (b == 0 and j == 1)
            cout = classes if last else (widths[b] if j > 1 else (widths[b - 1] if b > 0 else widths[0]))
            s += conv(n, prev, n, cout, 3, "xavier", pad=1)
            if not last:
                s += bn(n + "_bn", n) + relu(f"relu{b + 1}_{j}_D", n)
            prev = n
            if j == 1 and b in (4, 3, 2):
                s += drop(f"upsample{b}_drop", prev)
    s += softmax(prev)
    return s


if __name__ == "__main__":
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "configs")
    os.makedirs(root, exist_ok=True)
    open(os.path.join(root, "bayesian_segnet_basic.prototxt"), "w").write(basic())
    open(os.path.join(root, "bayesian_segnet.prototxt"), "w").write(standard())
    print("wrote configs/")
