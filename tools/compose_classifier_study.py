"""CPU study: how does composing conv_decode1 with the 1x1 classifier
(logits = (Wc W) * x + Wc b + bc, half weights, fp32 accumulation) compare with today's two-step fp16 path, both measured
against the same two convolutions evaluated in float64 on the same (half-rounded) input?  Oracle only; no GPU."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gen_prototxt  # noqa: E402
from oracle import segnet_oracle as S  # noqa: E402
from sivo_b200.caffemodel import synth_weights  # noqa: E402
from sivo_b200.prototxt import load_net  # noqa: E402
from sivo_b200.synth import stereo_frame  # noqa: E402

H, W, T = 96, 256, 2
net = load_net(gen_prototxt.basic(T=T, H=H, W=W))
w = synth_weights(net, 0)
left, _ = stereo_frame(0)
img = np.ascontiguousarray(left[100:100 + H, 300:300 + W])
prob, blobs = S.forward(net, w, img, seed=1234, frame=0, precision="fp16", return_blobs=True)
x = torch.as_tensor(np.asarray(blobs["upsample1"])).to(torch.float64)          # [T, 64, H, W], half-representable values
Wd, bd = [torch.from_numpy(a.astype(np.float64)) for a in w["conv_decode1"]]
Wc, bc = [torch.from_numpy(a.astype(np.float64)) for a in w["dense_softmax_inner_prod"]]
bd, bc = bd.reshape(-1), bc.reshape(-1)


def h(t):  # round to IEEE half, back to float64
    return t.to(torch.float16).to(torch.float64)


conv = torch.nn.functional.conv2d
truth = conv(conv(x, Wd, bd, padding=3), Wc, bc)                      # float64, unrounded weights: the reference's arithmetic
two_step = conv(h(conv(x, h(Wd), bd, padding=3)), h(Wc), bc)          # today's path: half weights, activation rounded to half
Wcomp = torch.einsum("oc,cikl->oikl", Wc[:, :, 0, 0], Wd)             # composed 15 x 64 x 7 x 7 weights (float64)
bcomp = Wc[:, :, 0, 0] @ bd + bc
composed = conv(x, h(Wcomp), bcomp, padding=3)


def report(name, y):
    err = (y - truth).abs()
    p, pt = torch.softmax(y, 1), torch.softmax(truth, 1)
    flips = (y.argmax(1) != truth.argmax(1)).double().mean().item()
    print(f"{name:10s} logits: max |err| {err.max():.3e}  rms {err.pow(2).mean().sqrt():.3e}   per-sample softmax max |err| "
          f"{(p - pt).abs().max():.3e}   per-sample argmax flips {flips:.2e}")


print(f"Basic {W}x{H}, T={T}; logits rms {truth.pow(2).mean().sqrt():.3f}")
report("two-step", two_step)
report("composed", composed)
