"""CPU: the variance oracle (oracle/variance_oracle.py) against a literal restatement of BayesianSegNet::computeVariance
(bayesian_segnet.cpp:205-260), its two documented rules (invalid classes give 0, float64 sample order), and the latency-mode
moments that add over sample ranges."""
import numpy as np
import pytest

from oracle.segnet_oracle import softmax_channels
from oracle.variance_oracle import mc_variance, mc_variance_from_moments, mc_variance_moments


def _prob(T, C, H, W, seed):
    import torch
    rng = np.random.default_rng(seed)
    logits = (rng.standard_normal((T, C, H, W)) * 2.5).astype(np.float32)
    return softmax_channels(torch.from_numpy(logits)).numpy()


def _literal(prob, classes):
    """bayesian_segnet.cpp:221-256 loop for loop: for every class i and pixel (j, k) whose detected class is i, the mean of the
    T-vector, then the sum of pow(x - avg, 2) in sample order, divided by size - 1.  Pixels of no class stay 0 (rule 1)."""
    T, C, H, W = prob.shape
    out = np.zeros((H, W))
    for i in range(C):
        for j in range(H):
            for k in range(W):
                if i == int(classes[j, k]):
                    vec = [float(prob[t, i, j, k]) for t in range(T)]
                    s = 0.0
                    for x in vec:
                        s += x
                    avg = s / T
                    acc = 0.0
                    for x in vec:
                        acc += (x - avg) * (x - avg)  # std::pow(d, 2): GCC folds it into d * d (libm pow is not always)
                    out[j, k] = acc / (T - 1)
    return out


@pytest.mark.parametrize("T", [2, 3, 12])
def test_mc_variance_equals_the_literal_loop(T):
    C, H, W = 15, 6, 9
    prob = _prob(T, C, H, W, seed=T)
    rng = np.random.default_rng(100 + T)
    classes = rng.integers(0, C, (H, W)).astype(np.uint8)
    classes[0, 0], classes[2, 3] = 255, C  # invalid classes: 0
    got = mc_variance(prob, classes)
    assert np.array_equal(got, _literal(prob, classes))
    assert got[0, 0] == 0.0 and got[2, 3] == 0.0
    assert (got[classes < C] > 0).all()


def test_invalid_classes_give_zero():
    prob = _prob(4, 15, 3, 5, seed=7)
    for bad in (15, 16, 200, 255):
        assert not mc_variance(prob, np.full((3, 5), bad, np.uint8)).any()


def test_identical_samples_give_zero_variance():
    one = _prob(1, 15, 4, 6, seed=3)
    prob = np.repeat(one, 6, axis=0)
    classes = np.random.default_rng(0).integers(0, 15, (4, 6)).astype(np.uint8)
    assert mc_variance(prob, classes).max() < 1e-30


def test_moments_over_sample_ranges_add_up_to_the_two_pass_variance():
    T, C, H, W = 12, 15, 8, 10
    prob = _prob(T, C, H, W, seed=11)
    classes = np.random.default_rng(5).integers(0, C + 3, (H, W)).astype(np.uint8)
    classes[1, 1] = 255
    want = mc_variance(prob, classes)
    for cuts in ([0, 12], [0, 6, 12], [0, 1, 5, 12], [0, 3, 4, 9, 11, 12], list(range(13))):
        total = sum(mc_variance_moments(prob[a:b], classes) for a, b in zip(cuts[:-1], cuts[1:]))
        got = mc_variance_from_moments(total, T)
        assert np.abs(got - want).max() <= 1e-12, cuts
        assert got[1, 1] == 0.0 and (got >= 0).all()
