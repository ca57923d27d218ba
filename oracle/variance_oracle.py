"""TEST INFRASTRUCTURE -- CPU oracle for `SIVO::BayesianSegNet::computeVariance` (src/bayesian_segnet/bayesian_segnet.cpp:205-260);
never imported by the product path.

For each pixel (row, col), with c = classes(row, col) and p_t = prob[t, c, row, col] cast to double:

    avg      = (sum_t p_t) / T
    variance = sum_t (p_t - avg)^2 / (T - 1)        (the SAMPLE variance, summed in double in sample order, :240-253)

The square is the rounded product d * d: GCC folds std::pow(d, 2) into it (a libm pow call can differ in the last bit).

Two rules the reference leaves open:
  1. a class >= C (e.g. VOID = 255) gives 0 -- the reference leaves that element of the matrix uninitialised;
  2. `prob` is whatever per-sample softmax the caller hands in: to compare with the device, the float32 softmax computed with the
     arithmetic of the reduction kernel the device runs (tests/test_gpu_variance.py), or the oracle's own forward() output.

Latency mode splits the samples over ranks: each shard reports the moments (sum p_t, sum p_t^2) of the given class, the moments
add over shards, and variance = max(0, (S2 - S1^2 / T) / (T - 1)).
"""
from __future__ import annotations

import numpy as np


def _class_probs(prob: np.ndarray, classes: np.ndarray):
    """prob [T, C, H, W], classes u8 [H, W] -> (p [T, H, W] float64 of each pixel's class (0 where invalid), valid [H, W])."""
    T, C, H, W = prob.shape
    cls = np.asarray(classes).astype(np.int64)
    assert cls.shape == (H, W)
    valid = cls < C
    idx = np.where(valid, cls, 0)
    p = np.take_along_axis(prob, np.broadcast_to(idx[None, None], (T, 1, H, W)), axis=1)[:, 0].astype(np.float64)
    return np.where(valid[None], p, 0.0), valid


def mc_variance(prob: np.ndarray, classes: np.ndarray) -> np.ndarray:
    """prob float32 [T, C, H, W], classes u8 [H, W] -> variance float64 [H, W] (two passes, sample order)."""
    T = prob.shape[0]
    if T < 2:
        raise ValueError("the sample variance needs T >= 2")
    p, valid = _class_probs(prob, classes)
    s = np.zeros(p.shape[1:], np.float64)
    for t in range(T):
        s = s + p[t]
    avg = s / T
    d2 = np.zeros_like(s)
    for t in range(T):
        d = p[t] - avg
        d2 = d2 + d * d
    return np.where(valid, d2 / (T - 1), 0.0)


def mc_variance_moments(prob: np.ndarray, classes: np.ndarray) -> np.ndarray:
    """One shard's moments: prob [n, C, H, W] of its samples -> float64 [H, W, 2] = (sum p_t, sum p_t^2); (0, 0) if invalid."""
    p, _ = _class_probs(prob, classes)
    s1 = np.zeros(p.shape[1:], np.float64)
    s2 = np.zeros_like(s1)
    for t in range(p.shape[0]):
        s1 = s1 + p[t]
        s2 = s2 + p[t] * p[t]
    return np.stack([s1, s2], axis=-1)


def mc_variance_from_moments(moments: np.ndarray, T: int) -> np.ndarray:
    """Moments summed over all T samples of the frame -> variance float64 [H, W]."""
    s1, s2 = moments[..., 0], moments[..., 1]
    return np.maximum(0.0, (s2 - s1 * s1 / T) / (T - 1))
