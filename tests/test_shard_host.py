"""Latency mode without a GPU: the sample split, the shard's dropout rows, the oracle's forward pass restricted to one
shard's samples and the sum-then-finalise reduction (SURVEY 8e, DESIGN §6)."""
from unittest import mock

import numpy as np
import pytest

from oracle import philox, segnet_oracle as S
from sivo_b200 import sample_ranges


@pytest.mark.parametrize("T", [1, 2, 3, 6, 7, 12])
def test_sample_ranges_cover_the_frame_contiguously_with_balanced_sizes(T):
    for G in range(1, T + 1):
        r = sample_ranges(T, G)
        assert len(r) == G
        assert r[0][0] == 0 and sum(n for _, n in r) == T
        for (b0, n0), (b1, _) in zip(r, r[1:]):
            assert b1 == b0 + n0  # contiguous, in order
        sizes = [n for _, n in r]
        assert min(sizes) >= 1 and max(sizes) - min(sizes) <= 1
        assert sizes == sorted(sizes, reverse=True)  # larger blocks first


def test_sample_ranges_example_and_errors():
    assert sample_ranges(6, 4) == [(0, 2), (2, 2), (4, 1), (5, 1)]
    assert sample_ranges(6, 2) == [(0, 3), (3, 3)]
    assert sample_ranges(6, 1) == [(0, 6)]
    with pytest.raises(ValueError):
        sample_ranges(6, 7)
    with pytest.raises(ValueError):
        sample_ranges(6, 0)


def keep_rows(seed, frame, layer, count, C, H, W, n0):
    """The keep-bit rule of oracle/philox.py (DESIGN §5) for MC samples n0 .. n0 + count - 1: the masks a shard that owns
    those samples draws (its local sample n is global sample n0 + n)."""
    pix = np.arange(H * W, dtype=np.uint32)[None, :, None]
    n = np.arange(n0, n0 + count, dtype=np.uint32)[:, None, None]
    ngroups = (C + 127) // 128
    g = np.arange(ngroups, dtype=np.uint32)[None, None, :]
    words = philox.philox4x32_10(pix, n | np.uint32(layer << 16) | (g << np.uint32(24)), np.uint32(frame & 0xFFFFFFFF),
                                 np.uint32((frame >> 32) & 0xFFFFFFFF), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    bits = (np.stack(words, axis=-1)[..., None] >> np.arange(32, dtype=np.uint32)) & np.uint32(1)
    bits = bits.reshape(count, H * W, ngroups * 128)[:, :, :C]
    return bits.astype(bool).transpose(0, 2, 1).reshape(count, C, H, W)


def forward_shard(net, w, img, samples, **kw):
    """The oracle's forward pass over one shard's samples only: batch `count`, each sample with the masks of its global index."""
    b, n = samples
    rows = lambda seed, frame, layer, T, C, H, W: keep_rows(seed, frame, layer, T, C, H, W, b)
    with mock.patch.object(S, "dropout_keep", rows):
        return S.forward(net, w, img, T=n, **kw)


@pytest.mark.parametrize("b,count", [(0, 6), (0, 3), (3, 3), (2, 2), (5, 1)])
def test_dropout_keep_rows_of_a_shard_equal_the_full_mask(b, count):
    full = philox.dropout_keep(1234, 77, 2, 6, 200, 5, 7)
    assert np.array_equal(keep_rows(1234, 77, 2, 6, 200, 5, 7, 0), full)  # the restated rule is the oracle's
    part = keep_rows(1234, 77, 2, count, 200, 5, 7, b)
    assert part.shape == (count, 200, 5, 7)
    assert np.array_equal(part, full[b:b + count])


@pytest.fixture(scope="module")
def small_basic(model_dir):
    from conftest import make_model
    net, w, _, _ = make_model(model_dir, "basic", T=6, H=32, W=64, width=8)
    rng = np.random.default_rng(11)
    img = rng.integers(0, 256, size=(32, 64, 3), dtype=np.uint8)
    full = S.forward(net, w, img, seed=1234, frame=4, T=6)
    return net, w, img, full


@pytest.mark.parametrize("ranges", [[(0, 3), (3, 3)], [(0, 2), (2, 2), (4, 1), (5, 1)], [(n, 1) for n in range(6)]])
def test_oracle_shards_concatenate_to_the_full_prob(small_basic, ranges):
    net, w, img, full = small_basic
    parts = [forward_shard(net, w, img, r, seed=1234, frame=4) for r in ranges]
    for (b, n), p in zip(ranges, parts):
        assert p.shape == (n,) + full.shape[1:]
    # CPU convolutions may order their sums differently for a different batch size: equal to ~1 float ulp
    assert np.abs(np.concatenate(parts) - full).max() < 1e-6
    assert not np.array_equal(parts[0][0], parts[-1][-1])  # the shards really draw different samples


def _finalize(sum_total, T):
    """The finalise step in float64: mean = sum * (1/T), first-max argmax, max, -sum p log2 p with 0 log 0 := 0."""
    mean = sum_total * (1.0 / T)
    classes = np.argmax(mean, axis=0).astype(np.uint8)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.where(mean == 0.0, 0.0, -mean * np.log2(mean))
    return classes, mean.max(axis=0), e.sum(axis=0)


def test_shard_sums_added_and_finalised_equal_mc_reduce(small_basic):
    net, w, img, full = small_basic
    rc, rf, re = S.mc_reduce(full)
    sums = [full[b:b + n].astype(np.float64).sum(axis=0) for b, n in sample_ranges(6, 4)]  # per shard, in sample order
    total = sums[0]
    for s in sums[1:]:
        total = total + s  # the cross-rank reduction
    cls, conf, ent = _finalize(total, 6)
    assert np.array_equal(cls, rc)
    assert np.abs(conf - rf).max() <= 1e-12
    assert np.abs(ent - re).max() <= 1e-12
