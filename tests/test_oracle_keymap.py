"""CPU: the semantic-key map of the Frame-tail device tests (oracle/keymap.py)."""
import numpy as np
import pytest

from oracle.keymap import SLACK, keymap, rejected_values, scatter


@pytest.mark.parametrize("n,cap,forced,duplicates", [(0, 40, (), False), (100, 2096, (0, 31, 32), True), (600, 2096, (255, 256, 511, 512), False),
                                                     (2000, 2096, (0, 31, 32, -1), True), (30, 30, (0,), True)])
def test_the_map_agrees_with_itself(n, cap, forced, duplicates):
    km = keymap(n, cap, np.random.default_rng(n), forced=forced, duplicates=duplicates)
    keep, src, dup = km.keep, km.src, km.dup
    n_junk = min(cap - n, max(16, (cap - n) // 8))
    assert km.n_keep == n + n_junk and len(keep) == max(km.n_keep, cap) + SLACK and keep.dtype == np.int32
    assert len(src) == len(dup) == km.n_keep and len(km.slots) == n and len(set(km.slots.tolist())) == n
    head = keep[:km.n_keep]
    valid = (head >= 0) & (head < cap)
    assert np.array_equal(valid, src >= 0)
    assert np.array_equal(head[valid], km.slots[src[valid]])
    assert np.array_equal(src[km.real], np.arange(n)) and np.array_equal(head[km.real], km.slots)
    assert not dup[~valid].any() and dup.any() == (duplicates and n_junk >= 4 and n > 0)
    assert set(head[~valid].tolist()) <= set(rejected_values(cap))
    if n_junk >= 16:  # enough junk: every rejected value appears
        assert set(head[~valid].tolist()) == set(rejected_values(cap))
    for j in forced:
        if j < km.n_keep and n_junk:
            assert src[j] == -1 and head[j] in rejected_values(cap), j
    slack = keep[km.n_keep:]
    assert ((slack >= 0) & (slack < cap)).all()


def test_without_junk_the_map_is_a_permutation():
    km = keymap(500, 2096, np.random.default_rng(1), forced=(0, 1), junk=False)
    assert km.n_keep == 500 and (km.src == np.arange(500)).all() and not km.dup.any()
    assert np.array_equal(km.keep[:500], km.slots)


def test_the_same_seed_gives_the_same_map():
    a, b = (keymap(300, 2096, np.random.default_rng(9), forced=(0, 31), duplicates=True) for _ in range(2))
    for f in ("keep", "src", "slots", "dup"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert a.n_keep == b.n_keep


def test_scatter_places_rows_at_their_slots_over_decoys():
    km = keymap(5, 20, np.random.default_rng(2))
    a = np.arange(10, dtype=np.float32).reshape(5, 2)
    out = scatter(a, km.slots, 20, -3.0)
    assert out.shape == (20 + SLACK, 2) and np.array_equal(out[km.slots], a)
    rest = np.setdiff1d(np.arange(20 + SLACK), km.slots)
    assert (out[rest] == -3.0).all()
