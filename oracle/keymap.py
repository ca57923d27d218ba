"""The semantic-key map the Frame-tail device calls read, embedded as their tests pass it.

Every device call reads semantic key j as extractor record keep_idx[j], for j < min(*n_keep, capacity); an entry below 0 or at
or above the capacity means "no key".  keymap() places n real keys in order on a permutation of the capacity's slots, with
rejected entries (and, on request, duplicates of earlier keys' slots) between them.  numpy only: the CPU tests use it."""
from dataclasses import dataclass

import numpy as np

SLACK = 64  # entries and rows past every bound, which a bound one too wide would read


def rejected_values(cap):
    """The rejected entries, in the order keymap cycles through them."""
    return (-1, -7, -2 ** 31, cap, cap + 3, cap + 5, cap + 7, 2 ** 31 - 1)


@dataclass
class KeyMap:
    keep: np.ndarray   # int32, max(n_keep, cap) + SLACK entries; those past n_keep are valid slots
    n_keep: int
    src: np.ndarray    # int64 per entry below n_keep: the real key it reads, -1 for a rejected entry
    slots: np.ndarray  # the slot of each real key
    dup: np.ndarray    # bool per entry below n_keep: a second entry on an earlier key's slot

    @property
    def real(self):
        """The entry of each real key."""
        return np.flatnonzero((self.src >= 0) & ~self.dup)


def keymap(n, cap, rng, forced=(), duplicates=False, junk=True) -> KeyMap:
    """n real keys on a permutation of cap slots.  Unless junk is False, min(cap - n, max(16, (cap - n) // 8)) entries go between
    them: the entries at the `forced` positions below n_keep (a negative one counts from n_keep) are rejected, the others sit at
    random positions.  Rejected entries cycle through rejected_values(cap); with `duplicates`, every fourth unforced one
    instead re-reads an earlier key's slot."""
    assert 0 <= n <= cap
    n_junk = min(cap - n, max(16, (cap - n) // 8)) if junk else 0
    n_keep = n + n_junk
    is_junk = np.zeros(n_keep, bool)
    pinned = np.zeros(n_keep, bool)
    if n_junk:
        fixed = sorted({j + n_keep if j < 0 else j for j in forced} & set(range(n_keep)))[:n_junk]
        rest = rng.permutation(np.setdiff1d(np.arange(n_keep), fixed))[:n_junk - len(fixed)]
        is_junk[fixed] = pinned[fixed] = True
        is_junk[rest] = True
    perm = rng.permutation(cap)
    keep = np.empty(max(n_keep, cap) + SLACK, np.int32)
    keep[n_keep:] = perm[rng.integers(0, cap, len(keep) - n_keep)]
    src = np.full(n_keep, -1, np.int64)
    dup = np.zeros(n_keep, bool)
    values = rejected_values(cap)
    c = r = q = 0  # real keys, unpinned junk entries and rejected entries so far
    for j in range(n_keep):
        if not is_junk[j]:
            keep[j], src[j] = perm[c], c
            c += 1
            continue
        if not pinned[j]:
            r += 1
            if duplicates and r % 4 == 0 and c > 0:
                i = int(rng.integers(c))
                keep[j], src[j], dup[j] = perm[i], i, True
                continue
        keep[j] = values[q % len(values)]
        q += 1
    return KeyMap(keep, n_keep, src, perm[:n].copy(), dup)


def scatter(a, slots, cap, decoy):
    """The rows of a at their slots of a cap + SLACK array whose every other row is `decoy` (anything that broadcasts to it)."""
    a = np.asarray(a)
    out = np.zeros((cap + SLACK,) + a.shape[1:], a.dtype)
    out[...] = decoy
    out[slots] = a
    return out
