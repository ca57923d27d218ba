"""TEST INFRASTRUCTURE -- seeded stereo scenes for Frame::ComputeStereoMatches whose every decision is known exactly.

Level 0 of the pyramid is the input image inside its reflected border, so an 11 x 11 window there is whatever the scene writes.
A key is matched against a patch of the right image copied from the left with an integer disparity (SAD 0 at the true shift,
thousands at every other shift of the random texture), plus `+k` at one non-centre pixel of the right window (best SAD exactly
k).  On a flat patch the SAD profile is built from single-pixel bumps instead: the profile is then a few multiples of k, with
the parabola's delta exactly 0 or 1/2 and first-minimum ties where wanted.  Key coordinates are chosen in float so that every
gate (row band, disparity window, window edges, disparity) sits exactly on its boundary or one ulp beside it, and descriptors
carry planted Hamming distances.  Every constructed left key names the stage (orb_oracle.STAGES) where its search must end;
tests/test_oracle_stereo.py holds the oracle to those stages."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle import orb_oracle as O
from sivo_b200.orb import KP_DTYPE as KP
ROWS, COLS = 240, 480
f32 = np.float32


@dataclass
class Scene:
    name: str
    left: np.ndarray
    right: np.ndarray
    kl: np.ndarray
    dl: np.ndarray
    kr: np.ndarray
    dr: np.ndarray
    mb: float
    mbf: float
    nlevels: int = 8
    scale_factor: float = 1.2
    want: dict = field(default_factory=dict)  # left key index -> the stage its search ends in

    def tables(self):
        return O.Tables(O.ExtractorParams(500, self.scale_factor, self.nlevels))

    def pyramids(self):
        t = self.tables()
        return O.compute_pyramid(self.left, t), O.compute_pyramid(self.right, t)

    def oracle(self, trace=None):
        t = self.tables()
        pl, pr = self.pyramids()
        return O.compute_stereo_matches(self.kl, self.dl, self.kr, self.dr, pl, pr, t.scale, t.inv_scale, self.mb, self.mbf,
                                        trace)


def ulp_up(v):
    return f32(np.nextafter(f32(v), f32(np.inf)))


def ulp_down(v):
    return f32(np.nextafter(f32(v), f32(-np.inf)))


class Builder:
    def __init__(self, name, seed, mb=1.0, mbf=40.0, nlevels=8, scale_factor=1.2, texture=True):
        self.name, self.mb, self.mbf = name, mb, mbf
        self.nlevels, self.scale_factor = nlevels, scale_factor
        self.rng = np.random.default_rng(seed)
        self.left = (self.rng.integers(40, 216, (ROWS, COLS)) if texture else np.full((ROWS, COLS), 128)).astype(np.uint8)
        self.right = self.left.copy()
        self.t = O.Tables(O.ExtractorParams(500, scale_factor, nlevels))
        self.kl, self.dl, self.kr, self.dr, self.want = [], [], [], [], {}
        self.slots = [(c, v) for v in range(12, ROWS - 11, 14) for c in range(60, COLS - 20, 70)]

    # ---- keys and descriptors
    def desc(self):
        return self.rng.integers(0, 256, 32).astype(np.uint8)

    def flip(self, d, nbits):
        bits = np.unpackbits(d)
        bits[self.rng.choice(256, nbits, replace=False)] ^= 1
        return np.packbits(bits)

    def left_key(self, x, y, octave, d, want=None):
        self.kl.append((f32(x), f32(y), octave))
        self.dl.append(d)
        if want is not None:
            self.want[len(self.kl) - 1] = want
        return len(self.kl) - 1

    def right_key(self, x, y, octave, d):
        self.kr.append((f32(x), f32(y), octave))
        self.dr.append(d)
        return len(self.kr) - 1

    def filler_right(self, n):
        """n right keys that are nobody's candidate (row band 0..4, far right, random descriptors): index padding."""
        for _ in range(n):
            self.right_key(COLS - 1, 2, 0, self.desc())

    def slot(self):
        return self.slots.pop(0)

    # ---- images
    def copy_patch(self, c, v, d):
        """Right rows v +- 5, columns c - d - 10 .. c - d + 10 = the left's columns c - 10 .. c + 10: the window at left column c
        has SAD 0 at right column c - d."""
        self.right[v - 5:v + 6, c - d - 10:c - d + 11] = self.left[v - 5:v + 6, c - 10:c + 11]

    def flat_patch(self, c, v, d, right_bumps, left_bumps=((1, 0, 30),)):
        """Flat left window at column c and flat right slide around column m = c - d, plus bumps (dy, dx, k) relative to the
        centres: every SAD is a sum of bump heights."""
        m = c - d
        self.left[v - 5:v + 6, c - 5:c + 6] = 128
        self.right[v - 5:v + 6, m - 10:m + 11] = 128
        for dy, dx, k in left_bumps:
            self.left[v + dy, c + dx] = 128 + k
        for dy, dx, k in right_bumps:
            self.right[v + dy, m + dx] = 128 + k

    def bump(self, c, v, d, k, dy=2, dx=-3):
        self.right[v + dy, c - d + dx] = np.uint8(int(self.right[v + dy, c - d + dx]) + k)

    # ---- the standard key: a left key at (x, v) with its right partner binc pixels left of the true match c - d
    def pair(self, x, v, d, binc=0, hd=10, octave=0, r_octave=None, r_y=None, want=None, r_x=None):
        dl = self.desc()
        il = self.left_key(x, v, octave, dl, want)
        rx = f32(round(float(x)) - d - binc) if r_x is None else r_x
        self.right_key(rx, v if r_y is None else r_y, octave if r_octave is None else r_octave, self.flip(dl, hd))
        return il

    def textured(self, d=8, k=20, binc=0, want="matched", **kw):
        c, v = self.slot()
        self.copy_patch(c, v, d)
        self.bump(c, v, d, k)
        return self.pair(c, v, d, binc=binc, want=want, **kw)

    def level_x(self, target, octave):
        """A float x with round(x * inv_scale[octave]) == target (the level-image column of a key at that octave)."""
        x = f32(f32(target) * self.t.scale[octave])
        for _ in range(64):
            r = O.round_half_away(f32(x * self.t.inv_scale[octave]))
            if r == target:
                return x
            x = ulp_down(x) if r > target else ulp_up(x)
        raise AssertionError("no float maps to that level column")

    def build(self):
        kl = np.zeros(len(self.kl), KP)
        for i, (x, y, o) in enumerate(self.kl):
            kl[i]["x"], kl[i]["y"], kl[i]["octave"] = x, y, o
            kl[i]["size"], kl[i]["response"] = 31, 1
        kr = np.zeros(len(self.kr), KP)
        for i, (x, y, o) in enumerate(self.kr):
            kr[i]["x"], kr[i]["y"], kr[i]["octave"] = x, y, o
            kr[i]["size"], kr[i]["response"] = 31, 1
        dl = np.array(self.dl, np.uint8).reshape(-1, 32)
        dr = np.array(self.dr, np.uint8).reshape(-1, 32)
        return Scene(self.name, self.left, self.right, kl, dl, kr, dr, self.mb, self.mbf, self.nlevels, self.scale_factor,
                     dict(self.want))


# ------------------------------------------------------------------------------------------------------- the scenes
def hamming_scene(seed=0):
    """Planted distances 74 / 75, exact ties across lanes and the 32-stride loop, the octave gate at the end octaves, the row
    band's floor / ceil on an integer and one ulp beside it, uR at both ends of the disparity window and one ulp outside,
    uL = -0.0 and maxU < 0."""
    b = Builder("hamming", seed)
    b.textured(hd=74)
    b.textured(hd=75, want="hamming")
    # ties: the right keys at i, i + 1 and i + 32 have the same distance; only the lowest index sits on the true match
    for lanes in ((0, 1), (0, 32), (0, 1, 32)):
        c, v = b.slot()
        b.copy_patch(c, v, 8)
        b.bump(c, v, 8, 20)
        dl = b.desc()
        b.left_key(c, v, 0, dl, "matched")
        b.filler_right((-len(b.kr)) % 32)
        base = len(b.kr)
        planted = b.flip(dl, 20)
        for j in range(max(lanes) + 1):
            if j in lanes:
                b.right_key(c - 8 if j == 0 else c - 8 - 5, v, 0, planted)  # the others leave binc = +5: refused
            else:
                b.right_key(COLS - 1, 2, 0, b.desc())
        assert b.kr[base][0] == c - 8
    # the same tie with the true match at the HIGHER index: the lowest index wins and its binc = +5 is refused
    c, v = b.slot()
    b.copy_patch(c, v, 8)
    dl = b.desc()
    b.left_key(c, v, 0, dl, "binc_edge")
    planted = b.flip(dl, 20)
    b.right_key(c - 8 - 5, v, 0, planted)
    b.filler_right(31)
    b.right_key(c - 8, v, 0, planted)
    # octave gate at octave 0: right octave 1 accepted, 2 refused
    for ro, want in ((1, None), (2, "hamming")):
        c, v = b.slot()
        b.copy_patch(c, v, 8)
        il = b.pair(c, v, 8, octave=0, r_octave=ro, want=want)
        if want is None:
            b.want[il] = "matched"  # the partner's octave only opens the gate; the SAD is at the left key's octave
    # octave gate at the last octave (level 7 is 134 x 67): right octaves 6 accepted, 5 refused
    top = b.nlevels - 1
    for j, (ro, want) in enumerate(((top - 1, "any"), (top - 2, "hamming"))):
        x, y = b.level_x(60 + 30 * j, top), b.level_x(20 + 12 * j, top)
        dl = b.desc()
        il = b.left_key(x, y, top, dl, None if want == "any" else want)
        b.right_key(ulp_down(x), y, ro, b.flip(dl, 5))
        if want == "any":
            b.want[il] = "past_hamming"
    # row band at octave 0 (band = 2): floor(R.y - 2) and ceil(R.y + 2) against the left row v
    for r_y, inside in ((lambda v: f32(v + 2), True), (lambda v: ulp_down(v + 3), True), (lambda v: f32(v + 3), False),
                        (lambda v: f32(v - 2), True), (lambda v: ulp_up(v - 3), True), (lambda v: f32(v - 3), False),
                        (lambda v: f32(v - 2.5), True)):
        c, v = b.slot()
        b.copy_patch(c, v, 8)
        b.bump(c, v, 8, 20)
        b.pair(c, v, 8, r_y=r_y(v), want="matched" if inside else "no_match")
    # the disparity window [uL - maxD, uL] (maxD = 40): uR on both ends and one ulp outside
    for d, nudge, want in ((0, None, "matched"), (0, ulp_up, "no_match"), (40, None, "disparity"), (40, ulp_down, "no_match")):
        c, v = b.slot()
        b.flat_patch(c, v, d, ((1, 0, 30), (-2, 4, 3)))
        rx = f32(c - d) if nudge is None else nudge(f32(c - d))
        b.pair(c, v, d, r_x=rx, want=want)
    # uL = -0.0 (maxU = -0.0 >= 0 holds: the right key at -0.0 is found, its slide leaves the image) and maxU < 0
    dl = b.desc()
    b.left_key(f32(-0.0), 100, 0, dl, "slide")
    b.left_key(ulp_down(0.0), 100, 0, dl, "no_candidate")
    b.right_key(f32(-0.0), 100, 0, dl)
    for _ in range(6):
        b.textured(k=25)
    return b.build()


def sad_scene(seed=1):
    """binc = +-4 accepted and +-5 refused, first-minimum ties, d3 == d2 (delta = 1/2 exactly), a flat window (binc = -5),
    the reference's endu test at su_r0 + 11 = cols - 1 and cols."""
    b = Builder("sad", seed)
    for binc, want in ((4, "matched"), (-4, "matched"), (5, "binc_edge"), (-5, "binc_edge")):
        b.textured(binc=binc, want=want)
    c, v = b.slot()
    b.flat_patch(c, v, 8, ((1, 0, 30), (1, 1, 30)))  # SAD k at shifts 0 and +1: delta = 1/2
    b.pair(c, v, 8, want="matched")
    c, v = b.slot()
    b.flat_patch(c, v, 8, ((1, 0, 30), (1, 3, 30)))  # SAD k at shifts 0 and +3: the first wins
    b.pair(c, v, 8, want="matched")
    c, v = b.slot()
    b.flat_patch(c, v, 8, ((1, 0, 30), (1, -3, 30)))  # SAD k at shifts -3 and 0: the first (-3) wins
    b.pair(c, v, 8, want="matched")
    c, v = b.slot()
    b.flat_patch(c, v, 8, (), ())  # every SAD 0: binc = -5
    b.pair(c, v, 8, want="binc_edge")
    # endu = su_r0 + 11 against cols at octave 0: su_r0 = cols - 12 passes, cols - 11 does not
    for r, (su_r0, want) in enumerate(((COLS - 12, "past_slide"), (COLS - 11, "slide_ref"))):
        dl = b.desc()
        b.left_key(COLS - 6, 40 + 30 * r, 0, dl, want)
        b.right_key(su_r0, 40 + 30 * r, 0, b.flip(dl, 3))
    for _ in range(8):
        b.textured(k=20)
    return b.build()


def window_scene(octave, seed=2):
    """Windows one pixel inside and outside every edge of the level image at `octave`: the right slide's first column
    (su_r0 = 10 / 9), the left window's last column (su_l = w - 6 / w - 5), its first and last rows (sv_l = 5 / 4, h - 6 /
    h - 5)."""
    b = Builder(f"window{octave}", seed + octave)
    w, h = O.level_sizes(COLS, ROWS, b.t)[octave]
    cases = [  # (su_l, sv_l, su_r0, stage)
        (14, h // 2, 10, "past_slide"), (14, h // 2, 9, "slide"),
        (w - 6, h // 2 - 8, w - 14, "past_slide"), (w - 5, h // 2 - 8, w - 14, "left_window"),
        (w // 2, 5, w // 2 - 3, "past_slide"), (w // 2 + 20, 4, w // 2 + 17, "slide"),
        (w // 2 - 20, h - 6, w // 2 - 23, "past_slide"), (w // 2 + 40, h - 5, w // 2 + 37, "slide"),
    ]
    if octave == 0:
        cases.append((14, h // 2 + 20, 0, "slide"))   # iniu = 0 passes the reference's test
        cases.append((14, h // 2 + 30, -1, "slide_ref"))
    for j, (su_l, sv_l, su_r0, want) in enumerate(cases):
        x, y, rx = b.level_x(su_l, octave), b.level_x(sv_l, octave), b.level_x(su_r0, octave)
        if octave == 0:
            x, y, rx = f32(su_l), f32(sv_l), f32(su_r0)
        dl = b.desc()
        b.left_key(x, y, octave, dl, want)
        b.right_key(rx, y, octave, b.flip(dl, 3 + j))
    return b.build()


def disparity_scene(seed=3):
    """maxD = 40 (mbf 40, mb 1): disparity exactly 0 (clamped to 0.01), -ulp refused, maxD - ulp accepted, maxD refused.  The
    flat patches make delta 0, so best_u = su_r0 + binc is an integer and the disparity uL - best_u is exact."""
    b = Builder("disparity", seed)
    b.slots = [sl for sl in b.slots if sl[0] != 60]
    rows = iter(range(12, ROWS - 11, 14))
    for d, x_of, want in ((0, lambda c: f32(c), "matched"), (0, lambda c: ulp_down(c), "disparity"),
                          (40, lambda c: f32(c - 40) + ulp_down(40), "matched"), (40, lambda c: f32(c), "disparity")):
        c, v = 55, next(rows)
        b.flat_patch(c, v, d, ((1, 0, 30), (-2, 4, 3)))
        il = b.pair(x_of(c), v, d, want=want, r_x=f32(c - d - 0.25) if d == 0 else f32(c - d + 0.25))
        assert round(float(b.kl[il][0])) == c
    for _ in range(6):
        b.textured(k=30)
    return b.build()


def small_maxd_scene(seed=4):
    """maxD = 0.5 px (mbf 0.5, mb 1): disparities 0, 0.25, 0.49 accepted and 0.5 refused; -0.25 refused."""
    b = Builder("small_maxd", seed, mbf=0.5)
    for off, want in ((0.0, "matched"), (0.25, "matched"), (0.49, "matched"), (-0.25, "disparity")):
        c, v = b.slot()
        b.flat_patch(c, v, 0, ((1, 0, 30), (-2, 4, 3)))
        b.pair(f32(c + off), v, 0, want=want, r_x=f32(f32(c + off) - f32(0.05)))
    c, v = b.slot()
    b.flat_patch(c, v, 0, ((1, 0, 30), (1, -1, 30)))  # delta = -1/2 at shift -1: best_u = c - 1.5, disparity 0.5 refused
    b.pair(f32(c), v, 0, want="disparity", r_x=f32(c - 0.05))
    return b.build()


def wide_maxd_scene(seed=5):
    """maxD = 1000 px, wider than the image: every right key in the band is a candidate."""
    b = Builder("wide_maxd", seed, mbf=1000.0)
    for j in range(30):
        b.textured(d=int(b.rng.integers(0, 30)), k=int(b.rng.integers(1, 40)), want=None)
    return b.build()


def median_scene(sads, seed=6, name="median"):
    """One textured key per entry of `sads` with best SAD exactly that value (0: no bump): the median cut on known values."""
    b = Builder(name, seed)
    cut = O.median_cut(np.array(sads))
    for k, c_ in zip(sads, cut):
        b.textured(k=k, want="cut" if c_ else "matched")
    return b.build()


def rule_scene(seed=7):
    """The rule: NaN and +-inf in x and y of left and right keys, |x| >= 2^31, rows -1, -0.5, 0, rows - 1 and rows."""
    b = Builder("rule", seed)
    b.slots = [sl for sl in b.slots if sl[0] != 60]
    nan, inf = f32(np.nan), f32(np.inf)
    for x, y in ((nan, 100), (100, nan), (inf, 100), (-inf, 100), (100, inf), (100, -inf), (nan, nan)):
        b.left_key(x, y, 0, b.desc(), "nonfinite")
    for y in (-1.0, f32(ROWS)):
        b.left_key(100, y, 0, b.desc(), "no_row")
    # rows -0.5 and 0 (row 0), rows - 1: a right partner at the same row; the windows leave the image
    for y in (-0.5, 0.0, f32(ROWS - 1)):
        dl = b.desc()
        b.left_key(200, y, 0, dl, "slide")
        b.right_key(195, y, 0, b.flip(dl, 4))
    # |x| >= 2^31 on both sides: matched in the Hamming stage, the windows are far outside
    for x in (f32(2.0 ** 31), f32(3e9), f32(-2.0 ** 31)):
        dl = b.desc()
        b.left_key(x, 120, 0, dl, "slide_ref" if x > 0 else "no_candidate")
        b.right_key(x, 120, 0, b.flip(dl, 4))
    # right keys with non-finite coordinates are no candidate, although their descriptors equal the left key's (a NaN y would
    # give the row band [0, 0] after a conversion to int)
    for (rx, ry), (lx, ly) in zip(((nan, 60), (50, nan), (inf, 74), (-inf, 88), (60, inf), (60, -inf)),
                                  ((60, 60), (60, 0), (60, 74), (60, 88), (70, 102), (70, 116))):
        dl = b.desc()
        b.left_key(lx, ly, 0, dl, "no_match")
        b.right_key(rx, ry, 0, dl)
    for _ in range(8):
        b.textured(k=15)
    return b.build()


def constructed_scenes():
    return [hamming_scene(), sad_scene(), window_scene(0), window_scene(3), window_scene(7), disparity_scene(), small_maxd_scene(),
            wide_maxd_scene(), rule_scene(),
            median_scene([5, 5, 10, 10, 10, 10, 20, 21], name="median_th21"),
            median_scene([0, 0, 0, 0, 0], name="median0"),
            median_scene([7], name="median_m1"), median_scene([7, 3], name="median_m2"), median_scene([9, 1, 30], name="median_m3"),
            median_scene([12, 12, 12, 12], name="median_equal")]


def fuzz_scene(seed, extra=None):
    """A seeded random scene: a texture whose right image is the left shifted by a per-band disparity, keys at every octave
    (on matches, near the level borders and outside the domain), descriptors with planted near-duplicates, random mb / mbf.
    `extra` = (kl, dl, kr, dr) of extractor keys to mix in, placed first."""
    rng = np.random.default_rng(1000 + seed)
    nlevels = int(rng.choice([4, 8]))
    sf = float(rng.choice([1.2, 1.5])) if nlevels == 4 else 1.2
    mb = float(rng.uniform(0.3, 1.5))
    mbf = float(mb * rng.uniform(5, 90))
    b = Builder(f"fuzz{seed}", seed + 5000, mb=mb, mbf=mbf, nlevels=nlevels, scale_factor=sf)
    band_h = int(rng.integers(8, 40))
    for y0 in range(0, ROWS, band_h):
        d = int(rng.integers(0, 40))
        b.right[y0:y0 + band_h, :COLS - d] = b.left[y0:y0 + band_h, d:]
    b.right = np.clip(b.right.astype(np.int64) + rng.integers(-3, 4, b.right.shape), 0, 255).astype(np.uint8)
    n = int(rng.integers(20, 120))
    for _ in range(n):
        o = int(rng.integers(0, nlevels))
        s = float(b.t.scale[o])
        kind = rng.random()
        if kind < 0.7:
            x, y = rng.uniform(0, COLS), rng.uniform(0, ROWS)
        elif kind < 0.9:  # near the level borders
            x = float(rng.choice([rng.uniform(-2, 16 * s), rng.uniform(COLS - 16 * s, COLS + 2)]))
            y = float(rng.choice([rng.uniform(-2, 16 * s), rng.uniform(ROWS - 16 * s, ROWS + 2)]))
        else:  # outside the domain
            x = float(rng.choice([np.nan, np.inf, -1e10, 3e9, rng.uniform(-50, 0)]))
            y = float(rng.choice([np.nan, -np.inf, ROWS, -1.0, rng.uniform(0, ROWS)]))
        dl = b.desc()
        b.left_key(x, y, o, dl)
        for _ in range(int(rng.integers(0, 4))):
            ro = int(np.clip(o + rng.integers(-2, 3), 0, nlevels - 1))
            rx = f32(x - rng.uniform(-2, mbf / mb + 2)) if np.isfinite(x) else f32(rng.uniform(0, COLS))
            ry = f32(y + rng.uniform(-3, 3) * s) if np.isfinite(y) else f32(rng.uniform(0, ROWS))
            b.right_key(rx, ry, ro, b.flip(dl, int(rng.choice([0, 10, 40, 74, 75, 99, 100, 120]))))
    sc = b.build()
    if extra is not None:
        ekl, edl, ekr, edr = extra
        sc.kl = np.concatenate([np.asarray(ekl, KP), sc.kl])
        sc.dl = np.concatenate([edl, sc.dl])
        sc.kr = np.concatenate([np.asarray(ekr, KP), sc.kr])
        sc.dr = np.concatenate([edr, sc.dr])
    return sc
