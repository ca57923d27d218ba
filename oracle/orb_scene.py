"""TEST INFRASTRUCTURE -- constructed input images for the ORB extractor's edge cases (tests/test_gpu_orb_edges.py against the
product, tests/test_oracle_orb.py against cv2); never imported by the product path.

Every image is built from a seed.  Each case names what it must reach, and the tests assert it from the oracle's own counts, so a
case cannot drift off the boundary it was built for:
  * density ladder: uniform noise blended into the KITTI crop at increasing strength, level 0 just below and just above the device
    quad tree's 8,192-candidate cap (kTreeKeyCap, orb.h), then pure noise, where levels 0-2 exceed it;
  * densest cell: the densest 3x3-NMS survivor lattice FAST admits, in the largest cell interior the grid makes (53 x 53);
  * min_th fallback: low-contrast dots (no corner at iniThFAST, many at minThFAST) next to high-contrast blocks;
  * saturation: binary 0 / 255 noise (8-bit responses tie heavily) and a one-pixel checkerboard (no level-0 corner at all);
  * geometry: the uncropped fixture, the smallest 8-level image, a level narrower than one cell, a portrait image, a wide strip with
    more than 16 initial quad-tree nodes, and the 4,058 / 4,059-px widths of the 12-bit coordinate packing.
"""
from __future__ import annotations

import numpy as np

from oracle import orb_oracle as O

H, W = 352, 1024  # the KITTI crop the extractor runs on in the Frame tail

TREE_KEY_CAP = 8192   # kTreeKeyCap: FAST candidates of one level the device quad tree holds
CELL_CAP = 1024       # kCellCap: per-cell candidate slots
MAX_PACKED_WIDTH = 4058  # level 0 + the 2 x 19-px border must fit 12 bits (4096)

# blend strengths of the density ladder, chosen with the oracle: level 0 of the KITTI crop lands just below / just above the cap
LADDER = {"below": 0.137, "above": 0.138, "full": 1.0}


def noise(rows: int, cols: int, seed: int) -> np.ndarray:
    return np.random.default_rng(seed).integers(0, 256, size=(rows, cols), dtype=np.uint8)


def blend(base: np.ndarray, strength: float, seed: int) -> np.ndarray:
    """(1 - strength) * base + strength * uniform noise, rounded."""
    n = noise(*base.shape, seed).astype(np.float64)
    return np.rint((1.0 - strength) * base.astype(np.float64) + strength * n).astype(np.uint8)


def densest_cell() -> np.ndarray:
    """A 91 x 91 image: at one pyramid level its FAST region is 59 px wide and high, so the grid is one cell whose interior is
    53 x 53 (cell interiors are at most 53 px on a side when the grid has one column, 45 with two, less with more).  The cell holds
    the densest lattice the strict 3x3 NMS allows, a survivor at every other pixel of every other row, 27 x 27 = 729:
    background 128, survivors 255 on even lattice rows and 0 on odd ones.  A survivor's ring (radius 3) meets the lattice only at
    its four (+-2, +-2) diagonal neighbours, which are of the opposite kind, so all 16 ring pixels are darker (or all brighter)
    than it: a corner of response 126 (127).  No background pixel has a 9-arc of one sign, so every survivor beats its 8
    neighbours.  Extract it with one pyramid level."""
    img = np.full((91, 91), 128, np.uint8)
    for i, y in enumerate(range(19, 72, 2)):
        img[y, 19:72:2] = 255 if i % 2 == 0 else 0
    return img


def low_contrast(seed: int) -> np.ndarray:
    """128 with isolated dots of +-12 on 2 % of the pixels: a dot is a corner of response 11, found at minThFAST = 7 but not at
    iniThFAST = 20.  In every fourth 60 x 60 block the dots are +-60, so cells that keep their iniThFAST corners sit next to cells
    that retry at minThFAST."""
    rng = np.random.default_rng(seed)
    by, bx = np.meshgrid(np.arange(H) // 60, np.arange(W) // 60, indexing="ij")
    amp = np.where((by + bx) % 4 == 0, 60, 12)
    sign = rng.choice([-1, 1], size=(H, W))
    dots = rng.random((H, W)) < 0.02
    return (128 + dots * sign * amp).astype(np.uint8)


def binary(seed: int) -> np.ndarray:
    return (np.random.default_rng(seed).integers(0, 2, size=(H, W)) * 255).astype(np.uint8)


def checkerboard() -> np.ndarray:
    """A one-pixel checkerboard: every ring pixel but the four at odd offsets (0, +-3), (+-3, 0) has the centre's value, so level 0
    has no corner at all; the resized levels are textured and have thousands."""
    y, x = np.mgrid[0:H, 0:W]
    return (((x + y) & 1) * 255).astype(np.uint8)


def min_rows(nlevels: int = 8, scale_factor: float = 1.2) -> int:
    """The fewest rows whose coarsest level is still 45 px (2 x 19 + 7) high: the smallest image the extractor accepts."""
    t = O.Tables(O.ExtractorParams(scale_factor=scale_factor, nlevels=nlevels))
    r = 45
    while O.level_sizes(W, r, t)[-1][1] < 45:
        r += 1
    return r


def level_stats(result: O.OrbResult, shape, params: O.ExtractorParams):
    """Per level: candidate count, the largest per-cell candidate count (from the cell rectangles of level_cells), the number of
    cells, and the initial quad-tree node count round(width / height) of the level's FAST region."""
    rows, cols = shape
    out = []
    for lvl, (lw, lh) in enumerate(O.level_sizes(cols, rows, O.Tables(params))):
        cells, (mbx, mby, Mbx, Mby) = O.level_cells(lw, lh)
        xs, ys, _ = result.candidates[lvl]
        gx, gy = xs + mbx, ys + mby  # level coordinates
        per_cell = [int(((gx >= x0 + 3) & (gx < x1 - 3) & (gy >= y0 + 3) & (gy < y1 - 3)).sum()) for (x0, y0, x1, y1) in cells]
        n_ini = max(int(np.float32(Mbx - mbx) / np.float32(Mby - mby) + np.float32(0.5)), 1)
        out.append({"candidates": len(xs), "cell_max": max(per_cell, default=0), "cells": len(cells), "n_ini": n_ini})
    return out


# ---------------------------------------------------------------------------------------------------------- the cases
P = O.ExtractorParams


def kitti_crop(gray: np.ndarray) -> np.ndarray:
    """The Frame tail's 1024 x 352 crop of the 1242 x 375 fixture (gray)."""
    return np.ascontiguousarray(gray[11:11 + H, 109:109 + W])


def dense(gray: np.ndarray) -> np.ndarray:
    """The ladder's densest frame below the cap: the dense image of the parameter sets."""
    return blend(kitti_crop(gray), LADDER["below"], 1)


# name -> (image from the uncropped gray fixture, extractor parameters)
CASES = {
    "ladder_below": (dense, P()),
    "ladder_above": (lambda g: blend(kitti_crop(g), LADDER["above"], 1), P()),
    "ladder_full": (lambda g: noise(H, W, 1), P()),
    "densest_cell": (lambda g: densest_cell(), P(1000, nlevels=1)),
    "min_th_fallback": (lambda g: low_contrast(2), P()),
    "binary": (lambda g: binary(3), P()),
    "checkerboard": (lambda g: checkerboard(), P()),
    "kitti_uncropped": (lambda g: np.ascontiguousarray(g), P()),
    "smallest_8_levels": (lambda g: np.ascontiguousarray(kitti_crop(g)[:min_rows()]), P()),
    "narrow_level": (lambda g: np.ascontiguousarray(kitti_crop(g)[:, :200]), P()),
    "portrait": (lambda g: np.ascontiguousarray(np.rot90(kitti_crop(g))[:, :160]), P()),
    "wide_4058": (lambda g: np.ascontiguousarray(np.tile(g[100:260], (1, 4))[:, :MAX_PACKED_WIDTH]), P()),
}
# the parameter sets of ORB-SLAM2's configurations (TUM 1000, EuRoC 1200, KITTI 2000; 5000 takes the host tree), the lower
# iniThFAST some use, and two other pyramids, on the KITTI crop and on the dense frame
PARAMS = {"nf1000": P(1000), "nf1200": P(1200), "nf2000": P(2000), "nf5000": P(5000), "th12_7": P(ini_th=12, min_th=7),
          "pyr1.5x5": P(scale_factor=1.5, nlevels=5), "pyr1.1x12": P(scale_factor=1.1, nlevels=12)}
for _k, _p in PARAMS.items():
    CASES["crop_" + _k] = (kitti_crop, _p)
    if _k != "nf2000":  # that one is ladder_below
        CASES["dense_" + _k] = (dense, _p)
