"""Building blocks of the projection-search tests: keypoint and map-point records in the library's layouts (KP_DTYPE and
MAP_POINT_DTYPE), descriptors with chosen bits set, and map points that project to chosen pixels."""
import numpy as np

from sivo_b200.orb import KP_DTYPE as KP
from sivo_b200.track import MAP_POINT_DTYPE as MP

SCALE = np.float32(1.2) ** np.arange(8, dtype=np.float32)
RESERVED = -0x5A5A5A5B  # every point's reserved field: junk, which both searches ignore


def keys(xy, octave=0, angle=0.0):
    k = np.zeros(len(xy), KP)
    k["x"], k["y"] = np.asarray(xy, np.float32).T
    k["octave"], k["angle"] = octave, angle
    return k


def desc_with(bits):
    d = np.zeros(32, np.uint8)
    for b in bits:
        d[b // 8] |= 1 << (b % 8)
    return d


def point_at(f, u, v, z, desc, observed=1, octave=0, angle=0.0):
    """A point that projects to (u, v) at depth z through the identity pose, seen head-on at its own distance."""
    p = np.zeros((), MP)
    x, y = (u - f.cx) * z / f.fx, (v - f.cy) * z / f.fy
    p["pos"] = (x, y, z)
    d = np.float32(np.sqrt(x * x + y * y + z * z))
    p["normal"] = np.array([x, y, z], np.float32) / d
    p["max_distance"], p["min_distance"] = d, d / SCALE[-1]
    p["desc"], p["observed"], p["octave"], p["angle"], p["reserved"] = desc, observed, octave, angle, RESERVED
    return p
