"""-m gpu: sivo_fuse_device, sivo_fuse and sivo_dbg_fuse held to oracle/fuse_oracle.py bit for bit at every boundary of the
Fuse rule (oracle/fuse_scene.py's edge_cases): z at +-0 and one ulp either side, u and v at the image bounds, both distance gates,
the viewing angle at 0.5 dist3D, PredictScale at exact powers and both clamps, octaves level - 2 .. level + 1 and an octave -1 key
at level 0, u_right 0 / -1 / NaN, e2 invSigma2 straddling 7.8 and 5.99, crowded windows with ties and 50 against 51 over several
cells and 32-key chunks, clipped corners, NaN positions and normals, and th other than 3."""
import numpy as np
import pytest

from fuse_support import camera, host_targets, records, run_device
from oracle import fuse_oracle as FO
from oracle import fuse_scene as S
from sivo_b200.mapping import dbg_fuse, fuse
from sivo_b200.orb import ORBextractor

pytestmark = pytest.mark.gpu
CASES = S.edge_cases()


@pytest.fixture(scope="module")
def left():
    return ORBextractor(2000, 1.2, 8, 20, 7)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_boundary(left, case):
    name, kfs, points, th = case
    want = FO.decide_all(kfs, points, S.EDGE_CAMERA, S.TABLES, th)
    m, d = fuse(left, host_targets(kfs), camera(S.EDGE_CAMERA), records(points), th)
    dm, dd, ds = dbg_fuse(left, host_targets(kfs), camera(S.EDGE_CAMERA), records(points), th)
    vm, vd = run_device(left, kfs, S.EDGE_CAMERA, points, th)
    for gm, gd in ((m, d), (dm, dd), (vm, vd)):
        np.testing.assert_array_equal(gm, want[0], err_msg=name)
        np.testing.assert_array_equal(gd, want[1], err_msg=name)
    np.testing.assert_array_equal(ds, want[2], err_msg=name)


def test_the_cases_reach_both_sides_of_each_boundary():
    stages = {name: FO.decide_all(kfs, pts, S.EDGE_CAMERA, S.TABLES, th)[2] for name, kfs, pts, th in CASES}
    assert {FO.DEPTH, FO.IMAGE} <= set(stages["depth"].ravel())
    assert {FO.IMAGE, FO.MATCHED} <= set(stages["image"].ravel())
    assert {FO.DISTANCE, FO.MATCHED} <= set(stages["distance"].ravel())
    assert {FO.ANGLE, FO.MATCHED, FO.IMAGE, FO.NO_CANDIDATE} <= set(stages["angle_nan"].ravel())
    assert {FO.ABOVE_TH_LOW, FO.MATCHED} <= set(stages["chi2"].ravel())
    assert {FO.ABOVE_TH_LOW, FO.MATCHED} <= set(stages["octaves"].ravel())
    assert {FO.ABOVE_TH_LOW, FO.MATCHED} <= set(stages["crowd"].ravel())
    dist = FO.decide_all(*[c for c in CASES if c[0] == "crowd"][0][1:3], S.EDGE_CAMERA, S.TABLES, 3.0)[1]
    assert {50, 51} <= set(dist.ravel())
