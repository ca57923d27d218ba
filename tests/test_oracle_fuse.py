"""CPU: oracle/fuse_oracle.py's Fuse decision against a direct transcription of ORBmatcher.cc:814-909, its replay against the
literal SearchInNeighbors on constructed and seeded maps, a map where the replay needs its re-search rule, and the
sivo_fuse_camera mirror against the header's layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import fuse_oracle as FO
from oracle import fuse_scene as S
from oracle import track_oracle as T
from oracle.orb_oracle import descriptor_distance
from sivo_b200 import _lib as L
from sivo_b200.mapping import FuseCamera

F32, F64 = np.float32, np.float64


def transcribed(kf, mp, cam, tables, th):
    """ORBmatcher.cc:814-909 line by line (stage numbers as SIVO_FUSE_STAGE_*)."""
    p3Dw = np.asarray(mp["pos"], F32)
    p3Dc = T.gemm_pc(kf.Rcw, p3Dw, kf.tcw)
    if p3Dc[2] < F32(0.0):
        return -1, 256, 0
    with np.errstate(all="ignore"):
        invz = F32(1) / p3Dc[2]
        x = p3Dc[0] * invz
        y = p3Dc[1] * invz
        u = cam.fx * x + cam.cx
        v = cam.fy * y + cam.cy
        if not (u >= cam.min_x and u < cam.max_x and v >= cam.min_y and v < cam.max_y):
            return -1, 256, 1
        ur = u - cam.mbf * invz
        maxDistance = F32(1.2) * F32(mp["max_distance"])
        minDistance = F32(0.8) * F32(mp["min_distance"])
        PO = p3Dw - kf.Ow
        dist3D = T.norm3(PO)
        if dist3D < minDistance or dist3D > maxDistance:
            return -1, 256, 2
        if T.dot3(PO, mp["normal"]) < 0.5 * F64(dist3D):
            return -1, 256, 3
        lq = T.logf(F32(mp["max_distance"]) / dist3D) / tables.log_scale
    if np.isnan(lq):
        return -1, 256, 4
    nPredictedLevel = min(max(int(np.ceil(lq)), 0), tables.nlevels - 1)
    radius = F32(th) * tables.scale[nPredictedLevel]
    vIndices = T.get_features_in_area(kf.grid, kf.kps, kf.geo, u, v, radius)
    if not vIndices:
        return -1, 256, 4
    bestDist, bestIdx = 256, -1
    for idx in vIndices:
        kpLevel = int(kf.kps["octave"][idx])
        if kpLevel < nPredictedLevel - 1 or kpLevel > nPredictedLevel or kpLevel < 0 or kpLevel >= tables.nlevels:
            continue
        kpx, kpy, kpr = F32(kf.kps["x"][idx]), F32(kf.kps["y"][idx]), F32(kf.u_right[idx])
        with np.errstate(all="ignore"):
            if kpr >= 0:
                ex, ey, er = u - kpx, v - kpy, ur - kpr
                if F64((ex * ex + ey * ey + er * er) * tables.inv_sigma2[kpLevel]) > 7.8:
                    continue
            else:
                ex, ey = u - kpx, v - kpy
                if F64((ex * ex + ey * ey) * tables.inv_sigma2[kpLevel]) > 5.99:
                    continue
        dist = descriptor_distance(mp["desc"], kf.desc[idx])
        if dist < bestDist:
            bestDist, bestIdx = dist, idx
    return (bestIdx, bestDist, 6) if bestDist <= 50 else (-1, bestDist, 5)


def test_decision_matches_a_direct_transcription():
    seen = set()
    for name, targets, points, th in S.edge_cases():
        for kf in targets:
            for p in points:
                got = FO.decide(kf, p, S.EDGE_CAMERA, S.TABLES, th)
                assert got == transcribed(kf, p, S.EDGE_CAMERA, S.TABLES, th), name
                seen.add(got[2])
    cur, targets, points = S.make_map(**S.CONSTRUCTED[0])
    for kf in [cur] + targets:
        for mp in points:
            r = FO.point_record(mp)
            got = FO.decide(kf, r, S.CAMERA, S.TABLES, 3.0)
            assert got == transcribed(kf, r, S.CAMERA, S.TABLES, 3.0)
            seen.add(got[2])
    assert seen == set(range(7))


def test_hand_built_decisions():
    cam, tab = S.EDGE_CAMERA, S.TABLES
    kf = S.edge_target([(320.0, 256.0, 0, -1.0, 10), (320.5, 256.0, 0, -1.0, 10), (321.0, 256.0, 0, -1.0, 7)])
    p = S.edge_point([0, 0, 1.0], max_d=1.0)
    assert FO.decide(kf, p, cam, tab, 3.0) == (2, 7, FO.MATCHED)  # the smallest distance
    kf = S.edge_target([(320.0, 256.0, 0, -1.0, 10), (320.5, 256.0, 0, -1.0, 10)])
    assert FO.decide(kf, p, cam, tab, 3.0) == (0, 10, FO.MATCHED)  # ties: the first in walk order
    assert FO.decide(kf, S.edge_point([0, 0, -1.0]), cam, tab, 3.0)[2] == FO.DEPTH
    assert FO.decide(kf, S.edge_point([0.625, 0, 1.0]), cam, tab, 3.0)[2] == FO.IMAGE  # u = max_x is out
    assert FO.decide(kf, S.edge_point([0, 0, 1.0], min_d=2.0), cam, tab, 3.0)[2] == FO.DISTANCE
    assert FO.decide(kf, S.edge_point([0, 0, 1.0], max_d=1.0, normal=[0, 0, -1]), cam, tab, 3.0)[2] == FO.ANGLE
    kf = S.edge_target([(320.0, 256.0, 0, -1.0, 51)])
    assert FO.decide(kf, p, cam, tab, 3.0) == (-1, 51, FO.ABOVE_TH_LOW)
    kf = S.edge_target([(320.0, 256.0, -1, -1.0, 1)])  # level 0 and an octave -1 key: never a candidate
    assert FO.decide(kf, p, cam, tab, 3.0) == (-1, 256, FO.ABOVE_TH_LOW)
    kf = S.edge_target([(300.0, 256.0, 0, -1.0, 1)])
    assert FO.decide(kf, p, cam, tab, 3.0)[2] == FO.NO_CANDIDATE


def _run(prm, how, research=True):
    cur, targets, points = S.make_map(**prm)
    events = set()
    if how == "literal":
        FO.search_in_neighbors(cur, targets, S.CAMERA, S.TABLES, 3.0, events)
        stats = None
    else:
        stats = FO.replay(cur, targets, FO.oracle_rows(S.CAMERA, S.TABLES, 3.0), research, events)
    return FO.map_state([cur] + targets, points), events, stats


@pytest.mark.parametrize("prm", S.CONSTRUCTED + [S.fuzz_params(s) for s in range(16)], ids=lambda p: f"seed{p['seed']}")
def test_replay_equals_literal_search_in_neighbors(prm):
    want, _, _ = _run(prm, "literal")
    got, _, stats = _run(prm, "replay")
    assert got == want
    assert stats["researched"][1] == 0  # the re-search never fires in phase 2


def test_constructed_maps_exercise_every_part_of_the_contract():
    events = set()
    for prm in S.CONSTRUCTED:
        events |= _run(prm, "literal")[1] | _run(prm, "replay")[1]
    assert events >= {"add", "replace_into_inkf", "replace_into_mp", "equal_obs", "bad_inkf", "same_key", "survivor_later",
                      "research_changed"}


def test_replay_without_the_research_rule_differs():
    differs = [prm["seed"] for prm in S.CONSTRUCTED if _run(prm, "replay", research=False)[0] != _run(prm, "literal")[0]]
    assert differs


def test_fuse_camera_mirror_matches_the_header(tmp_path):
    fields = [f for f, _ in FuseCamera._fields_]
    src = tmp_path / "layout.c"
    lines = ["#include <stddef.h>", "#include <stdio.h>", "#include <stdint.h>", '#include "sivo_b200.h"', "int main(void) {",
             '  printf("%zu\\n", sizeof(sivo_fuse_camera));']
    lines += [f'  printf("%zu %zu\\n", offsetof(sivo_fuse_camera, {f}), sizeof(((sivo_fuse_camera*)0)->{f}));' for f in fields]
    src.write_text("\n".join(lines + ["  return 0;", "}"]) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.dirname(L.HEADER), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert int(got[0]) == C.sizeof(FuseCamera)
    for i, f in enumerate(fields):
        d = getattr(FuseCamera, f)
        assert (int(got[1 + 2 * i]), int(got[2 + 2 * i])) == (d.offset, d.size), f
