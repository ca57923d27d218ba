"""CPU-only checks that the Python side holds the C ABI of include/sivo_b200.h: every entry point is typed from the header's
prototypes, and every struct mirror (ctypes Structure or numpy dtype) has the header's field offsets and size, as a C compiler
lays the header out."""
import ctypes as C
import os
import re
import subprocess

import pytest

from sivo_b200 import _lib as L
from sivo_b200.mapping import KeyframeKeys, MappingParams
from sivo_b200.orb import KP_DTYPE
from sivo_b200.pose import TRACE_DTYPE, PoseResult
from sivo_b200.reloc import PoseDebug
from sivo_b200.track import MAP_POINT_DTYPE, TrackFrame

MIRRORS = {"sivo_keypoint": KP_DTYPE, "sivo_map_point": MAP_POINT_DTYPE, "sivo_pose_result": PoseResult, "sivo_pose_trace_rec": TRACE_DTYPE,
           "sivo_keyframe_keys": KeyframeKeys, "sivo_mapping_params": MappingParams, "sivo_track_frame": TrackFrame,
           "sivo_info_camera": L.InfoCamera, "sivo_segnet_options": L.SegnetOptions, "sivo_pnp_pose_debug": PoseDebug}


def _header_without_comments():
    return re.sub(r"/\*.*?\*/", "", open(L.HEADER).read(), flags=re.S)


def test_every_declared_function_is_typed_with_the_headers_parameter_count():
    text = _header_without_comments()
    lib = L.lib()
    names = L.declared_symbols()
    assert len(names) == len(set(re.findall(r"\b(sivo_[a-z0-9_]+)\s*\(", text)))
    for name in names:
        params = re.search(rf"\b{name}\s*\(([^)]*)\)", text)[1].strip()
        count = 0 if params in ("", "void") else params.count(",") + 1
        assert getattr(lib, name).argtypes is not None and len(getattr(lib, name).argtypes) == count, name


def test_signatures_spelled_out():
    lib = L.lib()
    vp, i32 = C.c_void_p, C.c_int32
    want = {"sivo_dbg_pnp_draws": [i32, C.c_uint64, C.c_uint32, C.c_uint64, i32, i32, i32, vp],
            "sivo_segnet_blob": [vp, C.c_char_p, vp, C.c_size_t, vp, vp, vp, vp],
            "sivo_orb_create": [i32, C.c_float, i32, i32, i32, i32, vp],
            "sivo_segnet_set_frame": [vp, C.c_uint64],
            "sivo_info_select": [vp, vp, vp, vp, i32, vp, C.c_double, vp, vp, vp, vp],
            "sivo_segnet_op_timing": [vp, i32, vp, C.c_size_t, vp, vp, vp],
            "sivo_search_by_bow": [vp, vp, vp, vp, i32, vp, vp, i32, C.c_float, i32, vp, vp],
            "sivo_version": []}
    for name, argtypes in want.items():
        assert list(getattr(lib, name).argtypes) == argtypes, name
    for name in ("sivo_segnet_destroy", "sivo_orb_destroy", "sivo_vocabulary_destroy", "sivo_pnp_destroy"):
        assert getattr(lib, name).restype is None, name
    assert lib.sivo_orb_create.restype is C.c_int and lib.sivo_version.restype is C.c_char_p
    assert lib.sivo_last_error.restype is C.c_char_p


def test_parser_refuses_a_type_it_cannot_map():
    assert L.prototypes("int sivo_a(const char* p, uint8_t* const* q, float f);\nvoid sivo_b(void);") == {
        "sivo_a": (C.c_int, [C.c_char_p, C.c_void_p, C.c_float]), "sivo_b": (None, [])}
    for text in ("int sivo_bad(long n);", "int sivo_bad(sivo_keypoint kp);", "int sivo_bad(int);", "long sivo_bad(int n);",
                 "int sivo_ok(int n);\n/* a comment */ int sivo_bad(unsigned int n);"):
        with pytest.raises(ValueError, match="sivo_bad"):
            L.prototypes(text)


def _python_layout(mirror):
    """(sizeof, [(field, offset, size)]) of a ctypes Structure or a numpy structured dtype."""
    if isinstance(mirror, type) and issubclass(mirror, C.Structure):
        return C.sizeof(mirror), [(n, getattr(mirror, n).offset, getattr(mirror, n).size) for n, _ in mirror._fields_]
    return mirror.itemsize, [(n, mirror.fields[n][1], mirror.fields[n][0].itemsize) for n in mirror.names]


def test_struct_mirrors_match_the_header_layout(tmp_path):
    """A C program generated from the mirrors' own field lists prints what the compiler makes of the header."""
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "sivo_b200.h"', "int main(void) {"]
    want = []
    for struct, mirror in MIRRORS.items():
        size, fields = _python_layout(mirror)
        lines.append(f'  printf("{struct} %zu\\n", sizeof({struct}));')
        want.append(f"{struct} {size}")
        for name, offset, fsize in fields:
            lines.append(f'  printf("{struct}.{name} %zu %zu\\n", offsetof({struct}, {name}), sizeof((({struct}*)0)->{name}));')
            want.append(f"{struct}.{name} {offset} {fsize}")
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.dirname(L.HEADER), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")[:-1]
    assert got == want
