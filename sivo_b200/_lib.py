"""ctypes loader for libsivo_b200.so.  There is no CPU fallback: if the CUDA library is missing or a
call fails, this raises -- the product path never routes through oracle/."""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsivo_b200.so")
HEADER = os.path.join(_HERE, "..", "include", "sivo_b200.h")

OK, EINVAL, ENOENT, EFORMAT, ECUDA, ENOMEM, ERANGE = 0, -22, -2, -74, -5, -12, -34
PRECISION_FP16, PRECISION_FP32 = 0, 1
ENGINE_AUTO, ENGINE_SIMT, ENGINE_TCGEN05 = 0, 1, 2


class SivoError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"[{code}] {msg}")
        self.code = code


class Keypoint(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("size", C.c_float), ("angle", C.c_float),
                ("response", C.c_float), ("octave", C.c_int32), ("class_id", C.c_int32)]


class SegnetOptions(C.Structure):
    _fields_ = [("device", C.c_int32), ("T", C.c_int32), ("seed", C.c_uint64), ("precision", C.c_int32),
                ("engine", C.c_int32), ("keep_blobs", C.c_int32), ("reserved", C.c_int32)]


class InfoCamera(C.Structure):
    """sivo_info_camera: the Frame members the information selection reads (Rwc row-major, Sigma_cw row-major 6x6)."""
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("invfx", C.c_float),
                ("invfy", C.c_float), ("mb", C.c_float), ("Rwc", C.c_float * 9), ("Ow", C.c_float * 3), ("sigma_cw", C.c_double * 36)]


def build(verbose: bool = False) -> str:
    """Compiles the library in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
    r = subprocess.run(["make", "-C", os.path.join(_HERE, "csrc"), "-j8"], capture_output=True, text=True)
    if verbose or r.returncode:
        print(r.stdout[-4000:], r.stderr[-4000:])
    if r.returncode:
        raise RuntimeError("building libsivo_b200.so failed")
    return LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)")
        _lib = C.CDLL(LIB_PATH)
        _lib.sivo_last_error.restype = C.c_char_p
        _lib.sivo_version.restype = C.c_char_p
        _lib.sivo_segnet_destroy.restype = None
        _lib.sivo_orb_destroy.restype = None
        vp, i32, f32 = C.c_void_p, C.c_int, C.c_float
        _lib.sivo_segnet_semantic_keys_device.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp]
        _lib.sivo_stereo_match_device.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, f32, f32, vp, vp, vp]
        _lib.sivo_info_select.argtypes = [vp, vp, vp, vp, i32, vp, C.c_double, vp, vp, vp, vp]
        _lib.sivo_info_select_device.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.c_double, vp, vp, vp, vp, vp]
        _lib.sivo_dbg_info_terms.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp]
        _lib.sivo_search_local_points_device.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, f32, f32, vp, vp, vp, vp]
        _lib.sivo_search_last_frame_device.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, f32, vp, vp, vp]
        _lib.sivo_search_local_points.argtypes = [vp, vp, vp, vp, vp, i32, vp, i32, vp, f32, f32, vp, vp, vp]
        _lib.sivo_search_last_frame.argtypes = [vp, vp, vp, vp, i32, vp, i32, vp, vp, vp, f32, vp, vp]
        _lib.sivo_dbg_features_in_area.argtypes = [vp, vp, i32, f32, f32, f32, f32, vp, vp, i32, vp, vp, i32]
        _lib.sivo_pose_optimize_device.argtypes = [vp, vp, vp, vp, vp, vp, f32, f32, f32, f32, f32, vp, vp, vp, vp]
        _lib.sivo_pose_gather_device.argtypes = [vp, vp, vp, vp, i32, vp, vp]
        _lib.sivo_pose_optimize.argtypes = [vp, vp, vp, vp, i32, f32, f32, f32, f32, f32, vp, vp, vp]
        _lib.sivo_dbg_pose_system.argtypes = [vp, vp, vp, vp, i32, f32, f32, f32, f32, f32, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]
        _lib.sivo_dbg_pose_trace.argtypes = [vp, vp, vp, vp, i32, f32, f32, f32, f32, f32, vp, vp, vp, vp, i32]
        _lib.sivo_dbg_pose_se3.argtypes = [i32, i32, vp, vp, vp, vp, vp, vp]
        _lib.sivo_keyframe_gather_device.argtypes = [vp] * 19
        _lib.sivo_create_map_points_device.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp]
        _lib.sivo_create_map_points.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp, vp]
        _lib.sivo_dbg_create_map_points.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        _lib.sivo_vocabulary_destroy.restype = None
        _lib.sivo_vocabulary_load_text.argtypes = [C.c_char_p, i32, vp]
        _lib.sivo_vocabulary_create.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, i32, vp]
        _lib.sivo_dbg_vocabulary_parse.argtypes = [C.c_char_p, vp, vp, vp, vp, vp, vp, i32]
        _lib.sivo_compute_bow_device.argtypes = [vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp]
        _lib.sivo_compute_bow.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp]
        _lib.sivo_search_by_bow_device.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, i32, f32, i32, vp, vp, vp]
        _lib.sivo_search_by_bow.argtypes = [vp, vp, vp, vp, i32, vp, vp, i32, f32, i32, vp, vp]
        _lib.sivo_pnp_destroy.restype = None
        _lib.sivo_pnp_create.argtypes = [vp, i32, C.c_uint64, vp]
        _lib.sivo_pnp_setup_device.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, C.c_uint64, f32, f32, f32, f32, vp]
        _lib.sivo_pnp_iterate_device.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp]
        _lib.sivo_dbg_pnp_state.argtypes = [vp, vp, vp]
        d64 = C.c_double
        _lib.sivo_dbg_pnp_compute_pose.argtypes = [i32, vp, vp, vp, i32, f32, f32, f32, f32, vp, vp, vp, vp]
        _lib.sivo_dbg_pnp_hypotheses.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp]
        _lib.sivo_dbg_pnp_draws.argtypes = [i32, C.c_uint64, C.c_uint32, C.c_uint64, i32, i32, i32, vp]
        _lib.sivo_dbg_conv_unpooled.argtypes = [i32, vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, i32, i32, vp]
    return _lib


def check(rc: int) -> int:
    if rc < 0:
        raise SivoError(rc, lib().sivo_last_error().decode(errors="replace"))
    return rc


def declared_symbols() -> list:
    """Every function name declared in include/sivo_b200.h (for the export test)."""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sivo_[a-z0-9_]+)\s*\(", text)))
