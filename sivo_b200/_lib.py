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
