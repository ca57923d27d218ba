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


# Every C type in the header's prototypes: the scalars by name, `const char*` as a string, every other pointer (handles, struct
# and array pointers, `T**`, `T* const*`, the `char*` a string buffer is passed for) as an address.  A type outside these tables
# fails the load, so no declared function is ever called untyped.
_SCALARS = {"int": C.c_int32, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64, "size_t": C.c_size_t,
            "float": C.c_float, "double": C.c_double}
_RETURNS = {"int": C.c_int, "void": None, "const char*": C.c_char_p}


def _type(t: str) -> str:
    return re.sub(r" ?\* ?", "*", " ".join(t.split()))


def _param(decl: str, name: str):
    t = _type(re.sub(r"\b[A-Za-z_]\w*\s*$", "", decl))  # drop the parameter's name
    if "*" in t:
        return C.c_char_p if t == "const char*" else C.c_void_p
    if t.removeprefix("const ") not in _SCALARS:
        raise ValueError(f"{name}: parameter {decl.strip()!r} has no ctypes type")
    return _SCALARS[t.removeprefix("const ")]


def prototypes(text: str = None) -> dict:
    """{name: (restype, argtypes)} of every sivo_* function declared in `text` (default: include/sivo_b200.h).  Raises
    ValueError, naming the function, for a type outside the mapping."""
    if text is None:
        with open(HEADER) as f:
            text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", "", text, flags=re.M)
    out = {}
    for stmt in re.split(r"[;{}]", text):
        m = re.fullmatch(r"\s*(.*?)\b(sivo_[a-z0-9_]+)\s*\((.*)\)\s*", stmt, flags=re.S)
        if m is None:
            continue
        ret, name, params = _type(m[1]), m[2], m[3]
        if ret not in _RETURNS:
            raise ValueError(f"{name}: return type {ret!r} has no ctypes type")
        params = [] if _type(params) in ("", "void") else params.split(",")
        out[name] = (_RETURNS[ret], [_param(p, name) for p in params])
    return out


def declared_symbols() -> list:
    """Every function name declared in include/sivo_b200.h."""
    return sorted(prototypes())


def ptr(a):
    """The address of numpy array `a` for a pointer parameter (None: NULL).  The returned object keeps `a` alive."""
    return None if a is None else a.ctypes.data_as(C.c_void_p)


_lib = None


def lib() -> C.CDLL:
    """The library, every declared function typed from the header (argtypes / restype) before first use."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)")
        dll = C.CDLL(LIB_PATH)
        protos = prototypes()
        missing = [s for s in sorted(protos) if not hasattr(dll, s)]
        if missing:
            raise RuntimeError(f"{LIB_PATH} does not export {missing}")
        for name, (restype, argtypes) in protos.items():
            fn = getattr(dll, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = dll
    return _lib


def check(rc: int) -> int:
    if rc < 0:
        raise SivoError(rc, lib().sivo_last_error().decode(errors="replace"))
    return rc
