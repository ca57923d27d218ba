"""Compiles the unmodified C++ shim (integration/src/*.cpp) + tests/cpp/test_shim.cpp with g++ against integration/stubs
(minimal OpenCV / Eigen look-alikes; the image has neither) and links it to libsivo_b200.so.  The binaries go to a per-user
directory under the system's temporary directory, keyed by the checkout's path, so the suite writes nothing into the tree
(which may be read-only)."""
import hashlib
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD_DIR = os.path.join(tempfile.gettempdir(), f"sivo_b200_shim_{os.getuid()}_{hashlib.sha1(ROOT.encode()).hexdigest()[:12]}")
BIN = os.path.join(BUILD_DIR, "test_shim")
SOURCES = [os.path.join(ROOT, "integration", "src", "bayesian_segnet.cpp"), os.path.join(ROOT, "integration", "src", "ORBextractor.cc"),
           os.path.join(ROOT, "tests", "cpp", "test_shim.cpp")]


def build(force=False):
    deps = SOURCES + [os.path.join(ROOT, "sivo_b200", "libsivo_b200.so"), os.path.join(ROOT, "include", "sivo_b200.h")]
    for d, _, files in os.walk(os.path.join(ROOT, "integration")):
        deps += [os.path.join(d, f) for f in files]
    if not force and os.path.exists(BIN) and all(os.path.getmtime(BIN) >= os.path.getmtime(d) for d in deps):
        return BIN
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    lib_dir = os.path.join(ROOT, "sivo_b200")
    cmd = ["g++", "-std=c++11", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "integration", "stubs"),
           "-I" + os.path.join(ROOT, "integration", "include"), "-I" + os.path.join(ROOT, "include"), *SOURCES,
           "-L" + lib_dir, "-lsivo_b200", "-Wl,-rpath," + lib_dir, "-o", BIN]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("shim build failed:\n" + r.stderr[-4000:])
    return BIN
