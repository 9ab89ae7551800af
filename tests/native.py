"""Compiles and runs the native test code: the CPU oracle libraries loaded through ctypes, and the C++ adapter drivers of tests/cpp
-- TEST INFRASTRUCTURE ONLY.

Everything is compiled at most once per process, into one temporary directory (the source tree may be read-only) that is removed
when the process exits.
"""
import atexit
import ctypes
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GXX = "/usr/bin/g++"
# the CPU oracles' flags: -ffp-contract=off and no fast-math, so every product and sum is rounded on its own, in the order written
ORACLE_FLAGS = ["-O3", "-std=c++17", "-fopenmp", "-fPIC", "-ffp-contract=off", "-Wall", "-shared"]
LIBDIR = os.path.join(ROOT, "gtsam_points_b200", "lib")


@functools.cache
def _tmpdir():
    tmp = tempfile.mkdtemp(prefix="b2_native_")
    atexit.register(shutil.rmtree, tmp, True)
    return tmp


_LIBS = {}


def shared_library(sources, flags, cxx=GXX):
    """The shared library `cxx flags -o lib<first source>.so sources`, compiled on first use and loaded."""
    key = (tuple(sources), tuple(flags), cxx)
    if key not in _LIBS:
        so = os.path.join(_tmpdir(), "lib" + os.path.splitext(os.path.basename(sources[0]))[0] + ".so")
        subprocess.check_call([cxx, *flags, "-o", so, *sources])
        _LIBS[key] = ctypes.CDLL(so)
    return _LIBS[key]


@functools.cache
def _b2points():
    from gtsam_points_b200 import build

    return build.build()


@functools.cache
def adapter_driver(name, mock_gtsam):
    """tests/cpp/<name>.cpp built against libb2points.so: standalone, or with the GTSAM-typed branch of the adapters compiled against
    the header mocks of tests/cpp/mock_gtsam.  Returns the executable's path."""
    _b2points()
    exe = os.path.join(_tmpdir(), name + ("_gtsam" if mock_gtsam else ""))
    cmd = [GXX, "-std=c++17", "-O2", "-Wall", "-Wno-unused-variable", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "gtsam_points_b200", "cpp", "include")]
    if mock_gtsam:
        cmd += ["-I", os.path.join(ROOT, "tests", "cpp", "mock_gtsam")]
    cmd += [os.path.join(ROOT, "tests", "cpp", name + ".cpp"), "-o", exe, "-L", LIBDIR, "-lb2points", f"-Wl,-rpath,{LIBDIR}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return exe


def run_driver(exe, arrays, timeout):
    """Runs a driver on the case file of `arrays` -- per array a uint64 count, then that many float64 values (driver.hpp's Case reads
    them back) -- and returns its stdout, which must report OK."""
    with tempfile.TemporaryDirectory(dir=_tmpdir()) as d:
        case = os.path.join(d, "case.bin")
        with open(case, "wb") as f:
            for a in arrays:
                a = np.ascontiguousarray(a, dtype=np.float64).ravel()
                f.write(np.uint64(a.size).tobytes())
                f.write(a.tobytes())
        r = subprocess.run([exe, case], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "OK" in r.stdout
    return r.stdout
