"""ctypes binding of tests/transform_oracle.cpp, the CPU oracle's transform(frame, T) -- TEST INFRASTRUCTURE ONLY.

The library (the oracle's sources plus orc_transform) is compiled on first use by tests/native.py, with the compiler and flags that
oracle/Makefile builds liboracle.so with, read from the Makefile itself.
"""
import ctypes as C
import functools
import os
import shlex
import subprocess

import numpy as np

import native

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "transform_oracle.cpp")
ORACLE_DIR = os.path.join(os.path.dirname(HERE), "oracle")


def oracle_compile_command():
    """$(CXX) $(CXXFLAGS) of oracle/Makefile, as it would build liboracle.so."""
    out = subprocess.run(["make", "-s", "--no-print-directory", "-C", ORACLE_DIR, "--eval=print-cxx: ; @echo $(CXX) $(CXXFLAGS)", "print-cxx"], capture_output=True,
                         text=True, check=True).stdout
    return shlex.split(out.strip())


@functools.cache
def lib():
    cxx, *flags = oracle_compile_command()
    L = native.shared_library([SRC], flags + ["-shared"], cxx)
    vp, dp = C.c_void_p, C.POINTER(C.c_double)
    L.orc_cloud_create.restype = vp
    L.orc_cloud_create.argtypes = [dp, dp, C.c_size_t]
    L.orc_cloud_destroy.argtypes = [vp]
    L.orc_cloud_set_normals.argtypes = [vp, dp]
    L.orc_transform.argtypes = [dp, vp, dp, dp, dp]
    return L


def _dp(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


def transform(T, points, covs=None, normals=None):
    """orc_transform(T, cloud) -> (points n x 3, covs n x 3 x 3 or None, normals n x 3 or None).  points n x 3, covs n x 3 x 3,
    normals n x 3; T a 4x4 pose."""
    L = lib()
    p = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
    n = len(p)
    c = None if covs is None else np.ascontiguousarray(covs, dtype=np.float64).reshape(n, 9)
    nr = None if normals is None else np.ascontiguousarray(normals, dtype=np.float64).reshape(n, 3)
    dummy = np.zeros(9)  # non-NULL pointers for empty inputs
    h = L.orc_cloud_create(_dp(p if n else dummy), None if c is None else _dp(c if n else dummy), n)
    try:
        if nr is not None:
            L.orc_cloud_set_normals(h, _dp(nr if n else dummy))
        T16 = np.ascontiguousarray(T, dtype=np.float64).reshape(16)
        op = np.zeros((max(n, 1), 3))
        oc = None if c is None else np.zeros((max(n, 1), 9))
        on = None if nr is None else np.zeros((max(n, 1), 3))
        L.orc_transform(_dp(T16), h, _dp(op), _dp(oc), _dp(on))
    finally:
        L.orc_cloud_destroy(h)
    return op[:n].copy(), None if oc is None else oc[:n].reshape(n, 3, 3).copy(), None if on is None else on[:n].copy()
