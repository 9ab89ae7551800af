"""ctypes binding of tests/voxelgrid_oracle.cpp, the CPU restatement of voxelgrid_sampling -- TEST INFRASTRUCTURE ONLY.  The library
is compiled on first use by tests/native.py with the CPU oracles' flags.
"""
import ctypes as C
import functools
import os

import numpy as np

import native

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "voxelgrid_oracle.cpp")


@functools.cache
def lib():
    L = native.shared_library([SRC], native.ORACLE_FLAGS)
    dp = C.POINTER(C.c_double)
    L.orc_voxelgrid_sampling.restype = C.c_size_t
    L.orc_voxelgrid_sampling.argtypes = [C.c_double, dp, C.c_int, dp, C.c_int, dp, C.c_int, C.c_size_t, C.c_int, dp, dp, dp]
    L.orc_voxelgrid_max_threads.restype = C.c_int
    return L


def max_threads():
    return lib().orc_voxelgrid_max_threads()


def _dp(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


def voxelgrid_sampling(points, resolution, covs=None, normals=None, num_threads=1):
    """-> (points m x 3, covs m x 3 x 3 or None, normals m x 3 or None), voxels in ascending key order.  points N x 3 / N x 4,
    covs N x 3 x 3 / N x 4 x 4, normals N x 3 / N x 4."""
    p = np.ascontiguousarray(points, dtype=np.float64)
    n = len(p)
    c = None if covs is None else np.ascontiguousarray(covs, dtype=np.float64)
    c = None if c is None else c.reshape(n, c.shape[1] * c.shape[2])
    nr = None if normals is None else np.ascontiguousarray(normals, dtype=np.float64)
    op = np.zeros((max(n, 1), 3))
    oc = None if c is None else np.zeros((max(n, 1), 9))
    on = None if nr is None else np.zeros((max(n, 1), 3))
    dummy = np.zeros(16)  # non-NULL pointers for empty inputs
    m = lib().orc_voxelgrid_sampling(
        float(resolution), _dp(p if n else dummy), p.shape[1], None if c is None else _dp(c if n else dummy), 0 if c is None else c.shape[1],
        None if nr is None else _dp(nr if n else dummy), 0 if nr is None else nr.shape[1], n, int(num_threads), _dp(op), _dp(oc), _dp(on)
    )
    return op[:m].copy(), None if oc is None else oc[:m].reshape(m, 3, 3).copy(), None if on is None else on[:m].copy()
