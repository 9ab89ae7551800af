"""ctypes binding of tests/filter_oracle.cpp, the CPU restatement of the device frame filters -- TEST INFRASTRUCTURE ONLY.  The
library is compiled on first use by tests/native.py with the CPU oracles' flags."""
import ctypes as C
import functools
import os

import numpy as np

import native

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "filter_oracle.cpp")
_dp, _lp = C.POINTER(C.c_double), C.POINTER(C.c_int64)


@functools.cache
def lib():
    L = native.shared_library([SRC], native.ORACLE_FLAGS)
    L.orc_priority.restype = C.c_uint64
    L.orc_priority.argtypes = [C.c_uint64, C.c_uint64, C.c_int]
    L.orc_gather.restype = None
    L.orc_gather.argtypes = [_dp, C.c_int, _lp, C.c_size_t, _dp]
    L.orc_random_sampling.restype = C.c_size_t
    L.orc_random_sampling.argtypes = [C.c_size_t, C.c_double, C.c_uint64, _lp]
    L.orc_randomgrid_sampling.restype = C.c_size_t
    L.orc_randomgrid_sampling.argtypes = [_dp, C.c_int, C.c_size_t, C.c_double, C.c_double, C.c_uint64, C.c_int, _lp]
    L.orc_mean_knn_dists.restype = None
    L.orc_mean_knn_dists.argtypes = [_dp, C.c_int, C.c_size_t, C.c_int, C.c_int, _dp]
    L.orc_find_inliers.restype = C.c_size_t
    L.orc_find_inliers.argtypes = [_dp, C.c_size_t, C.c_double, C.c_int, _dp, _lp]
    return L


def _d(a):
    return a.ctypes.data_as(_dp)


def _l(a):
    return a.ctypes.data_as(_lp)


def _pts(points):
    p = np.ascontiguousarray(points, dtype=np.float64)
    return p if len(p) else np.zeros((1, 3))


def priority(seed, i, s):
    return int(lib().orc_priority(seed & (2**64 - 1), i, s))


def gather(rows, K):
    """rows[K] of an n x width array, through the oracle's loop."""
    r = np.ascontiguousarray(rows, dtype=np.float64)
    w = int(np.prod(r.shape[1:]))
    K = np.ascontiguousarray(K, dtype=np.int64)
    out = np.zeros((max(len(K), 1), w))
    lib().orc_gather(_d(r.reshape(len(r), w) if len(r) else np.zeros((1, w))), w, _l(K if len(K) else np.zeros(1, np.int64)), len(K), _d(out))
    return out[: len(K)].reshape((len(K),) + r.shape[1:])


def random_sampling(n, rate, seed=5489):
    out = np.zeros(max(n, 1), dtype=np.int64)
    m = lib().orc_random_sampling(n, float(rate), seed & (2**64 - 1), _l(out))
    return out[:m].copy()


def randomgrid_sampling(points, resolution, rate, seed=5489, apply_cap=True):
    p = _pts(points)
    n = len(points)
    out = np.zeros(max(n, 1), dtype=np.int64)
    m = lib().orc_randomgrid_sampling(_d(p), p.shape[1], n, float(resolution), float(rate), seed & (2**64 - 1), 1 if apply_cap else 0, _l(out))
    return out[:m].copy()


def mean_knn_dists(points, k, brute=False):
    p = _pts(points)
    out = np.zeros(max(len(points), 1))
    lib().orc_mean_knn_dists(_d(p), p.shape[1], len(points), int(k), 1 if brute else 0, _d(out))
    return out[: len(points)].copy()


def find_inliers(dists, std_thresh, sequential=False):
    """(K, thresh) of mean distances `dists`: chunked sums, or the reference's sequential ones."""
    d = np.ascontiguousarray(dists, dtype=np.float64)
    out = np.zeros(max(len(d), 1), dtype=np.int64)
    th = np.zeros(1)
    m = lib().orc_find_inliers(_d(d), len(d), float(std_thresh), 1 if sequential else 0, _d(th), _l(out))
    return out[:m].copy(), float(th[0])


def inliers(points, k, std_thresh, sequential=False):
    """(K, mean distances, thresh) of remove_outliers over `points`."""
    d = mean_knn_dists(points, k)
    K, th = find_inliers(d, std_thresh, sequential)
    return K, d, th
