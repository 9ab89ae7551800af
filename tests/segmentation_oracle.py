"""ctypes binding of tests/segmentation_oracle.cpp, the CPU restatement of region growing -- TEST INFRASTRUCTURE ONLY.  The library
is compiled on first use by tests/native.py with the CPU oracles' flags."""
import ctypes as C
import functools
import os

import numpy as np

import native

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "segmentation_oracle.cpp")
_dp, _lp, _vp = C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_void_p


@functools.cache
def lib():
    L = native.shared_library([SRC], native.ORACLE_FLAGS)
    L.orc_nearest.restype = C.c_longlong
    L.orc_nearest.argtypes = [_dp, C.c_size_t, _dp]
    L.orc_radius.restype = C.c_size_t
    L.orc_radius.argtypes = [_dp, C.c_size_t, _dp, C.c_double, C.c_size_t, C.c_int, _lp]
    L.orc_rg_create.restype = _vp
    L.orc_rg_create.argtypes = [_dp, _dp, C.c_size_t, C.c_longlong, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int]
    L.orc_rg_update.restype = C.c_int
    L.orc_rg_update.argtypes = [_vp, C.c_int]
    L.orc_rg_size.restype = C.c_size_t
    L.orc_rg_size.argtypes = [_vp]
    L.orc_rg_get.restype = None
    L.orc_rg_get.argtypes = [_vp, _lp]
    L.orc_rg_destroy.restype = None
    L.orc_rg_destroy.argtypes = [_vp]
    L.orc_mc_network.restype = C.c_longlong
    L.orc_mc_network.argtypes = [_dp, _dp, C.c_size_t, C.c_size_t, C.c_int, C.c_double, C.c_double, C.c_double, _lp, _dp, _lp]
    L.orc_mc_flow.restype = C.c_longlong
    L.orc_mc_flow.argtypes = [_dp, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, _lp, _lp, C.c_double, C.c_longlong, C.c_double, C.c_longlong, _lp,
                              C.POINTER(C.c_size_t)]
    return L


def _rows(a):
    a = np.ascontiguousarray(a, dtype=np.float64).reshape(-1, 3)
    return a if len(a) else np.zeros((1, 3))


def nearest(points, q):
    return int(lib().orc_nearest(_rows(points).ctypes.data_as(_dp), len(points), _rows(q).ctypes.data_as(_dp)))


def radius(points, q, r, max_nn=2**31 - 1, brute=False):
    p = _rows(points)
    out = np.zeros(max(len(points), 1), dtype=np.int64)
    m = lib().orc_radius(p.ctypes.data_as(_dp), len(points), _rows(q).ctypes.data_as(_dp), float(r), int(max_nn), 1 if brute else 0, out.ctypes.data_as(_lp))
    return out[:m].copy()


class RegionGrowing:
    """The reference's RegionGrowingContext with its init / update / cluster_indices; seed is the seed point's index (-1: the empty
    context of a cloud without points)."""

    def __init__(self, points, normals, seed, distance_threshold=0.5, angle_threshold=np.deg2rad(10.0), dilation_radius=0.5, max_cluster_size=1000000, brute=False):
        self._p, self._n = _rows(points), _rows(normals)
        self.h = lib().orc_rg_create(self._p.ctypes.data_as(_dp), self._n.ctypes.data_as(_dp), len(points), int(seed), float(distance_threshold), float(angle_threshold),
                                     float(dilation_radius), int(max_cluster_size), 1 if brute else 0)

    def update(self, max_steps=1000000):
        return bool(lib().orc_rg_update(self.h, int(max_steps)))

    @property
    def cluster_indices(self):
        m = lib().orc_rg_size(self.h)
        out = np.zeros(max(m, 1), dtype=np.int64)
        lib().orc_rg_get(self.h, out.ctypes.data_as(_lp))
        return out[:m].copy()

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_rg_destroy(self.h)
            self.h = None


def trace(points, normals, seed, steps, **kw):
    """[(converged, cluster)] after each update(max_steps) for max_steps in `steps`."""
    rg = RegionGrowing(points, normals, seed, **kw)
    return [(rg.update(s), rg.cluster_indices) for s in steps]


Q = 2.0**32


def mc_network(points, normals, s, k=20, distance_sigma=0.25, angle_sigma=np.deg2rad(10.0), background_mask_radius=3.0):
    """(t or -1, idx n x k, double weights n x k, quantised capacities n x k) of the min-cut network's k-NN arcs."""
    p, nr = _rows(points), _rows(normals)
    n = len(points)
    idx, q = np.zeros((max(n, 1), k), np.int64), np.zeros((max(n, 1), k), np.int64)
    w = np.zeros((max(n, 1), k))
    t = lib().orc_mc_network(p.ctypes.data_as(_dp), nr.ctypes.data_as(_dp), n, int(s), int(k), float(distance_sigma), float(angle_sigma), float(background_mask_radius),
                             idx.ctypes.data_as(_lp), w.ctypes.data_as(_dp), q.ctypes.data_as(_lp))
    return int(t), idx[:n], w[:n], q[:n]


def mc_flow(points, s, t, idx, q, background_mask_radius=3.0, background_weight=0.2, foreground_mask_radius=-1.0, foreground_weight=0.2, quantum=Q):
    """(maximum flow in quanta, the minimal source set) of an integer Dinic over the k-NN capacities q (caller-supplied), background
    arcs and, for foreground_mask_radius >= 0, the foreground arcs into s."""
    p = _rows(points)
    n = len(points)
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    q = np.ascontiguousarray(q, dtype=np.int64)
    out = np.zeros(max(n, 1), np.int64)
    m = C.c_size_t(0)
    flow = lib().orc_mc_flow(p.ctypes.data_as(_dp), n, int(s), int(t), idx.shape[1], idx.ctypes.data_as(_lp), q.ctypes.data_as(_lp), float(background_mask_radius),
                             int(np.floor(background_weight * quantum + 0.5)), float(foreground_mask_radius), int(np.floor(foreground_weight * quantum + 0.5)), out.ctypes.data_as(_lp), C.byref(m))
    return int(flow), out[: m.value].copy()
