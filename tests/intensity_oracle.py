"""ctypes binding of tests/intensity_oracle.cpp, the CPU restatement of how the reference carries point intensities -- TEST
INFRASTRUCTURE ONLY.  The library is compiled on first use by tests/native.py with the CPU oracles' flags."""
import ctypes as C
import functools
import os

import numpy as np

import native

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "intensity_oracle.cpp")
_dp, _ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)


@functools.cache
def lib():
    L = native.shared_library([SRC], native.ORACLE_FLAGS)
    L.orc_int_map_create.restype = C.c_void_p
    L.orc_int_map_create.argtypes = [C.c_double, C.c_size_t, C.c_size_t, C.c_int, C.c_double]
    L.orc_int_map_destroy.argtypes = [C.c_void_p]
    L.orc_int_map_insert.argtypes = [C.c_void_p, _dp, _dp, C.c_size_t]
    L.orc_int_map_num_voxels.restype = C.c_size_t
    L.orc_int_map_num_voxels.argtypes = [C.c_void_p]
    L.orc_int_map_num_points.restype = C.c_size_t
    L.orc_int_map_num_points.argtypes = [C.c_void_p]
    L.orc_int_map_export.argtypes = [C.c_void_p, _ip, _dp, _ip, _dp, _dp]
    L.orc_int_voxelgrid.restype = C.c_size_t
    L.orc_int_voxelgrid.argtypes = [C.c_double, _dp, _dp, C.c_size_t, _dp]
    L.orc_int_merge_frames.restype = C.c_size_t
    L.orc_int_merge_frames.argtypes = [C.c_double, _dp, _dp, C.c_size_t, _dp]
    return L


def _d(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _f64(a, cols=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a if cols is None else np.ascontiguousarray(a[:, :cols])


class Map:
    """IncrementalVoxelMap<GaussianVoxel> (max_points_in_cell = 0) or IncrementalVoxelMap<FlatContainer> (> 0), intensities only."""

    def __init__(self, resolution, lru_horizon=10, lru_clear_cycle=10, max_points_in_cell=0, min_dist_in_cell=0.1):
        self.h = lib().orc_int_map_create(float(resolution), int(lru_horizon), int(lru_clear_cycle), int(max_points_in_cell), float(min_dist_in_cell))
        self.flat = max_points_in_cell > 0

    def insert(self, points, intensities=None):
        p = _f64(points, 3)
        i = None if intensities is None else _f64(intensities)
        lib().orc_int_map_insert(self.h, _d(p), _d(i), len(p))

    def export(self):
        """Gaussian map: (coords V x 3, intensities V).  Flat map: (coords, counts V, points P x 3, intensities P)."""
        V, P = lib().orc_int_map_num_voxels(self.h), lib().orc_int_map_num_points(self.h)
        coords = np.zeros((V, 3), dtype=np.int32)
        if not self.flat:
            ints = np.zeros(V)
            lib().orc_int_map_export(self.h, coords.ctypes.data_as(_ip), _d(ints), None, None, None)
            return coords, ints
        counts, pts, ints = np.zeros(V, dtype=np.int32), np.zeros((P, 3)), np.zeros(P)
        lib().orc_int_map_export(self.h, coords.ctypes.data_as(_ip), None, counts.ctypes.data_as(_ip), _d(pts), _d(ints))
        return coords, counts, pts, ints

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_int_map_destroy(self.h)
            self.h = None


def voxelgrid(points, intensities, resolution):
    """Per voxel (ascending key order) the mean of its kept points' intensities, summed in caller order."""
    p, i = _f64(points, 3), _f64(intensities)
    out = np.zeros(max(len(p), 1))
    m = lib().orc_int_voxelgrid(float(resolution), _d(p), _d(i), len(p), _d(out))
    return out[:m].copy()


def merge_frames(key_points, intensities, resolution):
    """Per voxel (ascending key order) the maximum from 0.0 of its points' intensities; key_points: the points in the first frame's
    coordinates."""
    p, i = _f64(key_points, 3), _f64(intensities)
    out = np.zeros(len(p) + 1)
    m = lib().orc_int_merge_frames(float(resolution), _d(p), _d(i), len(p), _d(out))
    return out[:m].copy()
