"""ctypes binding of tests/occupancy_oracle.cpp, the CPU restatement of the reference's FastOccupancyGrid and VoxelRaycaster -- TEST
INFRASTRUCTURE ONLY.  The library is compiled on first use by tests/native.py with the CPU oracles' flags."""
import ctypes as C
import functools
import os

import numpy as np

import native

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "occupancy_oracle.cpp")
_dp, _vp, _u8p, _u64p, _i32p = C.POINTER(C.c_double), C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint64), C.POINTER(C.c_int32)


@functools.cache
def lib():
    L = native.shared_library([SRC], native.ORACLE_FLAGS)
    for name, res, args in (
        ("orc_grid_new", _vp, [C.c_double]),
        ("orc_grid_free", None, [_vp]),
        ("orc_grid_insert", None, [_vp, _dp, C.c_size_t, _dp]),
        ("orc_grid_overlap", C.c_uint64, [_vp, _dp, C.c_size_t, _dp, _u8p]),
        ("orc_grid_free_rays", None, [_vp, _dp, C.c_size_t, _dp]),
        ("orc_grid_num_cells", C.c_uint64, [_vp]),
        ("orc_grid_table_size", C.c_uint64, [_vp]),
        ("orc_grid_download", None, [_vp, _i32p]),
        ("orc_raycast", None, [_dp, _dp, C.c_size_t, C.c_double, _u64p, _i32p]),
        ("orc_naive_ray", C.c_size_t, [_dp, _dp, C.c_double, _i32p, C.c_size_t]),
        ("orc_reference_test_rays", None, [_dp, _dp]),
    ):
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return L


def _pts(points):
    p = np.ascontiguousarray(np.asarray(points, dtype=np.float64).reshape(-1, 3))
    return p, (p if len(p) else np.zeros((1, 3)))


def _pose(T):
    return None if T is None else np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(16))


class Grid:
    """The oracle FastOccupancyGrid(resolution)."""

    def __init__(self, resolution):
        self.h = lib().orc_grid_new(float(resolution))

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_grid_free(self.h)
            self.h = None

    def insert(self, points, T=None):
        p, buf = _pts(points)
        T = _pose(T)
        lib().orc_grid_insert(self.h, buf.ctypes.data_as(_dp), len(p), None if T is None else T.ctypes.data_as(_dp))

    def free_rays(self, points, T=None):
        p, buf = _pts(points)
        T = _pose(T)
        lib().orc_grid_free_rays(self.h, buf.ctypes.data_as(_dp), len(p), None if T is None else T.ctypes.data_as(_dp))

    def overlaps(self, points, T=None):
        """(count, flags) of the points posed by T."""
        p, buf = _pts(points)
        T = _pose(T)
        flags = np.zeros(max(len(p), 1), dtype=np.uint8)
        c = lib().orc_grid_overlap(self.h, buf.ctypes.data_as(_dp), len(p), None if T is None else T.ctypes.data_as(_dp), flags.ctypes.data_as(_u8p))
        return int(c), flags[: len(p)].copy()

    def num_occupied_cells(self):
        return int(lib().orc_grid_num_cells(self.h))

    def table_size(self):
        return int(lib().orc_grid_table_size(self.h))

    def cells(self):
        out = np.zeros((max(self.num_occupied_cells(), 1), 3), dtype=np.int32)
        lib().orc_grid_download(self.h, out.ctypes.data_as(_i32p))
        return out[: self.num_occupied_cells()].copy()


def raycast(starts, ends, voxel_size):
    """(offsets, coords) of VoxelRaycaster over every row, as b2_raycast returns them."""
    s, sb = _pts(starts)
    e, eb = _pts(ends)
    n = len(s)
    off = np.zeros(n + 1, dtype=np.uint64)
    lib().orc_raycast(sb.ctypes.data_as(_dp), eb.ctypes.data_as(_dp), n, float(voxel_size), off.ctypes.data_as(_u64p), None)
    coords = np.zeros((max(int(off[n]), 1), 3), dtype=np.int32)
    lib().orc_raycast(sb.ctypes.data_as(_dp), eb.ctypes.data_as(_dp), n, float(voxel_size), off.ctypes.data_as(_u64p), coords.ctypes.data_as(_i32p))
    return off, coords[: int(off[n])].copy()


def naive_ray(start, end, voxel_size):
    """The reference test's naive_ray_traversal: voxels visited by 1e-4 steps, end voxel excluded."""
    s = np.ascontiguousarray(start, dtype=np.float64)
    e = np.ascontiguousarray(end, dtype=np.float64)
    m = lib().orc_naive_ray(s.ctypes.data_as(_dp), e.ctypes.data_as(_dp), float(voxel_size), None, 0)
    out = np.zeros((max(m, 1), 3), dtype=np.int32)
    lib().orc_naive_ray(s.ctypes.data_as(_dp), e.ctypes.data_as(_dp), float(voxel_size), out.ctypes.data_as(_i32p), m)
    return out[:m].copy()


def reference_test_rays():
    """The reference test's rays as it draws them: RandomTest's 125 (5 resolutions x 25) and CornerTest's 200, each n x 6 (start, end)."""
    rnd, corner = np.zeros((125, 6)), np.zeros((200, 6))
    lib().orc_reference_test_rays(rnd.ctypes.data_as(_dp), corner.ctypes.data_as(_dp))
    return rnd, corner
