"""Occupancy grid and voxel ray traversal on the device.

Names follow the reference (paths relative to its root):
  FastOccupancyGrid  include/gtsam_points/ann/fast_occupancy_grid.hpp, ann/impl/fast_occupancy_grid_impl.hpp
  raycast            include/gtsam_points/util/voxel_raycaster.hpp (VoxelRaycaster, begin() up to end_voxel() excluded)
The grid takes device clouds (PointCloud) and 4x4 poses; see b2_occgrid_* and b2_raycast in include/b2points.h for the keying, the
ray arithmetic and the differences from the reference.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .types import Context, PointCloud, _pose16, default_context

_u64p, _u8p, _i32p = C.POINTER(C.c_uint64), C.POINTER(C.c_uint8), C.POINTER(C.c_int32)


class FastOccupancyGrid:
    """FastOccupancyGrid(resolution) on the device (b2_occgrid).  Poses are 4x4 (None: the stored points as they are)."""

    def __init__(self, resolution: float, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self.h = None
        h = C.c_void_p()
        capi.check(capi.lib().b2_occgrid_create(self.ctx.h, float(resolution), C.byref(h)))
        self.h = h

    def info(self) -> capi.OccGridInfo:
        info = capi.OccGridInfo()
        capi.check(capi.lib().b2_occgrid_get_info(self.h, C.byref(info)))
        return info

    @property
    def resolution(self) -> float:
        return float(self.info().resolution)

    def insert(self, points: PointCloud, pose=None):
        """insert(points, pose): the cells of the posed points become occupied."""
        T = _pose16(pose)
        capi.check(capi.lib().b2_occgrid_insert(self.h, points.h, None if T is None else capi.dptr(T)))

    def free_rays(self, points: PointCloud, pose=None):
        """Clears every occupied cell crossed by a ray from the pose's translation to a posed point, end voxels excluded (set_free along
        VoxelRaycaster).  The usual scan update is free_rays(scan, pose) then insert(scan, pose)."""
        T = _pose16(pose)
        capi.check(capi.lib().b2_occgrid_free_rays(self.h, points.h, None if T is None else capi.dptr(T)))

    def _overlap(self, points: PointCloud, poses, flags: bool):
        if poses is None:
            Ts, m = None, 1
        else:
            Ts = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(-1, 16))
            m = len(Ts)
        counts = np.zeros(max(m, 1), dtype=np.uint64)
        n = points.size()
        out = np.zeros((m, n), dtype=np.uint8) if flags else None
        capi.check(
            capi.lib().b2_occgrid_overlap(self.h, points.h, None if Ts is None else capi.dptr(Ts), m, counts.ctypes.data_as(_u64p),
                                          None if out is None else out.ctypes.data_as(_u8p))
        )
        return counts[:m], out

    def calc_overlap(self, points: PointCloud, pose=None) -> int:
        """The number of posed points whose cell is occupied."""
        return int(self._overlap(points, None if pose is None else [pose], False)[0][0])

    def calc_overlap_rate(self, points: PointCloud, pose=None) -> float:
        """calc_overlap / n in double; 0 for an empty cloud (the reference gives 0 / 0)."""
        n = points.size()
        return self.calc_overlap(points, pose) / float(n) if n else 0.0

    def get_overlaps(self, points: PointCloud, pose=None) -> np.ndarray:
        """Per point (caller order) 1 if its posed cell is occupied, else 0 (uint8)."""
        return self._overlap(points, None if pose is None else [pose], True)[1][0]

    def calc_overlaps(self, points: PointCloud, poses, flags: bool = False):
        """calc_overlap under every pose of `poses` (m x 4 x 4) in one launch: the m counts (uint64), and with flags=True also the
        m x n per-point flags."""
        counts, out = self._overlap(points, poses, flags)
        return (counts, out) if flags else counts

    def num_occupied_cells(self) -> int:
        return int(self.info().num_occupied_cells)

    def occupied_cells(self) -> np.ndarray:
        """The occupied cells' integer coordinates (int32, k x 3) in ascending key order: z, then y, then x."""
        out = np.zeros((self.num_occupied_cells(), 3), dtype=np.int32)
        capi.check(capi.lib().b2_occgrid_download(self.h, out.ctypes.data_as(_i32p) if len(out) else None))
        return out

    def __del__(self):
        try:
            if getattr(self, "h", None):
                capi.lib().b2_occgrid_destroy(self.h)
                self.h = None
        except Exception:
            pass


def raycast(starts, ends, voxel_size: float, ctx: Context | None = None):
    """VoxelRaycaster(start_i, end_i, voxel_size) for every row: (offsets (n + 1, uint64), coords (offsets[n] x 3, int32)); row i is
    coords[offsets[i]:offsets[i + 1]], the voxels from begin() up to, not including, end_voxel()."""
    ctx = ctx or default_context()
    s = np.ascontiguousarray(np.asarray(starts, dtype=np.float64).reshape(-1, 3))
    e = np.ascontiguousarray(np.asarray(ends, dtype=np.float64).reshape(-1, 3))
    if s.shape != e.shape:
        raise ValueError("raycast: starts and ends differ in shape")
    n = len(s)
    off = np.zeros(n + 1, dtype=np.uint64)
    sp, ep = (capi.dptr(s), capi.dptr(e)) if n else (None, None)
    L = capi.lib()
    capi.check(L.b2_raycast(ctx.h, sp, ep, n, float(voxel_size), off.ctypes.data_as(_u64p), 0, None))
    total = int(off[n])
    coords = np.zeros((total, 3), dtype=np.int32)
    if total:
        capi.check(L.b2_raycast(ctx.h, sp, ep, n, float(voxel_size), off.ctypes.data_as(_u64p), total, coords.ctypes.data_as(_i32p)))
    return off, coords
