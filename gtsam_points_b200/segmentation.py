"""Segmentation on the device: region growing over a device cloud with normals.

Names follow the reference (paths relative to its root):
  RegionGrowingParams    include/gtsam_points/segmentation/region_growing.hpp (defaults: 0.5, 10 degrees, 0.5, 1000000, 1000000)
  region_growing_init    segmentation/impl/region_growing_impl.hpp
  region_growing_update  segmentation/impl/region_growing_impl.hpp
  MinCutParams           include/gtsam_points/segmentation/min_cut.hpp (defaults: 0.25, 10 degrees, 0.2, 3.0, 0.2, 0.2, 20)
  min_cut                segmentation/impl/min_cut_impl.hpp
The whole visit order is computed on the device when the context is created; update() reveals it step by step exactly as the
reference's steps would, converged flag and dilation included.  See b2_region_growing_create in include/b2points.h for the
arithmetic and the differences from the reference.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np

from . import capi
from .types import KdTree, PointCloud


@dataclass
class RegionGrowingParams:
    distance_threshold: float = 0.5
    angle_threshold: float = 10.0 * math.pi / 180.0
    dilation_radius: float = 0.5
    max_cluster_size: int = 1000000
    max_steps: int = 1000000

    def _fixed(self):
        """The parameters the visit order depends on: all but max_steps."""
        return (float(self.distance_threshold), float(self.angle_threshold), float(self.dilation_radius), int(self.max_cluster_size))


class RegionGrowing:
    """RegionGrowingContext on the device (b2_region_growing).  The parameters other than max_steps are fixed at init()."""

    def __init__(self, h, params: RegionGrowingParams):
        self.h, self.params = h, params

    @classmethod
    def init(cls, cloud: PointCloud, seed_point, params: RegionGrowingParams | None = None, tree: KdTree | None = None) -> "RegionGrowing":
        """region_growing_init: the cloud must carry normals; tree None builds one, else a KdTree.from_cloud(cloud)."""
        params = params or RegionGrowingParams()
        seed = np.ascontiguousarray(np.asarray(seed_point, dtype=np.float64).reshape(-1)[:3])
        if seed.size != 3:
            raise ValueError("seed_point needs 3 coordinates")
        d, a, r, m = params._fixed()
        h = C.c_void_p()
        capi.check(capi.lib().b2_region_growing_create(cloud.h, None if tree is None else tree.h, capi.dptr(seed), d, a, r, m, C.byref(h)))
        return cls(h, RegionGrowingParams(d, a, r, m, int(params.max_steps)))

    def update(self, params: RegionGrowingParams | int | None = None) -> bool:
        """region_growing_update: at most max_steps steps (params.max_steps, an int, or the init params' max_steps); True when the
        queue is empty.  Parameters other than max_steps that differ from init's raise B2Error (B2_ERR_INVALID_ARGUMENT)."""
        if params is None:
            steps = self.params.max_steps
        elif isinstance(params, RegionGrowingParams):
            if params._fixed() != self.params._fixed():
                raise capi.B2Error(1, "region_growing_update: only max_steps may change after init (the visit order depends on the others)")
            steps = params.max_steps
        else:
            steps = params
        conv = C.c_int32(0)
        capi.check(capi.lib().b2_region_growing_update(self.h, max(min(int(steps), 2**31 - 1), -(2**31)), C.byref(conv)))
        return bool(conv.value)

    @property
    def cluster_indices(self) -> np.ndarray:
        """The cluster: visited points in visit order, or the dilation set in ascending order once it has run (int64)."""
        size = C.c_uint64(0)
        capi.check(capi.lib().b2_region_growing_get(self.h, C.byref(size), None))
        out = np.zeros(max(size.value, 1), dtype=np.int64)
        capi.check(capi.lib().b2_region_growing_get(self.h, C.byref(size), out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out[: size.value].copy()

    def __del__(self):
        try:
            if getattr(self, "h", None):
                capi.lib().b2_region_growing_destroy(self.h)
                self.h = None
        except Exception:
            pass


def region_growing_init(cloud: PointCloud, seed_point, params: RegionGrowingParams | None = None, tree: KdTree | None = None) -> RegionGrowing:
    return RegionGrowing.init(cloud, seed_point, params, tree)


def region_growing_update(context: RegionGrowing, params: RegionGrowingParams | int | None = None) -> bool:
    return context.update(params)


@dataclass
class MinCutParams:
    distance_sigma: float = 0.25
    angle_sigma: float = 10.0 * math.pi / 180.0
    foreground_mask_radius: float = 0.2
    background_mask_radius: float = 3.0
    foreground_weight: float = 0.2
    background_weight: float = 0.2
    k_neighbors: int = 20


@dataclass
class MinCutResult:
    source_index: int = -1
    sink_index: int = -1
    max_flow: float = 0.0
    max_flow_q: int = 0  # the maximum flow in capacity quanta of 2^-32
    flags: int = 0  # B2_MIN_CUT_NO_SEED / _FEW_NEIGHBORS / _NO_SINK
    cluster_indices: np.ndarray | None = None
    capacities: np.ndarray | None = None  # n x k quantised k-NN capacities, when asked for


def min_cut(cloud: PointCloud, source, params: MinCutParams | None = None, tree: KdTree | None = None, capacities: bool = False) -> MinCutResult:
    """min_cut on a device cloud with normals (b2_min_cut): source is a point index (int) or a seed point (3 coordinates, its nearest
    point is the source).  The cluster is the minimal minimum-cut source set, ascending."""
    p = params or MinCutParams()
    cp = capi.MinCutParamsC(float(p.distance_sigma), float(p.angle_sigma), float(p.foreground_mask_radius), float(p.background_mask_radius), float(p.foreground_weight),
                            float(p.background_weight), int(p.k_neighbors), 0)
    n = int(cloud.info().num_points)
    out = np.zeros(max(n, 1), dtype=np.int64)
    caps = np.zeros(max(n * max(int(p.k_neighbors), 1), 1), dtype=np.int64) if capacities else None
    res = capi.MinCutResultC()
    if isinstance(source, (int, np.integer)):
        idx, seed = int(source), None
    else:
        idx, seed = -1, np.ascontiguousarray(np.asarray(source, dtype=np.float64).reshape(-1)[:3])
    lp = C.POINTER(C.c_int64)
    capi.check(capi.lib().b2_min_cut(cloud.h, None if tree is None else tree.h, idx, None if seed is None else capi.dptr(seed), C.byref(cp), C.byref(res),
                                     out.ctypes.data_as(lp), None if caps is None else caps.ctypes.data_as(lp)))
    return MinCutResult(int(res.source_index), int(res.sink_index), float(res.max_flow), int(res.max_flow_q), int(res.flags), out[: res.cluster_size].copy(),
                        None if caps is None else caps[: n * int(p.k_neighbors)].reshape(n, int(p.k_neighbors)))
