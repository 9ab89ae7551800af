"""Host-side mirrors of the reference's data types for the scan-matching path.

Names and argument meaning follow the reference (paths relative to its root):
  PointCloud            include/gtsam_points/types/point_cloud.hpp:19-119 (+ PointCloudCPU / PointCloudGPU)
  GaussianVoxelMapGPU   include/gtsam_points/types/gaussian_voxelmap_gpu.hpp:39-108
  KdTree                include/gtsam_points/ann/kdtree.hpp, ann/nearest_neighbor_search.hpp:16-57
  iVox                  include/gtsam_points/ann/ivox.hpp (IncrementalVoxelMap<FlatContainer>, ann/incremental_voxelmap.hpp)
  iVoxCovarianceEstimation  include/gtsam_points/ann/ivox_covariance_estimation.hpp (IncrementalCovarianceVoxelMap)
All device work goes through the C ABI (include/b2points.h); nothing here computes on the CPU.
"""
from __future__ import annotations

import ctypes as C
import threading

import numpy as np

from . import capi

_ctx_lock = threading.Lock()
_default_ctx = {}


class Context:
    """Device + stream (b2_ctx).  `stream` is an integer cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream) or None."""

    def __init__(self, device: int = 0, stream: int | None = None):
        h = C.c_void_p()
        capi.check(capi.lib().b2_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(h)))
        self.h = h
        self.device = device

    def synchronize(self):
        capi.check(capi.lib().b2_ctx_synchronize(self.h))

    @property
    def stream(self) -> int:
        return capi.lib().b2_ctx_stream(self.h) or 0

    def close(self):
        if getattr(self, "h", None):
            capi.lib().b2_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def default_context(device: int = 0) -> Context:
    with _ctx_lock:
        if device not in _default_ctx:
            _default_ctx[device] = Context(device)
        return _default_ctx[device]


def current_access_time() -> int:
    """OffloadableGPU::current_access_time: the process-wide access clock that touch() advances."""
    out = C.c_uint64()
    capi.check(capi.lib().b2_access_time_current(C.byref(out)))
    return out.value


class OffloadableGPU:
    """OffloadableGPU (include/gtsam_points/types/offloadable.hpp): the device copy can be moved to pinned host memory
    (offload_gpu) and back (reload_gpu), and touch() records an access and reloads if needed.  Each returns whether it moved
    anything.  While offloaded, calls that read the device copy raise B2Error (B2_ERR_INVALID_STATE) -- except overlap_gpu and
    factor launches with set_enable_offloading(True), which touch what they read.  Which objects to offload is the caller's
    choice; nothing is evicted automatically."""

    _residency_api = ""  # the C ABI prefix of the handle: b2_cloud / b2_voxelmap

    def _residency_call(self, op: str) -> bool:
        changed = C.c_int32()
        capi.check(getattr(capi.lib(), f"{self._residency_api}_{op}")(self.h, C.byref(changed)))
        return bool(changed.value)

    def offload_gpu(self) -> bool:
        return self._residency_call("offload")

    def reload_gpu(self) -> bool:
        return self._residency_call("reload")

    def touch(self) -> bool:
        return self._residency_call("touch")

    def residency(self) -> capi.Residency:
        out = capi.Residency()
        capi.check(getattr(capi.lib(), f"{self._residency_api}_residency")(self.h, C.byref(out)))
        return out

    def loaded_on_gpu(self) -> bool:
        return bool(self.residency().loaded_on_gpu)

    def last_accessed_time(self) -> int:
        return int(self.residency().last_access)

    def memory_usage_gpu(self) -> int:
        """Device bytes the object holds now: 0 while offloaded."""
        return int(self.residency().device_bytes)


class PointCloud(OffloadableGPU):
    """Points (N x 3 or N x 4 float64) with optional covariances (N x 3 x 3 or N x 4 x 4 float64), normals (N x 3 or N x 4) and
    intensities (N).

    The device copy (`points_gpu` / `covs_gpu` / `normals_gpu` / `intensities_gpu` in the reference) is created on construction.
    flags: capi.B2_CLOUD_* (default lossless storage, Morton-ordered on the device).
    """

    _residency_api = "b2_cloud"

    def __init__(self, points, covs=None, ctx: Context | None = None, flags: int = capi.B2_CLOUD_DEFAULT, normals=None, intensities=None):
        self.ctx = ctx or default_context()
        self.intensities = None if intensities is None else np.ascontiguousarray(intensities, dtype=np.float64)
        if self.intensities is not None and (self.intensities.ndim != 1 or len(self.intensities) != len(points)):
            raise ValueError("intensities must be N values, one per point")
        self.normals = None if normals is None else np.ascontiguousarray(normals, dtype=np.float64)
        if self.normals is not None and (self.normals.ndim != 2 or self.normals.shape[1] not in (3, 4) or len(self.normals) != len(points)):
            raise ValueError("normals must be N x 3 or N x 4, one per point")
        self._device_normals = self.normals  # the array the device copy was made from (None: the device has no normals)
        self.points = np.ascontiguousarray(points, dtype=np.float64)
        if self.points.ndim != 2 or self.points.shape[1] not in (3, 4):
            raise ValueError("points must be N x 3 or N x 4")
        self.covs = None
        cov_stride = 0
        if covs is not None:
            covs = np.ascontiguousarray(covs, dtype=np.float64)
            if covs.shape[1:] == (3, 3):
                cov_stride = 9
            elif covs.shape[1:] == (4, 4):
                cov_stride = 16
            else:
                raise ValueError("covs must be N x 3 x 3 or N x 4 x 4")
            if len(covs) != len(self.points):
                raise ValueError("points / covs size mismatch")
            self.covs = covs
        h = C.c_void_p()
        capi.check(
            capi.lib().b2_cloud_create_with_intensities(
                self.ctx.h, capi.dptr(self.points), self.points.shape[1], capi.dptr(self.covs) if self.covs is not None else None, cov_stride,
                capi.dptr(self.normals) if self.normals is not None else None, 0 if self.normals is None else self.normals.shape[1],
                None if self.intensities is None else capi.dptr(self.intensities), len(self.points), flags, C.byref(h)
            )
        )
        self.h = h

    @classmethod
    def _from_handle(cls, h, ctx: Context) -> "PointCloud":
        """Wraps a device cloud the library created (voxel grid, estimation): .points / .covs / .normals / .intensities are its stored
        values in caller order (b2_cloud_download), so every consumer of a PointCloud takes it as it is."""
        self = cls.__new__(cls)
        self.ctx, self.h = ctx, h
        info = self.info()
        n = int(info.num_points)
        self.points = np.zeros((n, 3))
        self.covs = np.zeros((n, 3, 3)) if info.cov_bytes else None
        self.normals = np.zeros((n, 3)) if info.normal_bytes else None
        capi.check(capi.lib().b2_cloud_download(h, capi.dptr(self.points), None if self.covs is None else capi.dptr(self.covs), None if self.normals is None else capi.dptr(self.normals)))
        self._device_normals = self.normals
        self.intensities = self.intensities_gpu() if self.intensity_bytes() else None
        return self

    def estimated(self, k_neighbors: int = 10, eigen_values=(1e-3, 1.0, 1.0), normals: bool = False, tree: "KdTree | None" = None,
                  flags: int = capi.B2_CLOUD_DEFAULT) -> "PointCloud":
        """A new device cloud with these points and the covariances of estimate_covariances over them (features/covariance_estimation.cpp:
        18-77), with normals=True also the normals of estimate_normals from the same neighbour search; the points never leave the
        device; intensities, if the cloud has them, are kept.  tree: None builds one; else a KdTree.from_cloud(self).  flags pick the
        storage of the estimated arrays and of the intensities."""
        ev = np.ascontiguousarray(eigen_values, dtype=np.float64)
        h = C.c_void_p()
        capi.check(capi.lib().b2_cloud_create_estimated(self.h, None if tree is None else tree.h, int(k_neighbors), capi.dptr(ev), 1 if normals else 0, flags, C.byref(h)))
        return PointCloud._from_handle(h, self.ctx)

    def size(self) -> int:
        return len(self.points)

    def __len__(self):
        return len(self.points)

    def has_points(self):
        return True

    def has_covs(self):
        return self.covs is not None

    def has_normals(self):
        return self.normals is not None

    def normals_gpu(self) -> np.ndarray:
        """The normals as stored on the device (after any float32 rounding), N x 3 in the caller's order."""
        out = np.zeros((len(self.points), 3))
        capi.check(capi.lib().b2_cloud_download_normals(self.h, capi.dptr(out)))
        return out

    def has_intensities(self):
        return self.intensities is not None

    def intensity_bytes(self) -> int:
        """Storage of the device copy's intensities: 4 or 8 bytes, 0 = none."""
        out = C.c_int()
        capi.check(capi.lib().b2_cloud_intensity_bytes(self.h, C.byref(out)))
        return out.value

    def intensities_gpu(self) -> np.ndarray:
        """The intensities as stored on the device (after any float32 rounding), N values in the caller's order."""
        out = np.zeros(len(self.points))
        capi.check(capi.lib().b2_cloud_download_intensities(self.h, capi.dptr(out)))
        return out

    def info(self) -> capi.CloudInfo:
        info = capi.CloudInfo()
        capi.check(capi.lib().b2_cloud_get_info(self.h, C.byref(info)))
        return info

    def __del__(self):
        try:
            if getattr(self, "h", None):
                capi.lib().b2_cloud_destroy(self.h)
                self.h = None
        except Exception:
            pass


class GaussianVoxelMapGPU(OffloadableGPU):
    """Gaussian voxel map on the device with the CPU map's index semantics (first-touch ids, exact lookups)."""

    _residency_api = "b2_voxelmap"

    # The device map is made by the first insert (or set_lru / touch).  Until then the map holds no device memory, so offload_gpu /
    # reload_gpu move nothing, and last_accessed_time() is the clock's value at construction (the reference's creation stamp); the
    # device map, once made, records the clock's value at its own creation, as every new device object does.  touch() makes the
    # device map, so that it has an object to record the access on.
    def _residency_call(self, op: str) -> bool:
        if op == "touch":
            self._ensure()
        if self.h is None:
            return False
        return super()._residency_call(op)

    def residency(self) -> capi.Residency:
        if self.h is None:
            return capi.Residency(loaded_on_gpu=1, last_access=self._created_at)
        return super().residency()

    def __init__(self, resolution: float, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self._resolution = float(resolution)
        self.h = None
        self._lru = None
        self._created_at = current_access_time()

    def voxel_resolution(self) -> float:
        return self._resolution

    def insert(self, frame: PointCloud):
        """GaussianVoxelMap::insert(const PointCloud&).  The first call builds the map; further calls are incremental with the
        CPU map's semantics (IncrementalVoxelMap::insert + LRU eviction, ann/impl/incremental_voxelmap_impl.hpp:31-68) -- the
        reference's own GPU map is one-shot only (types/gaussian_voxelmap_gpu.hpp:63).  The frame's intensities, if it has them,
        raise each voxel's intensity to their maximum (voxel_intensities())."""
        if frame.covs is None:
            raise ValueError("GaussianVoxelMapGPU.insert: the frame has no covariances")
        cov_stride = 9 if frame.covs.shape[1:] == (3, 3) else 16
        self._ensure()
        ints = getattr(frame, "intensities", None)
        capi.check(capi.lib().b2_voxelmap_insert_with_intensities(self.h, capi.dptr(frame.points), frame.points.shape[1], capi.dptr(frame.covs), cov_stride,
                                                                  None if ints is None else capi.dptr(ints), len(frame.points)))

    def insert_cloud(self, cloud: PointCloud, T=None):
        """insert() of a device cloud posed by T (map <- frame 4x4; None: as stored) without a host copy: the map afterwards equals
        insert() of the cloud's stored values posed as transform_gpu() poses them (b2_voxelmap_insert_cloud).  The cloud must have
        covariances."""
        self._ensure()
        T16 = _pose16(T)
        capi.check(capi.lib().b2_voxelmap_insert_cloud(self.h, cloud.h, None if T16 is None else capi.dptr(T16)))

    def _ensure(self):
        if self.h is None:
            h = C.c_void_p()
            capi.check(capi.lib().b2_voxelmap_create(self.ctx.h, self._resolution, C.byref(h)))
            self.h = h
            if self._lru is not None:
                capi.check(capi.lib().b2_voxelmap_set_lru(self.h, *self._lru))

    def set_lru(self, lru_horizon: int, lru_clear_cycle: int):
        """IncrementalVoxelMap::set_lru_horizon / set_lru_clear_cycle (ann/incremental_voxelmap.hpp); defaults 10 / 10."""
        self._lru = (int(lru_horizon), int(lru_clear_cycle))
        if self.h is not None:
            capi.check(capi.lib().b2_voxelmap_set_lru(self.h, *self._lru))

    def save_compact(self, path):
        """GaussianVoxelMapCPU::save_compact wire format (src/gtsam_points/types/gaussian_voxelmap_cpu.cpp:79-97)."""
        capi.check(capi.lib().b2_voxelmap_save_compact(self.h, str(path).encode()))

    @classmethod
    def load(cls, path, ctx: Context | None = None):
        """GaussianVoxelMapCPU::load / GaussianVoxelMapGPU::load: reads a save_compact file onto the device."""
        ctx = ctx or default_context()
        h = C.c_void_p()
        capi.check(capi.lib().b2_voxelmap_load(ctx.h, str(path).encode(), C.byref(h)))
        self = cls(1.0, ctx)
        self.h = h
        self._resolution = float(self.info().resolution)
        return self

    @classmethod
    def from_voxels(cls, resolution, coords, means, covs, num_points=None, ctx: Context | None = None, intensities=None):
        """Upload an existing map (e.g. the contents of a GaussianVoxelMapCPU); ids = the given order.  intensities: each voxel's
        intensity (None: 0)."""
        self = cls(resolution, ctx)
        coords = np.ascontiguousarray(coords, dtype=np.int32)
        means = np.ascontiguousarray(means, dtype=np.float64)
        covs = np.ascontiguousarray(covs, dtype=np.float64).reshape(len(coords), 9)
        npts = None if num_points is None else np.ascontiguousarray(num_points, dtype=np.int32)
        ints = None if intensities is None else np.ascontiguousarray(intensities, dtype=np.float64)
        if ints is not None and ints.shape != (len(coords),):
            raise ValueError("intensities must hold one value per voxel")
        h = C.c_void_p()
        capi.check(
            capi.lib().b2_voxelmap_create_from_voxels_with_intensities(
                self.ctx.h, float(resolution), coords.ctypes.data_as(C.POINTER(C.c_int32)), capi.dptr(means), capi.dptr(covs), None if npts is None else npts.ctypes.data_as(C.POINTER(C.c_int32)),
                None if ints is None else capi.dptr(ints), len(coords), C.byref(h)
            )
        )
        self.h = h
        return self

    def info(self) -> capi.VoxelMapInfo:
        info = capi.VoxelMapInfo()
        capi.check(capi.lib().b2_voxelmap_get_info(self.h, C.byref(info)))
        return info

    @property
    def num_voxels(self) -> int:
        return int(self.info().num_voxels)

    def download(self):
        """download_voxel_means / _covs / _num_points + voxel coordinates, in id order."""
        V = self.num_voxels
        coords = np.zeros((V, 3), dtype=np.int32)
        means = np.zeros((V, 3))
        covs = np.zeros((V, 3, 3))
        n = np.zeros(V, dtype=np.int32)
        capi.check(capi.lib().b2_voxelmap_download(self.h, coords.ctypes.data_as(C.POINTER(C.c_int32)), capi.dptr(means), capi.dptr(covs), n.ctypes.data_as(C.POINTER(C.c_int32))))
        return dict(coords=coords, means=means, covs=covs, n=n, resolution=self._resolution)

    def voxel_intensities(self) -> np.ndarray:
        """Each voxel's intensity in id order: the maximum, from 0.0, of the intensities of the points inserted into it
        (GaussianVoxel::intensity); all 0 for a map that never received intensities."""
        out = np.zeros(self.num_voxels)
        capi.check(capi.lib().b2_voxelmap_download_intensities(self.h, capi.dptr(out)))
        return out

    def lookup_voxel_index(self, points) -> np.ndarray:
        """voxel_coord + lookup_voxel_index for a batch of points; -1 where no voxel exists."""
        p = np.ascontiguousarray(points, dtype=np.float64)
        out = np.zeros(len(p), dtype=np.int32)
        capi.check(capi.lib().b2_voxelmap_lookup(self.h, capi.dptr(p), p.shape[1], len(p), out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def __del__(self):
        try:
            if getattr(self, "h", None):
                capi.lib().b2_voxelmap_destroy(self.h)
                self.h = None
        except Exception:
            pass


class iVox:
    """Incremental point voxel map on the device (iVox = IncrementalVoxelMap<FlatContainer>): the frame-to-map odometry target.

    insert() keeps up to max_num_points_in_cell points per voxel, at least min_dist_in_cell apart, in first-touch voxels and evicts
    voxels untouched for lru_horizon inserts every lru_clear_cycle inserts; knn_search() searches the neighbour voxels of the
    query (neighbor_voxel_mode 1 / 7 / 19 / 27).  Ids, slot contents and search results equal the reference's CPU container."""

    _create = "b2_ivox_create"  # the C entry point that makes the handle (a subclass names its own)

    def __init__(self, voxel_resolution: float, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self._resolution = float(voxel_resolution)
        h = C.c_void_p()
        capi.check(getattr(capi.lib(), self._create)(self.ctx.h, self._resolution, C.byref(h)))
        self.h = h
        self._min_dist, self._max_points = 0.1, 20

    def voxel_resolution(self) -> float:
        return self._resolution

    def insert(self, frame, covs=None, intensities=None):
        """IncrementalVoxelMap::insert(const PointCloud&) (ann/impl/incremental_voxelmap_impl.hpp:31-68).  `frame`: a PointCloud, or
        an N x 3 / N x 4 array with optional N x 3 x 3 / N x 4 x 4 `covs` and N `intensities`; covariances and intensities are
        stored with the points when given (all inserts into one map must agree on each)."""
        pts = frame.points if isinstance(frame, PointCloud) else np.ascontiguousarray(frame, dtype=np.float64)
        if isinstance(frame, PointCloud):
            covs, intensities = frame.covs, frame.intensities
        else:
            if covs is not None:
                covs = np.ascontiguousarray(covs, dtype=np.float64)
            if intensities is not None:
                intensities = np.ascontiguousarray(intensities, dtype=np.float64)
                if intensities.shape != (len(pts),):
                    raise ValueError("intensities must be N values, one per point")
        cov_stride = 0 if covs is None else (9 if covs.shape[1:] == (3, 3) else 16)
        capi.check(capi.lib().b2_ivox_insert_with_intensities(self.h, capi.dptr(pts), pts.shape[1], capi.dptr(covs) if covs is not None else None, cov_stride,
                                                              None if intensities is None else capi.dptr(intensities), len(pts)))

    def insert_cloud(self, cloud: PointCloud, T=None):
        """insert() of a device cloud posed by T (map <- frame 4x4; None: as stored) without a host copy -- the map update of
        frame-to-map odometry (advanced_scan_matching.cpp:84-95) in one call.  The map afterwards equals insert() of the cloud's
        stored values posed as transform_gpu() poses them (b2_ivox_insert_cloud); its covariances and intensities go in iff it has them."""
        T16 = _pose16(T)
        capi.check(capi.lib().b2_ivox_insert_cloud(self.h, cloud.h, None if T16 is None else capi.dptr(T16)))

    def clear(self):
        capi.check(capi.lib().b2_ivox_clear(self.h))

    def set_lru_horizon(self, lru_horizon: int):
        self._lru = (int(lru_horizon), getattr(self, "_lru", (10, 10))[1])
        capi.check(capi.lib().b2_ivox_set_lru(self.h, *self._lru))

    def set_lru_clear_cycle(self, lru_clear_cycle: int):
        self._lru = (getattr(self, "_lru", (10, 10))[0], int(lru_clear_cycle))
        capi.check(capi.lib().b2_ivox_set_lru(self.h, *self._lru))

    def set_lru(self, lru_horizon: int, lru_clear_cycle: int):
        self._lru = (int(lru_horizon), int(lru_clear_cycle))
        capi.check(capi.lib().b2_ivox_set_lru(self.h, *self._lru))

    def set_neighbor_voxel_mode(self, mode: int):
        capi.check(capi.lib().b2_ivox_set_neighbor_voxel_mode(self.h, int(mode)))

    def set_min_dist_in_cell(self, dist: float):
        capi.check(capi.lib().b2_ivox_set_insertion_setting(self.h, float(dist), self._max_points))
        self._min_dist = float(dist)

    def set_max_num_points_in_cell(self, num_points: int):
        capi.check(capi.lib().b2_ivox_set_insertion_setting(self.h, self._min_dist, int(num_points)))
        self._max_points = int(num_points)

    def info(self) -> capi.IvoxInfo:
        info = capi.IvoxInfo()
        capi.check(capi.lib().b2_ivox_get_info(self.h, C.byref(info)))
        return info

    @property
    def num_voxels(self) -> int:
        return int(self.info().num_voxels)

    def size(self) -> int:
        """Number of stored points (frame::size of the iVox)."""
        return int(self.info().num_points)

    def download(self):
        """Voxel coordinates, per-voxel point counts, and the points / covariances in id, then slot order."""
        info = self.info()
        V, P = int(info.num_voxels), int(info.num_points)
        coords = np.zeros((V, 3), dtype=np.int32)
        counts = np.zeros(V, dtype=np.int32)
        points = np.zeros((P, 3))
        covs = np.zeros((P, 3, 3))
        ip = C.POINTER(C.c_int32)
        capi.check(capi.lib().b2_ivox_download(self.h, coords.ctypes.data_as(ip), counts.ctypes.data_as(ip), capi.dptr(points), capi.dptr(covs)))
        return dict(coords=coords, counts=counts, points=points, covs=covs, resolution=self._resolution)

    def voxel_points(self) -> np.ndarray:
        """iVox::voxel_points(): every stored point, voxels in id order, points in slot order (N x 4, w = 1)."""
        p = self.download()["points"]
        return np.concatenate([p, np.ones((len(p), 1))], 1)

    def voxel_intensities(self) -> np.ndarray:
        """iVox::voxel_intensities(): the stored points' intensities in voxel_points() order.  Raises on a map whose points came
        without intensities, and on an iVoxCovarianceEstimation, which keeps none."""
        out = np.zeros(self.size())
        capi.check(capi.lib().b2_ivox_download_intensities(self.h, capi.dptr(out)))
        return out

    def voxel_covs(self) -> np.ndarray:
        """iVox::voxel_covs(): the stored covariances in voxel_points() order (N x 4 x 4)."""
        c = self.download()["covs"]
        out = np.zeros((len(c), 4, 4))
        out[:, :3, :3] = c
        return out

    def knn_search(self, queries, k: int = 1, max_sq_dist: float = np.finfo(np.float64).max):
        """IncrementalVoxelMap::knn_search for a batch of queries: indices voxel_id << 32 | point_id (int64) and squared distances,
        KnnResult order; slots beyond the number found hold (-1, max_sq_dist).  Returns arrays of shape (nq, k)."""
        q = np.ascontiguousarray(queries, dtype=np.float64)
        if q.ndim == 1:
            q = q[None]
        idx = np.zeros((len(q), k), dtype=np.int64)
        sqd = np.zeros((len(q), k))
        capi.check(capi.lib().b2_ivox_knn(self.h, capi.dptr(q), q.shape[1], len(q), int(k), float(max_sq_dist), idx.ctypes.data_as(C.POINTER(C.c_int64)), capi.dptr(sqd)))
        return idx, sqd

    def __del__(self):
        try:
            if getattr(self, "h", None):
                capi.lib().b2_ivox_destroy(self.h)
                self.h = None
        except Exception:
            pass


class iVoxCovarianceEstimation(iVox):
    """iVox that estimates each stored point's covariance and normal from the map's own neighbourhood as frames arrive
    (iVoxCovarianceEstimation = IncrementalCovarianceVoxelMap, include/gtsam_points/ann/incremental_covariance_voxelmap.hpp).

    insert() ignores input covariances.  Points in warm-up, and invalid points on their low-rate turn, are re-estimated from their
    num_neighbors nearest stored points; a point whose eigenvalues pass the running thresholds becomes valid.  knn_search() and the
    GICP factor see valid points only; knn_search_force() sees every stored point.  The pass is include/b2points.h's, step by step;
    its statistics are summed in a fixed blocked order, so set_num_threads() changes nothing."""

    VALID_BIT = 1 << 63
    _create = "b2_ivox_create_covariance_estimation"

    def set_num_neighbors(self, num_neighbors: int):
        capi.check(capi.lib().b2_ivox_set_num_neighbors(self.h, int(num_neighbors)))

    def set_min_num_neighbors(self, min_num_neighbors: int):
        capi.check(capi.lib().b2_ivox_set_min_num_neighbors(self.h, int(min_num_neighbors)))

    def set_warmup_cycles(self, warmup_cycles: int):
        capi.check(capi.lib().b2_ivox_set_warmup_cycles(self.h, int(warmup_cycles)))

    def set_lowrate_cycles(self, lowrate_cycles: int):
        """Must be a power of two; otherwise raises and keeps the old value."""
        capi.check(capi.lib().b2_ivox_set_lowrate_cycles(self.h, int(lowrate_cycles)))

    def set_remove_invalid_age_thresh(self, remove_invalid_age_thresh: int):
        capi.check(capi.lib().b2_ivox_set_remove_invalid_age_thresh(self.h, int(remove_invalid_age_thresh)))

    def set_eig_stddev_thresh_scale(self, eig_stddev_thresh_scale: float):
        capi.check(capi.lib().b2_ivox_set_eig_stddev_thresh_scale(self.h, float(eig_stddev_thresh_scale)))

    def set_num_threads(self, num_threads: int):
        """Accepted for the reference's interface; the device pass has no thread count."""

    def download_state(self):
        """The full state in id, then slot order: coords, counts, points, flags (uint64), normals, covs (3 x 3)."""
        info = self.info()
        V, P = int(info.num_voxels), int(info.num_points)
        coords = np.zeros((V, 3), dtype=np.int32)
        counts = np.zeros(V, dtype=np.int32)
        points, normals, covs = np.zeros((P, 3)), np.zeros((P, 3)), np.zeros((P, 3, 3))
        flags = np.zeros(P, dtype=np.uint64)
        ip = C.POINTER(C.c_int32)
        capi.check(capi.lib().b2_ivox_download_state(self.h, coords.ctypes.data_as(ip), counts.ctypes.data_as(ip), capi.dptr(points),
                                                     flags.ctypes.data_as(C.POINTER(C.c_uint64)), capi.dptr(normals), capi.dptr(covs)))
        return dict(coords=coords, counts=counts, points=points, flags=flags, normals=normals, covs=covs)

    def insert_timings(self) -> dict:
        """Device time (ms, CUDA events) of the last insert's phases: base insert, estimation pass, statistics, removal."""
        ms = np.zeros(4)
        capi.check(capi.lib().b2_ivox_insert_timings(self.h, capi.dptr(ms)))
        return dict(zip(("base_insert", "estimation", "statistics", "removal"), ms.tolist()))

    def eig_stats(self):
        """The ring of eigenvalue statistics, oldest first: counts (10), sums (10 x 3), sums of squares (10 x 3)."""
        cnt = np.zeros(10, dtype=np.uint64)
        sums, sums_sq = np.zeros((10, 3)), np.zeros((10, 3))
        capi.check(capi.lib().b2_ivox_eig_stats(self.h, cnt.ctypes.data_as(C.POINTER(C.c_uint64)), capi.dptr(sums), capi.dptr(sums_sq)))
        return cnt, sums, sums_sq

    def _valid(self):
        st = self.download_state()
        valid = (st["flags"] & np.uint64(self.VALID_BIT)) != 0
        vid = np.repeat(np.arange(len(st["counts"]), dtype=np.int64), st["counts"])
        slot = np.arange(len(vid), dtype=np.int64) - np.repeat(np.cumsum(st["counts"]) - st["counts"], st["counts"])
        return st, valid, (vid << 32) | slot

    def valid_indices(self) -> np.ndarray:
        """voxel_id << 32 | point_id of every valid point, in id, then slot order."""
        _, valid, idx = self._valid()
        return idx[valid]

    def voxel_points(self) -> np.ndarray:
        """The valid points (N x 4, w = 1) in valid_indices() order."""
        st, valid, _ = self._valid()
        p = st["points"][valid]
        return np.concatenate([p, np.ones((len(p), 1))], 1)

    def voxel_normals(self) -> np.ndarray:
        """The valid points' normals (N x 4, w = 0) in valid_indices() order; signs are not oriented."""
        st, valid, _ = self._valid()
        n = st["normals"][valid]
        return np.concatenate([n, np.zeros((len(n), 1))], 1)

    def voxel_covs(self) -> np.ndarray:
        """The valid points' covariances (N x 4 x 4) in valid_indices() order."""
        st, valid, _ = self._valid()
        c = st["covs"][valid]
        out = np.zeros((len(c), 4, 4))
        out[:, :3, :3] = c
        return out

    def knn_search_force(self, queries, k: int = 1, max_sq_dist: float = np.finfo(np.float64).max):
        """knn_search over every stored point, valid or not (same outputs as knn_search)."""
        q = np.ascontiguousarray(queries, dtype=np.float64)
        if q.ndim == 1:
            q = q[None]
        idx = np.zeros((len(q), k), dtype=np.int64)
        sqd = np.zeros((len(q), k))
        capi.check(capi.lib().b2_ivox_knn_force(self.h, capi.dptr(q), q.shape[1], len(q), int(k), float(max_sq_dist), idx.ctypes.data_as(C.POINTER(C.c_int64)), capi.dptr(sqd)))
        return idx, sqd


def overlap_gpu(targets, source: PointCloud, Ts_target_source) -> float:
    """overlap_gpu (include/gtsam_points/types/gaussian_voxelmap_gpu.hpp:116-125): fraction of source points p for which
    T_j p falls into a voxel of target j for some j.  `targets` / `Ts_target_source`: one map + one 4x4, or equally long lists."""
    if isinstance(targets, GaussianVoxelMapGPU):
        targets, Ts_target_source = [targets], [Ts_target_source]
    Ts = np.ascontiguousarray(np.asarray(Ts_target_source, dtype=np.float64).reshape(len(targets), 16))
    arr = (C.c_void_p * len(targets))(*[t.h for t in targets])
    out = C.c_double()
    capi.check(capi.lib().b2_overlap(arr, len(targets), source.h, capi.dptr(Ts), C.cast(C.byref(out), C.POINTER(C.c_double))))
    return out.value


def _pose16(T):
    """A 4x4 pose as the 16 row-major doubles the C ABI takes (None stays None)."""
    return None if T is None else np.ascontiguousarray(np.asarray(T, dtype=np.float64).reshape(16))


def transform_gpu(cloud: PointCloud, T, flags: int = capi.B2_CLOUD_DEFAULT) -> PointCloud:
    """transform(frame, T) (point_cloud_cpu_funcs.cpp:469-488) of a device cloud into a new device cloud (b2_cloud_create_transformed):
    points T p, covariances T C T^T, normals R n, from the stored values, bit-identical to the CPU transform(); the caller order is
    kept.  flags: the new cloud's storage as for PointCloud -- a rotated cloud is rarely float32-exact, so it is float64 unless
    B2_CLOUD_COMPACT_F32 is given."""
    h = C.c_void_p()
    capi.check(capi.lib().b2_cloud_create_transformed(cloud.h, capi.dptr(_pose16(T)), int(flags), C.byref(h)))
    return PointCloud._from_handle(h, cloud.ctx)


def merge_frames_gpu(poses, frames, downsample_resolution: float, ctx: "Context | None" = None) -> PointCloud:
    """merge_frames_gpu (include/gtsam_points/types/gaussian_voxelmap_gpu.hpp:127-150): merges posed frames (poses: world <- frame
    4x4 each) into one cloud downsampled on a voxel grid laid out in the first frame's coordinates; means of the world points and
    of the rotated covariances, bit-identical to the CPU merge_frames.  Returns a device-resident PointCloud whose .covs are the
    full merged 3x3s (b2_merge_frames's output: the lower triangle of a rotated sum is not bit-symmetric to the upper one, and a
    device cloud keeps only the upper; b2_merge_frames_to_cloud gives the device cloud without the host copy)."""
    ctx = ctx or frames[0].ctx
    P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(len(frames), 16))
    total = sum(len(f.points) for f in frames)
    xyz = np.zeros((max(total, 1), 3), dtype=np.float64)
    cov = np.zeros((max(total, 1), 9), dtype=np.float64)
    m = C.c_size_t()
    arr = (C.c_void_p * len(frames))(*[f.h for f in frames])
    capi.check(capi.lib().b2_merge_frames(ctx.h, capi.dptr(P), arr, len(frames), float(downsample_resolution), capi.dptr(xyz), capi.dptr(cov), C.byref(m)))
    return PointCloud(xyz[: m.value].copy(), cov[: m.value].reshape(-1, 3, 3).copy(), ctx=ctx)


def voxelgrid_sampling(points, resolution: float, covs=None, normals=None, ctx: Context | None = None, flags: int = capi.B2_CLOUD_DEFAULT,
                       intensities=None) -> PointCloud:
    """voxelgrid_sampling (types/point_cloud_cpu.hpp:136) of a host scan into a device cloud: one point per occupied voxel of
    `resolution`, in ascending voxel-key order, each value the mean of the voxel's points in input order (covs N x 3 x 3 /
    N x 4 x 4, normals N x 3 / N x 4 and intensities N averaged alongside).  Points with a non-finite coordinate or outside the 21-bit voxel
    key range are dropped.  flags: capi.B2_CLOUD_* storage of the result.  See b2_cloud_create_voxelgrid for the differences from
    the reference."""
    ctx = ctx or default_context()
    p = np.ascontiguousarray(points, dtype=np.float64)
    if p.ndim != 2 or p.shape[1] not in (3, 4):
        raise ValueError("points must be N x 3 or N x 4")
    cov_stride, nrm_stride = 0, 0
    if covs is not None:
        covs = np.ascontiguousarray(covs, dtype=np.float64)
        if covs.shape[1:] not in ((3, 3), (4, 4)) or len(covs) != len(p):
            raise ValueError("covs must be N x 3 x 3 or N x 4 x 4, one per point")
        cov_stride = 9 if covs.shape[1] == 3 else 16
    if normals is not None:
        normals = np.ascontiguousarray(normals, dtype=np.float64)
        if normals.ndim != 2 or normals.shape[1] not in (3, 4) or len(normals) != len(p):
            raise ValueError("normals must be N x 3 or N x 4, one per point")
        nrm_stride = normals.shape[1]
    if intensities is not None:
        intensities = np.ascontiguousarray(intensities, dtype=np.float64)
        if intensities.shape != (len(p),):
            raise ValueError("intensities must be N values, one per point")
    h = C.c_void_p()
    capi.check(
        capi.lib().b2_cloud_create_voxelgrid_with_intensities(
            ctx.h, float(resolution), capi.dptr(p), p.shape[1], None if covs is None else capi.dptr(covs), cov_stride, None if normals is None else capi.dptr(normals),
            nrm_stride, None if intensities is None else capi.dptr(intensities), len(p), flags, C.byref(h)
        )
    )
    return PointCloud._from_handle(h, ctx)


def _lptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def sample(cloud: PointCloud, indices, flags: int = capi.B2_CLOUD_DEFAULT) -> PointCloud:
    """sample(frame, indices) (point_cloud_cpu_funcs.cpp:27-75) of a device cloud into a new device cloud: row r is the input's caller
    index indices[r] (duplicates allowed; an index outside [0, n) raises).  The result is the cloud b2_cloud_create makes of the same
    downloaded rows under `flags`; no point data leaves the device (b2_cloud_create_sampled)."""
    idx = np.ascontiguousarray(indices, dtype=np.int64).ravel()
    h = C.c_void_p()
    capi.check(capi.lib().b2_cloud_create_sampled(cloud.h, _lptr(idx), len(idx), int(flags), C.byref(h)))
    return PointCloud._from_handle(h, cloud.ctx)


def _random_sampled(cloud: PointCloud, rate: float, seed: int, flags: int):
    """(new cloud, K) of b2_cloud_create_random_sampled."""
    out = np.zeros(max(len(cloud), 1), dtype=np.int64)
    h = C.c_void_p()
    capi.check(capi.lib().b2_cloud_create_random_sampled(cloud.h, float(rate), int(seed) & (2**64 - 1), int(flags), _lptr(out), C.byref(h)))
    res = PointCloud._from_handle(h, cloud.ctx)
    return res, out[: len(res)].copy()


def random_sampling(cloud: PointCloud, rate: float, seed: int = 5489, flags: int = capi.B2_CLOUD_DEFAULT) -> PointCloud:
    """random_sampling(frame, rate, mt) (point_cloud_cpu_funcs.cpp:77-93) on the device: rate >= 0.99 keeps every point, else the
    int(n * rate) points with the smallest SplitMix64 priorities of `seed` (include/b2points.h), in caller order."""
    return _random_sampled(cloud, rate, seed, flags)[0]


def _randomgrid(cloud: PointCloud, resolution: float, rate: float, seed: int, flags: int):
    """(new cloud, K) of b2_cloud_create_randomgrid."""
    out = np.zeros(max(len(cloud), 1), dtype=np.int64)
    h = C.c_void_p()
    capi.check(capi.lib().b2_cloud_create_randomgrid(cloud.h, float(resolution), float(rate), int(seed) & (2**64 - 1), int(flags), _lptr(out), C.byref(h)))
    res = PointCloud._from_handle(h, cloud.ctx)
    return res, out[: len(res)].copy()


def randomgrid_sampling(cloud: PointCloud, resolution: float, rate: float, seed: int = 5489, flags: int = capi.B2_CLOUD_DEFAULT) -> PointCloud:
    """randomgrid_sampling(frame, resolution, rate, mt) (point_cloud_cpu_funcs.cpp:297-456) on the device: in every voxel of
    `resolution` at most ceil(rate n / V) points by priority, at most int(n rate 1.2) in all, in caller order.  See
    b2_cloud_create_randomgrid for the three deliberate differences from the reference."""
    return _randomgrid(cloud, resolution, rate, seed, flags)[0]


def _inliers(cloud: PointCloud, k: int, std_thresh: float, tree, flags: int):
    """(new cloud, K, mean neighbour distances in caller order, threshold) of b2_cloud_create_inliers."""
    n = len(cloud)
    idx = np.zeros(max(n, 1), dtype=np.int64)
    dists = np.zeros(max(n, 1))
    thresh = np.zeros(1)
    h = C.c_void_p()
    capi.check(capi.lib().b2_cloud_create_inliers(cloud.h, None if tree is None else tree.h, int(k), float(std_thresh), int(flags), capi.dptr(dists), capi.dptr(thresh),
                                                  _lptr(idx), C.byref(h)))
    res = PointCloud._from_handle(h, cloud.ctx)
    return res, idx[: len(res)].copy(), dists[:n].copy(), float(thresh[0])


def remove_outliers(cloud: PointCloud, k: int = 10, std_thresh: float = 1.0, tree: "KdTree | None" = None, flags: int = capi.B2_CLOUD_DEFAULT) -> PointCloud:
    """remove_outliers(frame, k, std_thresh) (point_cloud_cpu_funcs.cpp:576-650) on the device: keeps the points whose mean distance to
    their k nearest neighbours (themselves included) is below mean + std_thresh * stddev of those distances.  tree: None builds one;
    else a KdTree.from_cloud(cloud)."""
    return _inliers(cloud, k, std_thresh, tree, flags)[0]


def find_inlier_points(cloud: PointCloud, k: int = 10, std_thresh: float = 1.0, tree: "KdTree | None" = None) -> np.ndarray:
    """find_inlier_points (point_cloud_cpu_funcs.cpp:576-613) with its k-NN on the device: the caller indices remove_outliers keeps,
    ascending (int64)."""
    return _inliers(cloud, k, std_thresh, tree, capi.B2_CLOUD_DEFAULT)[1]


class KdTree:
    """NearestNeighborSearch over a point set: exact k-NN and radius search on the device."""

    @classmethod
    def from_cloud(cls, cloud: PointCloud) -> "KdTree":
        """The tree over a device cloud's stored points, built without a host copy (b2_kdtree_create_from_cloud); indices are the
        cloud's caller indices.  It is the tree PointCloud.estimated(tree=...) accepts for that cloud."""
        self = cls.__new__(cls)
        self.ctx, self.points = cloud.ctx, cloud.points
        h = C.c_void_p()
        capi.check(capi.lib().b2_kdtree_create_from_cloud(cloud.h, C.byref(h)))
        self.h = h
        return self

    def __init__(self, points, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self.points = np.ascontiguousarray(points.points if isinstance(points, PointCloud) else points, dtype=np.float64)
        h = C.c_void_p()
        capi.check(capi.lib().b2_kdtree_create(self.ctx.h, capi.dptr(self.points), self.points.shape[1], len(self.points), C.byref(h)))
        self.h = h

    def knn_search(self, queries, k: int = 1, max_sq_dist: float = np.finfo(np.float64).max):
        """Batched NearestNeighborSearch::knn_search (ann/nearest_neighbor_search.hpp:31-35): indices int64 and squared
        distances, sorted by distance; slots beyond the number found hold (-1, max_sq_dist) (ann/knn_result.hpp:44-72).
        k = 1 returns 1-D arrays, k > 1 arrays of shape (nq, k)."""
        q = np.ascontiguousarray(queries, dtype=np.float64)
        if q.ndim == 1:
            q = q[None]
        if k == 1:
            idx = np.zeros(len(q), dtype=np.int64)
            sqd = np.zeros(len(q))
            capi.check(capi.lib().b2_kdtree_knn1(self.h, capi.dptr(q), q.shape[1], len(q), float(max_sq_dist), idx.ctypes.data_as(C.POINTER(C.c_int64)), capi.dptr(sqd)))
            return idx, sqd
        idx = np.zeros((len(q), k), dtype=np.int64)
        sqd = np.zeros((len(q), k))
        capi.check(capi.lib().b2_kdtree_knn(self.h, capi.dptr(q), q.shape[1], len(q), int(k), float(max_sq_dist), idx.ctypes.data_as(C.POINTER(C.c_int64)), capi.dptr(sqd)))
        return idx, sqd

    def radius_search(self, query, radius: float, max_num_neighbors: int = 2**31 - 1):
        """NearestNeighborSearch::radius_search (ann/nearest_neighbor_search.hpp:45-56) for one query point: indices and squared
        distances of every point with squared distance < radius^2, sorted by (distance, index), at most the nearest
        max_num_neighbors."""
        _, idx, sqd = self.radius_search_batch(np.asarray(query, dtype=np.float64)[None], radius, max_num_neighbors)
        return idx, sqd

    def radius_search_batch(self, queries, radius: float, max_num_neighbors: int = 2**31 - 1):
        """radius_search for every row of `queries` (nq x 3 or nq x 4) -> (offsets, idx, sqd): query i's neighbours are
        idx[offsets[i]:offsets[i + 1]] (int64) with squared distances sqd[...], sorted by (distance, index)."""
        q = np.ascontiguousarray(queries, dtype=np.float64)
        off = np.zeros(len(q) + 1, dtype=np.uint64)
        args = (self.h, capi.dptr(q), q.shape[1], len(q), float(radius), max(int(max_num_neighbors), 0), off.ctypes.data_as(C.POINTER(C.c_uint64)))
        capi.check(capi.lib().b2_kdtree_radius_search(*args, 0, None, None))
        m = int(off[-1])
        idx = np.zeros(max(m, 1), dtype=np.int64)
        sqd = np.zeros(max(m, 1))
        capi.check(capi.lib().b2_kdtree_radius_search(*args, m, idx.ctypes.data_as(C.POINTER(C.c_int64)), capi.dptr(sqd)))
        return off.astype(np.int64), idx[:m], sqd[:m]

    def estimate_covariances(self, k_neighbors: int = 10, eigen_values=(1e-3, 1.0, 1.0)) -> np.ndarray:
        """estimate_covariances over this tree's points (src/gtsam_points/features/covariance_estimation.cpp:18-77) -> n x 3 x 3."""
        out = np.zeros((len(self.points), 3, 3))
        ev = np.ascontiguousarray(eigen_values, dtype=np.float64)
        capi.check(capi.lib().b2_kdtree_estimate_covariances(self.h, int(k_neighbors), capi.dptr(ev), capi.dptr(out)))
        return out

    def estimate_normals(self, k_neighbors: int = 10, eigen_values=(1e-3, 1.0, 1.0), with_covs: bool = False):
        """estimate_normals over this tree's points (src/gtsam_points/features/normal_estimation.cpp:52-55) -> n x 3, and with
        with_covs also the n x 3 x 3 covariances of estimate_covariances, from the same neighbour search."""
        nrm = np.zeros((len(self.points), 3))
        cov = np.zeros((len(self.points), 3, 3)) if with_covs else None
        ev = np.ascontiguousarray(eigen_values, dtype=np.float64)
        capi.check(capi.lib().b2_kdtree_estimate_normals(self.h, int(k_neighbors), capi.dptr(ev), capi.dptr(nrm), capi.dptr(cov) if with_covs else None))
        return (nrm, cov) if with_covs else nrm

    def __del__(self):
        try:
            if getattr(self, "h", None):
                capi.lib().b2_kdtree_destroy(self.h)
                self.h = None
        except Exception:
            pass


def estimate_covariances(points, k_neighbors: int = 10, eigen_values=(1e-3, 1.0, 1.0), ctx: Context | None = None) -> np.ndarray:
    """gtsam_points::estimate_covariances(points, k_neighbors, eigen_values) on the device (features/covariance_estimation.hpp:41-66):
    k-NN over a kd-tree built on the spot, covariance of the neighbourhood, EIG regularisation.  Returns n x 3 x 3."""
    ctx = ctx or default_context()
    p = np.ascontiguousarray(points.points if isinstance(points, PointCloud) else points, dtype=np.float64)
    out = np.zeros((len(p), 3, 3))
    ev = np.ascontiguousarray(eigen_values, dtype=np.float64)
    capi.check(capi.lib().b2_estimate_covariances(ctx.h, capi.dptr(p), p.shape[1], len(p), int(k_neighbors), capi.dptr(ev), capi.dptr(out)))
    return out


def estimate_normals(points, k_or_covs=10, ctx: Context | None = None) -> np.ndarray:
    """gtsam_points::estimate_normals on the device (features/normal_estimation.hpp, src/.../normal_estimation.cpp:18-62), both
    overloads: estimate_normals(points, k) estimates the covariances of the k nearest neighbours first; estimate_normals(points,
    covs) takes N x 3 x 3 / N x 4 x 4 covariances.  A PointCloud with covariances uses them (normal_estimation.cpp:57-62).
    Per point the eigenvector of the smallest eigenvalue, negated if p . n > 1.  Returns n x 3."""
    ctx = ctx or default_context()
    if isinstance(points, PointCloud) and points.covs is not None and np.isscalar(k_or_covs):
        k_or_covs = points.covs
    p = np.ascontiguousarray(points.points if isinstance(points, PointCloud) else points, dtype=np.float64)
    out = np.zeros((len(p), 3))
    if np.isscalar(k_or_covs):
        capi.check(capi.lib().b2_estimate_normals(ctx.h, capi.dptr(p), p.shape[1], len(p), int(k_or_covs), None, capi.dptr(out), None))
        return out
    covs = np.ascontiguousarray(k_or_covs, dtype=np.float64)
    if covs.shape[1:] not in ((3, 3), (4, 4)) or len(covs) != len(p):
        raise ValueError("covs must be N x 3 x 3 or N x 4 x 4, one per point")
    capi.check(capi.lib().b2_estimate_normals_from_covs(ctx.h, capi.dptr(p), p.shape[1], capi.dptr(covs), 9 if covs.shape[1] == 3 else 16, len(p), capi.dptr(out)))
    return out
