"""Host-side mirrors of the reference's factor / factor-set interface for the scan-matching path.

  IntegratedVGICPFactor   include/gtsam_points/factors/integrated_vgicp_factor.hpp:25-113 (+ _gpu.hpp:29-155)
  IntegratedGICPFactor    include/gtsam_points/factors/integrated_gicp_factor.hpp:32-152
  NonlinearFactorSetGPU   include/gtsam_points/cuda/nonlinear_factor_set_gpu.hpp:20-119, optimizers/linearization_hook.hpp:11-29
  HessianFactor           stand-in for gtsam::HessianFactor as filled at src/gtsam_points/factors/integrated_matching_cost_factor.cpp:46-52

`values` is a mapping key -> 4x4 pose matrix (gtsam::Values of Pose3).  Same names, argument meaning and call
order as the reference; errors the reference answers with abort() surface as exceptions (capi.B2Error / ValueError).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import capi
from .types import Context, GaussianVoxelMapGPU, KdTree, PointCloud, default_context, iVox


def pose_inverse(T):
    """gtsam::Pose3::inverse(): (R^T, -R^T t)."""
    T = np.asarray(T, dtype=np.float64)
    Ti = np.eye(4)
    Ti[:3, :3] = T[:3, :3].T
    Ti[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return Ti


@dataclass
class HessianFactor:
    """What IntegratedMatchingCostFactor::linearize hands to GTSAM: HessianFactor(k_t, k_s, H_t, H_ts, -b_t, H_s, -b_s, error)
    for binary factors, HessianFactor(k_s, H_s, -b_s, error) for unary ones."""

    keys: tuple
    H_target: np.ndarray | None
    H_target_source: np.ndarray | None
    g_target: np.ndarray | None  # = -b_target
    H_source: np.ndarray = field(default=None)
    g_source: np.ndarray = field(default=None)  # = -b_source
    f: float = 0.0

    def augmented_information(self) -> np.ndarray:
        """gtsam::HessianFactor::augmentedInformation(): [[G, -g], [-g^T, f]] with linear term g as passed in."""
        if len(self.keys) == 2:
            n = 12
            A = np.zeros((n + 1, n + 1))
            A[0:6, 0:6] = self.H_target
            A[0:6, 6:12] = self.H_target_source
            A[6:12, 0:6] = self.H_target_source.T
            A[6:12, 6:12] = self.H_source
            g = np.concatenate([self.g_target, self.g_source])
        else:
            n = 6
            A = np.zeros((n + 1, n + 1))
            A[0:6, 0:6] = self.H_source
            g = self.g_source
        A[:n, n] = g
        A[n, :n] = g
        A[n, n] = self.f
        return A


class IntegratedMatchingCostFactor:
    """Base: key handling and calc_delta (src/gtsam_points/factors/integrated_matching_cost_factor.cpp:11-69)."""

    def __init__(self, *args):
        # (target_key, source_key) or (fixed_target_pose, source_key)
        a0, a1 = args
        if isinstance(a0, (int, np.integer)):
            self.is_binary = True
            self._keys = (int(a0), int(a1))
            self.fixed_target_pose = np.eye(4)
        else:
            self.is_binary = False
            self._keys = (int(a1),)
            self.fixed_target_pose = np.array(a0, dtype=np.float64).reshape(4, 4)
        self.h = None
        self._last = None

    def keys(self):
        return self._keys

    def dim(self) -> int:
        return 6

    def calc_delta(self, values) -> np.ndarray:
        if self.is_binary:
            return pose_inverse(values[self._keys[0]]) @ np.asarray(values[self._keys[1]], dtype=np.float64)
        return pose_inverse(self.fixed_target_pose) @ np.asarray(values[self._keys[0]], dtype=np.float64)

    # -- NonlinearFactor interface -----------------------------------------------------------------------------
    def linearize(self, values) -> HessianFactor:
        delta = np.ascontiguousarray(self.calc_delta(values))
        buf = np.zeros(capi.B2_LINEARIZED_DOUBLES)
        capi.check(capi.lib().b2_factor_linearize(self.h, capi.dptr(delta), capi.dptr(buf)))
        return self._to_hessian(buf)

    def error(self, values) -> float:
        delta = np.ascontiguousarray(self.calc_delta(values))
        e = C.c_double()
        capi.check(capi.lib().b2_factor_error(self.h, capi.dptr(delta), C.cast(C.byref(e), C.POINTER(C.c_double))))
        return e.value

    def _to_hessian(self, buf) -> HessianFactor:
        l = capi.unpack_linearized(buf)
        self._last = l
        if self.is_binary:
            return HessianFactor(self._keys, l["H_target"], l["H_target_source"], -l["b_target"], l["H_source"], -l["b_source"], l["error"])
        return HessianFactor(self._keys, None, None, None, l["H_source"], -l["b_source"], l["error"])

    # -- statistics ----------------------------------------------------------------------------------------------
    def num_inliers(self) -> int:
        return 0 if self._last is None else self._last["num_inliers"]

    def inlier_fraction(self) -> float:
        return self.num_inliers() / max(1, self.source.size())

    def correspondences(self) -> np.ndarray:
        out = np.zeros(self.source.size(), dtype=np.int64)
        capi.check(capi.lib().b2_factor_correspondences(self.h, out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def memory_usage(self) -> int:
        """Device bytes the factor owns itself (correspondence array + linearization point); clouds / maps are shared."""
        return self.source.size() * 4 + 16 * 8

    def memory_usage_gpu(self) -> int:
        """Device bytes the factor owns itself (b2_factor_device_bytes): correspondences, gathered kd-tree target records and the
        linearization point; the clouds and maps it reads report their own (memory_usage_gpu)."""
        out = C.c_uint64()
        capi.check(capi.lib().b2_factor_device_bytes(self.h, C.byref(out)))
        return out.value

    def set_enable_offloading(self, enable: bool):
        """IntegratedVGICPFactorGPU::set_enable_offloading, on every factor kind: each linearize / error touches what the factor
        reads (a VGICP factor's target map, then the source cloud), reloading what was offloaded.  Off (the default), a call that
        would read an offloaded object raises."""
        capi.check(capi.lib().b2_factor_set_enable_offloading(self.h, 1 if enable else 0))
        self._offloading = bool(enable)

    def _carry_settings(self, f):
        """clone(): the copy takes this factor's offloading setting"""
        if getattr(self, "_offloading", False):
            f.set_enable_offloading(True)
        return f

    # -- tuning knobs of the reference, accepted for drop-in compatibility ------------------------------------------
    def set_num_threads(self, n: int):
        """The device path has no thread knob (integrated_vgicp_factor.hpp:71-73, integrated_gicp_factor.hpp:95-97)."""

    def set_fused_cov_cache_mode(self, mode):
        """The kernel recomputes (C_B + R C_A R^T)^-1 from the linearization rotation (the reference's NONE behaviour):
        there is no cache to choose a layout for (integrated_gicp_factor.hpp:20-24, :106-109)."""

    def __del__(self):
        try:
            if getattr(self, "h", None):
                capi.lib().b2_factor_destroy(self.h)
                self.h = None
        except Exception:
            pass


class IntegratedVGICPFactor(IntegratedMatchingCostFactor):
    """IntegratedVGICPFactor(target_key, source_key, target_voxels, source) or (fixed_target_pose, source_key, ...)."""

    def __init__(self, a0, a1, target_voxels: GaussianVoxelMapGPU, source: PointCloud, ctx: Context | None = None):
        super().__init__(a0, a1)
        if target_voxels is None or target_voxels.h is None:
            raise ValueError("error: target voxelmap has not been created!!")
        if source is None or not source.has_covs():
            raise ValueError("error: source don't have covs!!")
        self.ctx = ctx or source.ctx
        self.target_voxels, self.source = target_voxels, source
        h = C.c_void_p()
        capi.check(capi.lib().b2_vgicp_factor_create(self.ctx.h, target_voxels.h, source.h, C.byref(h)))
        self.h = h

    def get_target(self):
        return self.target_voxels

    def set_enable_surface_validation(self, enable: bool):
        """IntegratedVGICPFactorGPU::set_enable_surface_validation (integrated_vgicp_factor_gpu.hpp:88): source points whose normal
        faces away from the sensor at the association pose get no correspondence.  The source cloud must carry normals."""
        capi.check(capi.lib().b2_factor_set_enable_surface_validation(self.h, 1 if enable else 0))
        self._surface_validation = bool(enable)

    def clone(self):
        """NonlinearFactor::clone (integrated_vgicp_factor.hpp:90): a new factor over the same (shared) map and cloud."""
        a0 = self._keys[0] if self.is_binary else self.fixed_target_pose
        a1 = self._keys[1] if self.is_binary else self._keys[0]
        f = IntegratedVGICPFactor(a0, a1, self.target_voxels, self.source, ctx=self.ctx)
        if getattr(self, "_surface_validation", False):
            f.set_enable_surface_validation(True)
        return self._carry_settings(f)


IntegratedVGICPFactorGPU = IntegratedVGICPFactor


class IntegratedGICPFactor(IntegratedMatchingCostFactor):
    """IntegratedGICPFactor(target_key, source_key, target, source[, target_tree]) or (fixed_target_pose, source_key, ...).

    `target` may also be an iVox, which is then target and search structure at once (IntegratedGICPFactor_<iVox, PointCloud>,
    src/gtsam_points/factors/integrated_gicp_factor.cpp:11): correspondences are iVox indices voxel_id << 32 | point_id, and a
    factor whose map changed since its last linearize re-associates.  An iVoxCovarianceEstimation target (integrated_gicp_factor.cpp:12)
    serves only its valid points, with their estimated covariances."""

    def __init__(self, a0, a1, target, source: PointCloud, target_tree: KdTree | None = None, ctx: Context | None = None):
        super().__init__(a0, a1)
        if isinstance(target, iVox):
            if source is None or not source.has_covs():
                raise ValueError("error: source don't have covs!!")
            self.ctx = ctx or source.ctx
            self.target, self.source, self.target_tree = target, source, target
            h = C.c_void_p()
            capi.check(capi.lib().b2_gicp_ivox_factor_create(self.ctx.h, target.h, source.h, C.byref(h)))
            self.h = h
            return
        if target is None or not target.has_covs():
            raise ValueError("error: target don't have covs!!")
        if source is None or not source.has_covs():
            raise ValueError("error: source don't have covs!!")
        self.ctx = ctx or source.ctx
        self.target, self.source = target, source
        # default: a kd-tree over the target is built on the spot (integrated_gicp_factor_impl.hpp:47-51)
        self.target_tree = target_tree or KdTree(target, ctx=self.ctx)
        h = C.c_void_p()
        capi.check(capi.lib().b2_gicp_factor_create(self.ctx.h, target.h, self.target_tree.h, source.h, C.byref(h)))
        self.h = h

    def set_max_correspondence_distance(self, dist: float):
        capi.check(capi.lib().b2_factor_set_max_correspondence_distance(self.h, float(dist)))

    def set_correspondence_update_tolerance(self, angle: float, trans: float):
        """integrated_gicp_factor.hpp:103-109, impl:135-147: while the pose stays within (angle, trans) of the pose of the
        last correspondence update, linearize() keeps those correspondences and linearizes them at the new pose."""
        capi.check(capi.lib().b2_factor_set_correspondence_update_tolerance(self.h, float(angle), float(trans)))

    def clone(self):
        a0 = self._keys[0] if self.is_binary else self.fixed_target_pose
        a1 = self._keys[1] if self.is_binary else self._keys[0]
        return self._carry_settings(IntegratedGICPFactor(a0, a1, self.target, self.source, target_tree=self.target_tree, ctx=self.ctx))


class IntegratedICPFactor(IntegratedMatchingCostFactor):
    """IntegratedICPFactor(target_key, source_key, target, source[, target_tree][, use_point_to_plane]) or
    (fixed_target_pose, source_key, ...): include/gtsam_points/factors/integrated_icp_factor.hpp:27-145.  Point-to-plane
    needs target normals: those of the target PointCloud, which is then read on the device, or an `normals` attribute (n x 3) of
    any other target object.  Neither cloud needs covariances.

    `target` may also be an iVox, which is then target and search structure at once (IntegratedICPFactor_<iVox, PointCloud>,
    src/gtsam_points/factors/integrated_icp_factor.cpp:9-10): correspondences are iVox indices voxel_id << 32 | point_id, and a
    factor whose map changed since its last linearize re-associates.  Point-to-plane needs an iVoxCovarianceEstimation target,
    whose valid points and estimated normals it uses; a plain iVox keeps no normals."""

    def __init__(self, a0, a1, target: PointCloud, source: PointCloud, target_tree: KdTree | None = None, use_point_to_plane: bool = False, ctx: Context | None = None):
        super().__init__(a0, a1)
        if isinstance(target, iVox):
            if source is None:
                raise ValueError("error: source frame doesn't have required attributes for icp")
            self.ctx = ctx or source.ctx
            self.target, self.source, self.target_tree, self.use_point_to_plane = target, source, target, bool(use_point_to_plane)
            h = C.c_void_p()
            capi.check(capi.lib().b2_icp_ivox_factor_create(self.ctx.h, target.h, source.h, 1 if use_point_to_plane else 0, C.byref(h)))
            self.h = h
            return
        normals = getattr(target, "normals", None)
        if target is None or (use_point_to_plane and normals is None):
            raise ValueError("error: target frame doesn't have required attributes for icp")
        if source is None:
            raise ValueError("error: source frame doesn't have required attributes for icp")
        self.ctx = ctx or source.ctx
        self.target, self.source, self.use_point_to_plane = target, source, bool(use_point_to_plane)
        self.target_tree = target_tree or KdTree(target, ctx=self.ctx)
        nrm = None
        # a PointCloud's normals are already on the device -- unless `normals` was assigned or replaced after construction
        on_device = isinstance(target, PointCloud) and getattr(target, "_device_normals", None) is normals
        if use_point_to_plane and not on_device:
            nrm = np.ascontiguousarray(np.asarray(normals, dtype=np.float64)[:, :3])
        h = C.c_void_p()
        capi.check(capi.lib().b2_icp_factor_create(self.ctx.h, target.h, self.target_tree.h, source.h, 1 if use_point_to_plane else 0, capi.dptr(nrm) if nrm is not None else None, C.byref(h)))
        self.h = h

    def set_max_correspondence_distance(self, dist: float):
        capi.check(capi.lib().b2_factor_set_max_correspondence_distance(self.h, float(dist)))

    def set_correspondence_update_tolerance(self, angle: float, trans: float):
        capi.check(capi.lib().b2_factor_set_correspondence_update_tolerance(self.h, float(angle), float(trans)))

    def clone(self):
        a0 = self._keys[0] if self.is_binary else self.fixed_target_pose
        a1 = self._keys[1] if self.is_binary else self._keys[0]
        return self._carry_settings(IntegratedICPFactor(a0, a1, self.target, self.source, target_tree=self.target_tree, use_point_to_plane=self.use_point_to_plane, ctx=self.ctx))


class IntegratedPointToPlaneICPFactor(IntegratedICPFactor):
    """integrated_icp_factor.hpp:147-175: IntegratedICPFactor with use_point_to_plane = true."""

    def __init__(self, a0, a1, target: PointCloud, source: PointCloud, target_tree: KdTree | None = None, ctx: Context | None = None):
        super().__init__(a0, a1, target, source, target_tree=target_tree, use_point_to_plane=True, ctx=ctx)


class NonlinearFactorSetGPU:
    """Batches every device factor of a graph into one launch (NonlinearFactorSet interface)."""

    def __init__(self, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self.factors = []
        self.h = None
        self.num_linearizations = 0
        self.num_evaluations = 0
        self._results = None
        self._errors = None

    def size(self):
        return len(self.factors)

    def clear(self):
        self._destroy()
        self.factors = []

    def clear_counts(self):
        self.num_linearizations = 0
        self.num_evaluations = 0

    def linearization_count(self):
        return self.num_linearizations

    def evaluation_count(self):
        return self.num_evaluations

    def add(self, factor) -> bool:
        if isinstance(factor, (list, tuple)):
            return all([self.add(f) for f in factor])
        if isinstance(factor, IntegratedMatchingCostFactor):
            self._destroy()
            self.factors.append(factor)
            return True
        return False

    def _ensure(self):
        if self.h is None:
            arr = (C.c_void_p * len(self.factors))(*[f.h for f in self.factors])
            h = C.c_void_p()
            capi.check(capi.lib().b2_factor_set_create(self.ctx.h, arr, len(self.factors), C.byref(h)))
            self.h = h

    def linearize(self, values):
        if not self.factors:
            return
        self._ensure()
        self.num_linearizations += len(self.factors)
        deltas = np.ascontiguousarray(np.stack([f.calc_delta(values) for f in self.factors]))
        out = np.zeros((len(self.factors), capi.B2_LINEARIZED_DOUBLES))
        capi.check(capi.lib().b2_factor_set_linearize(self.h, capi.dptr(deltas), capi.dptr(out)))
        self._results = out
        return out

    def error(self, values):
        if not self.factors:
            return np.zeros(0)
        self._ensure()
        self.num_evaluations += len(self.factors)
        deltas = np.ascontiguousarray(np.stack([f.calc_delta(values) for f in self.factors]))
        out = np.zeros(len(self.factors))
        capi.check(capi.lib().b2_factor_set_error(self.h, capi.dptr(deltas), capi.dptr(out)))
        self._errors = out
        return out

    def calc_linear_factors(self, linearization_point):
        out = self.linearize(linearization_point)
        return [f._to_hessian(out[i]) for i, f in enumerate(self.factors)]

    def launch_count(self) -> int:
        return 0 if self.h is None else int(capi.lib().b2_factor_set_launch_count(self.h))

    def _destroy(self):
        if getattr(self, "h", None):
            capi.lib().b2_factor_set_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass
