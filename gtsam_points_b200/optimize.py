"""Pose optimization on the device: LevenbergMarquardtOptimizerExt (src/gtsam_points/optimizers/levenberg_marquardt_ext.cpp) on a
graph of one Pose3 variable made of unary matching-cost factors, run as one CUDA graph launch (b2_factor_set_optimize_pose).

  params = LevenbergMarquardtExtParams(maxIterations=30)
  result = optimize_pose_gpu([IntegratedVGICPFactor(T_target, 1, target_voxels, source)], T_init, params)
  result.pose  # the optimized source pose

The rules, and where they differ from GTSAM's, are documented at b2_factor_set_optimize_pose in include/b2points.h.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import capi
from .factors import IntegratedMatchingCostFactor, NonlinearFactorSetGPU

DEFAULT_TRACE_CAPACITY = 4096


@dataclass
class LevenbergMarquardtExtParams:
    """The LevenbergMarquardtParams fields the device loop reads, with GTSAM's names and defaults."""

    maxIterations: int = 100
    relativeErrorTol: float = 1e-5
    absoluteErrorTol: float = 1e-5
    errorTol: float = 0.0
    lambdaInitial: float = 1e-5
    lambdaFactor: float = 10.0
    lambdaUpperBound: float = 1e5
    lambdaLowerBound: float = 0.0
    minModelFidelity: float = 1e-3

    def to_c(self) -> capi.LmParamsC:
        p = capi.LmParamsC()
        p.max_iterations = int(self.maxIterations)
        p.relative_error_tol = float(self.relativeErrorTol)
        p.absolute_error_tol = float(self.absoluteErrorTol)
        p.error_tol = float(self.errorTol)
        p.lambda_initial = float(self.lambdaInitial)
        p.lambda_factor = float(self.lambdaFactor)
        p.lambda_upper_bound = float(self.lambdaUpperBound)
        p.lambda_lower_bound = float(self.lambdaLowerBound)
        p.min_model_fidelity = float(self.minModelFidelity)
        return p


@dataclass
class PoseOptimizationResult:
    pose: np.ndarray
    iterations: int          # accepted steps (GTSAM's iterations())
    outer_iterations: int    # linearizations
    inner_iterations: int    # tryLambda calls
    linearizations: int
    error_evaluations: int
    error0: float
    error: float
    lambda_: float
    termination: str         # capi.B2_LM_TERMINATION
    trace: list = field(default=None)  # one dict per tryLambda (trace=True), at most the capacity asked for
    trace_len: int = 0       # tryLambda calls, traced or not


def _trace_dict(e: capi.LmTraceEntryC) -> dict:
    return dict(
        outer=e.outer, solved=bool(e.solved), success=bool(e.success), stop=bool(e.stop), lam=e.lambda_,
        T_lin=np.array(e.T_lin[:]).reshape(4, 4), G=np.array(e.G[:]).reshape(6, 6), g=np.array(e.g[:]), error=e.error, half_f=e.half_f,
        d=np.array(e.d[:]), lin_change=e.lin_change, T_trial=np.array(e.T_trial[:]).reshape(4, 4), error_trial=e.error_trial, fidelity=e.fidelity,
    )


def _members(factors):
    """The factor list of `factors` (a NonlinearFactorSetGPU or a sequence of factors), checked to be unary on one source key."""
    fs = factors.factors if isinstance(factors, NonlinearFactorSetGPU) else list(factors)
    if not fs:
        raise ValueError("optimize_pose_gpu: no factors")
    for f in fs:
        if not isinstance(f, IntegratedMatchingCostFactor):
            raise ValueError(f"optimize_pose_gpu: {type(f).__name__} is not a device matching-cost factor")
        if f.is_binary:
            raise ValueError("optimize_pose_gpu: binary factors are not supported; construct them with a fixed target pose")
    keys = {f.keys()[0] for f in fs}
    if len(keys) != 1:
        raise ValueError(f"optimize_pose_gpu: the factors act on different source keys {sorted(keys)}; one pose variable is optimized")
    return fs


def optimize_pose_gpu(factors, T_init, params: LevenbergMarquardtExtParams | None = None, trace=False) -> PoseOptimizationResult:
    """Optimizes the source pose of unary factors from T_init on the device.  `factors`: a sequence of unary factors on one source key
    (a factor set is built for the call, so its graph is captured and instantiated for this call alone), or a NonlinearFactorSetGPU of
    them (reused, with its cached graph: what a per-frame caller wants).  trace: False, True
    (up to DEFAULT_TRACE_CAPACITY tryLambda entries) or a capacity."""
    fs = _members(factors)
    T_init = np.ascontiguousarray(np.asarray(T_init, dtype=np.float64))
    if T_init.shape != (4, 4) or not np.all(np.isfinite(T_init)):
        raise ValueError("optimize_pose_gpu: T_init must be a finite 4x4 pose")
    if isinstance(factors, NonlinearFactorSetGPU):
        fset = factors
    else:
        fset = NonlinearFactorSetGPU(fs[0].ctx)
        fset.add(fs)
    fset._ensure()
    targets = np.ascontiguousarray(np.stack([f.fixed_target_pose for f in fs]).astype(np.float64))
    p = (params or LevenbergMarquardtExtParams()).to_c()
    cap = 0 if trace is False else (DEFAULT_TRACE_CAPACITY if trace is True else int(trace))
    entries = (capi.LmTraceEntryC * max(cap, 1))() if cap > 0 else None
    T_out = np.zeros((4, 4))
    summary = capi.LmSummaryC()
    n = C.c_size_t(0)
    capi.check(capi.lib().b2_factor_set_optimize_pose(
        fset.h, capi.dptr(targets), capi.dptr(T_init), C.byref(p), capi.dptr(T_out), C.byref(summary),
        C.cast(entries, C.POINTER(capi.LmTraceEntryC)) if entries is not None else None, cap, C.byref(n)))
    fset.num_linearizations += summary.linearizations * len(fs)
    fset.num_evaluations += summary.error_evaluations * len(fs)
    tr = [_trace_dict(entries[i]) for i in range(min(cap, n.value))] if entries is not None else None
    return PoseOptimizationResult(
        pose=T_out, iterations=summary.iterations, outer_iterations=summary.outer_iterations, inner_iterations=summary.inner_iterations,
        linearizations=summary.linearizations, error_evaluations=summary.error_evaluations, error0=summary.error0, error=summary.error,
        lambda_=summary.lambda_, termination=capi.B2_LM_TERMINATION.get(summary.termination, str(summary.termination)), trace=tr, trace_len=n.value,
    )
