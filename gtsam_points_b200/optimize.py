"""Pose optimization on the device: LevenbergMarquardtOptimizerExt (src/gtsam_points/optimizers/levenberg_marquardt_ext.cpp) run
as one CUDA graph launch (b2_factor_set_optimize_poses), on one Pose3 variable made of unary matching-cost factors, or on a graph
of up to 32 Pose3 variables made of unary and binary matching-cost factors and Pose3 priors.

  params = LevenbergMarquardtExtParams(maxIterations=30)
  result = optimize_pose_gpu([IntegratedVGICPFactor(T_target, 1, target_voxels, source)], T_init, params)
  result.pose  # the optimized source pose

  result = optimize_graph_gpu([IntegratedVGICPFactor(0, 1, voxels0, cloud1)], {0: T0, 1: T1}, [PriorFactorPose3(0, T0, 1e6)])
  result.values  # {0: pose, 1: pose}

The rules, and where they differ from GTSAM's, are documented at b2_factor_set_optimize_poses in include/b2points.h.
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
    T_init = np.asarray(T_init, dtype=np.float64)
    if T_init.shape != (4, 4) or not np.all(np.isfinite(T_init)):
        raise ValueError("optimize_pose_gpu: T_init must be a finite 4x4 pose")
    # the N = 1 graph of unary members without priors
    _, _, member_vars, targets, pri, T_init = _graph_inputs(factors, {fs[0].keys()[0]: T_init}, [])
    cap = 0 if trace is False else (DEFAULT_TRACE_CAPACITY if trace is True else int(trace))
    T_out, result = _optimize(factors, fs, member_vars, targets, pri, 0, T_init, params, cap)
    if result["trace"] is not None:
        for e in result["trace"]:
            e["T_lin"], e["T_trial"] = e["T_lin"][0], e["T_trial"][0]
    return PoseOptimizationResult(pose=T_out[0], **result)


DEFAULT_GRAPH_TRACE_CAPACITY = 256


@dataclass
class PriorFactorPose3:
    """gtsam::PriorFactor<Pose3>(key, pose, noise) with a diagonal precision over the tangent [w, v]: a scalar (GTSAM's
    Isotropic::Precision(6, p)) or six values."""

    key: int
    pose: np.ndarray
    precision: object = 1.0


@dataclass
class GraphOptimizationResult:
    values: dict             # key -> optimized 4x4 pose
    keys: list               # the variables in index order (sorted keys of the initial values)
    iterations: int
    outer_iterations: int
    inner_iterations: int
    linearizations: int
    error_evaluations: int
    error0: float
    error: float
    lambda_: float
    termination: str
    trace: list = field(default=None)  # one dict per tryLambda (trace=True), N-pose arrays in variable order
    trace_len: int = 0


def _graph_trace_dict(e: capi.LmGraphTraceEntryC, x: np.ndarray, N: int) -> dict:
    n = 6 * N
    o = 16 * N
    return dict(
        outer=e.outer, solved=bool(e.solved), success=bool(e.success), stop=bool(e.stop), lam=e.lambda_, error=e.error, half_f=e.half_f,
        lin_change=e.lin_change, error_trial=e.error_trial, fidelity=e.fidelity,
        T_lin=x[:o].reshape(N, 4, 4).copy(), G=x[o:o + n * n].reshape(n, n).copy(), g=x[o + n * n:o + n * n + n].copy(),
        d=x[o + n * n + n:o + n * n + 2 * n].copy(), T_trial=x[o + n * n + 2 * n:].reshape(N, 4, 4).copy(),
    )


def _graph_inputs(factors, values, priors):
    """-> (member factors, sorted keys, member_vars F x 2, T_targets F x 16, prior array, T_init N x 16), or ValueError"""
    fn = "optimize_graph_gpu"
    fs = factors.factors if isinstance(factors, NonlinearFactorSetGPU) else list(factors)
    if not fs:
        raise ValueError(f"{fn}: no factors")
    if not isinstance(values, dict) or not values:
        raise ValueError(f"{fn}: values must be a non-empty dict from key to 4x4 pose")
    keys = sorted(values)
    if len(keys) > capi.B2_LM_MAX_POSES:
        raise ValueError(f"{fn}: {len(keys)} variables; at most {capi.B2_LM_MAX_POSES} are optimized")
    index = {k: i for i, k in enumerate(keys)}
    T_init = np.zeros((len(keys), 4, 4))
    for k in keys:
        T = np.asarray(values[k], dtype=np.float64)
        if T.shape != (4, 4) or not np.all(np.isfinite(T)):
            raise ValueError(f"{fn}: the value of key {k} must be a finite 4x4 pose")
        T_init[index[k]] = T
    used = np.zeros(len(keys), dtype=bool)
    member_vars = np.zeros((len(fs), 2), dtype=np.int32)
    targets = np.zeros((len(fs), 4, 4))
    for i, f in enumerate(fs):
        if not isinstance(f, IntegratedMatchingCostFactor):
            raise ValueError(f"{fn}: {type(f).__name__} is not a device matching-cost factor")
        for k in f.keys():
            if k not in index:
                raise ValueError(f"{fn}: factor {i} acts on key {k}, which has no value")
        if f.is_binary:
            t, s = index[f.keys()[0]], index[f.keys()[1]]
            if t == s:
                raise ValueError(f"{fn}: factor {i} has the same target and source key {f.keys()[0]}")
            member_vars[i] = (t, s)
            used[t] = True
        else:
            s = index[f.keys()[0]]
            member_vars[i] = (-1, s)
            targets[i] = f.fixed_target_pose
        used[s] = True
    pri = (capi.PosePriorC * max(len(priors), 1))()
    for j, p in enumerate(priors):
        if not isinstance(p, PriorFactorPose3):
            raise ValueError(f"{fn}: prior {j} is not a PriorFactorPose3")
        if p.key not in index:
            raise ValueError(f"{fn}: prior {j} acts on key {p.key}, which has no value")
        T = np.asarray(p.pose, dtype=np.float64)
        if T.shape != (4, 4) or not np.all(np.isfinite(T)):
            raise ValueError(f"{fn}: the pose of prior {j} must be a finite 4x4 pose")
        prec = np.broadcast_to(np.asarray(p.precision, dtype=np.float64), (6,)) if np.ndim(p.precision) == 0 else np.asarray(p.precision, dtype=np.float64)
        if prec.shape != (6,) or not np.all(np.isfinite(prec)) or not np.all(prec > 0.0):
            raise ValueError(f"{fn}: the precision of prior {j} must be a positive finite scalar or 6 such values")
        pri[j].var = index[p.key]
        pri[j].T_prior[:] = [float(x) for x in T.reshape(16)]
        pri[j].precision[:] = [float(x) for x in prec]
        used[index[p.key]] = True
    if not used.all():
        raise ValueError(f"{fn}: keys {[k for k in keys if not used[index[k]]]} are referenced by no factor and no prior")
    return fs, keys, member_vars, targets, pri, T_init


def optimize_graph_gpu(factors, values: dict, priors=(), params: LevenbergMarquardtExtParams | None = None, trace=False) -> GraphOptimizationResult:
    """Optimizes the poses of a graph of matching-cost factors and Pose3 priors on the device.  `values`: key -> initial 4x4 pose;
    the variables are its keys in sorted order.  Binary factors act on their keys(); unary factors on their source key, against
    their fixed_target_pose.  `factors`: a sequence of factors (a factor set is built for the call) or a NonlinearFactorSetGPU
    (reused, with its cached graph, across calls and graph shapes).  trace: False, True (up to DEFAULT_GRAPH_TRACE_CAPACITY
    tryLambda entries) or a capacity."""
    fs, keys, member_vars, targets, pri, T_init = _graph_inputs(factors, values, list(priors))
    cap = 0 if trace is False else (DEFAULT_GRAPH_TRACE_CAPACITY if trace is True else int(trace))
    T_out, result = _optimize(factors, fs, member_vars, targets, pri, len(priors), T_init, params, cap)
    return GraphOptimizationResult(values={k: T_out[i].copy() for i, k in enumerate(keys)}, keys=keys, **result)


def _optimize(factors, fs, member_vars, targets, pri, num_priors, T_init, params, cap):
    """b2_factor_set_optimize_poses on checked inputs (those of _graph_inputs) -> (T_out N x 4 x 4, the result's summary and trace
    fields).  `factors` is reused when it is a NonlinearFactorSetGPU; otherwise a set of `fs` is built for the call."""
    if isinstance(factors, NonlinearFactorSetGPU):
        fset = factors
    else:
        fset = NonlinearFactorSetGPU(fs[0].ctx)
        fset.add(fs)
    fset._ensure()
    N = len(T_init)
    p = (params or LevenbergMarquardtExtParams()).to_c()
    per = capi.lib().b2_lm_graph_trace_doubles(N)
    entries = (capi.LmGraphTraceEntryC * max(cap, 1))() if cap > 0 else None
    data = np.zeros(max(cap, 1) * per) if cap > 0 else None
    member_vars = np.ascontiguousarray(member_vars)
    targets = np.ascontiguousarray(targets)
    T_init = np.ascontiguousarray(T_init)
    T_out = np.zeros((N, 4, 4))
    summary = capi.LmSummaryC()
    n = C.c_size_t(0)
    capi.check(capi.lib().b2_factor_set_optimize_poses(
        fset.h, N, member_vars.ctypes.data_as(C.POINTER(C.c_int32)), capi.dptr(targets), C.cast(pri, C.POINTER(capi.PosePriorC)), num_priors,
        capi.dptr(T_init), C.byref(p), capi.dptr(T_out), C.byref(summary),
        C.cast(entries, C.POINTER(capi.LmGraphTraceEntryC)) if entries is not None else None, capi.dptr(data) if data is not None else None, cap, C.byref(n)))
    fset.num_linearizations += summary.linearizations * len(fs)
    fset.num_evaluations += summary.error_evaluations * len(fs)
    tr = [_graph_trace_dict(entries[i], data[i * per:(i + 1) * per], N) for i in range(min(cap, n.value))] if entries is not None else None
    return T_out, dict(
        iterations=summary.iterations, outer_iterations=summary.outer_iterations, inner_iterations=summary.inner_iterations,
        linearizations=summary.linearizations, error_evaluations=summary.error_evaluations, error0=summary.error0, error=summary.error,
        lambda_=summary.lambda_, termination=capi.B2_LM_TERMINATION.get(summary.termination, str(summary.termination)), trace=tr, trace_len=n.value,
    )
