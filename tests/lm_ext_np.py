"""Host restatement of b2_factor_set_optimize_pose (test infrastructure): LevenbergMarquardtOptimizerExt::optimize() on one Pose3
variable over unary factors, with the rules include/b2points.h states, and every floating-point operation in the device's order
(csrc/b2_optimize.cu, compiled without fused multiply-adds).  Python floats are IEEE doubles rounded per operation, so everything
here except Exp's sin / cos / sqrt reproduces the device's bits.

A factor is anything with linearize(delta) -> {"H_source", "b_source", "error"} and error(delta) -> float, where delta =
T_target^-1 T is a 4x4 pose (oracle_lib.Factor, or a test's synthetic factor).  error() after linearize() uses the correspondences
of that linearize.  optimize() evaluates all factors at once through an evaluator (linearize(deltas) -> records, error(deltas) ->
errors, in factor order): Factors() wraps a list of factors, and a device test passes one backed by a whole factor set.
"""
import math
from dataclasses import dataclass

import numpy as np

DBL_EPSILON = 2.220446049250313e-16
TERMINATION = {0: "none", 1: "max_iterations", 2: "non_finite", 3: "absolute_error_tol", 4: "relative_error_tol", 5: "error_tol"}


@dataclass
class Params:
    maxIterations: int = 100
    relativeErrorTol: float = 1e-5
    absoluteErrorTol: float = 1e-5
    errorTol: float = 0.0
    lambdaInitial: float = 1e-5
    lambdaFactor: float = 10.0
    lambdaUpperBound: float = 1e5
    lambdaLowerBound: float = 0.0
    minModelFidelity: float = 1e-3


def _flat(T):
    return [float(x) for x in np.asarray(T, dtype=np.float64).reshape(16)]


def _mat(v):
    return np.array(v, dtype=np.float64).reshape(4, 4)


def pose_inv(A):
    """[R^T | -((R_0r t0 + R_1r t1) + R_2r t2)]"""
    A = _flat(A)
    out = [0.0] * 16
    for r in range(3):
        for c in range(3):
            out[r * 4 + c] = A[c * 4 + r]
        out[r * 4 + 3] = -((A[0 * 4 + r] * A[3] + A[1 * 4 + r] * A[7]) + A[2 * 4 + r] * A[11])
    out[15] = 1.0
    return _mat(out)


def pose_mul(A, B):
    """((A_r0 B_0c + A_r1 B_1c) + A_r2 B_2c), plus A_r3 in the translation column; bottom row [0 0 0 1]"""
    A, B = _flat(A), _flat(B)
    out = [0.0] * 16
    for r in range(3):
        for c in range(4):
            s = (A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c]) + A[r * 4 + 2] * B[2 * 4 + c]
            out[r * 4 + c] = s + A[r * 4 + 3] if c == 3 else s
    out[15] = 1.0
    return _mat(out)


def delta_of(T_target, T):
    return pose_mul(pose_inv(T_target), T)


def se3_exp(xi):
    """synthetic.se3_exp's formula in the device's operation order."""
    w0, w1, w2, v0, v1, v2 = (float(x) for x in xi)
    W = [0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0]
    WW = [(W[r * 3 + 0] * W[0 * 3 + c] + W[r * 3 + 1] * W[1 * 3 + c]) + W[r * 3 + 2] * W[2 * 3 + c] for r in range(3) for c in range(3)]
    th2 = (w0 * w0 + w1 * w1) + w2 * w2
    th = math.sqrt(th2)
    eye = [1.0 if r == c else 0.0 for r in range(3) for c in range(3)]
    if th < 1e-10:
        R = [eye[k] + W[k] for k in range(9)]
        V = [eye[k] + 0.5 * W[k] for k in range(9)]
    else:
        s, co = math.sin(th), math.cos(th)
        a, b, c3 = s / th, (1.0 - co) / th2, (th - s) / (th2 * th)
        R = [(eye[k] + a * W[k]) + b * WW[k] for k in range(9)]
        V = [(eye[k] + b * W[k]) + c3 * WW[k] for k in range(9)]
    T = [0.0] * 16
    for r in range(3):
        for c in range(3):
            T[r * 4 + c] = R[r * 3 + c]
        T[r * 4 + 3] = (V[r * 3 + 0] * v0 + V[r * 3 + 1] * v1) + V[r * 3 + 2] * v2
    T[15] = 1.0
    return _mat(T)


def reduce(records):
    """G = sum H_source, g = -sum b_source, 0.5 sum f: set order, from 0.0"""
    G = [0.0] * 36
    g = [0.0] * 6
    f = 0.0
    for rec in records:
        H = np.asarray(rec["H_source"], dtype=np.float64).reshape(36)
        b = np.asarray(rec["b_source"], dtype=np.float64).reshape(6)
        G = [G[k] + float(H[k]) for k in range(36)]
        g = [g[k] + float(b[k]) for k in range(6)]
        f = f + float(rec["error"])
    return np.array(G).reshape(6, 6), -np.array(g), 0.5 * f


def sum_errors(errors):
    e = 0.0
    for x in errors:
        e = e + float(x)
    return e


def solve(G, g, lam):
    """Cholesky of G + lam I (lower triangle of G), then d and lin_change = d'g - 0.5 d'Gd.  -> (solved, d, lin_change)"""
    G = [float(x) for x in np.asarray(G).reshape(36)]
    g = [float(x) for x in np.asarray(g).reshape(6)]
    L = [0.0] * 36
    for j in range(6):
        s = G[j * 6 + j] + lam
        for k in range(j):
            s = s - L[j * 6 + k] * L[j * 6 + k]
        if not s > 0.0:
            return False, np.zeros(6), 0.0
        L[j * 6 + j] = math.sqrt(s)
        for i in range(j + 1, 6):
            v = G[i * 6 + j]
            for k in range(j):
                v = v - L[i * 6 + k] * L[j * 6 + k]
            L[i * 6 + j] = v / L[j * 6 + j]
    y = [0.0] * 6
    for i in range(6):
        s = g[i]
        for k in range(i):
            s = s - L[i * 6 + k] * y[k]
        y[i] = s / L[i * 6 + i]
    d = [0.0] * 6
    for i in range(5, -1, -1):
        s = y[i]
        for k in range(i + 1, 6):
            s = s - L[k * 6 + i] * d[k]
        d[i] = s / L[i * 6 + i]
    dg = 0.0
    for i in range(6):
        dg = dg + d[i] * g[i]
    dGd = 0.0
    for i in range(6):
        gd = 0.0
        for j in range(6):
            gd = gd + G[i * 6 + j] * d[j]
        dGd = dGd + d[i] * gd
    return True, np.array(d), dg - 0.5 * dGd


def _div(a, b):
    """IEEE a / b (Python raises on b == 0)"""
    if b != 0.0:
        return a / b
    if a != a or a == 0.0:
        return math.nan
    return math.copysign(math.inf, a) * math.copysign(1.0, b)


def decide(E, E_trial, lin_change, half_f, solved, p: Params):
    """tryLambda's verdict on one step -> (tried, success, stop, fidelity)"""
    tried = bool(solved) and lin_change >= 0.0
    success = stop = False
    fid = 0.0
    if tried:
        cost_change = E - E_trial
        if lin_change > DBL_EPSILON * half_f:
            fid = _div(cost_change, lin_change)
            success = fid > p.minModelFidelity
        stop = abs(cost_change) < p.relativeErrorTol * E
    return tried, success, stop, fid


def lambda_after(lam, success, stop, p: Params):
    """-> (new lambda, tryLambda's return value)"""
    if success:
        return max(lam / p.lambdaFactor, p.lambdaLowerBound), True
    if not stop:
        lam = lam * p.lambdaFactor
        return lam, lam >= p.lambdaUpperBound
    return lam, True


def termination(accepted, E_prev, E_new, p: Params):
    delta = abs(E_prev - E_new)
    if accepted > p.maxIterations:
        return 1
    if not math.isfinite(E_new):
        return 2
    if delta < p.absoluteErrorTol:
        return 3
    if _div(delta, abs(E_prev)) < p.relativeErrorTol:
        return 4
    if E_new < p.errorTol:
        return 5
    return 0


class Factors:
    """The evaluator of a list of factors, one call per factor."""

    def __init__(self, factors):
        self.factors = list(factors)

    def linearize(self, deltas):
        return [f.linearize(d) for f, d in zip(self.factors, deltas)]

    def error(self, deltas):
        return [f.error(d) for f, d in zip(self.factors, deltas)]


def optimize(evaluator, T_targets, T_init, p: Params | None = None):
    """-> dict(pose, iterations, outer_iterations, inner_iterations, error0, error, lambda_, termination, trace)"""
    p = p or Params()
    T = np.asarray(T_init, dtype=np.float64).copy()
    if isinstance(evaluator, (list, tuple)):
        evaluator = Factors(evaluator)

    def deltas(T_):
        return [delta_of(Tt, T_) for Tt in T_targets]

    error0 = sum_errors(evaluator.error(deltas(T)))
    lam, accepted, outer, inner = p.lambdaInitial, 0, 0, 0
    E_prev = error0
    E = error0
    trace = []
    while True:
        ds = deltas(T)
        records = evaluator.linearize(ds)
        E = sum_errors(evaluator.error(ds))
        G, g, half_f = reduce(records)
        while True:
            solved, d, lin = solve(G, g, lam)
            T_trial = pose_mul(T, se3_exp(d)) if solved and lin >= 0.0 else T.copy()
            Et = float("nan")
            if solved and lin >= 0.0:
                Et = sum_errors(evaluator.error(deltas(T_trial)))
            tried, success, stop, fid = decide(E, Et, lin, half_f, solved, p)
            trace.append(dict(outer=outer, solved=solved, success=success, stop=stop, lam=lam, T_lin=T.copy(), G=G, g=g, error=E, half_f=half_f, d=d,
                              lin_change=lin if solved else 0.0, T_trial=T_trial, error_trial=Et, fidelity=fid))
            inner += 1
            new_lam, done = lambda_after(lam, success, stop, p)
            if success:
                T, E = T_trial, Et
                accepted += 1
            lam = new_lam
            if done:
                break
        outer += 1
        reason = termination(accepted, E_prev, E, p)
        E_prev = E
        if reason:
            break
    return dict(pose=T, iterations=accepted, outer_iterations=outer, inner_iterations=inner, error0=error0, error=E, lambda_=lam,
                termination=TERMINATION[reason], trace=trace)
