"""Host restatement of b2_factor_set_optimize_poses (test infrastructure): LevenbergMarquardtOptimizerExt::optimize() on N Pose3
variables over unary and binary matching-cost factors and Pose3 priors, with the rules include/b2points.h states and every
floating-point operation in the device's order (csrc/b2_optimize.cu, compiled without fused multiply-adds): the pose products, the
assembly, the 6N Cholesky and substitutions, the prior, and the trial poses.  Python floats are IEEE doubles rounded per operation,
so everything here except the sin / cos / tan / atan2 / sqrt of Exp and of the prior reproduces the device's bits.

The members are given by an evaluator (linearize(deltas) -> records with H_target, H_source, H_target_source, b_target,
b_source and error, of which a unary member's needs only H_source, b_source and error; error(deltas) -> errors, in member
order), their topology [(target_var, source_var)] (target_var = -1: unary, against T_targets[i]) and the priors
[(var, T_prior, precision[6])].  Factors() wraps a list of factors (anything with linearize(delta) -> record and error(delta) ->
float, error() after linearize() using the correspondences of that linearize); a device test passes an evaluator backed by a
whole factor set.  One pose over unary factors is N = 1 with the topology [(-1, 0)] * F and no prior.
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


def mul3(A, B):
    return [(A[r * 3 + 0] * B[0 * 3 + c] + A[r * 3 + 1] * B[1 * 3 + c]) + A[r * 3 + 2] * B[2 * 3 + c] for r in range(3) for c in range(3)]


def skew3(w):
    return [0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0]


def se3_log(X):
    """Pose3::Logmap of a 4x4 in the device's order (se3_log) -> (xi [w, v] as a list, th)"""
    X = _flat(X)
    s = [0.5 * (X[9] - X[6]), 0.5 * (X[2] - X[8]), 0.5 * (X[4] - X[1])]
    c = 0.5 * (((X[0] + X[5]) + X[10]) - 1.0)
    sn = math.sqrt((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2])
    th = math.atan2(sn, c)
    if c >= 0.0:
        k = th / sn if sn > 0.0 else 1.0
        w = [k * s[j] for j in range(3)]
    else:
        omc = 1.0 - c
        i = 0
        for j in range(1, 3):
            if X[j * 5] > X[i * 5]:
                i = j
        a = [0.0] * 3
        a[i] = math.sqrt((X[i * 5] - c) / omc)
        for j in range(3):
            if j != i:
                a[j] = (0.5 * (X[i * 4 + j] + X[j * 4 + i])) / (omc * a[i])
        sgn = -1.0 if (a[0] * s[0] + a[1] * s[1]) + a[2] * s[2] < 0.0 else 1.0
        w = [th * (sgn * a[j]) for j in range(3)]
    t = [X[3], X[7], X[11]]
    W = skew3(w)
    Wt = [(W[r * 3 + 0] * t[0] + W[r * 3 + 1] * t[1]) + W[r * 3 + 2] * t[2] for r in range(3)]
    if th < 1e-10:
        v = [t[r] - 0.5 * Wt[r] for r in range(3)]
    else:
        h = 0.5 * th
        e = (1.0 - h / math.tan(h)) / (th * th)
        WWt = [(W[r * 3 + 0] * Wt[0] + W[r * 3 + 1] * Wt[1]) + W[r * 3 + 2] * Wt[2] for r in range(3)]
        v = [(t[r] - 0.5 * Wt[r]) + e * WWt[r] for r in range(3)]
    return w + v, th


def se3_log_derivative(xi, th):
    """Pose3::LogmapDerivative in the device's order (se3_log_derivative) -> 36 values, row-major"""
    W, V = skew3(xi[:3]), skew3(xi[3:])
    W2, WV, VW = mul3(W, W), mul3(W, V), mul3(V, W)
    WVW = mul3(WV, W)
    W2V, VW2, WVWW, WWVW = mul3(W2, V), mul3(V, W2), mul3(WVW, W), mul3(W, WVW)
    th2 = th * th
    if th < 1e-3:
        q = 1.0 / 12.0 + th2 / 720.0
    else:
        q = 1.0 / th2 - 1.0 / ((2.0 * th) * math.tan(0.5 * th))
    if th < 0.1:
        A = ((-th2 / 362880.0 + 1.0 / 5040.0) * th2 - 1.0 / 120.0) * th2 + 1.0 / 6.0
        B = ((th2 / 3628800.0 - 1.0 / 40320.0) * th2 + 1.0 / 720.0) * th2 - 1.0 / 24.0
        C = ((th2 / 39916800.0 - 1.0 / 362880.0) * th2 + 1.0 / 5040.0) * th2 - 1.0 / 120.0
    else:
        s, co = math.sin(th), math.cos(th)
        th3 = th2 * th
        th4 = th3 * th
        th5 = th4 * th
        A = (th - s) / th3
        B = ((1.0 - th2 / 2.0) - co) / th4
        C = ((th - s) - th3 / 6.0) / th5
    D = 0.5 * (B - 3.0 * C)
    Jw, Q = [0.0] * 9, [0.0] * 9
    for k in range(9):
        eye = 1.0 if k % 4 == 0 else 0.0
        Jw[k] = (eye + 0.5 * W[k]) + q * W2[k]
        T1 = (WV[k] + VW[k]) - WVW[k]
        T2 = (W2V[k] + VW2[k]) - 3.0 * WVW[k]
        T3 = WVWW[k] + WWVW[k]
        Q[k] = ((-0.5 * V[k] + A * T1) + B * T2) - D * T3
    Q2 = mul3(mul3(Jw, Q), Jw)
    J = [0.0] * 36
    for r in range(6):
        for c in range(6):
            k = (r % 3) * 3 + c % 3
            J[r * 6 + c] = (Jw[k] if c < 3 else 0.0) if r < 3 else (-Q2[k] if c < 3 else Jw[k])
    return J


def prior_eval(prior, T, jacobian=True):
    """prior_eval: -> (f, H (36 values) or None, b (6) or None); the prior's error is 0.5 f"""
    var, T_prior, p = prior
    p = [float(x) for x in p]
    r, th = se3_log(pose_mul(pose_inv(T_prior), T))
    u = [0.0] * 6
    f = 0.0
    for k in range(6):
        u[k] = p[k] * r[k]
        f = f + u[k] * r[k]
    if not jacobian:
        return f, None, None
    J = se3_log_derivative(r, th)
    H, b = [0.0] * 36, [0.0] * 6
    for k in range(6):
        s = 0.0
        for m in range(6):
            s = s + J[m * 6 + k] * u[m]
        b[k] = s
        for l in range(k + 1):
            h = 0.0
            for m in range(6):
                h = h + J[m * 6 + k] * (p[m] * J[m * 6 + l])
            H[k * 6 + l] = h
            H[l * 6 + k] = h
    return f, H, b


def deltas_at(topo, T_targets, T):
    """delta_i = T[target]^-1 T[source], or T_targets[i]^-1 T[source] for a unary member"""
    return [pose_mul(pose_inv(T_targets[i] if t < 0 else T[t]), T[s]) for i, (t, s) in enumerate(topo)]


def assemble(records, topo, priors, T, N):
    """lm_reduce: -> (G (6N x 6N), g (6N), half_f).  Blocks and segments sum their contributions in set order, then prior order."""
    n = 6 * N
    recs = [{k: [float(x) for x in np.asarray(r[k], dtype=np.float64).reshape(-1)] for k in ("H_target", "H_source", "H_target_source", "b_target", "b_source")
             if k in r} for r in records]
    plin = [prior_eval(pr, T[pr[0]]) for pr in priors]
    G = [0.0] * (n * n)
    for row in range(n):
        vr, ir = divmod(row, 6)
        for col in range(n):
            vc, ic = divmod(col, 6)
            s = 0.0
            for rec, (t, sv) in zip(recs, topo):
                if vr == sv and vc == sv:
                    s = s + rec["H_source"][ir * 6 + ic]
                elif t >= 0 and vr == t and vc == t:
                    s = s + rec["H_target"][ir * 6 + ic]
                elif t >= 0 and vr == t and vc == sv:
                    s = s + rec["H_target_source"][ir * 6 + ic]
                elif t >= 0 and vr == sv and vc == t:
                    s = s + rec["H_target_source"][ic * 6 + ir]
            if vr == vc:
                for (var, _, _), (_, H, _) in zip(priors, plin):
                    if var == vr:
                        s = s + H[ir * 6 + ic]
            G[row * n + col] = s
    g = [0.0] * n
    for row in range(n):
        v, ir = divmod(row, 6)
        s = 0.0
        for rec, (t, sv) in zip(recs, topo):
            if sv == v:
                s = s + rec["b_source"][ir]
            elif t == v:
                s = s + rec["b_target"][ir]
        for (var, _, _), (_, _, b) in zip(priors, plin):
            if var == v:
                s = s + b[ir]
        g[row] = -s
    f = 0.0
    for r in records:
        f = f + float(r["error"])
    for fp, _, _ in plin:
        f = f + fp
    return np.array(G).reshape(n, n), np.array(g), 0.5 * f


def total_error(member_errors, priors, T):
    """the members' errors in set order, then the priors' errors (0.5 f), from 0.0"""
    e = 0.0
    for x in member_errors:
        e = e + float(x)
    for pr in priors:
        e = e + 0.5 * prior_eval(pr, T[pr[0]], jacobian=False)[0]
    return e


def solve(G, g, lam):
    """Cholesky of G + lam I on G's lower triangle, substitutions, lin_change = d'g - 0.5 d'Gd -> (solved, d, lin_change).
    Every inner sum over ascending index: the left-looking form here and the device's right-looking one give the same bits."""
    G = np.asarray(G, dtype=np.float64)
    n = G.shape[0]
    Gl = [float(x) for x in G.reshape(-1)]
    gl = [float(x) for x in np.asarray(g).reshape(-1)]
    L = [0.0] * (n * n)
    for j in range(n):
        s = Gl[j * n + j] + lam
        for k in range(j):
            s = s - L[j * n + k] * L[j * n + k]
        if not s > 0.0:
            return False, np.zeros(n), 0.0
        L[j * n + j] = math.sqrt(s)
        for i in range(j + 1, n):
            v = Gl[i * n + j]
            for k in range(j):
                v = v - L[i * n + k] * L[j * n + k]
            L[i * n + j] = v / L[j * n + j]
    y = [0.0] * n
    for i in range(n):
        s = gl[i]
        for k in range(i):
            s = s - L[i * n + k] * y[k]
        y[i] = s / L[i * n + i]
    d = [0.0] * n
    for i in range(n - 1, -1, -1):
        s = y[i]
        for k in range(i + 1, n):
            s = s - L[k * n + i] * d[k]
        d[i] = s / L[i * n + i]
    dg = 0.0
    for i in range(n):
        dg = dg + d[i] * gl[i]
    dGd = 0.0
    for i in range(n):
        gd = 0.0
        for j in range(n):
            gd = gd + Gl[i * n + j] * d[j]
        dGd = dGd + d[i] * gd
    return True, np.array(d), dg - 0.5 * dGd


def trial_poses(T, d, tried):
    return [pose_mul(Tv, se3_exp(d[6 * v:6 * v + 6])) if tried else np.asarray(Tv, dtype=np.float64).copy() for v, Tv in enumerate(T)]


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


def optimize(evaluator, topo, T_targets, priors, T_init, p: Params | None = None):
    """-> dict(poses, iterations, outer_iterations, inner_iterations, error0, error, lambda_, termination, trace)"""
    p = p or Params()
    if isinstance(evaluator, (list, tuple)):
        evaluator = Factors(evaluator)
    N = len(T_init)
    T = [np.asarray(Tv, dtype=np.float64).copy() for Tv in T_init]
    E = error0 = total_error(evaluator.error(deltas_at(topo, T_targets, T)), priors, T)
    lam, accepted, outer, inner = p.lambdaInitial, 0, 0, 0
    E_prev = error0
    trace = []
    while True:
        ds = deltas_at(topo, T_targets, T)
        records = evaluator.linearize(ds)
        E = total_error(evaluator.error(ds), priors, T)
        G, g, half_f = assemble(records, topo, priors, T, N)
        while True:
            solved, d, lin = solve(G, g, lam)
            tried = solved and lin >= 0.0
            T_trial = trial_poses(T, d, tried)
            Et = float("nan")
            if tried:
                Et = total_error(evaluator.error(deltas_at(topo, T_targets, T_trial)), priors, T_trial)
            _, success, stop, fid = decide(E, Et, lin, half_f, solved, p)
            trace.append(dict(outer=outer, solved=solved, success=success, stop=stop, lam=lam, T_lin=np.stack(T), G=G, g=g, error=E, half_f=half_f,
                              d=d, lin_change=lin if solved else 0.0, T_trial=np.stack(T_trial), error_trial=Et, fidelity=fid))
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
    return dict(poses=np.stack(T), iterations=accepted, outer_iterations=outer, inner_iterations=inner, error0=error0, error=E, lambda_=lam,
                termination=TERMINATION[reason], trace=trace)
