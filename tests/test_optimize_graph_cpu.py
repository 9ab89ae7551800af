"""CPU checks of the multi-pose device optimizer's rules (b2_factor_set_optimize_poses) through their host restatement,
lm_graph_np:

* the prior's Logmap and its derivative J against an extended-precision (mpmath) Logmap and its central difference, 1e-12
  relative, at rotation angles below 1e-10, near 1e-5, 1 and pi - 1e-6, and far from the origin; and, independently of the Logmap's
  algebra, Exp(Log(X)) = X and agreement with mpmath's matrix logarithm where that is real;
* a G + lambda I that is not positive definite, and a graph with no prior (a free gauge) that ends finite;
* the restatement over the CPU oracle's factors passes the reference's 0.015 rad / 0.15 m gates on KITTI-07 in the four
  AlignmentTest shapes (src/test/test_matching_cost_factors.cpp:239-303) for GICP, VGICP and ICP, with test_alignment_gates' budgets;
* the ABI's defaults and the checks that run before the set is read (a set pointer that is never dereferenced shows it): NULL
  arguments, every parameter bound, poses and priors; and the Python argument errors.
"""
import ctypes as C
import math
import os

import mpmath as mp
import numpy as np
import pytest

import lm_graph_np as lg
import mini_lm
import oracle_lib as orc
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti07_frames.npz")


# ---- the prior against mpmath ---------------------------------------------------------------------------------------------------
def mp_exp(xi):
    """SE(3) Exp [w, v] in mpmath"""
    w = mp.matrix([xi[0], xi[1], xi[2]])
    v = mp.matrix([xi[3], xi[4], xi[5]])
    th = mp.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2)
    W = mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    eye = mp.eye(3)
    if th == 0:
        R, V = eye, eye
    else:
        R = eye + (mp.sin(th) / th) * W + ((1 - mp.cos(th)) / th ** 2) * W * W
        V = eye + ((1 - mp.cos(th)) / th ** 2) * W + ((th - mp.sin(th)) / th ** 3) * W * W
    t = V * v
    T = mp.eye(4)
    for r in range(3):
        for c in range(3):
            T[r, c] = R[r, c]
        T[r, 3] = t[r]
    return T


def mp_log(X):
    """SE(3) Logmap in mpmath: the same algebra as se3_log (above pi / 2 the axis from the symmetric part), without rounding"""
    s = [(X[2, 1] - X[1, 2]) / 2, (X[0, 2] - X[2, 0]) / 2, (X[1, 0] - X[0, 1]) / 2]
    c = (X[0, 0] + X[1, 1] + X[2, 2] - 1) / 2
    sn = mp.sqrt(s[0] ** 2 + s[1] ** 2 + s[2] ** 2)
    th = mp.atan2(sn, c)
    if c >= 0:
        k = th / sn if sn != 0 else mp.mpf(1)
        w = [k * x for x in s]
    else:
        i = max(range(3), key=lambda j: X[j, j])
        a = [mp.mpf(0)] * 3
        a[i] = mp.sqrt((X[i, i] - c) / (1 - c))
        for j in range(3):
            if j != i:
                a[j] = (X[i, j] + X[j, i]) / 2 / ((1 - c) * a[i])
        if sum(a[j] * s[j] for j in range(3)) < 0:
            a = [-x for x in a]
        w = [th * x for x in a]
    W = mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    t = mp.matrix([X[0, 3], X[1, 3], X[2, 3]])
    if th == 0:
        v = t - W * t / 2
    else:
        # V^-1 = I - W / 2 + (1 / th^2) (1 - (th / 2) cot(th / 2)) W^2
        v = t - W * t / 2 + ((1 - (th / 2) * mp.cot(th / 2)) / th ** 2) * (W * (W * t))
    return [w[0], w[1], w[2], v[0], v[1], v[2]]


def to_mp(T):
    return mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.asarray(T)])


def pose_with_angle(rng, angle, trans):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    xi = np.concatenate([angle * axis, rng.normal(size=3) * trans])
    with mp.workdps(40):
        T = mp_exp([mp.mpf(float(x)) for x in xi])
        return np.array([[float(T[r, c]) for c in range(4)] for r in range(4)])


@pytest.mark.parametrize("angle,trans", [(3e-11, 1.0), (0.0, 2.0), (1e-5, 1.0), (1.0, 1.0), (math.pi - 1e-6, 1.0), (2.5, 1.0), (0.05, 1.0),
                                         (0.3, 1.0), (1e-5, 3e4), (1.0, 3e4), (math.pi - 1e-6, 3e4)])
def test_prior_logmap_and_derivative_match_extended_precision(angle, trans):
    rng = np.random.default_rng(int(angle * 1e6) % 1000 + int(trans))
    X = pose_with_angle(rng, angle, trans)
    xi, th = lg.se3_log(X)
    J = np.array(lg.se3_log_derivative(xi, th)).reshape(6, 6)
    with mp.workdps(50):
        Xm = to_mp(X)
        ref = np.array([float(x) for x in mp_log(Xm)])
        h = mp.mpf("1e-20")
        Jref = np.zeros((6, 6))
        for k in range(6):
            e = [mp.mpf(0)] * 6
            e[k] = h
            plus = mp_log(Xm * mp_exp(e))
            e[k] = -h
            minus = mp_log(Xm * mp_exp(e))
            for r in range(6):
                Jref[r, k] = float((plus[r] - minus[r]) / (2 * h))
    scale = max(np.abs(ref).max(), 1e-300)
    assert np.abs(np.array(xi) - ref).max() <= 1e-12 * scale, (np.array(xi), ref)
    # references that do not share se3_log's algebra: Exp(Log(X)) = X, and where the principal matrix logarithm of the rounded X
    # is real (away from pi) mpmath's logm gives the twist [[W, v], [0, 0]] itself
    with mp.workdps(50):
        back = mp_exp([mp.mpf(x) for x in xi])
        assert max(abs(float(back[r, c]) - X[r, c]) for r in range(3) for c in range(4)) <= 1e-15 * max(1.0, np.abs(X).max())
        if angle < 3.0:
            M = mp.logm(to_mp(X))
            lg_ref = np.array([float(mp.re(x)) for x in ((M[2, 1] - M[1, 2]) / 2, (M[0, 2] - M[2, 0]) / 2, (M[1, 0] - M[0, 1]) / 2, M[0, 3], M[1, 3], M[2, 3])])
            assert np.abs(np.array(xi) - lg_ref).max() <= 1e-12 * scale, (np.array(xi), lg_ref)
    assert abs(th - np.linalg.norm(ref[:3])) <= 1e-12 * max(th, 1e-300)
    assert np.abs(J - Jref).max() <= 1e-12 * np.abs(Jref).max(), np.abs(J - Jref).max()


def test_prior_contribution_is_the_gauss_newton_model():
    rng = np.random.default_rng(3)
    T_prior = syn.random_pose(rng, 0.5, 2.0)
    T = T_prior @ syn.se3_exp(np.array([0.4, -0.2, 0.1, 0.3, 0.1, -0.2]))
    p = [1e6, 2e6, 3e6, 1e5, 2e5, 3e5]
    f, H, b = lg.prior_eval((0, T_prior, p), T)
    r, th = lg.se3_log(lg.pose_mul(lg.pose_inv(T_prior), T))
    J = np.array(lg.se3_log_derivative(r, th)).reshape(6, 6)
    P = np.diag(p)
    assert np.allclose(np.array(H).reshape(6, 6), J.T @ P @ J, rtol=1e-13, atol=0)
    assert np.allclose(b, J.T @ P @ np.array(r), rtol=1e-12)
    assert f == pytest.approx(float(np.array(r) @ P @ np.array(r)), rel=1e-14)
    # the model predicts the error of a small step
    d = 1e-4 * rng.normal(size=6)
    f2, _, _ = lg.prior_eval((0, T_prior, p), T @ syn.se3_exp(d))
    model = f + 2 * np.dot(b, d) + d @ np.array(H).reshape(6, 6) @ d
    assert abs(f2 - model) < 1e-6 * f


# ---- the restatement ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kitti():
    z = np.load(GOLD)
    pts = [z[f"points{i}"].astype(np.float64) for i in range(5)]
    threads = max(1, min(8, orc.max_threads()))
    covs = [orc.estimate_covariances(p, 10, num_threads=threads) for p in pts]
    clouds = [orc.Cloud(p, c) for p, c in zip(pts, covs)]
    return dict(pts=pts, covs=covs, clouds=clouds, poses=z["poses"], gt=z["poses_gt"], threads=threads)


def oracle_factor(kitti, method, t, s, threads=None):
    clouds, threads = kitti["clouds"], threads or kitti["threads"]
    if method == "VGICP":
        vm = orc.VoxelMap(1.0)
        vm.insert(clouds[t])
        return orc.Factor(vm, clouds[s], num_threads=threads)
    tree = orc.KdTree(clouds[t], threads)
    return orc.Factor(clouds[t], clouds[s], tree=tree, num_threads=threads, icp="point" if method == "ICP" else None)


def bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.int64), np.asarray(b, dtype=np.float64).view(np.int64))


def test_solve_matches_numpy_and_refuses_a_not_positive_definite_system():
    rng = np.random.default_rng(2)
    A = rng.normal(size=(30, 30))
    G = A @ A.T
    g = rng.normal(size=30)
    ok, d, lin = lg.solve(G, g, 1e-3)
    assert ok and np.allclose(d, np.linalg.solve(G + 1e-3 * np.eye(30), g), rtol=1e-9)
    assert lin == pytest.approx(d @ g - 0.5 * d @ G @ d, rel=1e-12)
    G[17, 17] = -50.0
    ok, d, lin = lg.solve(G, g, 1e-3)
    assert not ok and not d.any() and lin == 0.0


class QuadraticGraph:
    """binary members with cost |(t_s - t_t) - m|^2 over the translations (their exact model at identity rotations)"""

    def __init__(self, offsets):
        self.m = [np.asarray(o, dtype=np.float64) for o in offsets]

    def _r(self, d, m):
        return d[:3, 3] - m

    def linearize(self, deltas):
        out = []
        for d, m in zip(deltas, self.m):
            r = self._r(d, m)
            Hs = np.zeros((6, 6))
            Hs[3:, 3:] = 2 * np.eye(3)
            Hs[:3, :3] = 1e-3 * np.eye(3)
            bs = np.zeros(6)
            bs[3:] = 2 * r
            out.append(dict(H_source=Hs, H_target=Hs.copy(), H_target_source=-Hs, b_source=bs, b_target=-bs, error=float(r @ r)))
        return out

    def error(self, deltas):
        return [float(self._r(d, m) @ self._r(d, m)) for d, m in zip(deltas, self.m)]


def test_a_graph_without_prior_ends_finite_with_its_gauge_in_place():
    ev = QuadraticGraph([[1.0, 0, 0], [0, 1.0, 0]])
    T0 = [np.eye(4), np.eye(4), np.eye(4)]
    r = lg.optimize(ev, [(0, 1), (1, 2)], [None, None], [], T0)
    assert r["termination"] in ("absolute_error_tol", "relative_error_tol") and np.all(np.isfinite(r["poses"]))
    P = r["poses"]
    assert np.allclose(P[1][:3, 3] - P[0][:3, 3], [1, 0, 0], atol=1e-4) and np.allclose(P[2][:3, 3] - P[1][:3, 3], [0, 1, 0], atol=1e-4)
    # G is singular (a free translation): the damped steps have no component along the gauge, whose mean stays put
    assert np.allclose(sum(p[:3, 3] for p in P), 0.0, atol=1e-9)
    G = r["trace"][0]["G"]
    assert abs(np.linalg.eigvalsh(G).min()) < 1e-9


def test_a_not_positive_definite_system_raises_lambda():
    class Indefinite(QuadraticGraph):
        def linearize(self, deltas):
            out = super().linearize(deltas)
            out[0]["H_source"] = out[0]["H_source"].copy()
            out[0]["H_source"][0, 0] = -10.0
            return out

    ev = Indefinite([[1.0, 0, 0]])
    r = lg.optimize(ev, [(-1, 0)], [np.eye(4)], [(0, np.eye(4), [1.0] * 6)], [np.eye(4)], lg.Params(maxIterations=0))
    unsolved = [e for e in r["trace"] if not e["solved"]]
    assert unsolved and all(np.isnan(e["error_trial"]) and bits(e["T_trial"], e["T_lin"]) for e in unsolved)
    assert np.all(np.isfinite(r["poses"]))


def run_shapes(kitti, method, make_binary, make_unary):
    """FORWARD / BACKWARD (prior on frame i / i + 1), UNARY, MULTI_FRAME with test_alignment_gates' budgets"""
    poses, gt = kitti["poses"], kitti["gt"]
    p = lg.Params(maxIterations=100, relativeErrorTol=1e-6) if method == "ICP" else lg.Params(maxIterations=30, relativeErrorTol=1e-4)
    prior = lambda var, frame: (var, poses[frame], [1e6] * 6)  # noqa: E731

    def check(result, fixed, note):
        delta = gt[fixed[0]] @ np.linalg.inv(fixed[1])
        for k, T in result.items():
            err_r, err_t = mini_lm.pose_error(delta @ T, gt[k])
            assert err_r < 0.015 and err_t < 0.15, (method, note, k, err_r, err_t)

    for i in range(2):
        f = make_binary(i, i + 1)
        for note, pv in (("FORWARD", 0), ("BACKWARD", 1)):
            r = lg.optimize([f], [(0, 1)], [None], [prior(pv, i + pv)], [poses[i], poses[i + 1]], p)
            check({i + 1 - pv: r["poses"][1 - pv]}, (i + pv, r["poses"][pv]), f"{note}_{i}")
        r = lg.optimize([make_unary(i, i + 1)], [(-1, 0)], [poses[i]], [], [poses[i + 1]], p)
        check({i + 1: r["poses"][0]}, (i, poses[i]), f"UNARY_{i}")
    fs = [make_binary(i - 1, i) for i in range(1, 5)]
    r = lg.optimize(fs, [(i - 1, i) for i in range(1, 5)], [None] * 4, [prior(0, 0)], [poses[i] for i in range(5)], p)
    check({k: r["poses"][k] for k in range(1, 5)}, (0, r["poses"][0]), "MULTI_FRAME")


@pytest.mark.parametrize("method", ["GICP", "VGICP", "ICP"])
def test_restatement_on_oracle_factors_meets_the_reference_gates(kitti, method):
    run_shapes(kitti, method, lambda t, s: oracle_factor(kitti, method, t, s), lambda t, s: oracle_factor(kitti, method, t, s))


# ---- the ABI checks and the Python argument errors ---------------------------------------------------------------------------------
def test_abi_checks_before_the_set_is_read():
    import gtsam_points_b200 as g

    L = capi.lib()
    p = capi.LmParamsC()
    L.b2_lm_params_default(C.byref(p))
    assert bytes(p) == bytes(g.LevenbergMarquardtExtParams().to_c())
    bogus = C.c_void_p(1)
    vars2 = np.array([[0, 1]], dtype=np.int32)
    vp = vars2.ctypes.data_as(C.POINTER(C.c_int32))
    T2 = np.ascontiguousarray(np.stack([np.eye(4)] * 2))
    out = np.zeros((2, 4, 4))

    def call(set_=bogus, N=2, vars_=vp, priors=None, P=0, T=T2, params=p, T_out=out):
        st = L.b2_factor_set_optimize_poses(set_, N, vars_, None, priors, P, capi.dptr(T) if T is not None else None, C.byref(params) if params is not None else None,
                                            capi.dptr(T_out) if T_out is not None else None, None, None, None, 0, None)
        return st, L.b2_last_error().decode()

    for kw in (dict(set_=None), dict(vars_=None), dict(T=None), dict(params=None), dict(T_out=None), dict(P=1)):
        st, err = call(**kw)
        assert st == 1 and "NULL" in err, (kw, err)
    for N in (0, capi.B2_LM_MAX_POSES + 1):
        st, err = call(N=N)
        assert st == 1 and "num_poses" in err
    for kw, msg in [(dict(lambdaFactor=1.0), "lambda_factor"), (dict(absoluteErrorTol=0.0), "absolute_error_tol"), (dict(lambdaInitial=0.0), "lambda_initial"),
                    (dict(maxIterations=-1), "max_iterations"), (dict(relativeErrorTol=math.inf), "not finite"),
                    # lambda would underflow in max_iterations + 1 decreases (a closed form: no loop over the iterations)
                    (dict(maxIterations=2**31 - 1), "underflows"),
                    # more tryLambda calls than the bound allows: 1e-5 .. 1e5 in steps of 1 + 1e-12, and a 2^31-iteration budget
                    (dict(lambdaFactor=1.0 + 1e-12), "tryLambda calls"), (dict(maxIterations=2**31 - 1, lambdaLowerBound=1e-6), "tryLambda calls")]:
        st, err = call(params=g.LevenbergMarquardtExtParams(**kw).to_c())
        assert st == 1 and msg in err, (kw, err)
    bad = T2.copy()
    bad[1, 0, 3] = math.inf
    assert call(T=bad)[0] == 1 and "not finite" in L.b2_last_error().decode()

    def prior(var=0, prec=1e6, T=np.eye(4)):
        pr = (capi.PosePriorC * 1)()
        pr[0].var = var
        pr[0].T_prior[:] = list(np.asarray(T, dtype=np.float64).reshape(16))
        pr[0].precision[:] = [prec] * 6
        return pr

    for kw, msg in [(dict(var=2), "var"), (dict(var=-1), "var"), (dict(prec=0.0), "precision"), (dict(prec=-1.0), "precision"), (dict(prec=math.nan), "precision"),
                    (dict(T=np.full((4, 4), math.nan)), "not finite")]:
        st, err = call(priors=C.cast(prior(**kw), C.POINTER(capi.PosePriorC)), P=1)
        assert st == 1 and msg in err, (kw, err)
    assert L.b2_lm_graph_trace_doubles(1) == 80 and L.b2_lm_graph_trace_doubles(32) == 36 * 32 * 32 + 44 * 32
    assert L.b2_factor_set_lm_graph_builds(None) == 0


def _factor(cls, *keys_or_pose):
    from gtsam_points_b200.factors import IntegratedMatchingCostFactor

    f = cls.__new__(cls)
    IntegratedMatchingCostFactor.__init__(f, *keys_or_pose)
    return f


def test_python_argument_errors():
    import gtsam_points_b200 as g

    b01 = _factor(g.IntegratedVGICPFactor, 0, 1)
    vals = {0: np.eye(4), 1: np.eye(4)}
    cases = [
        (([], vals), "no factors"),
        (([b01], {}), "non-empty dict"),
        (([b01], {0: np.eye(4)}), "key 1, which has no value"),
        (([b01], {0: np.eye(4), 1: np.eye(3)}), "finite 4x4"),
        (([b01], {0: np.eye(4), 1: np.full((4, 4), np.nan)}), "finite 4x4"),
        (([_factor(g.IntegratedGICPFactor, 1, 1)], vals), "same target and source"),
        (([b01], {**vals, 2: np.eye(4)}), "referenced by no factor"),
        (([b01], {k: np.eye(4) for k in range(33)}), "at most 32"),
        (([mini_lm.PriorFactor(1, np.eye(4))], vals), "not a device matching-cost factor"),
        (([b01], vals, [g.PriorFactorPose3(5, np.eye(4))]), "key 5"),
        (([b01], vals, [g.PriorFactorPose3(0, np.eye(4), 0.0)]), "precision"),
        (([b01], vals, [g.PriorFactorPose3(0, np.eye(4), [1.0] * 5)]), "precision"),
        (([b01], vals, [g.PriorFactorPose3(0, np.eye(4), np.inf)]), "precision"),
        (([b01], vals, [g.PriorFactorPose3(0, np.eye(3))]), "finite 4x4"),
        (([b01], vals, [mini_lm.PriorFactor(0, np.eye(4))]), "not a PriorFactorPose3"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError, match=msg):
            g.optimize_graph_gpu(*args)
    # a prior alone may hold a variable; a unary factor's key is its source
    u2 = _factor(g.IntegratedGICPFactor, np.eye(4), 2)
    fs, keys, mv, targets, pri, T = __import__("gtsam_points_b200.optimize", fromlist=["_graph_inputs"])._graph_inputs(
        [b01, u2], {0: np.eye(4), 1: np.eye(4), 2: np.eye(4), 3: np.eye(4)}, [g.PriorFactorPose3(3, np.eye(4), [1, 2, 3, 4, 5, 6])])
    assert keys == [0, 1, 2, 3] and mv.tolist() == [[0, 1], [-1, 2]] and pri[0].var == 3 and list(pri[0].precision) == [1, 2, 3, 4, 5, 6]
