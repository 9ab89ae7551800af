"""CPU checks of the device optimizer's rules on one pose (b2_factor_set_optimize_poses with N = 1, unary members and no prior)
through their host restatement, lm_graph_np:

* scripted problems that drive each rule: the lambda schedule up to lambda_upper_bound, every termination reason, a G + lambda I
  that is not positive definite, lin_change < 0 (no trial evaluation), and a lin_change too small against 0.5 sum f to count;
* a quadratic problem where the steps are exact: one accepted step lands on the minimum;
* the restatement over the CPU oracle's factors on the reference's KITTI-07 frames (UNARY graphs of
  src/test/test_matching_cost_factors.cpp) meets the reference's 0.015 rad / 0.15 m gates;
* the Python argument errors of optimize_pose_gpu.
"""
import math
import os

import numpy as np
import pytest

import lm_graph_np as lg
import mini_lm
import oracle_lib as orc
from gtsam_points_b200 import synthetic as syn

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti07_frames.npz")


def one_pose(evaluator, T_targets, T_init, p=None):
    """the restatement on one pose over unary members, with the pose and the trace's poses as 4x4s"""
    r = lg.optimize(evaluator, [(-1, 0)] * len(T_targets), T_targets, [], [T_init], p)
    for e in r["trace"]:
        e["T_lin"], e["T_trial"] = e["T_lin"][0], e["T_trial"][0]
    return dict(r, pose=r["poses"][0])


class Scripted:
    """An evaluator with a fixed linear model (H, b, f) and a cost given as a function of the pose's tangent."""

    def __init__(self, H, b, f, cost):
        self.H, self.b, self.f, self.cost = np.asarray(H, dtype=np.float64), np.asarray(b, dtype=np.float64), f, cost
        self.trial_errors = 0

    def linearize(self, deltas):
        return [dict(H_source=self.H, b_source=self.b, error=self.f) for _ in deltas]

    def error(self, deltas):
        self.trial_errors += 1
        return [self.cost(deltas[0])]


def quadratic(center, scale=1.0, offset=0.0):
    """cost(T) = scale |t - c|^2 + offset over the translation, with its exact model at the identity rotation"""
    c = np.asarray(center, dtype=np.float64)

    class Quad:
        def linearize(self, deltas):
            t = deltas[0][:3, 3]
            H = np.zeros((6, 6))
            H[3:, 3:] = 2.0 * scale * np.eye(3)
            H[:3, :3] = 1e-3 * np.eye(3)
            b = np.zeros(6)
            b[3:] = 2.0 * scale * (t - c)
            return [dict(H_source=H, b_source=b, error=scale * float((t - c) @ (t - c)) + offset)]

        def error(self, deltas):
            t = deltas[0][:3, 3]
            return [scale * float((t - c) @ (t - c)) + offset]

    return Quad()


def test_pose_products_match_numpy_to_rounding():
    rng = np.random.default_rng(0)
    A, B = syn.random_pose(rng, 0.5, 3.0), syn.random_pose(rng, 0.5, 3.0)
    assert np.abs(lg.pose_mul(A, B) - A @ B).max() < 1e-14
    assert np.abs(lg.pose_inv(A) - np.linalg.inv(A)).max() < 1e-14
    for xi in (rng.uniform(-0.3, 0.3, 6), np.array([1e-12, 0, 0, 0.1, 0.2, 0.3]), np.zeros(6)):
        assert np.abs(lg.se3_exp(xi) - syn.se3_exp(xi)).max() < 1e-14


def test_quadratic_converges_in_one_exact_step():
    ev = quadratic([0.3, -0.2, 0.1])
    r = one_pose(ev, [np.eye(4)], np.eye(4))
    assert r["trace"][0]["success"] and r["iterations"] >= 1
    assert np.abs(r["pose"][:3, 3] - [0.3, -0.2, 0.1]).max() < 1e-4
    assert r["error"] < 1e-8 * r["error0"]
    assert r["termination"] in ("absolute_error_tol", "relative_error_tol")


def test_lambda_schedule_up_to_the_upper_bound_then_absolute_tol():
    # every trial is worse: tryLambda multiplies lambda by 10 until it reaches the upper bound and gives up; E equals error0, so the
    # absolute tolerance ends the loop after that one outer iteration
    ev = Scripted(np.eye(6), -np.ones(6), 2.0, lambda d: 1.0 if np.array_equal(d, np.eye(4)) else 5.0)
    r = one_pose(ev, [np.eye(4)], np.eye(4))
    lams = [e["lam"] for e in r["trace"]]
    expect = [1e-5]
    while expect[-1] * 10.0 < 1e5:
        expect.append(expect[-1] * 10.0)
    assert lams == expect and len(lams) == 10
    assert all(e["outer"] == 0 and e["solved"] and not e["success"] and not e["stop"] for e in r["trace"])
    assert r["lambda_"] >= 1e5 and r["iterations"] == 0
    assert r["termination"] == "absolute_error_tol" and r["outer_iterations"] == 1
    assert np.array_equal(r["pose"], np.eye(4))


def test_termination_reasons():
    ev = quadratic([0.3, -0.2, 0.1])
    assert one_pose(ev, [np.eye(4)], np.eye(4), lg.Params(maxIterations=0))["termination"] == "max_iterations"
    assert one_pose(ev, [np.eye(4)], np.eye(4), lg.Params(errorTol=1.0))["termination"] == "error_tol"
    r = one_pose(quadratic([0.3, -0.2, 0.1], offset=1.0), [np.eye(4)], np.eye(4), lg.Params(absoluteErrorTol=1e-300, relativeErrorTol=1e-3))
    assert r["termination"] == "relative_error_tol"
    nan = Scripted(np.eye(6), -np.ones(6), 2.0, lambda d: math.nan)
    r = one_pose(nan, [np.eye(4)], np.eye(4))
    assert r["termination"] == "non_finite" and math.isnan(r["error0"])
    assert lg.termination(0, 1.0, 1.0 - 1e-6, lg.Params()) == 3
    assert lg.termination(101, 1.0, 0.5, lg.Params()) == 1


def test_not_positive_definite_raises_lambda_until_solvable():
    H = np.diag([-1.0, 1, 1, 1, 1, 1])
    ev = Scripted(H, -np.ones(6), 2.0, lambda d: 1.0 if np.array_equal(d, np.eye(4)) else 0.5)
    r = one_pose(ev, [np.eye(4)], np.eye(4), lg.Params(maxIterations=0))
    tr = r["trace"]
    unsolved = [e for e in tr if not e["solved"]]
    assert len(unsolved) == 6 and all(e["lam"] <= 1.0 for e in unsolved)  # 1e-5 .. 1: G + lambda I has a pivot <= 0
    assert all(np.isnan(e["error_trial"]) and np.array_equal(e["T_trial"], e["T_lin"]) for e in unsolved)
    assert tr[len(unsolved)]["solved"] and tr[len(unsolved)]["lam"] == pytest.approx(10.0)
    assert lg.solve(H, np.ones(6), 0.5)[0] is False and lg.solve(H, np.ones(6), 2.0)[0] is True


def test_negative_lin_change_is_not_tried():
    # the solve reads G's lower triangle, d'Gd the whole matrix: a large upper entry makes lin_change negative
    H = np.eye(6)
    H[0, 1] = 1000.0
    solved, d, lin = lg.solve(H, np.ones(6), 1e-5)
    assert solved and lin < 0.0
    ev = Scripted(H, -np.ones(6), 2.0, lambda dd: 1.0)
    calls = ev.trial_errors
    r = one_pose(ev, [np.eye(4)], np.eye(4))
    neg = [e for e in r["trace"] if e["solved"] and e["lin_change"] < 0.0]
    assert neg and all(np.isnan(e["error_trial"]) and not e["success"] and not e["stop"] for e in neg)
    tried = sum(1 for e in r["trace"] if e["solved"] and e["lin_change"] >= 0.0)
    assert ev.trial_errors - calls == 1 + r["outer_iterations"] + tried  # error0, one per outer iteration, one per tried step


def test_tiny_lin_change_is_no_success():
    # the cost drops, but lin_change <= DBL_EPSILON * 0.5 sum f: no fidelity, no success; the cost change is not small -> lambda grows
    ev = Scripted(np.eye(6), -1e-3 * np.ones(6), 1e20, lambda d: 1e10 if np.array_equal(d, np.eye(4)) else 0.9e10)
    r = one_pose(ev, [np.eye(4)], np.eye(4))
    e = r["trace"][0]
    assert e["solved"] and 0.0 <= e["lin_change"] <= lg.DBL_EPSILON * e["half_f"]
    assert e["fidelity"] == 0.0 and not e["success"] and not e["stop"]
    assert r["trace"][1]["lam"] == e["lam"] * 10.0
    # the same step counts once lin_change clears the bar
    tried, success, stop, fid = lg.decide(1e10, 0.9e10, 1e9, 1.0, True, lg.Params())
    assert success and fid == pytest.approx(1.0)


@pytest.fixture(scope="module")
def kitti():
    z = np.load(GOLD)
    pts = [z[f"points{i}"].astype(np.float64) for i in range(3)]
    threads = max(1, min(8, orc.max_threads()))
    covs = [orc.estimate_covariances(p, 10, num_threads=threads) for p in pts]
    return dict(pts=pts, covs=covs, poses=z["poses"], gt=z["poses_gt"], threads=threads)


@pytest.mark.parametrize("method", ["ICP", "GICP", "VGICP"])
def test_restatement_on_oracle_factors_meets_the_reference_gates(kitti, method):
    clouds = [orc.Cloud(p, c) for p, c in zip(kitti["pts"], kitti["covs"])]
    for i in range(2):
        if method == "VGICP":
            vm = orc.VoxelMap(1.0)
            vm.insert(clouds[i])
            f = orc.Factor(vm, clouds[i + 1], num_threads=kitti["threads"])
        else:
            tree = orc.KdTree(clouds[i], kitti["threads"])
            f = orc.Factor(clouds[i], clouds[i + 1], tree=tree, num_threads=kitti["threads"], icp="point" if method == "ICP" else None)
        r = one_pose([f], [kitti["poses"][i]], kitti["poses"][i + 1])
        # UNARY test (test_matching_cost_factors.cpp:208-229): align the fixed pose with its ground truth, judge the optimized one
        delta = kitti["gt"][i] @ np.linalg.inv(kitti["poses"][i])
        err_r, err_t = mini_lm.pose_error(delta @ r["pose"], kitti["gt"][i + 1])
        assert err_r < 0.015 and err_t < 0.15, (method, i, err_r, err_t)


def _unary(cls, key):
    from gtsam_points_b200.factors import IntegratedMatchingCostFactor

    f = cls.__new__(cls)
    IntegratedMatchingCostFactor.__init__(f, np.eye(4), key)
    return f


def test_python_argument_errors():
    import gtsam_points_b200 as g
    from gtsam_points_b200.factors import IntegratedMatchingCostFactor

    binary = g.IntegratedVGICPFactor.__new__(g.IntegratedVGICPFactor)
    IntegratedMatchingCostFactor.__init__(binary, 0, 1)
    with pytest.raises(ValueError, match="binary"):
        g.optimize_pose_gpu([binary], np.eye(4))
    with pytest.raises(ValueError, match="different source keys"):
        g.optimize_pose_gpu([_unary(g.IntegratedGICPFactor, 1), _unary(g.IntegratedGICPFactor, 2)], np.eye(4))
    with pytest.raises(ValueError, match="no factors"):
        g.optimize_pose_gpu([], np.eye(4))
    with pytest.raises(ValueError, match="not a device matching-cost factor"):
        g.optimize_pose_gpu([mini_lm.PriorFactor(1, np.eye(4))], np.eye(4))
    for bad in (np.eye(3), np.full((4, 4), np.nan)):
        with pytest.raises(ValueError, match="T_init"):
            g.optimize_pose_gpu([_unary(g.IntegratedGICPFactor, 1)], bad)
    fset = g.NonlinearFactorSetGPU.__new__(g.NonlinearFactorSetGPU)
    fset.factors, fset.h = [binary], None
    with pytest.raises(ValueError, match="binary"):
        g.optimize_pose_gpu(fset, np.eye(4))

