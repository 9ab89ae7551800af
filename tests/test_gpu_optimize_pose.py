"""Pose optimization on the device (optimize_pose_gpu: b2_factor_set_optimize_poses with N = 1, unary members and no prior, -m gpu)
against the host restatement (lm_graph_np).

* step-locked parity for every factor kind and for mixed sets: each trace entry is replayed on the host from the device's own
  state -- G, g, 0.5 sum f and E from b2_factor_set_linearize / _error at the entry's linearization pose, E' from
  b2_factor_set_error at its trial pose, bit for bit; d, lin_change and the decision from the restatement, bit for bit; T' from
  the host Exp within 1e-14; lambda follows the schedule from entry to entry;
* end to end on the KITTI-07 frames: the device and the restatement driven through the same set agree on the iterations, the
  accept / reject sequence and the final pose (1e-9), and both meet the reference's 0.015 rad / 0.15 m gates;
* the correspondence-update tolerance: the device's frozen flags give the G the host rule gives, and a later linearize / error
  returns the bits the host-driven sequence leaves;
* repeated calls on one set, a call after an iVox insert, after a surface-validation switch (regrouping), after offload with
  offloading on, and trace truncation.
"""
import ctypes as C
import os

import numpy as np
import pytest

import lm_graph_np as lg
import mini_lm
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti07_frames.npz")


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


@pytest.fixture(scope="module")
def scene(g):
    z = np.load(GOLD)
    pts = [z[f"points{i}"].astype(np.float64) for i in range(5)]
    gt = z["poses_gt"]
    covs = [g.estimate_covariances(p, 10) for p in pts]
    normals = [g.estimate_normals(p, c) for p, c in zip(pts, covs)]
    clouds = [g.PointCloud(p, c, normals=n) for p, c, n in zip(pts, covs, normals)]
    return dict(pts=pts, covs=covs, normals=normals, clouds=clouds, gt=gt)


def world(scene, i):
    T = scene["gt"][i]
    R, t = T[:3, :3], T[:3, 3]
    return scene["pts"][i] @ R.T + t, R @ scene["covs"][i] @ R.T


def init_pose(scene, seed=5):
    return scene["gt"][1] @ syn.se3_exp(np.random.default_rng(seed).uniform(-0.05, 0.05, 6))


def ivox_target(g, scene, cov_est):
    iv = g.iVoxCovarianceEstimation(1.0) if cov_est else g.iVox(1.0)
    for i in (0, 2, 3, 4):
        p, c = world(scene, i)
        if cov_est:
            iv.insert(p)
        else:
            iv.insert(p, c)
    return iv


def make_factors(g, scene, kind):
    """-> (factors, T_targets, keep-alive objects); the source is frame 1"""
    src, gt = scene["clouds"][1], scene["gt"]
    tgt = scene["clouds"][0]
    if kind in ("vgicp", "vgicp_validated"):
        vm = g.GaussianVoxelMapGPU(1.0)
        vm.insert(tgt)
        f = g.IntegratedVGICPFactor(gt[0], 1, vm, src)
        if kind == "vgicp_validated":
            f.set_enable_surface_validation(True)
        return [f], [gt[0]], [vm]
    if kind in ("gicp", "icp", "icp_plane"):
        tree = g.KdTree(tgt)
        if kind == "gicp":
            f = g.IntegratedGICPFactor(gt[0], 1, tgt, src, tree)
        else:
            f = g.IntegratedICPFactor(gt[0], 1, tgt, src, tree, use_point_to_plane=kind == "icp_plane")
        return [f], [gt[0]], [tree]
    cov_est = kind.startswith("ivoxcov")
    iv = ivox_target(g, scene, cov_est)
    base = kind.split("_", 1)[1]
    if base == "gicp":
        f = g.IntegratedGICPFactor(np.eye(4), 1, iv, src)
    else:
        f = g.IntegratedICPFactor(np.eye(4), 1, iv, src, use_point_to_plane=base == "icp_plane")
    return [f], [np.eye(4)], [iv]


KINDS = ["vgicp", "vgicp_validated", "gicp", "icp", "icp_plane", "ivox_gicp", "ivox_icp", "ivoxcov_gicp", "ivoxcov_icp", "ivoxcov_icp_plane"]
MIXED = [("vgicp", "gicp"), ("ivox_icp", "gicp", "vgicp_validated"), ("ivoxcov_gicp", "ivoxcov_icp_plane", "icp")]


def make_set(g, scene, kinds):
    fs, targets, keep = [], [], []
    for k in kinds:
        f, t, kk = make_factors(g, scene, k)
        fs += f
        targets += t
        keep += kk
    fset = g.NonlinearFactorSetGPU(fs[0].ctx)
    fset.add(fs)
    fset._ensure()
    return fset, fs, targets, keep


class SetEvaluator:
    """lm_graph_np's evaluator over a whole factor set (b2_factor_set_linearize / _error)"""

    def __init__(self, fset):
        self.fset = fset

    def linearize(self, deltas):
        out = np.zeros((len(deltas), capi.B2_LINEARIZED_DOUBLES))
        capi.check(capi.lib().b2_factor_set_linearize(self.fset.h, capi.dptr(np.ascontiguousarray(np.stack(deltas))), capi.dptr(out)))
        return [capi.unpack_linearized(r) for r in out]

    def error(self, deltas):
        out = np.zeros(len(deltas))
        capi.check(capi.lib().b2_factor_set_error(self.fset.h, capi.dptr(np.ascontiguousarray(np.stack(deltas))), capi.dptr(out)))
        return list(out)


def deltas(targets, T):
    """the unary members' deltas at the one pose T"""
    return lg.deltas_at([(-1, 0)] * len(targets), targets, [T])


def assemble(records, T):
    """-> (G, g, half_f) of one pose over unary members"""
    return lg.assemble(records, [(-1, 0)] * len(records), [], [T], 1)


def bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.int64), np.asarray(b, dtype=np.float64).view(np.int64))


def replay(fset, targets, res, p=None):
    """Replays every trace entry on the host from the device's own state."""
    p = p or lg.Params()
    ev = SetEvaluator(fset)
    tr = res.trace
    assert len(tr) == res.trace_len == res.inner_iterations
    outer = -1
    for k, e in enumerate(tr):
        if e["outer"] != outer:
            assert e["outer"] == outer + 1
            outer = e["outer"]
            ds = deltas(targets, e["T_lin"])
            G, gv, half_f = assemble(ev.linearize(ds), e["T_lin"])
            E = lg.total_error(ev.error(ds), [], [e["T_lin"]])
            assert bits(G, e["G"]) and bits(gv, e["g"]) and bits(half_f, e["half_f"]), k
            assert bits(E, e["error"]), (k, E, e["error"])
        solved, d, lin = lg.solve(e["G"], e["g"], e["lam"])
        assert solved == e["solved"] and bits(d, e["d"]) and bits(lin, e["lin_change"]), k
        if solved and lin >= 0.0:
            T_host = lg.pose_mul(e["T_lin"], lg.se3_exp(d))
            assert np.abs(T_host - e["T_trial"]).max() <= 1e-14, k
            Et = lg.total_error(ev.error(deltas(targets, e["T_trial"])), [], [e["T_trial"]])
            assert bits(Et, e["error_trial"]), (k, Et, e["error_trial"])
        else:
            assert bits(e["T_trial"], e["T_lin"]) and np.isnan(e["error_trial"])
        _, success, stop, fid = lg.decide(e["error"], e["error_trial"], e["lin_change"], e["half_f"], e["solved"], p)
        assert (success, stop) == (e["success"], e["stop"]) and bits(fid, e["fidelity"]), k
        lam, done = lg.lambda_after(e["lam"], success, stop, p)
        if k + 1 < len(tr):
            assert bits(lam, tr[k + 1]["lam"]), k
            assert done == (tr[k + 1]["outer"] != e["outer"]), k
            nxt = e["T_trial"] if success else e["T_lin"]
            assert bits(tr[k + 1]["T_lin"], nxt), k
        else:
            assert done and bits(lam, res.lambda_)
    last = tr[-1]
    assert bits(res.pose, last["T_trial"] if last["success"] else last["T_lin"])


def gate(T, T_gt):
    err_r, err_t = mini_lm.pose_error(T, T_gt)
    assert err_r < 0.015 and err_t < 0.15, (err_r, err_t)


@pytest.mark.parametrize("kinds", [(k,) for k in KINDS] + MIXED, ids=lambda k: "+".join(k))
def test_step_locked_parity(g, scene, kinds):
    fset, fs, targets, keep = make_set(g, scene, kinds)
    res = g.optimize_pose_gpu(fset, init_pose(scene), trace=True)
    assert res.iterations >= 1 and res.termination != "none"
    assert res.linearizations == res.outer_iterations and res.error_evaluations == 1 + res.outer_iterations + res.inner_iterations
    replay(fset, targets, res)


@pytest.mark.parametrize("kinds", [("vgicp",), ("gicp",), ("ivoxcov_gicp",), ("vgicp", "gicp")], ids=lambda k: "+".join(k))
def test_end_to_end_matches_the_restatement_and_meets_the_gates(g, scene, kinds):
    T0 = init_pose(scene, seed=9)
    fset, fs, targets, keep = make_set(g, scene, kinds)
    launches = fset.launch_count()
    res = g.optimize_pose_gpu(fset, T0, trace=True)
    assert fset.launch_count() == launches  # the call's launches are its own
    fset2, _, _, keep2 = make_set(g, scene, kinds)
    ref = lg.optimize(SetEvaluator(fset2), [(-1, 0)] * len(targets), targets, [], [T0])
    assert res.iterations == ref["iterations"] and res.inner_iterations == ref["inner_iterations"]
    assert [e["success"] for e in res.trace] == [e["success"] for e in ref["trace"]]
    assert res.termination == ref["termination"]
    assert np.abs(res.pose - ref["poses"][0]).max() < 1e-9
    gate(res.pose, scene["gt"][1])
    gate(ref["poses"][0], scene["gt"][1])


def test_correspondence_update_tolerance_follows_the_host_rule(g, scene):
    T0 = init_pose(scene, seed=3)
    sets = []
    for _ in range(2):
        fset, fs, targets, keep = make_set(g, scene, ("gicp", "ivox_icp"))
        for f in fs:
            f.set_correspondence_update_tolerance(0.005, 0.05)
        fset._destroy()
        fset._ensure()  # any_tolerance is taken when the set is created
        sets.append((fset, fs, targets, keep))
    (fa, _, targets, _), (fb, _, _, _) = sets
    res = g.optimize_pose_gpu(fa, T0, trace=True)
    # the host-driven sequence of the same calls on the twin set
    ev = SetEvaluator(fb)
    ev.error(deltas(targets, T0))
    outer = -1
    for e in res.trace:
        if e["outer"] != outer:
            outer = e["outer"]
            G, gv, half_f = assemble(ev.linearize(deltas(targets, e["T_lin"])), e["T_lin"])
            assert bits(G, e["G"]) and bits(gv, e["g"]), outer
            ev.error(deltas(targets, e["T_lin"]))
        if e["solved"] and e["lin_change"] >= 0.0:
            ev.error(deltas(targets, e["T_trial"]))
    # afterwards both sets answer a linearize / error at a nearby pose with the same bits
    T1 = res.pose @ syn.se3_exp(np.full(6, 1e-3))
    for T in (T1, res.pose):
        la, lb = SetEvaluator(fa).linearize(deltas(targets, T)), ev.linearize(deltas(targets, T))
        for ra, rb in zip(la, lb):
            assert all(bits(ra[k], rb[k]) for k in ("H_source", "b_source", "error"))
        assert bits(SetEvaluator(fa).error(deltas(targets, T1)), ev.error(deltas(targets, T1)))


def test_repeated_calls_inserts_regroups_and_offload(g, scene):
    fset, fs, targets, keep = make_set(g, scene, ("ivox_gicp", "vgicp"))
    for seed in (1, 2):
        res = g.optimize_pose_gpu(fset, init_pose(scene, seed), trace=True)
        replay(fset, targets, res)
    # an iVox insert moves the map's generation: the members re-associate, the graph stays
    keep[0].insert(*world(scene, 1))
    res = g.optimize_pose_gpu(fset, init_pose(scene, 4), trace=True)
    replay(fset, targets, res)
    gate(res.pose, scene["gt"][1])
    # a surface-validation switch regroups the set: the graph is rebuilt
    fs[1].set_enable_surface_validation(True)
    res = g.optimize_pose_gpu(fset, init_pose(scene, 6), trace=True)
    replay(fset, targets, res)
    # offloading on: the VGICP member's map and the shared source leave the device; the call reloads them (new device addresses,
    # written into the descriptors in place) and runs the cached graph
    for f in fs:
        f.set_enable_offloading(True)
    vm, src = keep[1], scene["clouds"][1]
    vm.offload_gpu()
    src.offload_gpu()
    assert not vm.loaded_on_gpu() and not src.loaded_on_gpu()
    res = g.optimize_pose_gpu(fset, init_pose(scene, 7), trace=True)
    assert vm.loaded_on_gpu() and src.loaded_on_gpu()
    replay(fset, targets, res)
    gate(res.pose, scene["gt"][1])


def test_offloaded_objects_reload_and_give_the_same_result(g, scene):
    pts, covs = scene["pts"], scene["covs"]
    results = []
    for offload in (False, True):
        src = g.PointCloud(pts[1], covs[1])
        vm = g.GaussianVoxelMapGPU(1.0)
        vm.insert(g.PointCloud(pts[0], covs[0]))
        f = g.IntegratedVGICPFactor(scene["gt"][0], 1, vm, src)
        f.set_enable_offloading(True)
        if offload:
            vm.offload_gpu()
            src.offload_gpu()
            assert not vm.loaded_on_gpu() and not src.loaded_on_gpu()
        results.append(g.optimize_pose_gpu([f], init_pose(scene, 8), trace=True))
        assert vm.loaded_on_gpu() and src.loaded_on_gpu()
    a, b = results
    assert bits(a.pose, b.pose) and a.inner_iterations == b.inner_iterations
    # with offloading off, an offloaded source fails before any device work
    src = g.PointCloud(pts[1], covs[1])
    vm = g.GaussianVoxelMapGPU(1.0)
    vm.insert(g.PointCloud(pts[0], covs[0]))
    f = g.IntegratedVGICPFactor(scene["gt"][0], 1, vm, src)
    src.offload_gpu()
    with pytest.raises(capi.B2Error) as ei:
        g.optimize_pose_gpu([f], init_pose(scene))
    assert ei.value.status == 4


def test_trace_truncation(g, scene):
    fset, fs, targets, keep = make_set(g, scene, ("gicp",))
    full = g.optimize_pose_gpu(fset, init_pose(scene, 12), trace=True)
    fset2, _, _, keep2 = make_set(g, scene, ("gicp",))
    short = g.optimize_pose_gpu(fset2, init_pose(scene, 12), trace=2)
    none = g.optimize_pose_gpu(make_set(g, scene, ("gicp",))[0], init_pose(scene, 12))
    assert len(short.trace) == 2 and short.trace_len == full.trace_len and none.trace is None and none.trace_len == full.trace_len
    for a, b in zip(short.trace, full.trace):
        assert all(bits(a[k], b[k]) for k in ("G", "g", "d", "T_trial", "error_trial", "lam"))
    assert bits(short.pose, full.pose) and bits(none.pose, full.pose)


def test_summary_counts_and_params(g, scene):
    fset, fs, targets, keep = make_set(g, scene, ("vgicp",))
    p = g.LevenbergMarquardtExtParams(maxIterations=2, lambdaInitial=1e3, lambdaUpperBound=1e4)
    res = g.optimize_pose_gpu(fset, init_pose(scene), p, trace=True)
    replay(fset, targets, res, lg.Params(maxIterations=2, lambdaInitial=1e3, lambdaUpperBound=1e4))
    assert res.iterations <= 3
    s = capi.LmSummaryC()
    pc = p.to_c()
    pc.lambda_factor = 1.0
    T = np.eye(4)
    member_vars = np.array([[-1, 0]] * len(targets), dtype=np.int32)
    st = capi.lib().b2_factor_set_optimize_poses(fset.h, 1, member_vars.ctypes.data_as(C.POINTER(C.c_int32)), capi.dptr(np.ascontiguousarray(np.stack(targets))),
                                                 None, 0, capi.dptr(T), C.byref(pc), capi.dptr(np.zeros((4, 4))), C.byref(s), None, None, 0, None)
    assert st == 1
    # a lambda factor so close to 1 that the loop could run for days is refused, and the set still works
    with pytest.raises(capi.B2Error, match="tryLambda calls"):
        g.optimize_pose_gpu(fset, init_pose(scene), g.LevenbergMarquardtExtParams(lambdaFactor=1.0 + 1e-12))
    res = g.optimize_pose_gpu(fset, init_pose(scene), trace=True)
    replay(fset, targets, res)
