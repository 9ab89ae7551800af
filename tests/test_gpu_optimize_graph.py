"""Multi-pose optimization on the device (b2_factor_set_optimize_poses, -m gpu) against the host restatement (lm_graph_np).

* step-locked replay of every trace entry from the device's own state: the members' records from b2_factor_set_linearize at the
  deltas of T_lin, assembled on the host -- G and g bit for bit without priors; with priors only the prior-touched diagonal blocks
  (and E, E') may differ, within 1e-12 relative (atan2 / sin / cos / tan); d and lin_change re-solved from the entry's own G and g
  bit for bit, T' within 1e-14, every decision and lambda exactly.  Graphs: FORWARD, BACKWARD and MULTI_FRAME on KITTI-07, the
  demo's 5-frame full connection, a mixed-kind graph, a prior with a large rotational residual and a 32-pose ring;
* the four AlignmentTest shapes pass the reference's gates with CUDA factors for VGICP, GICP and ICP;
* the tolerance's frozen flags and the host state left for binary members, repeated calls with another topology and other priors
  (no re-capture unless a capacity grows), a call after an iVox insert, after a regroup and with offloaded objects;
* a graph with a free gauge ends finite, and every topology error is refused before device work.
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
    covs = [g.estimate_covariances(p, 10) for p in pts]
    normals = [g.estimate_normals(p, c) for p, c in zip(pts, covs)]
    clouds = [g.PointCloud(p, c, normals=n) for p, c, n in zip(pts, covs, normals)]
    maps = []
    for c in clouds:
        vm = g.GaussianVoxelMapGPU(1.0)
        vm.insert(c)
        maps.append(vm)
    trees = [g.KdTree(c) for c in clouds]
    return dict(pts=pts, covs=covs, clouds=clouds, maps=maps, trees=trees, poses=z["poses"], gt=z["poses_gt"])


def factor(g, scene, kind, a0, a1, t, s):
    c, m, tr = scene["clouds"], scene["maps"], scene["trees"]
    if kind == "VGICP":
        return g.IntegratedVGICPFactor(a0, a1, m[t], c[s])
    if kind == "GICP":
        return g.IntegratedGICPFactor(a0, a1, c[t], c[s], tr[t])
    return g.IntegratedICPFactor(a0, a1, c[t], c[s], tr[t], use_point_to_plane=kind == "ICP_PLANE")


class SetEvaluator:
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


def bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.int64), np.asarray(b, dtype=np.float64).view(np.int64))


def close(a, b, rel=1e-12):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() <= rel * max(np.abs(b).max(), 1e-300)


def graph_of(fs, values, priors):
    """-> (topology, T_targets, host priors) as optimize_graph_gpu maps them"""
    keys = sorted(values)
    ix = {k: i for i, k in enumerate(keys)}
    topo = [(ix[f.keys()[0]], ix[f.keys()[1]]) if f.is_binary else (-1, ix[f.keys()[0]]) for f in fs]
    targets = [None if f.is_binary else f.fixed_target_pose for f in fs]
    hp = [(ix[p.key], p.pose, np.broadcast_to(np.asarray(p.precision, dtype=np.float64), (6,))) for p in priors]
    return topo, targets, hp


def replay(fset, fs, values, priors, res, p=None, graph=None):
    """graph: (topology, T_targets, host priors) when the call's topology is not the factors' own keys"""
    p = p or lg.Params()
    topo, targets, hp = graph or graph_of(fs, values, priors)
    N = len(res.keys)
    ev = SetEvaluator(fset)
    tr = res.trace
    assert len(tr) == res.trace_len == res.inner_iterations
    prior_vars = {v for v, _, _ in hp}
    mask = np.zeros((6 * N, 6 * N), dtype=bool)
    for v in prior_vars:
        mask[6 * v:6 * v + 6, 6 * v:6 * v + 6] = True
    gmask = mask.any(axis=1)
    same = bits if not hp else (lambda a, b: close(a, b))  # noqa: E731
    outer = -1
    for k, e in enumerate(tr):
        T_lin = list(e["T_lin"])
        if e["outer"] != outer:
            assert e["outer"] == outer + 1
            outer = e["outer"]
            ds = lg.deltas_at(topo, targets, T_lin)
            G, gv, half_f = lg.assemble(ev.linearize(ds), topo, hp, T_lin, N)
            E = lg.total_error(ev.error(ds), hp, T_lin)
            assert bits(G[~mask], e["G"][~mask]) and bits(gv[~gmask], e["g"][~gmask]), k
            if hp:
                assert close(G[mask], e["G"][mask]) and close(gv[gmask], e["g"][gmask]), k
            assert same(half_f, e["half_f"]) and same(E, e["error"]), (k, E, e["error"])
        solved, d, lin = lg.solve(e["G"], e["g"], e["lam"])
        assert solved == e["solved"] and bits(d, e["d"]) and bits(lin, e["lin_change"]), k
        if solved and lin >= 0.0:
            T_host = np.stack(lg.trial_poses(T_lin, d, True))
            assert np.abs(T_host - e["T_trial"]).max() <= 1e-14 * max(1.0, np.abs(e["T_trial"]).max()), k
            T_trial = list(e["T_trial"])
            Et = lg.total_error(ev.error(lg.deltas_at(topo, targets, T_trial)), hp, T_trial)
            assert same(Et, e["error_trial"]), (k, Et, e["error_trial"])
        else:
            assert bits(e["T_trial"], e["T_lin"]) and np.isnan(e["error_trial"])
        _, success, stop, fid = lg.decide(e["error"], e["error_trial"], e["lin_change"], e["half_f"], e["solved"], p)
        assert (success, stop) == (e["success"], e["stop"]) and bits(fid, e["fidelity"]), k
        lam, done = lg.lambda_after(e["lam"], success, stop, p)
        if k + 1 < len(tr):
            assert bits(lam, tr[k + 1]["lam"]), k
            assert done == (tr[k + 1]["outer"] != e["outer"]), k
            assert bits(tr[k + 1]["T_lin"], e["T_trial"] if success else e["T_lin"]), k
        else:
            assert done and bits(lam, res.lambda_)
    last = tr[-1]
    final = last["T_trial"] if last["success"] else last["T_lin"]
    assert bits(np.stack([res.values[k] for k in res.keys]), final)


def raw_call(fset, topo, targets, priors, T_init, cap=256):
    """b2_factor_set_optimize_poses with an explicit topology and host priors [(var, pose, precision[6])] (keys 0..N-1) -> a result
    shaped as optimize_graph_gpu's"""
    from gtsam_points_b200 import optimize as opt

    N = len(T_init)
    mv = np.array(topo, dtype=np.int32)
    tg = np.stack([np.eye(4) if t is None else t for t in targets])
    pri = (capi.PosePriorC * max(len(priors), 1))()
    for j, (var, pose, prec) in enumerate(priors):
        pri[j].var = var
        pri[j].T_prior[:] = [float(x) for x in np.asarray(pose).reshape(16)]
        pri[j].precision[:] = [float(x) for x in prec]
    out, result = opt._optimize(fset, fset.factors, mv, tg, pri, len(priors), np.stack(T_init), None, cap)
    return opt.GraphOptimizationResult(values={k: out[k] for k in range(N)}, keys=list(range(N)), **result)


def run(g, fs, values, priors=(), **kw):
    fset = g.NonlinearFactorSetGPU(fs[0].ctx)
    fset.add(fs)
    fset._ensure()
    res = g.optimize_graph_gpu(fset, values, priors, trace=True, **kw)
    assert res.termination != "none" and res.error_evaluations == 1 + res.outer_iterations + res.inner_iterations
    return fset, res


def ring_scene(g, n=32, seed=3):
    """n frames on a circle looking at one synthetic scene, consecutive frames and the last and first linked by GICP factors"""
    pts, covs = syn.make_cloud(6000, stream=71, scale=0.3)
    rng = np.random.default_rng(seed)
    gt = []
    for k in range(n):
        a = 2 * np.pi * k / n
        T = syn.se3_exp(np.array([0.0, 0.0, a, 0.0, 0.0, 0.0]))
        T[:3, 3] = [3.0 * np.cos(a), 3.0 * np.sin(a), 0.1 * np.sin(3 * a)]
        gt.append(T)
    clouds, trees = [], []
    for T in gt:
        R, t = T[:3, :3], T[:3, 3]
        local = (pts - t) @ R
        c = g.PointCloud(local, R.T @ covs @ R)
        clouds.append(c)
        trees.append(g.KdTree(c))
    fs = [g.IntegratedGICPFactor(k, (k + 1) % n, clouds[k], clouds[(k + 1) % n], trees[k]) for k in range(n)]
    init = {k: gt[k] @ syn.se3_exp(rng.uniform(-0.02, 0.02, 6)) for k in range(n)}
    return fs, init, gt, (clouds, trees)


@pytest.mark.parametrize("shape", ["forward", "backward", "multi_frame", "full_connection", "mixed", "large_prior", "ring32"])
def test_step_locked_replay(g, scene, shape):
    poses = scene["poses"]
    P = g.PriorFactorPose3
    keep = None
    if shape in ("forward", "backward"):
        fs = [factor(g, scene, "VGICP", 0, 1, 0, 1)]
        values = {0: poses[0], 1: poses[1]}
        priors = [P(0, poses[0], 1e6)] if shape == "forward" else [P(1, poses[1], 1e6)]
    elif shape == "multi_frame":
        fs = [factor(g, scene, "VGICP", i - 1, i, i - 1, i) for i in range(1, 5)]
        values = {i: poses[i] for i in range(5)}
        priors = [P(0, poses[0], 1e6)]
    elif shape == "full_connection":  # demo_matching_cost_factors.cpp:233-257, full connection
        fs = [factor(g, scene, "GICP", i, j, i, j) for i in range(5) for j in range(i + 1, 5)]
        values = {i: poses[i] for i in range(5)}
        priors = [P(0, poses[0], 1e6)]
    elif shape == "mixed":
        iv = g.iVox(1.0)
        for i in (0, 2):
            R, t = scene["gt"][i][:3, :3], scene["gt"][i][:3, 3]
            iv.insert(scene["pts"][i] @ R.T + t, R @ scene["covs"][i] @ R.T)
        keep = iv
        fs = [factor(g, scene, "VGICP", 0, 1, 0, 1), factor(g, scene, "GICP", 1, 2, 1, 2), factor(g, scene, "ICP", 2, 3, 2, 3),
              factor(g, scene, "ICP_PLANE", 0, 2, 0, 2), g.IntegratedGICPFactor(np.eye(4), 3, iv, scene["clouds"][3])]
        values = {i: poses[i] for i in range(4)}
        priors = [P(0, poses[0], [1e6, 1e6, 1e6, 1e5, 1e5, 1e5])]
    elif shape == "large_prior":
        fs = [factor(g, scene, "GICP", 0, 1, 0, 1)]
        values = {0: poses[0], 1: poses[1]}
        priors = [P(0, poses[0] @ syn.se3_exp(np.array([2.0, -1.2, 0.8, 0.5, 0.2, -0.3])), 10.0), P(1, poses[1], 1e6)]
    else:
        fs, values, gt, keep = ring_scene(g)
        priors = [P(0, gt[0], 1e6)]
    fset, res = run(g, fs, values, priors)
    assert res.iterations >= 1
    replay(fset, fs, values, priors, res)
    del keep  # the targets outlive the call


@pytest.mark.parametrize("method", ["VGICP", "GICP", "ICP"])
def test_alignment_shapes_meet_the_reference_gates(g, scene, method):
    poses, gt = scene["poses"], scene["gt"]
    P = g.PriorFactorPose3
    params = g.LevenbergMarquardtExtParams(maxIterations=100, relativeErrorTol=1e-6) if method == "ICP" else g.LevenbergMarquardtExtParams(maxIterations=30, relativeErrorTol=1e-4)

    def check(result, fixed_key, note):
        delta = gt[fixed_key] @ np.linalg.inv(result[fixed_key])
        for k, T in result.items():
            err_r, err_t = mini_lm.pose_error(delta @ T, gt[k])
            assert err_r < 0.015 and err_t < 0.15, (method, note, k, err_r, err_t)

    for i in range(2):
        for note, pk in (("FORWARD", i), ("BACKWARD", i + 1)):
            r = g.optimize_graph_gpu([factor(g, scene, method, i, i + 1, i, i + 1)], {i: poses[i], i + 1: poses[i + 1]}, [P(pk, poses[pk], 1e6)], params)
            check(r.values, pk, f"{note}_{i}")
        r = g.optimize_graph_gpu([factor(g, scene, method, poses[i], i + 1, i, i + 1)], {i + 1: poses[i + 1]}, (), params)
        check({i: poses[i], **r.values}, i, f"UNARY_{i}")
    r = g.optimize_graph_gpu([factor(g, scene, method, i - 1, i, i - 1, i) for i in range(1, 5)], {i: poses[i] for i in range(5)}, [P(0, poses[0], 1e6)], params)
    check(r.values, 0, "MULTI_FRAME")
    r = g.optimize_graph_gpu([factor(g, scene, method, i, j, i, j) for i in range(5) for j in range(i + 1, 5)], {i: poses[i] for i in range(5)},
                             [P(0, poses[0], 1e6)], params)
    check(r.values, 0, "FULL_CONNECTION")


def test_binary_members_follow_the_tolerance_rule_and_leave_the_host_state(g, scene):
    poses = scene["poses"]
    values = {i: poses[i] for i in range(3)}
    priors = [g.PriorFactorPose3(0, poses[0], 1e6)]
    sets = []
    for _ in range(2):
        fs = [factor(g, scene, "GICP", 0, 1, 0, 1), factor(g, scene, "ICP", 1, 2, 1, 2)]
        for f in fs:
            f.set_correspondence_update_tolerance(0.005, 0.05)
        fset = g.NonlinearFactorSetGPU(fs[0].ctx)
        fset.add(fs)
        fset._ensure()
        sets.append((fset, fs))
    (fa, fs), (fb, _) = sets
    res = g.optimize_graph_gpu(fa, values, priors, trace=True)
    topo, targets, hp = graph_of(fs, values, priors)
    ev = SetEvaluator(fb)
    ev.error(lg.deltas_at(topo, targets, [values[k] for k in range(3)]))
    outer = -1
    for e in res.trace:
        T_lin = list(e["T_lin"])
        if e["outer"] != outer:
            outer = e["outer"]
            ds = lg.deltas_at(topo, targets, T_lin)
            G, gv, _ = lg.assemble(ev.linearize(ds), topo, hp, T_lin, 3)
            mask = np.zeros(G.shape, dtype=bool)
            mask[:6, :6] = True  # the prior's block
            assert bits(G[~mask], e["G"][~mask]) and bits(gv[6:], e["g"][6:]), outer
            ev.error(ds)
        if e["solved"] and e["lin_change"] >= 0.0:
            ev.error(lg.deltas_at(topo, targets, list(e["T_trial"])))
    final = [res.values[k] for k in range(3)]
    T1 = [T @ syn.se3_exp(np.full(6, 1e-3)) for T in final]
    for T in (T1, final):
        ds = lg.deltas_at(topo, targets, T)
        la, lb = SetEvaluator(fa).linearize(ds), ev.linearize(ds)
        for ra, rb in zip(la, lb):
            assert all(bits(ra[k], rb[k]) for k in ("H_target", "H_source", "H_target_source", "b_target", "b_source", "error"))
        assert bits(SetEvaluator(fa).error(lg.deltas_at(topo, targets, T1)), ev.error(lg.deltas_at(topo, targets, T1)))


def test_reuse_across_topologies_priors_inserts_regroups_and_offload(g, scene):
    poses, P = scene["poses"], g.PriorFactorPose3
    L = capi.lib()
    iv = g.iVox(1.0)
    R, t = scene["gt"][0][:3, :3], scene["gt"][0][:3, 3]
    iv.insert(scene["pts"][0] @ R.T + t, R @ scene["covs"][0] @ R.T)
    vm = g.GaussianVoxelMapGPU(1.0)
    vm.insert(scene["clouds"][1])
    src2 = g.PointCloud(scene["pts"][2], scene["covs"][2], normals=g.estimate_normals(scene["pts"][2], scene["covs"][2]))
    fs = [g.IntegratedVGICPFactor(1, 2, vm, src2), g.IntegratedGICPFactor(np.eye(4), 1, iv, scene["clouds"][1])]
    fset = g.NonlinearFactorSetGPU(fs[0].ctx)
    fset.add(fs)
    fset._ensure()
    builds = lambda: L.b2_factor_set_lm_graph_builds(fset.h)  # noqa: E731
    assert builds() == 0
    v3 = {1: poses[1], 2: poses[2]}
    res = g.optimize_graph_gpu(fset, v3, [P(1, poses[1], 1e6)], trace=True)
    replay(fset, fs, v3, [P(1, poses[1], 1e6)], res)
    assert builds() == 1
    # no prior, the same capacities: the same graph
    res = g.optimize_graph_gpu(fset, {1: poses[1], 2: poses[2]}, [], trace=True)
    replay(fset, fs, {1: poses[1], 2: poses[2]}, [], res)
    assert builds() == 1 and np.all(np.isfinite(np.stack(list(res.values.values()))))
    # more priors than before: the prior buffers grow, the graph is captured again; then fewer priors reuse it
    pri2 = [P(1, poses[1], 1e6), P(2, poses[2], 1.0)]
    res = g.optimize_graph_gpu(fset, {1: poses[1], 2: poses[2]}, pri2, trace=True)
    replay(fset, fs, {1: poses[1], 2: poses[2]}, pri2, res)
    assert builds() == 2
    res = g.optimize_graph_gpu(fset, {1: poses[1], 2: poses[2]}, pri2[:1], trace=True)
    assert builds() == 2
    # another topology at the same capacities, through the C ABI: the binary member with its variables swapped and the unary
    # member on the other variable.  The topology is a per-call input: the same graph, and the replay holds for the new shape
    topo = [(1, 0), (-1, 1)]
    graph = (topo, [None, np.eye(4)], [(0, poses[1], np.full(6, 1e6))])
    res = raw_call(fset, *graph, [poses[1], poses[2]])
    assert builds() == 2 and res.termination != "none"
    replay(fset, fs, None, None, res, graph=graph)
    res = g.optimize_graph_gpu(fset, {1: poses[1], 2: poses[2]}, pri2[:1], trace=True)
    replay(fset, fs, {1: poses[1], 2: poses[2]}, pri2[:1], res)
    assert builds() == 2
    # an iVox insert re-associates the members and keeps the graph
    R, t = scene["gt"][3][:3, :3], scene["gt"][3][:3, 3]
    iv.insert(scene["pts"][3] @ R.T + t, R @ scene["covs"][3] @ R.T)
    res = g.optimize_graph_gpu(fset, {1: poses[1], 2: poses[2]}, pri2[:1], trace=True)
    replay(fset, fs, {1: poses[1], 2: poses[2]}, pri2[:1], res)
    assert builds() == 2
    # a surface-validation switch regroups the set: the graph is rebuilt
    fs[0].set_enable_surface_validation(True)
    res = g.optimize_graph_gpu(fset, {1: poses[1], 2: poses[2]}, pri2[:1], trace=True)
    replay(fset, fs, {1: poses[1], 2: poses[2]}, pri2[:1], res)
    assert builds() == 3
    # offloaded objects with offloading on: the call reloads them and runs the cached graph
    for f in fs:
        f.set_enable_offloading(True)
    vm.offload_gpu()
    src2.offload_gpu()
    res = g.optimize_graph_gpu(fset, {1: poses[1], 2: poses[2]}, pri2[:1], trace=True)
    assert vm.loaded_on_gpu() and src2.loaded_on_gpu() and builds() == 3
    replay(fset, fs, {1: poses[1], 2: poses[2]}, pri2[:1], res)
    # a larger graph on the same set: a third variable held by a prior alone (more poses: captured again)
    v4 = {0: poses[0], 1: poses[1], 2: poses[2]}
    res = g.optimize_graph_gpu(fset, v4, [P(0, poses[0], 1e6)], trace=True)
    assert builds() == 4
    replay(fset, fs, v4, [P(0, poses[0], 1e6)], res)


def test_gauge_free_graph_ends_finite(g, scene):
    poses = scene["poses"]
    fs = [factor(g, scene, "GICP", i - 1, i, i - 1, i) for i in range(1, 4)]
    values = {i: poses[i] for i in range(4)}
    fset, res = run(g, fs, values)
    assert res.termination in ("absolute_error_tol", "relative_error_tol", "max_iterations")
    assert all(np.all(np.isfinite(T)) for T in res.values.values())
    replay(fset, fs, values, [], res)
    # the relative poses converge as with a prior on frame 0
    _, ref = run(g, [factor(g, scene, "GICP", i - 1, i, i - 1, i) for i in range(1, 4)], values, [g.PriorFactorPose3(0, poses[0], 1e6)])
    for k in range(1, 4):
        a = np.linalg.inv(res.values[0]) @ res.values[k]
        b = np.linalg.inv(ref.values[0]) @ ref.values[k]
        err_r, err_t = mini_lm.pose_error(a, b)
        assert err_r < 2e-3 and err_t < 2e-2, (k, err_r, err_t)


def test_topology_errors_are_refused_before_device_work(g, scene):
    fs = [factor(g, scene, "GICP", 0, 1, 0, 1), factor(g, scene, "GICP", scene["gt"][0], 1, 0, 1)]
    fset = g.NonlinearFactorSetGPU(fs[0].ctx)
    fset.add(fs)
    fset._ensure()
    L = capi.lib()
    p = g.LevenbergMarquardtExtParams().to_c()
    T = np.ascontiguousarray(np.stack([np.eye(4)] * 3))
    out = np.zeros((3, 4, 4))
    targets = np.ascontiguousarray(np.stack([np.eye(4)] * 2))

    def call(vars_, N=2, tg=targets):
        v = np.ascontiguousarray(np.asarray(vars_, dtype=np.int32))
        st = L.b2_factor_set_optimize_poses(fset.h, N, v.ctypes.data_as(C.POINTER(C.c_int32)), capi.dptr(tg) if tg is not None else None, None, 0, capi.dptr(T), C.byref(p),
                                            capi.dptr(out), None, None, None, 0, None)
        return st, L.b2_last_error().decode()

    for vars_, N, tg, msg in [([[0, 1], [-1, 2]], 2, targets, "source_var"), ([[2, 1], [-1, 1]], 2, targets, "target_var"), ([[-2, 1], [-1, 1]], 2, targets, "target_var"),
                              ([[1, 1], [-1, 1]], 2, targets, "target_var == source_var"), ([[0, 1], [-1, 1]], 3, targets, "variable 2"),
                              ([[0, 1], [-1, 1]], 2, None, "T_targets is NULL")]:
        st, err = call(vars_, N, tg)
        assert st == 1 and msg in err, (vars_, err)
    bad = targets.copy()
    bad[1, 0, 0] = np.nan
    assert call([[0, 1], [-1, 1]], 2, bad)[0] == 1
    assert L.b2_factor_set_lm_graph_builds(fset.h) == 0 and fset.launch_count() == 0
    # a valid call on the same set works, and T_targets may be NULL when every member is binary
    st, err = call([[0, 1], [-1, 1]], 2, targets)
    assert st == 0, err
    fset2 = g.NonlinearFactorSetGPU(fs[0].ctx)
    fset2.add([factor(g, scene, "GICP", 0, 1, 0, 1)])
    fset2._ensure()
    v = np.array([[0, 1]], dtype=np.int32)
    assert L.b2_factor_set_optimize_poses(fset2.h, 2, v.ctypes.data_as(C.POINTER(C.c_int32)), None, None, 0, capi.dptr(T), C.byref(p), capi.dptr(out), None, None, None, 0,
                                          None) == 0
