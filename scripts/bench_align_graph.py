"""What running the whole Levenberg-Marquardt loop of a pose graph on the device costs: b2_factor_set_optimize_poses (one CUDA graph
launch per optimization) against the same rules as a compiled host loop over the C ABI (scripts/bench_align_graph_host.cpp: one
blocking b2_factor_set_linearize per outer iteration, one blocking b2_factor_set_error for error0, each outer iteration's E and each
tried step, and the same dense 6N solve), alternated in one run on five graphs:

  vgicp1m          one pose: one unary VGICP factor, 1M source points, 0.5 m Gaussian voxel map of a 1M-point target (synthetic
                   clouds);
  ivoxcov          one pose: one unary GICP factor of a 20k-point KITTI-07 frame (frame 1) against an iVoxCovarianceEstimation
                   holding frames 0, 2, 3, 4 (the frame-to-map step of odometry);
  multi_frame      the five KITTI-07 frames, four binary VGICP factors (i - 1 -> i, 1.0 m voxels) and a Pose3 prior on frame 0
                   (the reference AlignmentTest's MULTI_FRAME graph);
  full_connection  the same frames with a binary VGICP factor between every pair (10 factors) and the prior: the full-connection
                   graph of demo_matching_cost_factors.cpp;
  ring32           32 frames of a 6000-point synthetic scene on a circle, a binary GICP factor between neighbours (32 factors,
                   closing the loop) and a prior on frame 0: the largest graph the optimizer takes.

Each arm has its own factor set over the same objects and starts every optimization from the same poses.  Reported per graph: median
wall time per optimization; the device arm's first call on a fresh set (graph capture and instantiation included) apart from its
steady state; iterations (accepted / tryLambda calls) and kernel launches per optimization in both arms (device: the graph's kernel
nodes executed, from the call's counts and the set's launches per group pass; host: the set's launch counter); the host arm's time
inside the C ABI calls; whether the two arms end on the same pose bits (the priors' transcendental functions may differ in the last
bits between CUDA and glibc, so a difference of a few ulps is expected there); and, from a separate torch.profiler run, the mean time
of the lm_solve and lm_reduce kernels.  Prints the card name, power limit and max SM clock of the same run, then one JSON line.

  python scripts/bench_align_graph.py [--reps 10] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import gtsam_points_b200 as g  # noqa: E402
import native  # noqa: E402
from gtsam_points_b200 import capi  # noqa: E402
from gtsam_points_b200 import synthetic as syn  # noqa: E402
from gtsam_points_b200.optimize import _graph_inputs  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    if not q.strip():
        raise RuntimeError("nvidia-smi reports no GPU: this benchmark measures on the device only")
    return q.strip().splitlines()[0]


def host_loop():
    """lm_graph_host of scripts/bench_align_graph_host.cpp, compiled into a temporary directory (the tree may be read-only)"""
    inc, lib = os.path.join(ROOT, "include"), os.path.join(ROOT, "gtsam_points_b200", "lib")
    L = native.shared_library([os.path.join(ROOT, "scripts", "bench_align_graph_host.cpp"), os.path.join(lib, "libb2points.so")],
                              ["-O3", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-I", inc, f"-Wl,-rpath,{lib}"])
    fn = L.lm_graph_host
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_int32), capi._dp, C.c_size_t, C.POINTER(capi.PosePriorC), C.c_size_t, capi._dp,
                   C.POINTER(capi.LmParamsC), capi._dp, C.POINTER(C.c_int64), C.POINTER(C.c_double)]
    return fn


def kitti(pairs):
    z = np.load(os.path.join(ROOT, "tests", "golden", "kitti07_frames.npz"))
    pts = [z[f"points{i}"].astype(np.float64) for i in range(5)]
    clouds = [g.PointCloud(p, g.estimate_covariances(p, 10)) for p in pts]
    maps = []
    for c in clouds:
        vm = g.GaussianVoxelMapGPU(1.0)
        vm.insert(c)
        maps.append(vm)
    make = lambda: [g.IntegratedVGICPFactor(t, s, maps[t], clouds[s]) for t, s in pairs]  # noqa: E731
    values = {i: z["poses"][i] for i in range(5)}
    return make, values, [g.PriorFactorPose3(0, z["poses"][0], 1e6)], (clouds, maps)


def vgicp1m():
    tp, tc = syn.make_cloud(1_000_000, stream=1, scale=0.25)
    sp, sc = syn.make_cloud(1_000_000, stream=2, scale=0.25)
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(g.PointCloud(tp, tc))
    src = g.PointCloud(sp, sc)
    make = lambda: [g.IntegratedVGICPFactor(np.eye(4), 1, vm, src)]  # noqa: E731
    return make, {1: syn.random_pose(np.random.default_rng(1), 0.02, 0.2)}, [], (vm, src)


def ivoxcov():
    z = np.load(os.path.join(ROOT, "tests", "golden", "kitti07_frames.npz"))
    gt = z["poses_gt"]
    iv = g.iVoxCovarianceEstimation(1.0)
    for i in (0, 2, 3, 4):
        p = z[f"points{i}"].astype(np.float64)
        iv.insert(p @ gt[i][:3, :3].T + gt[i][:3, 3])
    sp = z["points1"].astype(np.float64)
    sp = sp[np.random.default_rng(0).permutation(len(sp))[:20000]]
    src = g.PointCloud(sp, g.estimate_covariances(sp, 10))
    make = lambda: [g.IntegratedGICPFactor(np.eye(4), 1, iv, src)]  # noqa: E731
    return make, {1: gt[1] @ syn.se3_exp(np.random.default_rng(2).uniform(-0.05, 0.05, 6))}, [], (iv, src)


def multi_frame():
    return kitti([(i - 1, i) for i in range(1, 5)])


def full_connection():
    return kitti([(i, j) for i in range(5) for j in range(i + 1, 5)])


def ring32(n=32):
    pts, covs = syn.make_cloud(6000, stream=71, scale=0.3)
    rng = np.random.default_rng(3)
    gt, clouds, trees = [], [], []
    for k in range(n):
        a = 2 * np.pi * k / n
        T = syn.se3_exp(np.array([0.0, 0.0, a, 0.0, 0.0, 0.0]))
        T[:3, 3] = [3.0 * np.cos(a), 3.0 * np.sin(a), 0.1 * np.sin(3 * a)]
        gt.append(T)
        R, t = T[:3, :3], T[:3, 3]
        c = g.PointCloud((pts - t) @ R, R.T @ covs @ R)
        clouds.append(c)
        trees.append(g.KdTree(c))
    make = lambda: [g.IntegratedGICPFactor(k, (k + 1) % n, clouds[k], clouds[(k + 1) % n], trees[k]) for k in range(n)]  # noqa: E731
    values = {k: gt[k] @ syn.se3_exp(rng.uniform(-0.02, 0.02, 6)) for k in range(n)}
    return make, values, [g.PriorFactorPose3(0, gt[0], 1e6)], (clouds, trees)


def kernel_times(fset, values, priors):
    """mean device time (ms) of lm_solve_kernel and lm_reduce_kernel over a few optimizations, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            g.optimize_graph_gpu(fset, values, priors)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("lm_solve_kernel", "lm_reduce_kernel"):
            if k in e.key:
                total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                out[k] = total / max(e.count, 1) / 1e3
    return {k: out.get(k) for k in ("lm_solve_kernel", "lm_reduce_kernel")}


def run(name, setup, reps, warmup, lm_host):
    make, values, priors, keep = setup()
    fs_dev, fs_host = make(), make()
    dev_set, host_set = g.NonlinearFactorSetGPU(), g.NonlinearFactorSetGPU()
    dev_set.add(fs_dev)
    host_set.add(fs_host)
    dev_set._ensure()
    host_set._ensure()
    _, keys, mv, targets, pri, T0 = _graph_inputs(fs_host, values, priors)
    N, F = len(keys), len(fs_host)
    params = g.LevenbergMarquardtExtParams().to_c()
    # kernel launches of one pass over the set's groups (one b2_factor_set_error call)
    n0 = host_set.launch_count()
    capi.check(capi.lib().b2_factor_set_error(host_set.h, capi.dptr(np.ascontiguousarray(np.stack([np.eye(4)] * F))), capi.dptr(np.zeros(F))))
    groups = host_set.launch_count() - n0
    t = time.perf_counter()
    g.optimize_graph_gpu(dev_set, values, priors)  # the first call on the set captures and instantiates its graph
    first_ms = (time.perf_counter() - t) * 1e3
    dev_t, host_t, abi_t, dev_it, host_it, dev_l, host_l, same, diffs = [], [], [], [], [], [], [], [], []
    for r in range(warmup + reps):
        t = time.perf_counter()
        res = g.optimize_graph_gpu(dev_set, values, priors)
        td = time.perf_counter() - t
        n0 = host_set.launch_count()
        T_host, counts, abi = np.zeros((N, 4, 4)), (C.c_int64 * 3)(), C.c_double()
        t = time.perf_counter()
        capi.check(lm_host(host_set.h, N, mv.ctypes.data_as(C.POINTER(C.c_int32)), capi.dptr(targets), F, pri, len(priors), capi.dptr(T0), C.byref(params),
                           capi.dptr(T_host), counts, C.byref(abi)))
        th = time.perf_counter() - t
        if r < warmup:
            continue
        T_dev = np.stack([res.values[k] for k in keys])
        dev_t.append(td * 1e3)
        host_t.append(th * 1e3)
        abi_t.append(abi.value * 1e3)
        dev_it.append((res.iterations, res.inner_iterations))
        host_it.append((counts[0], counts[2]))
        # setup + error groups + init; per outer: linearize + error groups + reduce; per inner: solve + error groups + decide
        dev_l.append(2 + groups + res.outer_iterations * (2 * groups + 1) + res.inner_iterations * (groups + 2))
        host_l.append(host_set.launch_count() - n0)
        same.append(bool(np.array_equal(T_dev.view(np.int64), T_host.view(np.int64))))
        diffs.append(float(np.abs(T_dev - T_host).max()))
    kt = kernel_times(dev_set, values, priors)
    out = dict(workload=name, poses=N, factors=F, priors=len(priors), device_ms=statistics.median(dev_t), device_first_call_ms=first_ms,
               host_ms=statistics.median(host_t), host_abi_ms=statistics.median(abi_t), device_iterations=dev_it[-1], host_iterations=host_it[-1],
               device_kernel_nodes=dev_l[-1], host_launches=host_l[-1], same_pose_bits=all(same), max_pose_diff=max(diffs),
               lm_solve_ms=kt["lm_solve_kernel"], lm_reduce_ms=kt["lm_reduce_kernel"])
    print(f"{name} (N={N}, F={F}): device {out['device_ms']:.3f} ms (first call {first_ms:.3f} ms; {dev_it[-1][0]} accepted / {dev_it[-1][1]} tryLambda, "
          f"{dev_l[-1]} kernel nodes; lm_solve {kt['lm_solve_kernel']} ms, lm_reduce {kt['lm_reduce_kernel']} ms)  host loop {out['host_ms']:.3f} ms, "
          f"of which {out['host_abi_ms']:.3f} ms in C ABI calls ({host_it[-1][0]} / {host_it[-1][1]}, {host_l[-1]} launches)  same pose bits {all(same)}, "
          f"max |dT| {out['max_pose_diff']:.2e}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    c = card()
    print("card:", c)
    lm_host = host_loop()
    workloads = (("vgicp1m", vgicp1m), ("ivoxcov", ivoxcov), ("multi_frame", multi_frame), ("full_connection", full_connection), ("ring32", ring32))
    results = [run(n, f, a.reps, a.warmup, lm_host) for n, f in workloads]
    print(json.dumps(dict(card=c, results=results)))


if __name__ == "__main__":
    main()
