"""What running the whole Levenberg-Marquardt loop on the device saves: b2_factor_set_optimize_pose (one CUDA graph launch per
optimization) against the same rules as a compiled host loop over the C ABI (scripts/bench_align_host.cpp: one blocking
b2_factor_set_linearize per outer iteration, one blocking b2_factor_set_error for error0, each outer iteration's E and each tried
step), alternated in one run on two workloads:

  vgicp1m   one VGICP factor, 1M source points, 0.5 m Gaussian voxel map of a 1M-point target (synthetic clouds);
  ivoxcov   one GICP factor of a 20k-point KITTI-07 frame (frame 1) against an iVoxCovarianceEstimation holding frames 0, 2, 3, 4
            (the frame-to-map step of odometry).

Each arm has its own factor set over the same objects and starts every optimization from the same pose.  Reported per arm: median
wall time per optimization, iterations (accepted / tryLambda calls) and kernel launches per optimization (host arm: the set's launch
counter; device arm: the graph's kernel nodes executed, from the call's counts).  The host arm's time inside the C ABI calls is
reported apart from its total, so what its own loop costs is visible; the device arm's first call on a fresh set (graph capture and
instantiation included) is reported apart from the steady state.  Prints the card name, power limit and max SM clock of the same run,
then one JSON line.

  python scripts/bench_align.py [--reps 10] [--warmup 2]
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    if not q.strip():
        raise RuntimeError("nvidia-smi reports no GPU: this benchmark measures on the device only")
    return q.strip().splitlines()[0]


def host_loop():
    """lm_host of scripts/bench_align_host.cpp, compiled into a temporary directory (the tree may be read-only)"""
    inc, lib = os.path.join(ROOT, "include"), os.path.join(ROOT, "gtsam_points_b200", "lib")
    # the library after the source on the link line, so that the linker resolves the C ABI calls against it
    L = native.shared_library([os.path.join(ROOT, "scripts", "bench_align_host.cpp"), os.path.join(lib, "libb2points.so")],
                              ["-O3", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-I", inc, f"-Wl,-rpath,{lib}"])
    fn = L.lm_host
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, capi._dp, C.c_size_t, capi._dp, C.POINTER(capi.LmParamsC), capi._dp, C.POINTER(C.c_int64), C.POINTER(C.c_double)]
    return fn


def vgicp1m():
    tp, tc = syn.make_cloud(1_000_000, stream=1, scale=0.25)
    sp, sc = syn.make_cloud(1_000_000, stream=2, scale=0.25)
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(g.PointCloud(tp, tc))
    src = g.PointCloud(sp, sc)
    make = lambda: g.IntegratedVGICPFactor(np.eye(4), 1, vm, src)  # noqa: E731
    return make, np.eye(4), syn.random_pose(np.random.default_rng(1), 0.02, 0.2), (vm, src)


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
    make = lambda: g.IntegratedGICPFactor(np.eye(4), 1, iv, src)  # noqa: E731
    return make, np.eye(4), gt[1] @ syn.se3_exp(np.random.default_rng(2).uniform(-0.05, 0.05, 6)), (iv, src)


def run(name, setup, reps, warmup, lm_host):
    make, T_target, T0, keep = setup()
    dev_set, host_set = g.NonlinearFactorSetGPU(), g.NonlinearFactorSetGPU()
    dev_set.add(make())
    host_set.add(make())
    dev_set._ensure()
    host_set._ensure()
    groups = 1
    params = g.LevenbergMarquardtExtParams().to_c()
    targets = np.ascontiguousarray(T_target.reshape(1, 4, 4))
    T0 = np.ascontiguousarray(T0)
    t = time.perf_counter()
    g.optimize_pose_gpu(dev_set, T0)  # the first call on the set captures and instantiates its graph
    first_ms = (time.perf_counter() - t) * 1e3
    dev_t, host_t, abi_t, dev_it, host_it, dev_l, host_l, poses = [], [], [], [], [], [], [], []
    for r in range(warmup + reps):
        t = time.perf_counter()
        res = g.optimize_pose_gpu(dev_set, T0)
        td = time.perf_counter() - t
        n0 = host_set.launch_count()
        T_host, counts, abi = np.zeros((4, 4)), (C.c_int64 * 3)(), C.c_double()
        t = time.perf_counter()
        capi.check(lm_host(host_set.h, capi.dptr(targets), 1, capi.dptr(T0), C.byref(params), capi.dptr(T_host), counts, C.byref(abi)))
        th = time.perf_counter() - t
        if r < warmup:
            continue
        dev_t.append(td * 1e3)
        host_t.append(th * 1e3)
        abi_t.append(abi.value * 1e3)
        dev_it.append((res.iterations, res.inner_iterations))
        host_it.append((counts[0], counts[2]))
        # setup + error groups + init; per outer: linearize + error groups + reduce; per inner: solve + error groups + decide
        dev_l.append(2 + groups + res.outer_iterations * (2 * groups + 1) + res.inner_iterations * (groups + 2))
        host_l.append(host_set.launch_count() - n0)
        poses.append(float(np.abs(res.pose - T_host).max()))
    out = dict(workload=name, device_ms=statistics.median(dev_t), device_first_call_ms=first_ms, host_ms=statistics.median(host_t),
               host_abi_ms=statistics.median(abi_t), device_iterations=dev_it[-1], host_iterations=host_it[-1], device_launches=dev_l[-1],
               host_launches=host_l[-1], max_pose_diff=max(poses))
    print(f"{name}: device {out['device_ms']:.3f} ms (first call on the set {first_ms:.3f} ms; {dev_it[-1][0]} accepted / {dev_it[-1][1]} tryLambda, "
          f"{dev_l[-1]} kernels)  host loop {out['host_ms']:.3f} ms, of which {out['host_abi_ms']:.3f} ms in C ABI calls ({host_it[-1][0]} / {host_it[-1][1]}, "
          f"{host_l[-1]} launches)  max |dT| {out['max_pose_diff']:.2e}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    c = card()
    print("card:", c)
    lm_host = host_loop()
    results = [run("vgicp1m", vgicp1m, a.reps, a.warmup, lm_host), run("ivoxcov", ivoxcov, a.reps, a.warmup, lm_host)]
    print(json.dumps(dict(card=c, results=results)))


if __name__ == "__main__":
    main()
