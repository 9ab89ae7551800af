"""Frame-to-map odometry timing of iVoxCovarianceEstimation on one GPU: align a frame against the map with GICP, insert it at its
pose (without covariances: the map estimates them).

Workloads: a synthetic scene (synthetic.make_cloud) scanned along a trajectory at 20k and 120k points per frame, and the five
KITTI-07 submaps of tests/golden.  Per frame it reports medians of:
  * insert, end to end, and its device phases by CUDA events (b2_ivox_insert_timings): base insert, estimation pass,
    statistics, removal of old invalid points with the valid view;
  * linearize and error of a GICP factor on the map: kernel time by CUDA events on the context's stream, and end to end;
  * the host restatement (tests/ivox_cov_np.py) doing the same insert (numpy, one process; KITTI and the 20k loop only by default);
  * with --factor icp or plane, also linearize and error of a point-to-point or point-to-plane ICP factor on the same map and
    frame (icp_* / plane_* keys), next to GICP in the same run.  A point-to-plane factor turns on the map's plane view, which
    every later insert rewrites in its last phase (removal_ms): the insert columns then include it.
Prints the card name, power limit and max SM clock of the same run.

  python scripts/bench_ivox_cov.py [--frames 12] [--sizes 20000 120000] [--host-max 20000] [--factor gicp|icp|plane]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import gtsam_points_b200 as g  # noqa: E402
import ivox_cov_np  # noqa: E402
from gtsam_points_b200 import capi  # noqa: E402
from gtsam_points_b200 import synthetic as syn  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def synthetic_frames(n, count, seed=7):
    rng = np.random.default_rng(seed)
    T, out = np.eye(4), []
    for f in range(count):
        p, c = syn.make_cloud(n, stream=f, scale=1.0)
        T = T @ syn.se3_exp(np.concatenate([rng.uniform(-0.02, 0.02, 3), [0.8, rng.uniform(-0.1, 0.1), 0.0]]))
        out.append((np.asarray(p, dtype=np.float64), np.asarray(c, dtype=np.float64), T.copy()))
    return out


def kitti_frames():
    z = np.load(os.path.join(ROOT, "tests", "golden", "kitti07_frames.npz"))
    out = []
    for i in range(5):
        p = z[f"points{i}"].astype(np.float64)
        c = g.estimate_covariances(p, 10)  # source covariances of the alignment; the map itself gets points only
        out.append((p, c, z["poses_gt"][i]))
    return out


def kernel_ms(stream, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b)


def wall_ms(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def factor_times(stream, fac, delta, d_out):
    """(linearize kernel, linearize end to end, error kernel, error end to end) in ms; the factor has been linearized once."""
    lin_k = kernel_ms(stream, lambda: capi.check(capi.lib().b2_factor_issue_linearize(fac.h, capi.dptr(delta), C.c_void_p(d_out.data_ptr()))))
    lin_e = wall_ms(lambda: fac.linearize({1: delta}))
    err_k = kernel_ms(stream, lambda: capi.check(capi.lib().b2_factor_issue_error(fac.h, capi.dptr(delta), C.c_void_p(d_out.data_ptr()))))
    err_e = wall_ms(lambda: fac.error({1: delta}))
    return lin_k, lin_e, err_k, err_e


def run(name, fr, host, factor="gicp"):
    stream = torch.cuda.current_stream()
    ctx = g.Context(0, stream.cuda_stream)
    m = g.iVoxCovarianceEstimation(1.0, ctx=ctx)
    ref = ivox_cov_np.IvoxCovNp(1.0) if host else None
    d_out = torch.zeros(capi.B2_LINEARIZED_DOUBLES, dtype=torch.float64, device="cuda")
    keys = ("insert_e2e_ms", "base_insert_ms", "estimation_ms", "statistics_ms", "removal_ms", "lin_kernel_ms", "lin_e2e_ms", "err_kernel_ms", "err_e2e_ms", "host_insert_ms")
    extra = tuple(f"{factor}_{k}" for k in ("lin_kernel_ms", "lin_e2e_ms", "err_kernel_ms", "err_e2e_ms")) if factor != "gicp" else ()
    rec = {k: [] for k in keys + extra}
    warm = 1 if len(fr) <= 5 else 2
    for f, (p, c, T) in enumerate(fr):
        R, t = T[:3, :3], T[:3, 3]
        world = p @ R.T + t
        if f > 0 and len(m.valid_indices()) > 0:
            src = g.PointCloud(p, c, ctx=ctx)
            delta = np.ascontiguousarray(T @ syn.random_pose(np.random.default_rng(f), 0.01, 0.1))
            fac = g.IntegratedGICPFactor(np.eye(4), 1, m, src, ctx=ctx)
            fac.linearize({1: delta})
            lin_k, lin_e, err_k, err_e = factor_times(stream, fac, delta, d_out)
            if extra:
                ifac = g.IntegratedICPFactor(np.eye(4), 1, m, g.PointCloud(p, ctx=ctx), use_point_to_plane=factor == "plane", ctx=ctx)
                ifac.linearize({1: delta})
                times = factor_times(stream, ifac, delta, d_out)
            if f >= warm:
                rec["lin_kernel_ms"].append(lin_k)
                rec["lin_e2e_ms"].append(lin_e)
                rec["err_kernel_ms"].append(err_k)
                rec["err_e2e_ms"].append(err_e)
                for k, v in zip(extra, times if extra else ()):
                    rec[k].append(v)
        e2e = wall_ms(lambda: m.insert(world))
        ph = m.insert_timings()
        h = wall_ms(lambda: ref.insert(world)) if ref is not None else None
        if f >= warm:
            rec["insert_e2e_ms"].append(e2e)
            rec["base_insert_ms"].append(ph["base_insert"])
            rec["estimation_ms"].append(ph["estimation"])
            rec["statistics_ms"].append(ph["statistics"])
            rec["removal_ms"].append(ph["removal"])
            if h is not None:
                rec["host_insert_ms"].append(h)
    info = m.info()
    out = {k: (float(np.median(v)) if v else None) for k, v in rec.items()}
    out.update(workload=name, frames=len(fr), timed_frames=len(fr) - warm, map_voxels=int(info.num_voxels), map_points=int(info.num_points), valid_points=int(len(m.valid_indices())))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--sizes", type=int, nargs="+", default=[20000, 120000])
    ap.add_argument("--host-max", type=int, default=20000, help="largest synthetic frame size the host restatement also runs")
    ap.add_argument("--factor", choices=("gicp", "icp", "plane"), default="gicp", help="icp / plane: also time that ICP factor on the map, next to GICP")
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    for n in a.sizes:
        print(json.dumps(run(f"synthetic {n} pts/frame", synthetic_frames(n, a.frames), n <= a.host_max, a.factor)))
    print(json.dumps(run("KITTI-07 submaps", kitti_frames(), True, a.factor)))


if __name__ == "__main__":
    main()
