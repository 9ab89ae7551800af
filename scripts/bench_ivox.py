"""Frame-to-map odometry timing of the iVox path on one GPU (the loop of the reference's advanced_scan_matching example:
align a frame against the map with GICP, transform it, insert it).

A synthetic scene (synthetic.make_cloud) is scanned along a trajectory, N points per frame, and inserted into an iVox at
1.0 m resolution.  Per frame it times:
  * insert (host points and covariances in, map updated);
  * linearize and error of an iVox GICP factor: kernel time by CUDA events on the context's stream, and end to end;
  * the alternative a kd-tree user has: rebuild a device kd-tree (and the GICP target cloud) over the same map points,
    then linearize -- end to end, and its linearize kernel;
  * the oracle's kd-tree GICP over the same map points on the host cores (tree build + linearize);
  * with --factor icp, also linearize and error of a point-to-point ICP factor on the same map and frame (icp_* keys), next to
    GICP in the same run.
Medians over the timed frames; map size at the end.  Prints the card name, power limit and max SM clock of the same run.

  python scripts/bench_ivox.py [--frames 12] [--sizes 20000 120000] [--factor gicp|icp]
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
import oracle_lib as orc  # noqa: E402
from gtsam_points_b200 import capi  # noqa: E402
from gtsam_points_b200 import synthetic as syn  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def frames(n, count, seed=7):
    rng = np.random.default_rng(seed)
    T, out = np.eye(4), []
    for f in range(count):
        p, c = syn.make_cloud(n, stream=f, scale=1.0)
        T = T @ syn.se3_exp(np.concatenate([rng.uniform(-0.02, 0.02, 3), [0.8, rng.uniform(-0.1, 0.1), 0.0]]))
        out.append((np.asarray(p, dtype=np.float64), np.asarray(c, dtype=np.float64), T.copy()))
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


def run(n, count, threads, factor="gicp"):
    stream = torch.cuda.current_stream()
    ctx = g.Context(0, stream.cuda_stream)
    ivox = g.iVox(1.0, ctx=ctx)
    d_out = torch.zeros(capi.B2_LINEARIZED_DOUBLES, dtype=torch.float64, device="cuda")
    rec = {k: [] for k in ("insert_ms", "lin_kernel_ms", "lin_e2e_ms", "err_kernel_ms", "err_e2e_ms", "kd_rebuild_lin_e2e_ms", "kd_lin_kernel_ms", "host_oracle_ms")}
    icp_keys = ("icp_lin_kernel_ms", "icp_lin_e2e_ms", "icp_err_kernel_ms", "icp_err_e2e_ms")
    if factor == "icp":
        rec.update({k: [] for k in icp_keys})
    fr = frames(n, count)
    for f, (p, c, T) in enumerate(fr):
        R, t = T[:3, :3], T[:3, 3]
        world_p, world_c = p @ R.T + t, R @ c @ R.T
        world_c = 0.5 * (world_c + world_c.transpose(0, 2, 1))
        if f > 0:
            # align this frame (a slightly perturbed pose) against the map before it is inserted
            src = g.PointCloud(p, c, ctx=ctx)
            delta = np.ascontiguousarray(T @ syn.random_pose(np.random.default_rng(f), 0.01, 0.1))
            fac = g.IntegratedGICPFactor(np.eye(4), 1, ivox, src, ctx=ctx)
            fac.linearize({1: delta})  # first call builds the factor's launch set
            lin_k, lin_e, err_k, err_e = factor_times(stream, fac, delta, d_out)
            if factor == "icp":
                ifac = g.IntegratedICPFactor(np.eye(4), 1, ivox, g.PointCloud(p, ctx=ctx), ctx=ctx)
                ifac.linearize({1: delta})
                icp = factor_times(stream, ifac, delta, d_out)
            m = ivox.download()
            mp, mc = m["points"], m["covs"]

            def kd_path():
                tgt = g.PointCloud(mp, mc, ctx=ctx)
                kf = g.IntegratedGICPFactor(np.eye(4), 1, tgt, src, target_tree=g.KdTree(tgt, ctx=ctx), ctx=ctx)
                kf.linearize({1: delta})
                return kf

            kd_e = wall_ms(kd_path)
            kf = kd_path()
            kd_k = kernel_ms(stream, lambda: capi.check(capi.lib().b2_factor_issue_linearize(kf.h, capi.dptr(delta), C.c_void_p(d_out.data_ptr()))))

            def host():
                oc, os_ = orc.Cloud(mp, mc), orc.Cloud(p, c)
                of = orc.Factor(oc, os_, tree=orc.KdTree(oc, threads), num_threads=threads)
                of.linearize(delta)

            host_ms = wall_ms(host) if f % 3 == 1 else None
            if f >= 2:  # frame 1 warms up
                rec["lin_kernel_ms"].append(lin_k)
                rec["lin_e2e_ms"].append(lin_e)
                rec["err_kernel_ms"].append(err_k)
                rec["err_e2e_ms"].append(err_e)
                rec["kd_rebuild_lin_e2e_ms"].append(kd_e)
                rec["kd_lin_kernel_ms"].append(kd_k)
                if factor == "icp":
                    for k, v in zip(icp_keys, icp):
                        rec[k].append(v)
                if host_ms is not None:
                    rec["host_oracle_ms"].append(host_ms)
        ins = wall_ms(lambda: ivox.insert(world_p, world_c))
        if f >= 2:
            rec["insert_ms"].append(ins)
    info = ivox.info()
    out = {k: (float(np.median(v)) if v else None) for k, v in rec.items()}
    out.update(n_per_frame=n, frames=count, timed_frames=count - 2, map_voxels=int(info.num_voxels), map_points=int(info.num_points), host_threads=threads)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--sizes", type=int, nargs="+", default=[20000, 120000])
    ap.add_argument("--factor", choices=("gicp", "icp"), default="gicp", help="icp: also time point-to-point ICP on the map, next to GICP")
    a = ap.parse_args()
    threads = max(1, min(os.cpu_count() or 1, orc.max_threads()))
    print(json.dumps({"card": card()}))
    for n in a.sizes:
        print(json.dumps(run(n, a.frames, threads, a.factor)))


if __name__ == "__main__":
    main()
