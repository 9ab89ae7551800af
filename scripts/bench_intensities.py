"""What carrying intensities costs on one GPU: a 1M-point posed insert into the Gaussian voxel map (b2_voxelmap_insert_cloud) and a
1M-point voxel-grid downsampling (b2_cloud_create_voxelgrid[_with_intensities]), each with and without per-point intensities.

Inputs: synthetic frames (synthetic.make_cloud with covariances) of 1M points, each with a random pose; the intensities are random
doubles that are not float32-exact (float64 storage, the costlier case).
  (1) wall time: medians per C ABI call over --reps calls after one warm-up call per arm, the two arms alternating.  Every call ends
      in a stream synchronise inside the library.  The voxel-grid call includes its host-to-device upload of the scan (points,
      covariances and, in the second arm, intensities); no result is downloaded.  The two maps' voxels are asserted equal.
  (2) device time: a profiled run of its own (torch.profiler, CUDA activities) of --reps calls per arm: per call, the summed device
      time of every kernel, of the kernels that differ between the arms (voxel_sum_kernel, insert_voxels_kernel and the intensity
      kernels), and of the host-to-device copies.
Prints the card name, power limit and max SM clock of the same run, then one JSON line per case.

  python scripts/bench_intensities.py [--reps 9]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import gtsam_points_b200 as g  # noqa: E402
from gtsam_points_b200 import capi  # noqa: E402
from gtsam_points_b200 import synthetic as syn  # noqa: E402

WATCHED = ("voxel_sum_kernel", "insert_voxels_kernel", "intensities_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def wall_ms(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def voxelgrid_call(ctx, pts, covs, ints, res):
    """b2_cloud_create_voxelgrid_with_intensities (ints None: without), the new cloud destroyed at once."""
    h = C.c_void_p()
    capi.check(capi.lib().b2_cloud_create_voxelgrid_with_intensities(ctx.h, res, capi.dptr(pts), 3, capi.dptr(covs), 9, None, 0, None if ints is None else capi.dptr(ints),
                                                                     len(pts), 0, C.byref(h)))
    n = C.c_int()
    capi.check(capi.lib().b2_cloud_intensity_bytes(h, C.byref(n)))
    capi.lib().b2_cloud_destroy(h)
    return n.value


def device_us(fn, reps):
    """Per call: (all kernels, each watched kernel, host-to-device copies) in us of device time, from a profiled run of `reps` calls."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    total, h2d, watched = 0.0, 0.0, defaultdict(float)
    for e in prof.events():
        if e.device_time <= 0:
            continue
        if "Memcpy HtoD" in e.name:
            h2d += e.device_time
        elif "Memcpy" not in e.name and "Memset" not in e.name:
            total += e.device_time
            for w in WATCHED:
                if w in e.name:
                    watched[w] += e.device_time
    return dict(kernels_us=round(total / reps, 1), h2d_us=round(h2d / reps, 1), **{k + "_us": round(v / reps, 1) for k, v in sorted(watched.items())})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--n", type=int, default=1_000_000)
    args = ap.parse_args()
    print(f"# {card()}", flush=True)
    rng = np.random.default_rng(0)
    ctx = g.default_context()

    # Gaussian voxel map, posed insert of a device cloud
    frames = []
    for r in range(args.reps + 1):
        pts, covs = syn.make_cloud(args.n, stream=10 + r, scale=1.0)
        ints = rng.uniform(0.0, 255.0, len(pts)) / 3.0
        frames.append((g.PointCloud(pts, covs), g.PointCloud(pts, covs, intensities=ints), syn.random_pose(rng, 0.2, 2.0)))
    plain_map, int_map = g.GaussianVoxelMapGPU(1.0), g.GaussianVoxelMapGPU(1.0)
    t_plain, t_int = [], []
    for r, (plain, with_ints, T) in enumerate(frames):
        a = wall_ms(lambda: plain_map.insert_cloud(plain, T))
        b = wall_ms(lambda: int_map.insert_cloud(with_ints, T))
        if r:
            t_plain.append(a)
            t_int.append(b)
    x, y = plain_map.download(), int_map.download()
    assert all(np.array_equal(x[k], y[k]) for k in x if k != "resolution")
    plain, with_ints, T = frames[-1]
    m1, m2 = g.GaussianVoxelMapGPU(1.0), g.GaussianVoxelMapGPU(1.0)
    print(json.dumps(dict(case="voxelmap_insert_cloud", n=args.n, voxels=plain_map.num_voxels, wall_ms_without=round(float(np.median(t_plain)), 3),
                          wall_ms_with=round(float(np.median(t_int)), 3), device_without=device_us(lambda: m1.insert_cloud(plain, T), args.reps),
                          device_with=device_us(lambda: m2.insert_cloud(with_ints, T), args.reps))), flush=True)

    # voxel-grid downsampling of a host scan
    pts, covs = syn.make_cloud(args.n, stream=99, scale=1.0)
    pts, covs = np.ascontiguousarray(pts[:, :3]), np.ascontiguousarray(covs[:, :3, :3])
    ints = rng.uniform(0.0, 255.0, len(pts)) / 3.0
    t_plain, t_int = [], []
    for r in range(args.reps + 1):
        a = wall_ms(lambda: voxelgrid_call(ctx, pts, covs, None, 0.25))
        b = wall_ms(lambda: voxelgrid_call(ctx, pts, covs, ints, 0.25))
        if r:
            t_plain.append(a)
            t_int.append(b)
    assert voxelgrid_call(ctx, pts, covs, ints, 0.25) == 8
    voxels = len(g.voxelgrid_sampling(pts, 0.25, covs=covs))
    print(json.dumps(dict(case="voxelgrid_sampling", n=args.n, voxels=voxels, wall_ms_without=round(float(np.median(t_plain)), 3),
                          wall_ms_with=round(float(np.median(t_int)), 3), device_without=device_us(lambda: voxelgrid_call(ctx, pts, covs, None, 0.25), args.reps),
                          device_with=device_us(lambda: voxelgrid_call(ctx, pts, covs, ints, 0.25), args.reps))), flush=True)


if __name__ == "__main__":
    main()
