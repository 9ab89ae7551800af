"""Region growing timing on one GPU: a device cloud with normals in, the converged cluster out.

Inputs: the KITTI-00 frame 0 of tests/golden (62k points) with normals estimated on the device, seeded on the road ahead and at
its point 0 (a small cluster, to show the fixed cost); a submap of the five KITTI-07 frames
of tests/golden merged in their poses (54k points), normals estimated on the device, seeded on the road; and a synthetic 1.2M-point plane with normals
+z.  Per input it takes the median, min and max over --reps calls (after one warm-up call) of the wall time of
  (a) the device call: b2_region_growing_create (with its kd-tree), one update to convergence, and the cluster read back;
  (b) the host trip: b2_cloud_download of points and normals, then the CPU oracle (tests/segmentation_oracle.cpp, single-threaded
      like the reference's region_growing_update) to convergence.  Both take one update with max_steps = 2^31 - 1.
Both arms are checked to give the same cluster before anything is timed.  Prints the card name, power limit and max SM clock of the
same run, then one JSON line per input.

  python scripts/bench_segmentation.py [--reps 7]
"""
import argparse
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
import segmentation_oracle as so  # noqa: E402
from gtsam_points_b200 import capi  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def inputs():
    gold = os.path.join(ROOT, "tests", "golden")
    k00 = np.load(os.path.join(gold, "kitti00_pair.npz"))["frame0"].astype(np.float64)[:, :3]
    frame = g.PointCloud(k00).estimated(10, normals=True)
    ground = np.array([5.0, 0.0, -1.7])  # the road in front of the sensor
    yield "kitti00_frame_ground", frame, ground, (0.5, np.deg2rad(10.0), 0.5)
    yield "kitti00_frame_small", frame, k00[0], (0.5, np.deg2rad(10.0), 0.5)
    f = np.load(os.path.join(gold, "kitti07_frames.npz"))
    parts = []
    for i in range(5):
        T = f["poses"][i]
        p = f[f"points{i}"].astype(np.float64)
        parts.append(p @ T[:3, :3].T + T[:3, 3])
    sub = np.vstack(parts)
    T0 = f["poses"][0]
    yield "kitti07_submap_ground", g.PointCloud(sub).estimated(10, normals=True), T0[:3, :3] @ ground + T0[:3, 3], (0.5, np.deg2rad(10.0), 0.5)
    rng = np.random.default_rng(9)
    n = 1_200_000
    plane = np.c_[rng.uniform(0, 60, (n, 2)), rng.normal(0, 0.002, n)]
    yield "plane_1.2M", g.PointCloud(plane, normals=np.tile([0.0, 0.0, 1.0], (n, 1))), np.array([30.0, 30.0, 0.0]), (0.1, np.deg2rad(10.0), 0.1)


def device(cloud, seed_point, prm):
    rg = g.RegionGrowing.init(cloud, seed_point, g.RegionGrowingParams(*prm))
    assert rg.update(2**31 - 1)
    return rg.cluster_indices


def host(cloud, seed_point, prm):
    n = int(cloud.info().num_points)
    p, nr = np.zeros((n, 3)), np.zeros((n, 3))
    capi.check(capi.lib().b2_cloud_download(cloud.h, capi.dptr(p), None, capi.dptr(nr)))
    rg = so.RegionGrowing(p, nr, so.nearest(p, seed_point), *prm)
    assert rg.update(2**31 - 1)
    return rg.cluster_indices


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    print(card())
    for name, cloud, seed_point, prm in inputs():
        d, h = device(cloud, seed_point, prm), host(cloud, seed_point, prm)
        assert np.array_equal(d, h)
        td = timed(lambda: device(cloud, seed_point, prm), a.reps)
        th = timed(lambda: host(cloud, seed_point, prm), a.reps)
        print(json.dumps(dict(input=name, points=int(cloud.info().num_points), cluster=int(len(d)), device_ms=td, host_trip_ms=th, speedup=th[0] / td[0])))
    min_cut_rows(a.reps)


def min_cut_rows(reps):
    """min_cut (defaults, background radius 3 m) on crops of 10k, 100k and 1M points of a box on a ground plane: the device call
    against download + the CPU oracle (brute-force k-NN network and integer Dinic) where the oracle is affordable."""
    rng = np.random.default_rng(4)
    for n in (10_000, 100_000, 1_000_000):
        side = np.sqrt(n / 400.0)
        nb = n // 10
        ground = np.c_[rng.uniform(-side / 2, side / 2, (n - nb, 2)), rng.normal(0, 0.003, n - nb)]
        f = rng.uniform(0, 1, (nb, 3))
        ax = rng.integers(0, 3, nb)
        f[np.arange(nb), ax] = rng.integers(0, 2, nb)
        nrm = np.vstack([np.tile([0, 0, 1.0], (n - nb, 1)), np.eye(3)[ax]])
        cloud = g.PointCloud(np.vstack([ground, f - np.array([0.5, 0.5, 0.0])]), normals=nrm)
        seed = np.array([0.0, 0.0, 0.9])
        res = g.min_cut(cloud, seed)
        row = dict(input=f"min_cut_box_on_ground_{n}", points=n, cluster=int(len(res.cluster_indices)), max_flow=res.max_flow,
                   device_ms=timed(lambda: g.min_cut(cloud, seed), reps))
        if n <= 10_000:
            def host_mc():
                p, nr = np.zeros((n, 3)), np.zeros((n, 3))
                capi.check(capi.lib().b2_cloud_download(cloud.h, capi.dptr(p), None, capi.dptr(nr)))
                s = so.nearest(p, seed)
                t, idx, w, q = so.mc_network(p, nr, s)
                return so.mc_flow(p, s, t, idx, q)
            assert np.array_equal(host_mc()[1], res.cluster_indices)
            row["host_trip_ms"] = timed(host_mc, reps)
        print(json.dumps(row))


if __name__ == "__main__":
    main()
