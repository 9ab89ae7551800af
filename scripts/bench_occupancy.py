"""Occupancy grid timing on one GPU: FastOccupancyGrid insert, batched overlap and free_rays on device clouds.

Inputs: the KITTI-00 pair of tests/golden (frame 0: 62k points; the pair concatenated: 124k points) and a synthetic 1M-point cloud
(synthetic.make_cloud).  Cases, each against the host trip -- b2_cloud_download, the CPU oracle (tests/occupancy_oracle.cpp, one
thread), and the upload of its result to the device:
  insert_<input>_<res>:        create a grid and insert the cloud posed by KITTI-00's T_final (host trip: download, oracle insert,
                               upload of the occupied cells);
  overlap_<input>_P<m>:        counts of the 124k-point cloud under m = 1 and 64 poses against a grid of frame 0 at 0.5 m (host trip:
                               download, one oracle calc_overlap per pose, upload of the counts);
  free_rays_<res>:             free_rays of frame 1 at T_final on a grid of frame 0 (host trip: download, oracle free_rays, upload of
                               the occupied cells).  Clearing is idempotent, so repeated calls do the same work.
Medians over --reps calls after one warm-up call, wall time around calls that end in a stream synchronise.  The device arm and the
oracle are checked to agree before anything is timed.  Then, in a separate profiled run, the overlap kernel's mean time at 64 poses and
its achieved rate over the bytes its lookups read (from shapes: per (pose, point) one point, one 8-byte table key and one 8-byte bitmap
word), against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet.  Prints the card name, power limit and max SM clock of the same
run, then one JSON line per case.

  python scripts/bench_occupancy.py [--reps 7]
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

import occupancy_oracle as oo  # noqa: E402
import gtsam_points_b200 as g  # noqa: E402
from gtsam_points_b200 import capi  # noqa: E402
from gtsam_points_b200 import synthetic as syn  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def wall_ms(fn):
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def download(cloud):
    p = np.zeros((cloud.size(), 3))
    capi.check(capi.lib().b2_cloud_download(cloud.h, capi.dptr(p), None, None))
    return p


def upload(a):
    torch.as_tensor(np.ascontiguousarray(a)).to("cuda")
    torch.cuda.synchronize()


def timed(name, n, device, host, reps, **extra):
    device()
    host()
    dev = [wall_ms(device) for _ in range(reps)]
    hst = [wall_ms(host) for _ in range(reps)]
    d, h = float(np.median(dev)), float(np.median(hst))
    row = dict(case=name, points=n, device_ms=round(d, 3), host_trip_ms=round(h, 3), speedup=round(h / d, 2), **extra)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_occupancy: no CUDA device")
    ctx = g.Context(0, torch.cuda.current_stream().cuda_stream)
    print(json.dumps({"card": card(), "host_threads": os.cpu_count()}), flush=True)
    k00 = np.load(os.path.join(ROOT, "tests", "golden", "kitti00_pair.npz"))
    T = k00["T_final"]
    f0, f1 = g.PointCloud(k00["frame0"], ctx=ctx), g.PointCloud(k00["frame1"], ctx=ctx)
    pair = g.PointCloud(np.concatenate([k00["frame0"], k00["frame1"]]), ctx=ctx)
    big = g.PointCloud(syn.make_cloud(1_000_000, stream=4, scale=1.0)[0], ctx=ctx)

    # insert
    for name, cloud in (("kitti00_frame0", f0), ("synthetic_1M", big)):
        rows = download(cloud)
        for res in (0.25, 0.5):
            def dev(cloud=cloud, res=res):
                grid = g.FastOccupancyGrid(res, ctx)
                grid.insert(cloud, T)
                return grid

            def host(cloud=cloud, res=res):
                orc = oo.Grid(res)
                orc.insert(download(cloud), T)
                upload(orc.cells())
                return orc

            assert np.array_equal(dev().occupied_cells(), host().cells()), (name, res)
            timed(f"insert_{name}_{res}", len(rows), dev, host, a.reps, cells=int(dev().num_occupied_cells()))

    # batched overlap
    grid, orc = g.FastOccupancyGrid(0.5, ctx), oo.Grid(0.5)
    grid.insert(f0)
    orc.insert(download(f0))
    rng = np.random.default_rng(1)
    poses64 = np.stack([T] + [syn.random_pose(rng, 0.05, 0.5) for _ in range(63)])
    for m in (1, 64):
        Ts = poses64[:m]

        def dev(Ts=Ts):
            return grid.calc_overlaps(pair, Ts)

        def host(Ts=Ts):
            p = download(pair)
            c = np.array([orc.overlaps(p, X)[0] for X in Ts], dtype=np.uint64)
            upload(c)
            return c

        assert np.array_equal(dev(), host()), m
        timed(f"overlap_kitti00_pair_P{m}", pair.size(), dev, host, a.reps, poses=m)

    # free_rays
    for res in (0.25, 0.5):
        grid_f, orc_f = g.FastOccupancyGrid(res, ctx), oo.Grid(res)
        grid_f.insert(f0)
        orc_f.insert(download(f0))

        def dev(grid_f=grid_f):
            grid_f.free_rays(f1, T)

        def host(orc_f=orc_f):
            orc_f.free_rays(download(f1), T)
            upload(orc_f.cells())

        dev(), host()
        assert np.array_equal(grid_f.occupied_cells(), orc_f.cells()), res
        timed(f"free_rays_kitti00_{res}", f1.size(), dev, host, a.reps, cells_after=int(grid_f.num_occupied_cells()))

    # overlap kernel time and achieved rate at 64 poses (profiled run of its own)
    from torch.profiler import ProfilerActivity, profile

    calls = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            grid.calc_overlaps(pair, poses64)
        torch.cuda.synchronize()
    durs = [e.device_time for e in prof.events() if "overlap_kernel" in e.name]
    n, P = pair.size(), len(poses64)
    point_bytes = int(pair.info().point_bytes)
    bytes_read = n * P * (3 * point_bytes + 8 + 8)
    if durs:
        us = float(np.mean(durs))
        rate = bytes_read / (us * 1e-6)
        print(json.dumps(dict(case="overlap_kernel_P64", points=n, poses=P, launches=len(durs), kernel_us=round(us, 2), bytes_read=bytes_read,
                              achieved_tb_s=round(rate / 1e12, 3), share_of_3_35_tb_s=round(rate / HBM_BYTES_PER_S, 3))), flush=True)
    else:
        print(json.dumps(dict(case="overlap_kernel_P64", error="no overlap_kernel events in the profile")), flush=True)


if __name__ == "__main__":
    main()
