"""Frame filtering timing on one GPU: a device cloud in, a filtered device cloud out.

Inputs: the KITTI-00 frame 0 of tests/golden (62k points) and synthetic clouds of 120k and 1M points (synthetic.make_cloud).  Cases:
remove_outliers at k = 10 (std_thresh 1), randomgrid_sampling at 0.5 m and rate 0.5, random_sampling at rate 0.5.  Per input and
case it takes medians over --reps calls (after one warm-up call) of the wall time of
  (a) the device call, device cloud to device cloud (b2_cloud_create_inliers / _randomgrid / _random_sampled; the outlier call
      builds its temporary kd-tree);
  (b) the host trip: b2_cloud_download, the CPU oracle (tests/filter_oracle.cpp: the outlier k-NN on every host thread, the
      samplers single-threaded), then b2_cloud_create of the selected rows.
Both arms are checked to select the same indices before anything is timed.  Prints the card name, power limit and max SM clock of
the same run, then one JSON line per input and case.

  python scripts/bench_filter.py [--reps 9]
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

import filter_oracle as fo  # noqa: E402
import gtsam_points_b200 as g  # noqa: E402
from gtsam_points_b200 import capi  # noqa: E402
from gtsam_points_b200 import synthetic as syn  # noqa: E402

SEED = 5489


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def wall_ms(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def inputs():
    k00 = np.load(os.path.join(ROOT, "tests", "golden", "kitti00_pair.npz"))
    return [("kitti00_frame0", k00["frame0"]), ("synthetic_120k", syn.make_cloud(120000, stream=3, scale=1.0)[0]),
            ("synthetic_1M", syn.make_cloud(1000000, stream=4, scale=1.0)[0])]


CASES = {
    "remove_outliers_k10": (lambda cloud, idx: capi.lib().b2_cloud_create_inliers(cloud.h, None, 10, 1.0, 0, None, None, idx[0], idx[1]),
                            lambda p: fo.inliers(p, 10, 1.0)[0]),
    "randomgrid_0.5m_rate0.5": (lambda cloud, idx: capi.lib().b2_cloud_create_randomgrid(cloud.h, 0.5, 0.5, SEED, 0, idx[0], idx[1]),
                                lambda p: fo.randomgrid_sampling(p, 0.5, 0.5, SEED)),
    "random_rate0.5": (lambda cloud, idx: capi.lib().b2_cloud_create_random_sampled(cloud.h, 0.5, SEED, 0, idx[0], idx[1]),
                       lambda p: fo.random_sampling(len(p), 0.5, SEED)),
}


def run(ctx, name, pts, case, reps):
    L = capi.lib()
    cloud = g.PointCloud(pts, ctx=ctx)
    n = len(pts)
    call, oracle = CASES[case]
    K_dev = np.zeros(n, dtype=np.int64)

    def device(want_indices=False):
        h = C.c_void_p()
        capi.check(call(cloud, (K_dev.ctypes.data_as(C.POINTER(C.c_int64)) if want_indices else None, C.byref(h))))
        info = capi.CloudInfo()
        capi.check(L.b2_cloud_get_info(h, C.byref(info)))
        L.b2_cloud_destroy(h)
        return int(info.num_points)

    def host_trip():
        p = np.zeros((n, 3))
        capi.check(L.b2_cloud_download(cloud.h, capi.dptr(p), None, None))
        K = oracle(p)
        rows = np.ascontiguousarray(p[K])
        h = C.c_void_p()
        capi.check(L.b2_cloud_create(ctx.h, capi.dptr(rows), 3, None, 9, len(K), 0, C.byref(h)))
        L.b2_cloud_destroy(h)
        return K

    m = device(True)
    K_host = host_trip()
    assert np.array_equal(K_dev[:m], K_host), (name, case)
    dev, host = [], []
    for _ in range(reps):
        dev.append(wall_ms(device))
        host.append(wall_ms(host_trip))
    d, h = float(np.median(dev)), float(np.median(host))
    return dict(input=name, points=n, case=case, selected=m, device_ms=round(d, 3), host_trip_ms=round(h, 3), speedup=round(h / d, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_filter: no CUDA device")
    ctx = g.Context(0, torch.cuda.current_stream().cuda_stream)
    print(json.dumps({"card": card(), "host_threads": os.cpu_count()}), flush=True)
    for name, pts in inputs():
        for case in CASES:
            print(json.dumps(run(ctx, name, pts, case, a.reps)), flush=True)


if __name__ == "__main__":
    main()
