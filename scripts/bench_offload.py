"""What GPU memory offloading costs on one GPU, at the cfg4 shape: F VGICP factors of 200k source points, each with its own 0.5 m
Gaussian voxel map built from a 200k-point target (BASELINE.md, the per-GPU share of the ISAM2-style relinearize).

  (1) offload and reload per object (b2_cloud_* / b2_voxelmap_*): wall time per C ABI call (each returns after its stream has
      synchronised), the bytes moved (the object's pinned host copy) and the achieved rate.  The first offload of an object copies
      it to the host; a repeat offload of an object that still holds its host copy only frees device memory; a reload copies back
      (and, for a map, rebuilds the bucket table).  Medians over the k offloaded factors' objects.
  (2) b2_factor_set_linearize over the F factors (host poses, host records), medians over --reps calls of each arm:
        resident   every object on the device;
        reload     the maps and sources of k factors offloaded before the call (not timed), offloading on: the call reloads them;
        next       the resident call that follows a reload call.
      The three arms' records are asserted bit-identical at the same poses.
Prints the card name, power limit and max SM clock of the same run, then one JSON line.

  python scripts/bench_offload.py [--factors 32] [--offloaded 8] [--points 200000] [--reps 7]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import gtsam_points_b200 as g  # noqa: E402
from gtsam_points_b200 import capi  # noqa: E402
from gtsam_points_b200 import synthetic as syn  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    if not q.strip():
        raise RuntimeError("nvidia-smi reports no GPU: this benchmark measures on the device only")
    return q.strip().splitlines()[0]


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t) * 1e3, out


def move(obj, op):
    """One offload / reload C ABI call on a PointCloud or GaussianVoxelMapGPU: (ms, moved anything)."""
    api = "b2_cloud" if isinstance(obj, g.PointCloud) else "b2_voxelmap"
    ch = C.c_int32()
    ms, st = timed(lambda: getattr(capi.lib(), f"{api}_{op}")(obj.h, C.byref(ch)))
    capi.check(st)
    assert ch.value == 1
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--factors", type=int, default=32)
    ap.add_argument("--offloaded", type=int, default=8)
    ap.add_argument("--points", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    F, k, n = args.factors, args.offloaded, args.points
    print(card(), flush=True)
    ctx = g.default_context()
    maps, srcs, factors = [], [], []
    for i in range(F):  # bench_configs.py cfg4: every factor has its own scene sampling
        tp, tc = syn.make_cloud(n, stream=100 + 2 * i, scene_seed=1000 + i)
        sp, sc = syn.make_cloud(n, stream=101 + 2 * i, scene_seed=1000 + i)
        vm = g.GaussianVoxelMapGPU(0.5, ctx)
        vm.insert(g.PointCloud(tp, tc, ctx=ctx, flags=capi.B2_CLOUD_NO_REORDER))
        src = g.PointCloud(sp, sc, ctx=ctx)
        maps.append(vm), srcs.append(src)
        factors.append(g.IntegratedVGICPFactor(2 * i, 2 * i + 1, vm, src, ctx=ctx))
    for f in factors:
        f.set_enable_offloading(True)
    s = g.NonlinearFactorSetGPU(ctx)
    s.add(factors)
    s._ensure()
    rng = np.random.default_rng(5)
    deltas = np.ascontiguousarray(np.stack([syn.random_pose(rng, 0.01, 0.1) for _ in range(F)]).reshape(F, 16))
    L = capi.lib()

    def linearize():
        out = np.zeros((F, capi.B2_LINEARIZED_DOUBLES))
        capi.check(L.b2_factor_set_linearize(s.h, capi.dptr(deltas), capi.dptr(out)))
        return out

    # (1) per object: first offload (copy + free), reload, repeat offload (free only), reload
    per = {"cloud": {}, "map": {}}
    for name, objs in (("cloud", srcs[:k]), ("map", maps[:k])):
        rec = {"offload_first_ms": [], "reload_ms": [], "offload_repeat_ms": [], "reload_again_ms": []}
        for o in objs:
            rec["offload_first_ms"].append(move(o, "offload"))
            rec["reload_ms"].append(move(o, "reload"))
            rec["offload_repeat_ms"].append(move(o, "offload"))
            rec["reload_again_ms"].append(move(o, "reload"))
        nbytes = int(np.median([o.residency().host_bytes for o in objs]))
        med = {key: float(np.median(v)) for key, v in rec.items()}
        per[name] = dict(med, bytes=nbytes, device_bytes=int(np.median([o.memory_usage_gpu() for o in objs])),
                         offload_first_GBps=nbytes / (med["offload_first_ms"] * 1e-3) / 1e9, reload_GBps=nbytes / (med["reload_ms"] * 1e-3) / 1e9)

    # (2) set linearize: resident / reload inside the call / next resident
    ref = linearize()  # warm-up (module load, first descriptors)
    arms = {"resident": [], "reload": [], "next": []}
    for _ in range(args.reps):
        ms, out = timed(linearize)
        arms["resident"].append(ms)
        assert out.tobytes() == ref.tobytes()
        for o in maps[:k] + srcs[:k]:
            o.offload_gpu()
        ms, out = timed(linearize)
        arms["reload"].append(ms)
        assert out.tobytes() == ref.tobytes() and all(o.loaded_on_gpu() for o in maps[:k] + srcs[:k])
        ms, out = timed(linearize)
        arms["next"].append(ms)
        assert out.tobytes() == ref.tobytes()
    lin = {a: float(np.median(v)) for a, v in arms.items()}
    moved = sum(o.residency().host_bytes for o in maps[:k] + srcs[:k])
    print(json.dumps({
        "workload": f"{F} VGICP factors x {n} source points, own 0.5 m map each; {k} maps + {k} sources offloaded",
        "per_object": per,
        "linearize_ms": lin,
        "reload_in_call_bytes": moved,
        "reload_in_call_extra_ms": lin["reload"] - lin["resident"],
        "reload_in_call_GBps": moved / ((lin["reload"] - lin["resident"]) * 1e-3) / 1e9 if lin["reload"] > lin["resident"] else None,
        "inliers_mean": float(ref[:, 121].mean()), "reps": args.reps,
    }), flush=True)


if __name__ == "__main__":
    main()
