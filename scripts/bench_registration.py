"""Global registration timing on one GPU: FPFH, feature matching, RANSAC, GNC and the whole chains, against the CPU oracle's chains.

Inputs: the KITTI-00 pair of tests/golden voxelised at 0.5 m (about 9.3k points each, the reference test's input), and a synthetic
submap pair (synthetic.make_cloud, --synthetic points each before voxelising at 0.5 m; the source moved by a known pose), both with
normals from 10 neighbours estimated on the device.  Per input it takes medians over --reps repetitions of
  (a) the device stages, each between device synchronisations: FPFH of both clouds (radius 5 m), the feature 1-NN of every source row
      among the target rows, RANSAC (5000 hypotheses, dof 6) on the device features, and the chain end to end; GNC (default
      parameters, dof 6): its matching alone (both feature 1-NN passes and the compaction: max_iterations = 0), the whole call, and
      FPFH + GNC end to end; gnc_loop is the whole call's median minus the matching's; the same stages by CUDA events on the
      context's stream;
  (b) the same chains on the CPU oracles (tests/registration_oracle.cpp) on all host cores, timed once
      (it takes minutes at the synthetic size): brute-force FPFH, then RANSAC with a brute-force 1-NN per sample, or GNC with
      brute-force matching.
Then, per input, a second JSON line with the PFH and keypoint stages (radius 5 m, 10000 neighbours), medians over --reps between
device synchronisations: PFH and FPFH of the target over all points and at 1 % and 10 % of its points (a seeded random choice), and
PFH of both clouds followed by RANSAC or GNC, end to end.  The pair counts are summed from the neighbour counts of the device radius
search (m (m - 1) / 2 per row for PFH, m - 1 per SPFH row for FPFH), and pairs per second is that count over the median time.  With
the CPU oracle (tests/registration_oracle.cpp), its PFH over all points and its PFH and FPFH at 10 % are timed once each.
Prints the card name, power limit and max SM clock of the same run, then the JSON lines.

  python scripts/bench_registration.py [--reps 5] [--synthetic 100000] [--no-cpu] [--pfh-only]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import gtsam_points_b200 as g  # noqa: E402
import registration_cases as rc  # noqa: E402
import registration_oracle as ro  # noqa: E402
from gtsam_points_b200 import synthetic as syn  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0] if q.strip() else torch.cuda.get_device_name(0)


def inputs(n_synth):
    d = rc.kitti00()
    yield "kitti00_0.5m", d["frame0"], (rc.pose_inverse(rc.offset_pose()) @ d["T_final"], d["frame1"])
    tp = syn.make_cloud(n_synth, stream=11, scale=1.0)[0]
    sp = syn.make_cloud(n_synth, stream=12, scale=1.0)[0]
    yield f"synthetic_{n_synth}", tp, (rc.pose_inverse(rc.offset_pose()), sp)


def timed(ctx, fn):
    """(wall ms between device synchronisations, CUDA-event ms on the context's stream, result)"""
    stream = torch.cuda.ExternalStream(ctx.stream)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ctx.synchronize()
    t = time.perf_counter()
    a.record(stream)
    out = fn()
    b.record(stream)
    ctx.synchronize()
    wall = (time.perf_counter() - t) * 1e3
    b.synchronize()
    return wall, a.elapsed_time(b), out


def run(name, tp, src, reps, cpu):
    ctx = g.default_context()
    T_src, sp = src
    tgt = g.voxelgrid_sampling(tp, 0.5).estimated(10, normals=True)
    source = g.transform_gpu(g.voxelgrid_sampling(sp, 0.5).estimated(10, normals=True), T_src)
    params = g.RANSACParams(dof=6)
    gparams, gmatch = g.GNCParams(dof=6), g.GNCParams(dof=6, max_iterations=0)
    stages = {k: ([], []) for k in ("fpfh", "match", "ransac", "end_to_end", "gnc_match", "gnc", "gnc_end_to_end")}

    def chain():
        tf, sf = g.estimate_fpfh(tgt, 5.0), g.estimate_fpfh(source, 5.0)
        return g.estimate_pose_ransac(tgt, source, tf, sf, params)

    def gnc_chain():
        tf, sf = g.estimate_fpfh(tgt, 5.0), g.estimate_fpfh(source, 5.0)
        return g.estimate_pose_gnc(tgt, source, tf, sf, gparams)

    chain()  # warm-up: module load, every shape
    gnc_chain()
    res = gres = None
    for _ in range(reps):
        w, e, (tf, sf) = timed(ctx, lambda: (g.estimate_fpfh(tgt, 5.0), g.estimate_fpfh(source, 5.0)))
        stages["fpfh"][0].append(w), stages["fpfh"][1].append(e)
        w, e, _ = timed(ctx, lambda: sf.nearest(tf))
        stages["match"][0].append(w), stages["match"][1].append(e)
        w, e, res = timed(ctx, lambda: g.estimate_pose_ransac(tgt, source, tf, sf, params))
        stages["ransac"][0].append(w), stages["ransac"][1].append(e)
        w, e, _ = timed(ctx, chain)
        stages["end_to_end"][0].append(w), stages["end_to_end"][1].append(e)
        w, e, _ = timed(ctx, lambda: g.estimate_pose_gnc(tgt, source, tf, sf, gmatch))
        stages["gnc_match"][0].append(w), stages["gnc_match"][1].append(e)
        w, e, gres = timed(ctx, lambda: g.estimate_pose_gnc(tgt, source, tf, sf, gparams))
        stages["gnc"][0].append(w), stages["gnc"][1].append(e)
        w, e, _ = timed(ctx, gnc_chain)
        stages["gnc_end_to_end"][0].append(w), stages["gnc_end_to_end"][1].append(e)
    et, er = rc.pose_error(res.T_target_source, rc.offset_pose())
    out = dict(input=name, target_points=len(tgt), source_points=len(source), error_m=round(et, 4), error_rad=round(er, 5), inlier_rate=round(res.inlier_rate, 4))
    et, er = rc.pose_error(gres.T_target_source, rc.offset_pose())
    out.update(gnc_error_m=round(et, 4), gnc_error_rad=round(er, 5), gnc_inlier_rate=round(gres.inlier_rate, 4))
    for k, (w, e) in stages.items():
        out[f"gpu_{k}_ms"] = round(statistics.median(w), 3)
        out[f"gpu_{k}_event_ms"] = round(statistics.median(e), 3)
    out["gpu_gnc_loop_ms"] = round(out["gpu_gnc_ms"] - out["gpu_gnc_match_ms"], 3)
    if cpu:
        threads = ro.max_threads()  # compiles the oracle on first use: outside the timed window
        t = time.perf_counter()
        tf_c, _, _ = ro.fpfh(tgt.points, tgt.normals, 5.0, 10000, threads)
        sf_c, _, _ = ro.fpfh(source.points, source.normals, 5.0, 10000, threads)
        t_fpfh = time.perf_counter() - t
        ro.ransac(tgt.points, source.points, tf_c, sf_c, dof=6, num_threads=threads)
        out["cpu_oracle_end_to_end_ms"] = round((time.perf_counter() - t) * 1e3, 1)
        t = time.perf_counter()
        ro.gnc(tgt.points, source.points, tf_c, sf_c, dof=6, num_threads=threads)
        out["cpu_oracle_gnc_end_to_end_ms"] = round((t_fpfh + time.perf_counter() - t) * 1e3, 1)
        out["cpu_threads"] = threads
    return out


def neighbour_counts(cloud, queries, radius=5.0, max_nn=10000):
    off, _, _ = g.KdTree.from_cloud(cloud).radius_search_batch(queries, radius, max_nn)
    return np.diff(off).astype(np.int64)


def run_pfh(name, tp, src, reps, cpu):
    ctx = g.default_context()
    T_src, sp = src
    tgt = g.voxelgrid_sampling(tp, 0.5).estimated(10, normals=True)
    source = g.transform_gpu(g.voxelgrid_sampling(sp, 0.5).estimated(10, normals=True), T_src)
    rng = np.random.default_rng(3)
    kp = {f: np.sort(rng.choice(len(tgt), max(1, len(tgt) * f // 100), replace=False)) for f in (1, 10)}
    m_all = neighbour_counts(tgt, tgt.points)
    pairs = {"pfh_all": int((m_all * (m_all - 1) // 2).sum()), "fpfh_all": int(np.maximum(m_all - 1, 0).sum())}
    for f, idx in kp.items():
        m = m_all[idx]
        pairs[f"pfh_kp{f}"] = int((m * (m - 1) // 2).sum())
        # SPFH runs on the distinct union of the keypoints' neighbours
        _, nbr, _ = g.KdTree.from_cloud(tgt).radius_search_batch(tgt.points[idx], 5.0, 10000)
        pairs[f"fpfh_kp{f}"] = int(np.maximum(m_all[np.unique(nbr)] - 1, 0).sum())
    stages = {
        "pfh_all": lambda: g.estimate_pfh(tgt, 5.0),
        "fpfh_all": lambda: g.estimate_fpfh(tgt, 5.0),
        "pfh_kp1": lambda: g.estimate_pfh(tgt, 5.0, indices=kp[1]),
        "fpfh_kp1": lambda: g.estimate_fpfh(tgt, 5.0, indices=kp[1]),
        "pfh_kp10": lambda: g.estimate_pfh(tgt, 5.0, indices=kp[10]),
        "fpfh_kp10": lambda: g.estimate_fpfh(tgt, 5.0, indices=kp[10]),
        "pfh_ransac_end_to_end": lambda: g.estimate_pose_ransac(tgt, source, g.estimate_pfh(tgt, 5.0), g.estimate_pfh(source, 5.0), g.RANSACParams(dof=6)),
        "pfh_gnc_end_to_end": lambda: g.estimate_pose_gnc(tgt, source, g.estimate_pfh(tgt, 5.0), g.estimate_pfh(source, 5.0), g.GNCParams(dof=6)),
    }
    for fn in stages.values():  # warm-up: module load, every shape
        fn()
    times, results = {k: [] for k in stages}, {}
    for _ in range(reps):
        for k, fn in stages.items():
            w, _, results[k] = timed(ctx, fn)
            times[k].append(w)
    out = dict(input=name, target_points=len(tgt), source_points=len(source), mean_neighbours=round(float(m_all.mean()), 1), max_neighbours=int(m_all.max()),
               keypoints_1pct=len(kp[1]), keypoints_10pct=len(kp[10]))
    for k, w in times.items():
        out[f"gpu_{k}_ms"] = round(statistics.median(w), 3)
        if k in pairs:
            out[f"{k}_pairs"] = pairs[k]
            out[f"{k}_pairs_per_s"] = float(f"{pairs[k] / (statistics.median(w) * 1e-3):.4g}")
    for k in ("pfh_ransac_end_to_end", "pfh_gnc_end_to_end"):
        et, er = rc.pose_error(results[k].T_target_source, rc.offset_pose())
        out[f"{k}_error_m"], out[f"{k}_error_rad"] = round(et, 4), round(er, 5)
    if cpu:
        threads = ro.max_threads()
        for k, fn in (("pfh_all", lambda: ro.pfh(tgt.points, tgt.normals, 5.0, 10000, threads)),
                      ("pfh_kp10", lambda: ro.pfh(tgt.points, tgt.normals, 5.0, 10000, threads, indices=kp[10])),
                      ("fpfh_kp10", lambda: ro.fpfh_at(tgt.points, tgt.normals, kp[10], 5.0, 10000, threads))):
            t = time.perf_counter()
            fn()
            out[f"cpu_oracle_{k}_ms"] = round((time.perf_counter() - t) * 1e3, 1)
        out["cpu_threads"] = threads
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--synthetic", type=int, default=100000)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--pfh-only", action="store_true", help="only the PFH and keypoint stages")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU path only")
    print("card:", card())
    for name, tp, src in inputs(a.synthetic):
        if not a.pfh_only:
            print(json.dumps(run(name, tp, src, a.reps, not a.no_cpu)), flush=True)
        print(json.dumps(run_pfh(name, tp, src, a.reps, not a.no_cpu)), flush=True)


if __name__ == "__main__":
    main()
