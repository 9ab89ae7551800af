"""Every C ABI call hands the caller's current CUDA context back on return (pytest -m gpu).

Each entry point that touches a device opens b2::DeviceScope on its handle's device: the device is current for the call, and on
return the calling thread has again whatever context it had before, none included.  One call or more of every handle family,
the failing call of two of them (which fail after they have selected their device) and every destroy are driven with the
current context checked after each call:

* in a fresh process whose thread has no current context, on device 0: the thread has none after any call;
* in a fresh process whose thread has a context of its own on device 0 (not the primary context the library works in): that
  context is current again after every call;

and with two or more GPUs also:

* with device 0 current, on a context on device 1, and the mirror case: the current device is still the caller's after every
  call, read through PyTorch and through the driver;
* a fresh process that only uses device 1 does not create device 0's primary context;
* a VGICP linearize record, k-NN indices and a voxel-map download on device 1 equal the same calls on device 0 bit for bit.

With one GPU the cross-device tests skip: the library's device is then the caller's, and only the scope's same-device path runs
in the rest of the suite.
"""
import ctypes as C
import gc
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def env():
    """Two or more GPUs, PyTorch and the driver library; PyTorch's current device is put back afterwards for the tests that
    follow in this process."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device: the library's device is always the caller's")
    import gtsam_points_b200 as g

    before = torch.cuda.current_device()
    yield dict(g=g, torch=torch, cu=C.CDLL("libcuda.so.1"))
    torch.cuda.set_device(before)


def current_context(cu):
    """The calling thread's current context, read through the driver (None: no context is current)."""
    ctx = C.c_void_p()
    assert cu.cuCtxGetCurrent(C.byref(ctx)) == 0
    return ctx.value


def driver_device(cu):
    """The device of the calling thread's current context, read through the driver (None: no context is current)."""
    if current_context(cu) is None:
        return None
    dev = C.c_int()
    assert cu.cuCtxGetDevice(C.byref(dev)) == 0
    return dev.value


def make_current(env, device):
    env["torch"].cuda.set_device(device)
    env["torch"].zeros(1, device="cuda")  # the caller's own context exists and is current
    assert driver_device(env["cu"]) == device


def scene():
    tp, tc = syn.make_cloud(6000, stream=1, scale=0.25)
    sp, sc = syn.make_cloud(3000, stream=2, scale=0.25)
    delta = syn.random_pose(np.random.default_rng(7), 0.02, 0.2)
    return tp, tc, sp, sc, delta


def drive_every_family(g, device, check, tmp_path):
    """Calls of every handle family on a new context on `device`, check(name) after each; destroys everything at the end."""
    L = capi.lib()

    def step(name, fn, *args, **kw):
        out = fn(*args, **kw)
        check(name)
        return out

    ctx = step("b2_ctx_create", g.Context, device)
    step("b2_ctx_synchronize", ctx.synchronize)
    d_buf, host, back = C.c_void_p(), np.arange(64.0), np.zeros(64)
    step("b2_device_malloc", lambda: capi.check(L.b2_device_malloc(ctx.h, host.nbytes, C.byref(d_buf))))
    step("b2_memcpy_h2d", lambda: capi.check(L.b2_memcpy_h2d(ctx.h, d_buf, capi.dptr(host), host.nbytes)))
    step("b2_memcpy_d2h", lambda: capi.check(L.b2_memcpy_d2h(ctx.h, capi.dptr(back), d_buf, host.nbytes)))
    assert np.array_equal(back, host)
    step("b2_device_free", lambda: capi.check(L.b2_device_free(ctx.h, d_buf)))

    tp, tc, sp, sc, delta = scene()
    q = tp[::40] + 0.05
    values = {0: np.eye(4), 1: delta}

    # clouds
    tgt = step("b2_cloud_create", g.PointCloud, tp, tc, ctx=ctx)
    src = step("b2_cloud_create", g.PointCloud, sp, sc, ctx=ctx)
    step("b2_cloud_create_transformed", g.transform_gpu, src, delta)
    step("b2_cloud_create_voxelgrid", g.voxelgrid_sampling, tp, 0.5, covs=tc, ctx=ctx)
    tgt_n = step("b2_cloud_create_estimated", tgt.estimated, normals=True)
    step("b2_cloud_download_normals", tgt_n.normals_gpu)
    step("b2_cloud_create_sampled", g.sample, tgt, np.arange(0, len(tp), 3))
    step("b2_cloud_create_random_sampled", g.random_sampling, tgt, 0.3)
    step("b2_cloud_create_randomgrid", g.randomgrid_sampling, tgt, 1.0, 0.3)
    step("b2_cloud_create_inliers", g.remove_outliers, tgt)
    step("b2_merge_frames", g.merge_frames_gpu, np.stack([np.eye(4), delta]), [tgt, src], 0.5, ctx=ctx)
    merged = C.c_void_p()
    poses = np.ascontiguousarray(np.stack([np.eye(4), delta]).reshape(2, 16))
    frames = (C.c_void_p * 2)(tgt.h, src.h)
    step("b2_merge_frames_to_cloud", lambda: capi.check(L.b2_merge_frames_to_cloud(ctx.h, capi.dptr(poses), frames, 2, 0.5, 0, C.byref(merged))))
    step("b2_cloud_destroy", L.b2_cloud_destroy, merged)

    # Gaussian voxel map
    vm = g.GaussianVoxelMapGPU(0.5, ctx=ctx)
    step("b2_voxelmap_insert", vm.insert, tgt)
    step("b2_voxelmap_insert_cloud", vm.insert_cloud, src, delta)
    step("b2_voxelmap_lookup", vm.lookup_voxel_index, q)
    step("b2_overlap", g.overlap_gpu, vm, src, delta)
    step("b2_voxelmap_save_compact", vm.save_compact, tmp_path / "map.bin")
    loaded = step("b2_voxelmap_load", g.GaussianVoxelMapGPU.load, tmp_path / "map.bin", ctx=ctx)
    step("b2_voxelmap_download", vm.download)
    from_points = C.c_void_p()
    step("b2_voxelmap_create_from_points", lambda: capi.check(L.b2_voxelmap_create_from_points(ctx.h, 0.5, capi.dptr(tp), 3, capi.dptr(tc), 9, len(tp), C.byref(from_points))))
    step("b2_voxelmap_destroy", L.b2_voxelmap_destroy, from_points)

    # iVox and iVoxCovarianceEstimation
    iv = g.iVox(0.5, ctx=ctx)
    step("b2_ivox_insert", iv.insert, tp, tc)
    step("b2_ivox_insert_cloud", iv.insert_cloud, src, delta)
    step("b2_ivox_knn", iv.knn_search, q, 5)
    step("b2_ivox_download", iv.download)
    step("b2_ivox_get_info", iv.info)
    ic = g.iVoxCovarianceEstimation(0.5, ctx=ctx)
    step("b2_ivox_insert (covariance estimation)", ic.insert, tp)
    step("b2_ivox_insert_cloud (covariance estimation)", ic.insert_cloud, src, delta)
    step("b2_ivox_knn (covariance estimation)", ic.knn_search, q, 5)
    step("b2_ivox_knn_force", ic.knn_search_force, q, 5)
    step("b2_ivox_download_state", ic.download_state)
    step("b2_ivox_insert_timings", ic.insert_timings)

    # kd-tree
    tree = step("b2_kdtree_create", g.KdTree, tp, ctx=ctx)
    step("b2_kdtree_knn1", tree.knn_search, q, 1)
    step("b2_kdtree_knn", tree.knn_search, q, 5)
    step("b2_kdtree_radius_search", tree.radius_search_batch, q, 1.0)
    step("b2_kdtree_estimate_covariances", tree.estimate_covariances)
    step("b2_kdtree_estimate_normals", tree.estimate_normals)
    step("b2_estimate_normals", g.estimate_normals, tp, 10, ctx=ctx)
    step("b2_estimate_normals_from_covs", g.estimate_normals, tp, tc, ctx=ctx)
    step("b2_estimate_covariances", g.estimate_covariances, tp, ctx=ctx)
    tree_n = step("b2_kdtree_create_from_cloud", g.KdTree.from_cloud, tgt_n)

    # features and global registration
    src_n = step("b2_cloud_create_estimated", src.estimated, normals=True)
    ft = step("b2_features_create_fpfh", g.estimate_fpfh, tgt_n, 2.5, 30, tree=tree_n)
    fs = step("b2_features_create_fpfh", g.estimate_fpfh, src_n, 2.5, 30)
    step("b2_features_create_fpfh_at", g.estimate_fpfh, tgt_n, 2.5, 30, indices=[3, 1, 3])
    step("b2_features_create_pfh", g.estimate_pfh, src_n, 2.5, 30, indices=np.arange(0, len(sp), 50))
    step("b2_features_nearest", fs.nearest, ft)
    step("b2_features_create", g.Features.from_array, np.ones((4, 8)), ctx=ctx)
    step("b2_features_download", fs.download)
    step("b2_estimate_pose_ransac", g.estimate_pose_ransac, tgt_n, src_n, ft, fs, g.RANSACParams(max_iterations=64))
    step("b2_estimate_pose_gnc", g.estimate_pose_gnc, tgt_n, src_n, ft, fs, g.GNCParams(max_iterations=8))

    # segmentation
    rg = step("b2_region_growing_create", g.RegionGrowing.init, tgt_n, tp[0], tree=tree_n)
    step("b2_region_growing_update", rg.update)
    step("b2_region_growing_get", lambda: rg.cluster_indices)
    step("b2_min_cut", g.min_cut, tgt_n, 0)

    # occupancy
    grid = step("b2_occgrid_create", g.FastOccupancyGrid, 0.5, ctx=ctx)
    step("b2_occgrid_insert", grid.insert, tgt)
    step("b2_occgrid_overlap", grid.calc_overlaps, src, np.stack([np.eye(4), delta]), True)
    step("b2_occgrid_free_rays", grid.free_rays, src, delta)
    step("b2_occgrid_get_info", grid.info)
    step("b2_occgrid_download", grid.occupied_cells)
    step("b2_raycast", g.raycast, tp[:100], tp[100:200], 0.5, ctx=ctx)

    # factors, a factor set and a one-rank exchange
    vgicp = step("b2_vgicp_factor_create", g.IntegratedVGICPFactor, 0, 1, vm, src)
    gicp = step("b2_gicp_factor_create", g.IntegratedGICPFactor, 0, 1, tgt, src, target_tree=tree)
    icp = step("b2_icp_factor_create", g.IntegratedPointToPlaneICPFactor, 0, 1, tgt_n, src, target_tree=tree_n)
    gicp_iv = step("b2_gicp_ivox_factor_create", g.IntegratedGICPFactor, 0, 1, iv, src)
    icp_iv = step("b2_icp_ivox_factor_create", g.IntegratedPointToPlaneICPFactor, 0, 1, ic, src)
    for factor in (vgicp, gicp, icp, gicp_iv, icp_iv):
        step("b2_factor_linearize", factor.linearize, values)
        step("b2_factor_error", factor.error, values)
        step("b2_factor_correspondences", factor.correspondences)
    d_out = C.c_void_p()
    capi.check(L.b2_device_malloc(ctx.h, capi.B2_LINEARIZED_DOUBLES * 8, C.byref(d_out)))
    dlt = np.ascontiguousarray(delta.reshape(16))
    step("b2_factor_issue_linearize", lambda: capi.check(L.b2_factor_issue_linearize(vgicp.h, capi.dptr(dlt), d_out)))
    step("b2_factor_sync", lambda: capi.check(L.b2_factor_sync(vgicp.h)))
    step("b2_factor_issue_error", lambda: capi.check(L.b2_factor_issue_error(vgicp.h, capi.dptr(dlt), d_out)))
    step("b2_factor_sync", lambda: capi.check(L.b2_factor_sync(vgicp.h)))
    fset = g.NonlinearFactorSetGPU(ctx=ctx)
    fset.add([vgicp, gicp, icp, gicp_iv, icp_iv])
    step("b2_factor_set_linearize", fset.linearize, values)
    step("b2_factor_set_error", fset.error, values)
    deltas = np.ascontiguousarray(np.stack([f.calc_delta(values) for f in fset.factors]))
    ex = C.c_void_p()
    step("b2_exchange_create", lambda: capi.check(L.b2_exchange_create(ctx.h, 1, 0, len(deltas), C.byref(ex))))
    step("b2_exchange_linearize", lambda: capi.check(L.b2_exchange_linearize(ex, fset.h, capi.dptr(deltas), 0, 1)))
    step("b2_exchange_barrier", lambda: capi.check(L.b2_exchange_barrier(ex)))
    step("b2_factor_set_sync", lambda: capi.check(L.b2_factor_set_sync(fset.h)))
    step("b2_exchange_destroy", L.b2_exchange_destroy, ex)
    step("b2_device_free", lambda: capi.check(L.b2_device_free(ctx.h, d_out)))

    # calls that fail after selecting their device: a non-finite coordinate found by the device scan
    bad = tp.copy()
    bad[17, 1] = np.nan
    for name, fn in (("b2_kdtree_create", g.KdTree), ("b2_cloud_create", g.PointCloud)):
        with pytest.raises(capi.B2Error, match="non-finite coordinate"):
            fn(bad, ctx=ctx)
        check(name + " (failed)")

    # destroy every handle (the wrappers' __del__), then the context: no handle may outlive it
    del factor, vgicp, gicp, icp, gicp_iv, icp_iv, fset, rg, grid, ft, fs, tree, tree_n, iv, ic, vm, loaded, tgt, src, tgt_n, src_n
    gc.collect()
    check("*_destroy")
    step("b2_ctx_destroy", ctx.close)


@pytest.mark.parametrize("caller,device", [(0, 1), (1, 0)])
def test_every_family_keeps_the_callers_device(env, caller, device, tmp_path):
    make_current(env, caller)
    seen = []

    def check(name):
        assert env["torch"].cuda.current_device() == caller, f"after {name}: PyTorch's current device"
        assert driver_device(env["cu"]) == caller, f"after {name}: the driver's current context"
        seen.append(name)

    drive_every_family(env["g"], device, check, tmp_path)
    assert len(seen) > 100


# Drives every family on a device from a thread that has no current context ("none") or a context of its own on device 0
# ("own"), in a process of its own.  argv: repository root, mode, device, scratch directory.
CHILD = r"""
import ctypes as C, gc, pathlib, sys
root, mode, device, scratch = sys.argv[1], sys.argv[2], int(sys.argv[3]), pathlib.Path(sys.argv[4])
sys.path[:0] = [root, root + "/tests"]
import gtsam_points_b200 as g
from test_gpu_device_scope import current_context, drive_every_family

cu = C.CDLL("libcuda.so.1")
assert cu.cuInit(0) == 0
mine = None
if mode == "own":
    dev, ctx = C.c_int(), C.c_void_p()
    assert cu.cuDeviceGet(C.byref(dev), 0) == 0 and cu.cuCtxCreate_v2(C.byref(ctx), 0, dev) == 0
    mine = ctx.value
assert current_context(cu) == mine
seen = []

def check(name):
    assert current_context(cu) == mine, "after " + name
    seen.append(name)

drive_every_family(g, device, check, scratch)
gc.collect()
check("the end")
assert len(seen) > 100
if mode == "none" and device != 0:
    flags, active = C.c_uint(), C.c_int()
    assert cu.cuDevicePrimaryCtxGetState(0, C.byref(flags), C.byref(active)) == 0
    assert active.value == 0, "device 0's primary context was created"
print("child ok")
"""


def run_child(mode, device, tmp_path):
    r = subprocess.run([sys.executable, "-s", "-c", CHILD, ROOT, mode, str(device), str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "child ok" in r.stdout, r.stdout[-4000:] + r.stderr[-4000:]


@pytest.mark.parametrize("mode", ["none", "own"])
def test_every_family_keeps_the_threads_context(mode, tmp_path):
    run_child(mode, 0, tmp_path)


def test_a_process_on_device_1_gets_no_context_on_device_0(env, tmp_path):
    run_child("none", 1, tmp_path)


def test_results_on_device_1_equal_device_0(env):
    g = env["g"]
    make_current(env, 0)
    tp, tc, sp, sc, delta = scene()
    q = sp[::7]
    out = []
    for device in (0, 1):
        ctx = g.Context(device)
        vm = g.GaussianVoxelMapGPU(0.5, ctx=ctx)
        vm.insert(g.PointCloud(tp, tc, ctx=ctx))
        f = g.IntegratedVGICPFactor(0, 1, vm, g.PointCloud(sp, sc, ctx=ctx))
        f.linearize({0: np.eye(4), 1: delta})
        idx, sq = g.KdTree(tp, ctx=ctx).knn_search(q, 8)
        out.append((f._last.copy(), f.correspondences(), idx, sq, vm.download()))
        del f, vm
        gc.collect()
        ctx.close()
    (lin0, corr0, idx0, sq0, map0), (lin1, corr1, idx1, sq1, map1) = out
    for k in lin0:
        assert np.array_equal(lin0[k], lin1[k]), k
    assert np.array_equal(corr0, corr1)
    assert np.array_equal(idx0, idx1) and np.array_equal(sq0, sq1)
    for k in ("coords", "means", "covs", "n"):
        assert np.array_equal(map0[k], map1[k]), k
