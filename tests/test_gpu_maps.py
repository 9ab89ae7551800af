"""Device voxel-map utilities against the CPU oracle (pytest -m gpu): incremental insert + LRU, save_compact / load across
the two implementations, overlap.  Mirrors src/test/test_voxelmap.cpp:92-153,231-239 on the reference's KITTI-07 submaps."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import golden_util
import oracle_lib as orc
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


@pytest.fixture(scope="module")
def gold():
    return golden_util.load()


def assert_maps_equal(got, ref):
    assert np.array_equal(got["coords"], ref["coords"])  # ids = first-touch order, survivors re-indexed in order
    assert np.array_equal(got["n"], ref["n"])
    assert np.array_equal(got["means"], ref["means"])  # same float64 operation sequence as GaussianVoxel::add / finalize
    assert np.array_equal(got["covs"], ref["covs"])


def test_incremental_insert_and_lru_match_cpu_map_bitwise(g):
    """25 overlapping frames along a trajectory, lru_horizon 3 / lru_clear_cycle 4: after EVERY insert the device map equals
    IncrementalVoxelMap<GaussianVoxel> (ann/impl/incremental_voxelmap_impl.hpp:31-68) bit for bit, evictions included."""
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.set_lru(3, 4)
    ovm = orc.VoxelMap(0.5)
    ovm.set_lru(3, 4)
    sizes = []
    for step in range(25):
        pts, covs = syn.make_cloud(6000 + 37 * step, stream=100 + step, scale=0.2)
        pts = pts + np.array([1.5 * step, 0.3 * step, 0.0])
        vm.insert(g.PointCloud(pts, covs))
        ovm.insert(orc.Cloud(pts, covs))
        assert_maps_equal(vm.download(), ovm.export())
        sizes.append(vm.num_voxels)
        q = pts[::7] + 0.01
        assert np.array_equal(vm.lookup_voxel_index(q), ovm.lookup(q))
    assert max(sizes) > sizes[-1] or any(b < a for a, b in zip(sizes, sizes[1:]))  # the LRU sweep removed voxels at some point


def test_xyzw_4x4_insert_equals_xyz_3x3_insert_bitwise(g):
    """The same clouds inserted as (xyz, 3 x 3 covariances) and as (xyzw with w = 1, 4 x 4 covariances): after EVERY insert the two
    maps download bit-identical voxels and answer lookups identically, LRU evictions included."""
    a, b = g.GaussianVoxelMapGPU(0.5), g.GaussianVoxelMapGPU(0.5)
    a.set_lru(3, 4)
    b.set_lru(3, 4)
    sizes = []
    for step in range(25):
        pts, covs = syn.make_cloud(6000 + 37 * step, stream=200 + step, scale=0.2)
        pts = pts + np.array([1.5 * step, 0.3 * step, 0.0])
        covs4 = np.zeros((len(covs), 4, 4))
        covs4[:, :3, :3] = covs
        covs4[:, 3, 3] = 1.0
        a.insert(g.PointCloud(pts, covs))
        b.insert(g.PointCloud(np.hstack([pts, np.ones((len(pts), 1))]), covs4))
        got_a, got_b = a.download(), b.download()
        for k in ("coords", "n", "means", "covs"):
            assert np.array_equal(got_a[k], got_b[k]), (step, k)
        sizes.append(a.num_voxels)
        q = pts[::7] + 0.01
        assert np.array_equal(a.lookup_voxel_index(q), b.lookup_voxel_index(q))
    assert max(sizes) > sizes[-1] or any(y < x for x, y in zip(sizes, sizes[1:]))  # the LRU sweep removed voxels at some point


def test_factor_sees_map_growth(g):
    """A factor built over a map keeps working, with the new contents, after further insert() calls (descriptor refresh)."""
    tp, tc = syn.make_cloud(30000, stream=1, scale=0.25)
    sp, sc = syn.make_cloud(9000, stream=2, scale=0.25)
    half = len(tp) // 2
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(g.PointCloud(tp[:half], tc[:half]))
    ovm = orc.VoxelMap(0.5)
    ovm.insert(orc.Cloud(tp[:half], tc[:half]))
    src = g.PointCloud(sp, sc)
    f = g.IntegratedVGICPFactor(0, 1, vm, src)
    of = orc.Factor(ovm, orc.Cloud(sp, sc), num_threads=2)
    delta = syn.random_pose(np.random.default_rng(4), 0.02, 0.2)
    values = {0: np.eye(4), 1: delta}
    for stage in range(2):
        f.linearize(values)
        ref = of.linearize(delta)
        assert np.array_equal(f.correspondences(), of.correspondences())
        for k in ("H_target", "H_source", "H_target_source", "b_target", "b_source"):
            assert np.abs(f._last[k] - ref[k]).max() <= 1e-9 * np.abs(ref[k]).max(), (stage, k)
        if stage == 0:
            vm.insert(g.PointCloud(tp[half:], tc[half:]))
            ovm.insert(orc.Cloud(tp[half:], tc[half:]))


def test_save_compact_load_across_implementations(g, gold, tmp_path):
    """save_compact written by the device map loads in the CPU restatement and vice versa (same 56-byte records);
    checks of src/test/test_voxelmap.cpp:108-151: resolution, count, means / covs within 1e-3, identical index lookups."""
    tgt = g.PointCloud(gold["target_points"], gold["target_covs"])
    vm = g.GaussianVoxelMapGPU(1.0)
    vm.insert(tgt)
    ovm = orc.VoxelMap(1.0)
    ovm.insert(orc.Cloud(gold["target_points"], gold["target_covs"]))
    a, b = tmp_path / "gpu.bin", tmp_path / "cpu.bin"
    vm.save_compact(a)
    ovm.save_compact(b)
    assert open(a, "rb").read() == open(b, "rb").read()  # byte-identical files
    from_cpu = g.GaussianVoxelMapGPU.load(b)
    from_gpu = orc.VoxelMap.load(a)
    ref = ovm.export()
    for got in (from_cpu.download(), from_gpu.export()):
        assert np.array_equal(got["coords"], ref["coords"]) and np.array_equal(got["n"], ref["n"])
        assert np.linalg.norm(got["means"] - ref["means"], axis=1).max() < 1e-3 and np.abs(got["covs"] - ref["covs"]).max() < 1e-3
    assert from_cpu.voxel_resolution() == 1.0 and from_cpu.num_voxels == ovm.num_voxels
    assert np.array_equal(from_cpu.lookup_voxel_index(ref["means"]), ovm.lookup(ref["means"]))
    # a loaded map is a valid VGICP target
    src = g.PointCloud(gold["source_points"], gold["source_covs"])
    f = g.IntegratedVGICPFactor(0, 1, from_cpu, src)
    f.linearize({0: np.eye(4), 1: gold["delta"]})
    assert f.num_inliers() > 0.5 * len(gold["source_points"])


def test_overlap_gpu_equals_cpu_overlap(g, gold):
    """src/test/test_voxelmap.cpp:92-106,231-239: self-overlap >= 0.99; the device value equals the CPU value EXACTLY (float64
    with the CPU's operation order; the reference's float32 GPU path only promises 0.01), single map and map list."""
    tp, tc, sp, sc = gold["target_points"], gold["target_covs"], gold["source_points"], gold["source_covs"]
    tgt, src = g.PointCloud(tp, tc), g.PointCloud(sp, sc)
    vm = g.GaussianVoxelMapGPU(1.0)
    vm.insert(tgt)
    vm2 = g.GaussianVoxelMapGPU(1.0)
    vm2.insert(src)
    ovm, ovm2 = orc.VoxelMap(1.0), orc.VoxelMap(1.0)
    otgt, osrc = orc.Cloud(tp, tc), orc.Cloud(sp, sc)
    ovm.insert(otgt)
    ovm2.insert(osrc)
    assert g.overlap_gpu(vm, tgt, np.eye(4)) >= 0.99
    rng = np.random.default_rng(9)
    for _ in range(4):
        T = syn.random_pose(rng, 0.2, 1.0)
        assert g.overlap_gpu(vm, src, T) == ovm.overlap(osrc, T)
        Ts = np.stack([T, syn.random_pose(rng, 0.3, 3.0)])
        assert g.overlap_gpu([vm, vm2], src, Ts) == orc.overlap_multi([ovm, ovm2], osrc, Ts)


def test_merge_frames_gpu_equals_cpu_merge_frames(g, gold):
    """merge_frames_gpu vs merge_frames (gaussian_voxelmap_cpu_funcs.cpp:25-113): same voxels in the same (key) order, means of
    world points and rotated covariances BIT-identical (same summation order), Morton-reordered and caller-order storage alike;
    the merged cloud is a usable frame (src/test/test_voxelmap.cpp:108-131 merges frames and checks the overlap with the inputs)."""
    tp, tc, sp, sc = gold["target_points"], gold["target_covs"], gold["source_points"], gold["source_covs"]
    poses = np.stack([gold["T_target"], gold["T_source_gt"]])
    for flags in (capi.B2_CLOUD_DEFAULT, capi.B2_CLOUD_NO_REORDER):
        frames = [g.PointCloud(tp, tc, flags=flags), g.PointCloud(sp, sc, flags=flags)]
        for res in (0.5, 0.2):
            merged = g.merge_frames_gpu(poses, frames, res)
            xyz, cov = orc.merge_frames(poses, [orc.Cloud(tp, tc), orc.Cloud(sp, sc)], res)
            assert len(merged.points) == len(xyz) and len(xyz) < len(tp) + len(sp)
            assert np.array_equal(merged.points, xyz)
            assert np.array_equal(merged.covs, cov.reshape(-1, 3, 3))
    # every input point lies in a voxel of a map built from the merged frame at the same resolution-ish scale
    vm = g.GaussianVoxelMapGPU(1.0)
    vm.insert(merged)
    assert g.overlap_gpu(vm, g.PointCloud(tp, tc), poses[0]) > 0.9
