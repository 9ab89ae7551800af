"""iVox on the device (-m gpu) against the Python restatement of the reference's container (tests/ivox_np.py).

* the device map equals the restatement bit for bit -- voxel coords, ids, counts, points, covariances -- after every insert of a
  25-frame trajectory with LRU (3, 4) and small cells (rejections, full cells, evictions), in every neighbour mode;
* knn (k = 1, 5, 20): distances exact, indices where the distance is unique in the row;
* the GICP factor on an iVox: correspondences bit-identical to the restatement's association, H / b / error within 1e-9 of
  np_ref.linearize, error() after linearize equals the linearized error, the tolerance-frozen path, bit-reproducible runs;
* a map mutation between calls re-associates (no stale indices), for linearize and for error();
* one factor set mixing VGICP, GICP and iVox-GICP factors equals the per-factor results;
* the KITTI-07 frame-to-map odometry loop through the device factor and map meets the reference's gates, with an LM pose track
  equal to the restatement-driven track to 1e-7 per iteration.
"""
import numpy as np
import pytest

import ivox_np
import mini_lm
import np_ref
from test_ivox_cpu import UnaryAdapter, kitti07, odometry, trajectory_frames

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def make_pair(g, mode, max_points=4, min_dist=0.3):
    dev = g.iVox(1.0)
    dev.set_lru(3, 4)
    dev.set_neighbor_voxel_mode(mode)
    dev.set_min_dist_in_cell(min_dist)
    dev.set_max_num_points_in_cell(max_points)
    ref = ivox_np.IvoxNp(1.0)
    ref.mode = mode
    ref.lru_horizon, ref.lru_clear_cycle = 3, 4
    ref.min_sq, ref.max_points = min_dist * min_dist, max_points
    return dev, ref


def assert_same_map(dev, ref):
    a, b = dev.download(), ref.export()
    for k in ("coords", "counts", "points", "covs"):
        assert a[k].shape == b[k].shape, k
        assert np.array_equal(a[k], b[k]), k


def assert_same_knn(dev, ref, q, k, max_sq):
    idx, sqd = dev.knn_search(q, k, max_sq)
    for i in range(len(q)):
        ri, rd = ref.knn(q[i], k, max_sq)
        assert np.array_equal(sqd[i], np.array(rd)), i
        for j in range(k):
            if np.count_nonzero(sqd[i] == sqd[i][j]) == 1:
                assert idx[i][j] == ri[j], (i, j)


def as_layout(pts, covs, layout):
    """The frame in one of the insert input layouts: xyz with 3x3 covariances, xyzw (w = 1) with 4x4, or xyz without covariances."""
    if layout == "xyzw-4x4":
        covs4 = np.zeros((len(covs), 4, 4))
        covs4[:, :3, :3] = covs
        covs4[:, 3, 3] = 1.0
        return np.hstack([pts, np.ones((len(pts), 1))]), covs4
    return pts, (None if layout == "xyz" else covs)


@pytest.mark.parametrize(
    "mode,layout",
    [pytest.param(m, "xyz-3x3", id=str(m)) for m in (1, 7, 19, 27)] + [pytest.param(7, layout, id=f"7-{layout}") for layout in ("xyzw-4x4", "xyz")],
)
def test_map_and_knn_match_restatement(g, mode, layout):
    dev, ref = make_pair(g, mode)
    rng = np.random.default_rng(mode)
    for f, frame in enumerate(trajectory_frames()):
        pts, covs = as_layout(*frame, layout)
        dev.insert(pts, covs)
        ref.insert(pts, covs)
        assert_same_map(dev, ref)
        if f % 6 == 5:
            ex = ref.export()
            q = ex["points"][rng.integers(0, len(ex["points"]), 200)] + rng.normal(scale=0.3, size=(200, 3))
            for k in (1, 5, 20):
                assert_same_knn(dev, ref, q, k, 1.5)
    assert dev.num_voxels == len(ref.voxels) > 0


def test_clear_and_settings(g):
    dev = g.iVox(0.5)
    with pytest.raises(g.B2Error):
        dev.set_neighbor_voxel_mode(5)
    with pytest.raises(g.B2Error):
        dev.set_max_num_points_in_cell(33)
    pts, covs = trajectory_frames(num_frames=1)[0]
    dev.insert(pts, covs)
    with pytest.raises(g.B2Error):
        dev.set_max_num_points_in_cell(21)  # slots were laid out for 20 by the first insert
    with pytest.raises(g.B2Error):
        dev.insert(pts)  # no mixing of inserts with and without covariances
    dev.set_max_num_points_in_cell(5)
    dev.clear()
    assert dev.num_voxels == 0
    ref = ivox_np.IvoxNp(0.5)
    ref.max_points = 5
    dev.insert(pts, covs)
    ref.insert(pts, covs)
    assert_same_map(dev, ref)


def build_map(g, frames, mode=7):
    dev, ref = make_pair(g, mode, max_points=20, min_dist=0.1)
    dev.set_lru(10, 10)
    ref.lru_horizon, ref.lru_clear_cycle = 10, 10
    for pts, covs in frames:
        dev.insert(pts, covs)
        ref.insert(pts, covs)
    return dev, ref


def source_frame(n=3000, stream=99):
    from gtsam_points_b200 import synthetic as syn

    pts, covs = syn.make_cloud(n, stream=stream, scale=1.0)
    return np.asarray(pts, dtype=np.float64), np.asarray(covs, dtype=np.float64)


def check_lin(dev_l, ref_l, tol=1e-9):
    for k in ("H_target", "H_source", "H_target_source", "b_target", "b_source"):
        scale = max(1.0, float(np.abs(ref_l[k]).max()))
        assert np.abs(dev_l[k] - ref_l[k]).max() <= tol * scale, k
    assert abs(dev_l["error"] - ref_l["error"]) <= tol * max(1.0, abs(ref_l["error"]))
    assert dev_l["num_inliers"] == ref_l["num_inliers"]


@pytest.mark.parametrize("mode", [1, 7, 27])
def test_factor_matches_restatement(g, mode):
    from gtsam_points_b200 import synthetic as syn

    dev, ref = build_map(g, trajectory_frames(num_frames=3), mode)
    src, scov = source_frame()
    cloud = g.PointCloud(src, scov)
    f = g.IntegratedGICPFactor(np.eye(4), 1, dev, cloud)
    rf = ivox_np.GicpIvoxNp(ref, src, scov)
    rng = np.random.default_rng(mode)
    delta = syn.random_pose(rng, rot=0.05, trans=0.3)
    f.linearize({1: delta})
    dl = f._last
    rl = rf.linearize(delta)
    assert np.array_equal(f.correspondences(), rf.corr)
    check_lin(dl, rl)
    # error() at the linearization point equals the linearized error; elsewhere the frozen correspondences are re-used
    assert abs(f.error({1: delta}) - dl["error"]) <= 1e-12 * max(1.0, abs(dl["error"]))
    delta2 = delta @ syn.se3_exp(np.full(6, 0.01))
    assert abs(f.error({1: delta2}) - rf.error(delta2)) <= 1e-9 * max(1.0, rf.error(delta2))
    # bit-reproducible
    f.linearize({1: delta})
    again = f._last
    for k in dl:
        assert np.array_equal(np.asarray(dl[k]), np.asarray(again[k])), k


def test_tolerance_frozen_path(g):
    from gtsam_points_b200 import synthetic as syn

    dev, ref = build_map(g, trajectory_frames(num_frames=3))
    src, scov = source_frame()
    f = g.IntegratedGICPFactor(np.eye(4), 1, dev, g.PointCloud(src, scov))
    f.set_correspondence_update_tolerance(0.1, 0.5)
    delta = syn.random_pose(np.random.default_rng(1), rot=0.05, trans=0.3)
    f.linearize({1: delta})
    corr0 = f.correspondences()
    delta2 = delta @ syn.se3_exp(np.array([0.01, 0, 0, 0.05, 0, 0]))
    f.linearize({1: delta2})  # within tolerance: the correspondences of delta are kept and linearized at delta2
    assert np.array_equal(f.correspondences(), corr0)
    ex, fi = ref.export(), ref.flat_index()
    flat = np.array([fi[c] if c >= 0 else -1 for c in corr0])
    check_lin(f._last, np_ref.linearize(delta2, src, scov, ex["points"], ex["covs"], flat))


def test_map_mutation_reassociates(g):
    from gtsam_points_b200 import synthetic as syn

    frames = trajectory_frames(num_frames=6)
    dev, ref = build_map(g, frames[:3])
    src, scov = source_frame()
    f = g.IntegratedGICPFactor(np.eye(4), 1, dev, g.PointCloud(src, scov))
    f.set_correspondence_update_tolerance(10.0, 100.0)  # would freeze forever if the map change were ignored
    delta = syn.random_pose(np.random.default_rng(2), rot=0.05, trans=0.3)
    f.linearize({1: delta})
    for pts, covs in frames[3:]:
        dev.insert(pts, covs)
        ref.insert(pts, covs)
    # error() before the next linearize associates at the evaluation pose
    rf = ivox_np.GicpIvoxNp(ref, src, scov)
    e_ref = rf.linearize(delta)["error"]
    assert abs(f.error({1: delta}) - e_ref) <= 1e-9 * max(1.0, abs(e_ref))
    dev.set_neighbor_voxel_mode(27)
    ref.mode = 27
    f.linearize({1: delta})
    rl = rf.linearize(delta)
    assert np.array_equal(f.correspondences(), rf.corr)
    check_lin(f._last, rl)
    dev.clear()
    dev.insert(*frames[0])
    ref.clear()
    ref.insert(*frames[0])
    f.linearize({1: delta})
    rf.linearize(delta)
    assert np.array_equal(f.correspondences(), rf.corr)


def test_mixed_factor_set(g):
    from gtsam_points_b200 import synthetic as syn

    frames = trajectory_frames(num_frames=3)
    dev, _ = build_map(g, frames)
    tgt_pts = np.concatenate([p for p, _ in frames])
    tgt_cov = np.concatenate([c for _, c in frames])
    target = g.PointCloud(tgt_pts, tgt_cov)
    vm = g.GaussianVoxelMapGPU(1.0)
    vm.insert(target)
    srcs = [g.PointCloud(*source_frame(2000, stream=s)) for s in (50, 51, 52)]
    factors = [
        g.IntegratedVGICPFactor(0, 1, vm, srcs[0]),
        g.IntegratedGICPFactor(0, 2, target, srcs[1]),
        g.IntegratedGICPFactor(0, 3, dev, srcs[2]),
        g.IntegratedGICPFactor(0, 1, dev, srcs[0]),
    ]
    rng = np.random.default_rng(4)
    values = {0: np.eye(4), 1: syn.random_pose(rng), 2: syn.random_pose(rng), 3: syn.random_pose(rng)}
    fs = g.NonlinearFactorSetGPU()
    fs.add(factors)
    out = fs.linearize(values)
    errs = fs.error(values)
    for i, f in enumerate(factors):
        f.linearize(values)
        single = f._last
        l = g.capi.unpack_linearized(out[i])
        check_lin(l, single, 1e-12)
        assert abs(errs[i] - f.error(values)) <= 1e-12 * max(1.0, abs(errs[i]))


def test_kitti07_frame_to_map_odometry_device(g):
    pts, covs, poses_gt = kitti07()
    dev = g.iVox(1.0)
    keep = []

    def make_factor(src, scov):
        cloud = g.PointCloud(src, scov)
        key = len(keep) + 1
        f = g.IntegratedGICPFactor(np.eye(4), key, dev, cloud)
        keep.append((cloud, f))
        return f

    est_dev, hist_dev = odometry(pts, covs, poses_gt, make_factor, lambda p, c: dev.insert(p, c))
    for i in range(1, 5):
        err_r, err_t = mini_lm.pose_error(est_dev[i], poses_gt[i])
        assert err_r < 0.015 and err_t < 0.15, (i, err_r, err_t)

    ref = ivox_np.IvoxNp(1.0)
    state = {}

    def make_ref(src, scov):
        f = ivox_np.GicpIvoxNp(ref, src, scov)
        state["key"] = state.get("key", 0) + 1
        return UnaryAdapter(state["key"], f.linearize, f.error)

    est_ref, hist_ref = odometry(pts, covs, poses_gt, make_ref, ref.insert)
    for a, b in zip(hist_dev, hist_ref):  # the LM pose track, iteration by iteration
        assert len(a) == len(b)
        for Ta, Tb in zip(a, b):
            assert np.abs(Ta - Tb).max() < 1e-7
