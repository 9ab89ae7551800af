"""CPU checks of the ICP-on-iVox restatement (ivox_icp_np.IcpIvoxNp) the GPU tests compare against.

* oracle tie-in: with neighbour mode 27 and a max correspondence distance of at most the voxel size, the iVox 1-NN is exact, so
  point-to-point ICP on an iVox equals the oracle's kd-tree ICP over the map's stored points, and point-to-plane ICP on an
  iVoxCovarianceEstimation equals the oracle's point-to-plane ICP over the map's valid points and estimated normals: identical
  correspondences, H / b / error within 1e-12 relative;
* odometry: the KITTI-07 frame-to-map loop of test_ivox_cpu.py with point-to-point ICP on an iVox filled without covariances,
  and with point-to-plane ICP on an iVoxCovarianceEstimation, against the reference's 0.015 rad / 0.15 m gates.  Both loops
  miss a gate on some frame; the tests record the numbers and fail if the loops start to meet the gates.
"""
import numpy as np
import pytest

import ivox_cov_np
import ivox_icp_np
import ivox_np
import mini_lm
import oracle_lib as orc
from gtsam_points_b200 import synthetic as syn
from test_ivox_cpu import UnaryAdapter, kitti07, odometry, trajectory_frames

KEYS = ("H_target", "H_source", "H_target_source", "b_target", "b_source")


def assert_close(rl, ol, tol=1e-12):
    for k in KEYS:
        assert np.abs(rl[k] - ol[k]).max() <= tol * max(1.0, np.abs(ol[k]).max()), k
    assert abs(rl["error"] - ol["error"]) <= tol * abs(ol["error"])
    assert rl["num_inliers"] == ol["num_inliers"]


def source_and_pose(stream=40, n=1500):
    src, _ = syn.make_cloud(n, stream=stream, scale=1.0)
    return np.asarray(src, dtype=np.float64), syn.random_pose(np.random.default_rng(3), 0.05, 0.3)


def test_point_to_point_against_oracle_kdtree_icp():
    iv = ivox_np.IvoxNp(1.0)
    iv.mode = 27
    for pts, _ in trajectory_frames(num_frames=4):
        iv.insert(pts)  # no covariances: ICP needs none
    ex, fi = iv.export(), iv.flat_index()
    cloud = orc.Cloud(ex["points"])
    src, delta = source_and_pose()
    rf = ivox_icp_np.IcpIvoxNp(iv, src)
    rl = rf.linearize(delta)
    of = orc.Factor(cloud, orc.Cloud(src), tree=orc.KdTree(cloud, 2), num_threads=2, icp="point")
    ol = of.linearize(delta)
    flat = np.array([fi[c] if c >= 0 else -1 for c in rf.corr])
    assert (flat >= 0).sum() > 100
    assert np.array_equal(flat, of.correspondences())
    assert_close(rl, ol)
    d2 = delta @ syn.se3_exp(np.array([0.01, -0.005, 0.002, 0.05, 0.02, -0.03]))
    assert abs(rf.error(d2) - of.error(d2)) <= 1e-12 * abs(of.error(d2))


def test_point_to_plane_against_oracle_kdtree_icp():
    m = ivox_cov_np.IvoxCovNp(1.0)
    m.mode = 27
    for pts, _ in trajectory_frames(num_frames=4):
        m.insert(pts)
    vpts, vnormals, to_valid = ivox_icp_np.valid_cloud(m)
    assert 0 < len(vpts) < len(m.export()["points"])  # some points are invalid and must not be found
    cloud = orc.Cloud(vpts)
    cloud.set_normals(vnormals)
    src, delta = source_and_pose()
    rf = ivox_icp_np.IcpIvoxNp(m, src, point_to_plane=True)
    rl = rf.linearize(delta)
    of = orc.Factor(cloud, orc.Cloud(src), tree=orc.KdTree(cloud, 2), num_threads=2, icp="plane")
    ol = of.linearize(delta)
    corr = np.array([to_valid[int(c)] if c >= 0 else -1 for c in rf.corr])
    assert (corr >= 0).sum() > 100
    assert np.array_equal(corr, of.correspondences())
    assert_close(rl, ol)
    d2 = delta @ syn.se3_exp(np.array([0.01, -0.005, 0.002, 0.05, 0.02, -0.03]))
    assert abs(rf.error(d2) - of.error(d2)) <= 1e-12 * abs(of.error(d2))


def test_point_to_plane_needs_normals():
    iv = ivox_np.IvoxNp(1.0)
    iv.insert(np.zeros((1, 3)))
    try:
        ivox_icp_np.IcpIvoxNp(iv, np.zeros((1, 3)), point_to_plane=True)
    except ValueError as e:
        assert "target frame doesn't have required attributes for icp" in str(e)
    else:
        raise AssertionError("a plain iVox has no normals")


def run_odometry(m, point_to_plane):
    pts, covs, poses_gt = kitti07()
    state = {}

    def make_factor(src, scov):
        f = ivox_icp_np.IcpIvoxNp(m, src, point_to_plane=point_to_plane)
        state["key"] = state.get("key", 0) + 1
        return UnaryAdapter(state["key"], f.linearize, f.error)

    estimates, _ = odometry(pts, covs, poses_gt, make_factor, lambda p, c: m.insert(p))
    return [mini_lm.pose_error(estimates[i], poses_gt[i]) for i in range(1, 5)]


@pytest.mark.xfail(strict=True, reason="frames 2 and 4 miss the 0.15 m gate (0.356 m, 0.315 m; frame 4 also 0.042 rad); DESIGN.md 4.4")
def test_kitti07_frame_to_map_odometry_point_to_point_numpy():
    """Point-to-point ICP on a plain iVox filled without covariances.  Recorded per frame 1-4 (rad, m): (0.0013, 0.032),
    (0.0090, 0.356), (0.0033, 0.149), (0.0422, 0.315): 1-NN point-to-point with the loop's U(-0.1, 0.1) start misses two
    frames, where GICP and point-to-plane converge."""
    for i, (err_r, err_t) in enumerate(run_odometry(ivox_np.IvoxNp(1.0), False), 1):
        assert err_r < 0.015 and err_t < 0.15, (i, err_r, err_t)


@pytest.mark.xfail(strict=True, reason="frame 4 misses the 0.015 rad gate by 3 % (0.01539 rad, 0.055 m); DESIGN.md 4.4")
def test_kitti07_frame_to_map_odometry_point_to_plane_numpy():
    """Point-to-plane ICP on an iVoxCovarianceEstimation: its valid points and estimated normals.  Recorded per frame 1-4 (rad,
    m): (0.00045, 0.021), (0.00022, 0.017), (0.0019, 0.036), (0.0154, 0.055)."""
    for i, (err_r, err_t) in enumerate(run_odometry(ivox_cov_np.IvoxCovNp(1.0), True), 1):
        assert err_r < 0.015 and err_t < 0.15, (i, err_r, err_t)
