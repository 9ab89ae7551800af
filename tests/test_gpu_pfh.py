"""PFH and features at chosen points on the device (b2_features_create_pfh, b2_features_create_fpfh_at) against the CPU oracle
(orc_pfh / orc_fpfh_at in tests/registration_oracle.cpp), and RANSAC and GNC on PFH features."""
import numpy as np
import pytest

import gtsam_points_b200 as g
import registration_cases as rc
import registration_oracle as ro
from gtsam_points_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def kitti():
    """The KITTI-00 pair voxelised at 0.5 m with normals (k = 10) on the device, the source posed by T_final, then by the inverse of
    the reference test's offset."""
    d = rc.kitti00()
    tgt = g.voxelgrid_sampling(d["frame0"], 0.5).estimated(10, normals=True)
    src = g.voxelgrid_sampling(d["frame1"], 0.5).estimated(10, normals=True)
    src = g.transform_gpu(src, rc.pose_inverse(rc.offset_pose()) @ d["T_final"])
    return tgt, src


def counts(rows, nn):
    """The integer counts behind PFH rows: row = count * (100 / (m (m - 1) / 2))."""
    pairs = (nn * (nn - 1) // 2).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        c = np.rint(rows * (pairs / 100.0)[:, None])
    return np.where(nn[:, None] > 1, c, 0.0).astype(np.int64)


def check_pfh(got, want, edge, nn, max_differ):
    """Rows the oracle does not flag are bit-identical; a flagged row that differs keeps its total and moves counts only along theta
    (bin = b_theta + 5 b_phi + 25 b_alpha), between adjacent theta bins."""
    differ = np.nonzero((got != want).any(axis=1))[0]
    assert set(differ.tolist()) <= set(np.nonzero(edge)[0].tolist()), differ[:10]
    if len(differ):
        cg, cw = counts(got[differ], nn[differ]), counts(want[differ], nn[differ])
        d = (cg - cw).reshape(len(differ), 25, 5)  # [row, phi + 5 alpha, theta]
        assert not d.sum(axis=2).any()  # the same total in every (phi, alpha): counts moved along theta only
    print(f"{len(got)} rows, {edge.sum()} flagged at a theta bin edge, {len(differ)} differ, mean |N| {nn.mean():.1f}, max |N| {nn.max()}")
    assert len(differ) <= max_differ
    return differ


def test_pfh_matches_the_oracle_on_kitti00_all_points(kitti):
    for cloud in kitti:
        got = g.estimate_pfh(cloud, 2.0).download()
        want, edge, nn = ro.pfh(cloud.points, cloud.normals, 2.0, 10000)
        assert got.shape == (len(cloud), 125)
        check_pfh(got, want, edge, nn, 20)
        assert np.array_equal(g.estimate_pfh(cloud, 2.0).download(), got)  # bit-reproducible


def test_pfh_and_fpfh_at_keypoints_match_the_oracle_on_kitti00(kitti):
    tgt, _ = kitti
    rng = np.random.default_rng(4)
    idx = rng.choice(len(tgt), 400, replace=False)
    got = g.estimate_pfh(tgt, 5.0, indices=idx).download()
    want, edge, nn = ro.pfh(tgt.points, tgt.normals, 5.0, 10000, indices=idx)
    check_pfh(got, want, edge, nn, 10)
    assert np.array_equal(g.estimate_pfh(tgt, 5.0, indices=idx).download(), got)
    f_got = g.estimate_fpfh(tgt, 5.0, indices=idx).download()
    f_want, f_edge, _ = ro.fpfh_at(tgt.points, tgt.normals, idx, 5.0, 10000)
    assert np.array_equal(f_got[~f_edge], f_want[~f_edge])
    assert np.array_equal(f_got, g.estimate_fpfh(tgt, 5.0).download()[idx])


@pytest.mark.parametrize("seed", [1, 2])
def test_pfh_on_synthetic_scenes(seed):
    P, N = rc.small_scene(1500, seed=seed, extent=10.0)
    P = np.concatenate([P, [[80.0, 80.0, 80.0], P[3]]])  # isolated: a zero row; a coincident point: bin 62
    N = np.concatenate([N, [[0.0, 0.0, 1.0], N[9]]])
    rows = {}
    for flags in (capi.B2_CLOUD_DEFAULT, capi.B2_CLOUD_NO_REORDER):
        cloud = g.PointCloud(P, normals=N, flags=flags)
        for max_nn in (10000, 16):
            rows[flags, max_nn] = g.estimate_pfh(cloud, 1.5, max_nn, tree=g.KdTree.from_cloud(cloud) if max_nn == 16 else None).download()
    for max_nn in (10000, 16):
        want, edge, nn = ro.pfh(P, N, 1.5, max_nn)
        assert np.array_equal(rows[capi.B2_CLOUD_DEFAULT, max_nn], rows[capi.B2_CLOUD_NO_REORDER, max_nn])
        got = rows[capi.B2_CLOUD_DEFAULT, max_nn]
        check_pfh(got, want, edge, nn, 5)
        assert not got[1500].any() and nn[1500] == 1
        assert got[1501, 62] > 0.0
        if max_nn == 16:
            assert nn.max() == 16
    assert not np.array_equal(rows[capi.B2_CLOUD_DEFAULT, 16], rows[capi.B2_CLOUD_DEFAULT, 10000])


def test_features_at_indices_equal_the_all_points_rows():
    P, N = rc.small_scene(900, seed=6, extent=8.0)
    P = np.concatenate([P, [[60.0, 0.0, 0.0]]])
    N = np.concatenate([N, [[1.0, 0.0, 0.0]]])
    for flags in (capi.B2_CLOUD_DEFAULT, capi.B2_CLOUD_NO_REORDER):
        cloud = g.PointCloud(P, normals=N, flags=flags)
        tree = g.KdTree.from_cloud(cloud)
        for est, dim in ((g.estimate_fpfh, 33), (g.estimate_pfh, 125)):
            for max_nn in (10000, 20):
                full = est(cloud, 1.2, max_nn).download()
                for idx in ([900, 5, 17, 5, 899, 0, 17], [412], list(range(900, -1, -7)), np.arange(901)):
                    got = est(cloud, 1.2, max_nn, tree=tree, indices=np.asarray(idx)).download()
                    assert got.shape == (len(idx), dim) and np.array_equal(got, full[np.asarray(idx)])
                empty = est(cloud, 1.2, max_nn, indices=np.zeros(0, dtype=np.int64))
                assert len(empty) == 0 and empty.dim == dim and empty.download().shape == (0, dim)
            assert not est(cloud, 1.2, 0, indices=[3, 4]).download().any()


def test_feature_errors():
    P, N = rc.small_scene(50, seed=1)
    bare = g.PointCloud(P)
    cloud = g.PointCloud(P, normals=N)
    other = g.PointCloud(P, normals=N)
    for est in (g.estimate_fpfh, g.estimate_pfh):
        for idx in ([0, 50], [-1], [3, 2**40]):
            with pytest.raises(capi.B2Error) as e:
                est(cloud, 1.0, indices=idx)
            assert e.value.status == 1
        with pytest.raises(capi.B2Error) as e:
            est(bare, 1.0, indices=[1])
        assert e.value.status == 4
        with pytest.raises(capi.B2Error) as e:
            est(cloud, 1.0, tree=g.KdTree.from_cloud(other), indices=[1])
        assert e.value.status == 1
        with pytest.raises(capi.B2Error) as e:
            est(cloud, float("nan"), indices=[1])
        assert e.value.status == 1
    with pytest.raises(capi.B2Error) as e:
        g.estimate_pfh(bare, 1.0)
    assert e.value.status == 4


def test_pfh_rows_split_over_many_ctas():
    """Keypoints inside a dense cluster: each row has millions of pairs, spread over hundreds of CTAs whose counts are summed."""
    rng = np.random.default_rng(11)
    P = rng.uniform(-1.0, 1.0, (4000, 3))
    Nr = rng.normal(size=(4000, 3)) + [0.0, 0.0, 3.0]
    Nr /= np.linalg.norm(Nr, axis=1)[:, None]
    P = np.round(P, 6)
    cloud = g.PointCloud(P, normals=Nr)
    idx = np.array([0, 1234, 3999])
    got = g.estimate_pfh(cloud, 5.0, 10000, indices=idx).download()
    want, edge, nn = ro.pfh(P, Nr, 5.0, 10000, indices=idx)
    assert (nn == 4000).all()
    check_pfh(got, want, edge, nn, 3)


def test_pfh_counts_are_64_bit():
    """One keypoint among 70 000 coincident points: 2 449 965 000 pairs, all the zero feature, in bin 62 -- beyond 32-bit counts."""
    n = 70000
    P = np.tile([[1.0, 2.0, 3.0]], (n, 1))
    N = np.tile([[0.0, 0.0, 1.0]], (n, 1))
    cloud = g.PointCloud(P, normals=N)
    row = g.estimate_pfh(cloud, 0.5, 100000, indices=[17]).download()[0]
    pairs = n * (n - 1) // 2
    assert pairs > 2**31
    assert row[62] == np.float64(pairs) * (100.0 / np.float64(pairs))
    assert not np.delete(row, 62).any()


def test_registration_on_pfh(kitti):
    """PFH at 5 m feeds RANSAC (dof 6 and 4) and GNC.  With the oracle's PFH rows on both sides, the device follows the oracle chains;
    the device's own PFH rows then drive the same calls end to end.  Both meet the reference test's gate (0.5 m, 0.1 rad)."""
    tgt, src = kitti
    tf, _, _ = ro.pfh(tgt.points, tgt.normals, 5.0, 10000)
    sf, _, _ = ro.pfh(src.points, src.normals, 5.0, 10000)
    TF, SF = g.Features.from_array(tf), g.Features.from_array(sf)
    dev_tf, dev_sf = g.estimate_pfh(tgt, 5.0), g.estimate_pfh(src, 5.0)
    assert dev_tf.dim == 125 and len(dev_tf) == len(tgt)
    for dof in (6, 4):
        K = 2000
        want = ro.ransac(tgt.points, src.points, tf, sf, max_iterations=K, dof=dof)
        res = g.estimate_pose_ransac(tgt, src, TF, SF, g.RANSACParams(max_iterations=K, dof=dof), hypothesis_inliers=True)
        ws, got = want["status"], res.hypothesis_inliers
        assert np.array_equal(np.minimum(got, 0), np.minimum(ws, 0))
        ok = (ws >= 0) & ~want["degenerate"]
        assert np.all(np.abs(got[ok] - ws[ok]) <= want["slack"][ok])
        assert np.abs(res.T_target_source[:3] - want["T"][res.hypothesis]).max() <= 1e-9
        oracle_err = rc.pose_error(want["T_target_source"], rc.offset_pose())
        dev = g.estimate_pose_ransac(tgt, src, dev_tf, dev_sf, g.RANSACParams(dof=dof))
        dev_err = rc.pose_error(dev.T_target_source, rc.offset_pose())
        print(f"RANSAC dof {dof}: oracle chain {oracle_err[0]:.3f} m {oracle_err[1]:.4f} rad; device PFH end to end {dev_err[0]:.3f} m {dev_err[1]:.4f} rad")
        et, er = rc.pose_error(res.T_target_source, rc.offset_pose())
        assert oracle_err[0] <= 0.5 and oracle_err[1] <= 0.1  # the oracle chain meets the reference test's gate, so the device must too
        assert et <= 0.5 and er <= 0.1 and dev_err[0] <= 0.5 and dev_err[1] <= 0.1
    for dof in (6, 4):
        want = ro.gnc(tgt.points, src.points, tf, sf, dof=dof)
        res, C = g.estimate_pose_gnc(tgt, src, TF, SF, g.GNCParams(dof=dof), correspondences=True)
        assert np.array_equal(C, want["C"])
        assert np.abs(res.T_target_source - want["T_target_source"]).max() <= 1e-9
        oracle_err = rc.pose_error(want["T_target_source"], rc.offset_pose())
        dev = g.estimate_pose_gnc(tgt, src, dev_tf, dev_sf, g.GNCParams(dof=dof))
        dev_err = rc.pose_error(dev.T_target_source, rc.offset_pose())
        print(f"GNC dof {dof}: oracle chain {oracle_err[0]:.3f} m {oracle_err[1]:.4f} rad; device PFH end to end {dev_err[0]:.3f} m {dev_err[1]:.4f} rad")
        et, er = rc.pose_error(res.T_target_source, rc.offset_pose())
        assert oracle_err[0] <= 0.5 and oracle_err[1] <= 0.1  # the oracle chain meets the reference test's gate, so the device must too
        assert et <= 0.5 and er <= 0.1 and dev_err[0] <= 0.5 and dev_err[1] <= 0.1
