"""GNC global registration on the device (b2_estimate_pose_gnc) against the CPU oracle (orc_gnc in tests/registration_oracle.cpp),
the reference's end-to-end gate (src/test/test_global_registration.cpp) run entirely on the device, and the feature 1-NN's split
of the targets over CTAs when the queries are few."""
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
    the reference test's offset; with the oracle's FPFH rows of both."""
    d = rc.kitti00()
    tgt = g.voxelgrid_sampling(d["frame0"], 0.5).estimated(10, normals=True)
    src = g.voxelgrid_sampling(d["frame1"], 0.5).estimated(10, normals=True)
    src = g.transform_gpu(src, rc.pose_inverse(rc.offset_pose()) @ d["T_final"])
    tf, _, _ = ro.fpfh(tgt.points, tgt.normals, 5.0, 10000)
    sf, _, _ = ro.fpfh(src.points, src.normals, 5.0, 10000)
    return tgt, src, tf, sf


CASES = {
    "dof6": dict(dof=6),
    "dof4": dict(dof=4),
    "no_reciprocal": dict(reciprocal_check=False, max_init_samples=2000),
    "tuples": dict(tuple_check=True, max_num_tuples=300),
    "tuples_no_reciprocal_dof4": dict(reciprocal_check=False, tuple_check=True, max_num_tuples=500, max_init_samples=3000, dof=4),
    "swapped": dict(swap=True),
    "swapped_no_reciprocal_tuples": dict(swap=True, reciprocal_check=False, tuple_check=True, max_num_tuples=800, max_init_samples=4000),
    "all_samples": dict(max_init_samples=20000, max_iterations=10),
}


@pytest.mark.parametrize("case", list(CASES))
def test_gnc_matches_the_oracle(kitti, case):
    tgt, src, tf, sf = kitti
    kw = dict(CASES[case])
    if kw.pop("swap", False):
        tgt, src, tf, sf = src, tgt, sf, tf
    assert (len(src) < len(tgt)) != case.startswith("swapped")
    want = ro.gnc(tgt.points, src.points, tf, sf, **kw)
    TF, SF = g.Features.from_array(tf), g.Features.from_array(sf)
    params = g.GNCParams(**kw)
    res, C = g.estimate_pose_gnc(tgt, src, TF, SF, params, correspondences=True)
    assert C.dtype == np.int64 and np.array_equal(C, want["C"])
    if "tuple_check" in kw:
        assert want["draws"] is not None and len(want["C"]) < len(want["matched"])
    assert np.abs(res.T_target_source - want["T_target_source"]).max() <= 1e-9
    assert abs(res.num_inliers - want["num_inliers"]) <= want["slack"].sum()
    assert res.hypothesis == -1 and res.inlier_rate == res.num_inliers / len(C)
    et, er = rc.pose_error(res.T_target_source, rc.offset_pose() if not case.startswith("swapped") else rc.pose_inverse(rc.offset_pose()))
    print(f"{case}: |C| {len(C)} of {len(want['samples'])} samples, inliers {res.num_inliers}, error {et:.3f} m {er:.4f} rad")
    if kw.get("dof") == 4:
        assert np.array_equal(res.T_target_source[2, :3], [0.0, 0.0, 1.0]) and np.array_equal(res.T_target_source[:2, 2], [0.0, 0.0])
    again, C2 = g.estimate_pose_gnc(tgt, src, TF, SF, params, correspondences=True)
    assert again.T_target_source.tobytes() == res.T_target_source.tobytes() and np.array_equal(C2, C) and again.num_inliers == res.num_inliers


@pytest.mark.parametrize("dof", [6, 4])
def test_reference_gate_on_the_device(kitti, dof):
    tgt, src, _, _ = kitti
    tf, sf = g.estimate_fpfh(tgt, 5.0), g.estimate_fpfh(src, 5.0)
    res = g.estimate_pose_gnc(tgt, src, tf, sf, g.GNCParams(dof=dof))
    et, er = rc.pose_error(res.T_target_source, rc.offset_pose())
    print(f"dof {dof}: error {et:.3f} m {er:.4f} rad, inlier rate {res.inlier_rate:.3f}")
    assert et <= 0.5 and er <= 0.1
    if dof == 4:
        assert np.abs(res.T_target_source[:3, 2] - [0.0, 0.0, 1.0]).max() <= 1e-6


def test_gnc_invalid_inputs(kitti):
    tgt, src, tf, sf = kitti
    TF, SF = g.Features.from_array(tf), g.Features.from_array(sf)
    empty = g.PointCloud(np.zeros((0, 3)), normals=np.zeros((0, 3)))
    f_empty = g.Features.from_array(np.ones((0, 33)))
    cases = [
        (tgt, src, TF, SF, g.GNCParams(dof=5)),
        (tgt, src, TF, SF, g.GNCParams(max_init_samples=0)),
        (tgt, src, TF, SF, g.GNCParams(max_num_tuples=-1)),
        (tgt, src, TF, SF, g.GNCParams(tuple_thresh=0.0)),
        (tgt, src, TF, SF, g.GNCParams(tuple_thresh=1.5)),
        (tgt, src, TF, SF, g.GNCParams(div_factor=0.0)),
        (tgt, src, TF, SF, g.GNCParams(div_factor=float("inf"))),
        (tgt, src, TF, SF, g.GNCParams(max_corr_dist=float("nan"))),
        (tgt, src, TF, SF, g.GNCParams(inner_iterations=-1)),
        (tgt, src, TF, SF, g.GNCParams(max_iterations=-1)),
        (tgt, src, SF, SF, g.GNCParams()),
        (tgt, src, TF, g.Features.from_array(np.ones((len(src), 32))), g.GNCParams()),
        (empty, src, f_empty, SF, g.GNCParams()),
        (tgt, empty, TF, f_empty, g.GNCParams()),
    ]
    for t, s, ft, fs, p in cases:
        with pytest.raises(capi.B2Error) as e:
            g.estimate_pose_gnc(t, s, ft, fs, p)
        assert e.value.status == 1
    # NULL arguments, and a correspondence buffer that is too small: the count is still written
    import ctypes as C

    cp = capi.GncParams(5000, 1, 0, 1000, 0.9, 1.4, 0.25, 3, 64, 6, 0, 5489)
    res = capi.RegistrationResultC()
    lib = capi.lib()
    assert lib.b2_estimate_pose_gnc(tgt.h, src.h, TF.h, SF.h, None, C.byref(res), None, 0, None) == 1
    assert lib.b2_estimate_pose_gnc(tgt.h, src.h, None, SF.h, C.byref(cp), C.byref(res), None, 0, None) == 1
    assert lib.b2_estimate_pose_gnc(tgt.h, src.h, TF.h, SF.h, C.byref(cp), None, None, 0, None) == 1
    pairs = np.zeros((4, 2), dtype=np.int64)
    num = C.c_size_t()
    assert lib.b2_estimate_pose_gnc(tgt.h, src.h, TF.h, SF.h, C.byref(cp), C.byref(res), pairs.ctypes.data_as(C.POINTER(C.c_int64)), 4, C.byref(num)) == 1
    assert num.value == len(ro.gnc(tgt.points, src.points, tf, sf)["C"]) > 4


def test_gnc_identity_cases():
    P, N = rc.small_scene(240, seed=5)
    F, _, _ = ro.fpfh(P, N, 2.0, 10000, num_threads=2)
    rng = np.random.default_rng(7)
    perm = rng.permutation(240)[:200]
    Ti = rc.pose_inverse(rc.offset_pose())
    S = (Ti[:3, :3] @ P[perm].T).T + Ti[:3, 3]
    sf = np.roll(F[perm], 1, axis=0)  # wrong matches: no tuple keeps its edge ratios exactly
    kw = dict(reciprocal_check=False, tuple_check=True, max_num_tuples=10, tuple_thresh=1.0)
    assert len(ro.gnc(P, S, F, sf, num_threads=2, **kw)["C"]) == 0
    tgt, src = g.PointCloud(P), g.PointCloud(S)
    TF, SF = g.Features.from_array(F), g.Features.from_array(sf)
    res, C = g.estimate_pose_gnc(tgt, src, TF, SF, g.GNCParams(**kw), correspondences=True)
    assert len(C) == 0 and np.array_equal(res.T_target_source, np.eye(4)) and res.inlier_rate == 0.0 and res.num_inliers == 0
    for p in (g.GNCParams(max_iterations=0), g.GNCParams(inner_iterations=0)):
        res, C = g.estimate_pose_gnc(tgt, src, TF, g.Features.from_array(F[perm]), p, correspondences=True)
        assert len(C) > 0 and np.array_equal(res.T_target_source, np.eye(4)) and res.inlier_rate == 0.0 and res.num_inliers == 0


@pytest.mark.parametrize("nq,nt", [(1, 5000), (40, 20000), (130, 777)])
def test_feature_nearest_split_targets(nq, nt):
    """Few queries against many targets: the targets are split over CTAs and the partial minima merged; ties across slice boundaries
    still go to the smallest index."""
    rng = np.random.default_rng(nq)
    T = rng.integers(0, 3, size=(nt, 8)).astype(np.float64)
    Q = rng.integers(0, 3, size=(nq, 8)).astype(np.float64)
    T[nt - 1] = T[nt // 2] = T[300] = Q[0]  # an exact match in several slices
    acc = np.zeros((nq, nt))
    for d in range(8):
        diff = Q[:, None, d] - T[None, :, d]
        acc = acc + diff * diff
    idx, sq = g.Features.from_array(Q).nearest(g.Features.from_array(T))
    assert np.array_equal(idx, np.argmin(acc, axis=1)) and np.array_equal(sq, acc.min(axis=1))
    assert sq[0] == 0.0 and idx[0] == np.nonzero((T == Q[0]).all(axis=1))[0].min()
