"""The C++ adapters' GNC path (GNCParams, estimate_pose_gnc_gpu) compiles against the C ABI -- standalone and against the header mocks
(tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_gnc.cpp) is checked against the CPU registration oracle."""
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_gnc_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_gnc", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_features_create", "b2_estimate_pose_gnc"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_gnc_driver(mock_gtsam):
    import normals_ref
    import registration_cases as rc
    import registration_oracle as ro
    import voxelgrid_oracle as vo

    exe = native.adapter_driver("test_gnc", mock_gtsam)
    d = rc.kitti00()
    tgt = vo.voxelgrid_sampling(d["frame0"], 0.5)[0]
    src = vo.voxelgrid_sampling(d["frame1"], 0.5)[0]
    tn, sn = normals_ref.estimate_normals(tgt, 10)[0], normals_ref.estimate_normals(src, 10)[0]
    P = rc.pose_inverse(rc.offset_pose()) @ d["T_final"]
    src = (P[:3, :3] @ src.T).T + P[:3, 3]
    sn = (P[:3, :3] @ sn.T).T
    tf, _, _ = ro.fpfh(tgt, tn, 5.0, 10000)
    sf, _, _ = ro.fpfh(src, sn, 5.0, 10000)
    r = ro.gnc(tgt, src, tf, sf)
    want = np.concatenate([r["T_target_source"].ravel(), [r["num_inliers"], r["slack"].sum()]])

    native.run_driver(exe, [np.concatenate([tgt, np.ones((len(tgt), 1))], 1), np.concatenate([src, np.ones((len(src), 1))], 1), tf, sf, r["C"].astype(np.float64), want], timeout=300)
