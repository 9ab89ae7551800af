"""The C++ adapters' global registration path (FeaturesGPU, estimate_fpfh_gpu, estimate_pose_ransac_gpu) compiles against the C ABI --
standalone and against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_registration.cpp) is checked
against the CPU registration oracle."""
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_registration_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_registration", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_features_create", "b2_features_create_fpfh", "b2_estimate_pose_ransac", "b2_features_download"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_registration_driver(mock_gtsam):
    import normals_ref
    import registration_cases as rc
    import registration_oracle as ro
    import voxelgrid_oracle as vo

    exe = native.adapter_driver("test_registration", mock_gtsam)
    d = rc.kitti00()
    tgt = vo.voxelgrid_sampling(d["frame0"], 0.5)[0]
    src = vo.voxelgrid_sampling(d["frame1"], 0.5)[0]
    tn, sn = normals_ref.estimate_normals(tgt, 10)[0], normals_ref.estimate_normals(src, 10)[0]
    P = rc.pose_inverse(rc.offset_pose()) @ d["T_final"]
    src = (P[:3, :3] @ src.T).T + P[:3, 3]
    sn = (P[:3, :3] @ sn.T).T
    # the default storage of a device cloud is lossless, so the oracle and the device see the same values
    tf, te, _ = ro.fpfh(tgt, tn, 5.0, 10000)
    sf, se, _ = ro.fpfh(src, sn, 5.0, 10000)
    r = ro.ransac(tgt, src, tf, sf, max_iterations=1000)
    want = np.concatenate([r["T_target_source"].ravel(), [r["num_inliers"], r["hypothesis"]]])

    def pad(a, w):
        return np.concatenate([a, np.full((len(a), 1), w)], 1)

    native.run_driver(exe, [pad(tgt, 1.0), pad(tn, 0.0), pad(src, 1.0), pad(sn, 0.0), tf, sf, np.concatenate([te, se]).astype(np.float64), want], timeout=300)
