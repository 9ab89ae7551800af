"""The C++ adapters' frame-preparation path (voxelgrid_sampling_gpu, estimate_covariances_gpu, KdTreeGPU from a device cloud)
compiles against the C ABI -- standalone and against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver
(tests/cpp/test_preprocess.cpp) is checked against the CPU voxel-grid oracle and the host-array factor path."""
import os
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_preprocess_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_preprocess", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_cloud_create_voxelgrid", "b2_cloud_create_estimated", "b2_kdtree_create_from_cloud", "b2_cloud_download"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_preprocess_driver(mock_gtsam):
    import voxelgrid_oracle as vo
    from gtsam_points_b200 import synthetic as syn

    exe = native.adapter_driver("test_preprocess", mock_gtsam)
    k00 = np.load(os.path.join(native.ROOT, "tests", "golden", "kitti00_pair.npz"))
    tp, sp = k00["frame0"], k00["frame1"]
    res = 0.25
    want = vo.voxelgrid_sampling(tp, res)[0]
    delta = syn.random_pose(np.random.default_rng(3), 0.02, 0.3)

    def pad4(p):
        return np.concatenate([p, np.ones((len(p), 1))], 1)

    native.run_driver(exe, [pad4(tp), pad4(sp), np.array([res]), want, delta], timeout=180)
