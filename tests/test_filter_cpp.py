"""The C++ adapters' frame filters (sample_gpu, random_sampling_gpu, randomgrid_sampling_gpu, remove_outliers_gpu,
find_inlier_points_gpu) compile against the C ABI -- standalone and against the header mocks (tests/cpp/mock_gtsam).  On a GPU box
the driver (tests/cpp/test_filter.cpp) is checked against the CPU oracle's selections."""
import os
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_filter_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_filter", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_cloud_create_sampled", "b2_cloud_create_random_sampled", "b2_cloud_create_randomgrid", "b2_cloud_create_inliers"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_filter_driver(mock_gtsam):
    import filter_oracle as fo

    exe = native.adapter_driver("test_filter", mock_gtsam)
    pts = np.load(os.path.join(native.ROOT, "tests", "golden", "kitti00_pair.npz"))["frame0"].astype(np.float64)
    seed, rate, res, grid_rate, k, std_thresh = 42, 0.3, 0.5, 0.5, 10, 1.0
    want_random = fo.random_sampling(len(pts), rate, seed)
    want_grid = fo.randomgrid_sampling(pts, res, grid_rate, seed)
    want_inliers = fo.inliers(pts, k, std_thresh)[0]
    indices = np.random.default_rng(1).integers(0, len(pts), 500)
    xyz1 = np.concatenate([pts, np.ones((len(pts), 1))], 1)
    prm = np.array([seed, rate, res, grid_rate, k, std_thresh], dtype=np.float64)
    native.run_driver(exe, [xyz1, prm, want_random, want_grid, want_inliers, indices], timeout=180)
