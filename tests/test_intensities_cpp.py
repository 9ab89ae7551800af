"""The C++ adapters' intensities (PointCloudGPU::from_frame / add_intensities, GaussianVoxelMapGPU with download_voxel_intensities,
iVoxGPU::voxel_intensities) compile against the C ABI -- standalone and against the header mocks (tests/cpp/mock_gtsam).  On a GPU
box the driver (tests/cpp/test_intensities.cpp) is checked against the CPU oracle (tests/intensity_oracle.cpp)."""
import os
import subprocess

import numpy as np
import pytest

import intensity_oracle as io
import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_intensity_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_intensities", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_cloud_create_with_intensities", "b2_cloud_create_with_added_intensities", "b2_cloud_download_intensities", "b2_voxelmap_insert_with_intensities", "b2_voxelmap_download_intensities",
              "b2_ivox_insert_with_intensities", "b2_ivox_download_intensities"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_intensity_driver(mock_gtsam):
    exe = native.adapter_driver("test_intensities", mock_gtsam)
    pts = np.load(os.path.join(native.ROOT, "tests", "golden", "kitti00_pair.npz"))["frame0"].astype(np.float64)
    rng = np.random.default_rng(3)
    ints = rng.normal(30.0, 20.0, len(pts)) / 3.0
    covs = np.zeros((len(pts), 4, 4))
    covs[:, :3, :3] = np.eye(3) * 0.01
    vm = io.Map(0.5)
    vm.insert(pts, ints)
    ivox = io.Map(0.5, max_points_in_cell=20, min_dist_in_cell=0.1)
    ivox.insert(pts, ints)
    xyz1 = np.concatenate([pts, np.ones((len(pts), 1))], 1)
    native.run_driver(exe, [xyz1, covs, ints, vm.export()[1], ivox.export()[3]], timeout=180)
