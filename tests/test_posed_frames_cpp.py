"""The C++ adapters' map updates from device clouds (GaussianVoxelMapGPU::insert_cloud, iVoxGPU::insert_cloud, transform_gpu,
merge_frames_gpu) compile against the C ABI -- standalone and against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the
driver (tests/cpp/test_posed_frames.cpp) checks them against the host-array path over the numpy-posed arrays."""
import subprocess

import numpy as np
import pytest

import adversarial as adv
import native
import posed_ref


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_posed_frames_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_posed_frames", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_voxelmap_insert_cloud", "b2_ivox_insert_cloud", "b2_cloud_create_transformed", "b2_merge_frames_to_cloud"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_posed_frames_driver(mock_gtsam):
    from gtsam_points_b200 import synthetic as syn

    exe = native.adapter_driver("test_posed_frames", mock_gtsam)
    rng = np.random.default_rng(8)
    pts = rng.uniform(-8, 8, (4000, 3))
    covs = adv.spd(len(pts), 3)
    T = syn.random_pose(rng, 0.5, 3.0)
    q, qc, _ = posed_ref.transform(T, pts, covs)
    native.run_driver(exe, [pts, covs, T, q, qc], timeout=180)
