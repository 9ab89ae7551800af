"""GPU memory offloading through the C++ adapters (OffloadableGPU, set_enable_offloading) compiles against the C ABI -- standalone and
against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_offload.cpp) runs the optimizers' call
order with offloading on over offloaded objects and checks it against the same factors over resident ones, bit for bit."""
import subprocess

import numpy as np
import pytest

import native
from gtsam_points_b200 import synthetic as syn


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_offload_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_offload", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_cloud_offload", "b2_cloud_reload", "b2_cloud_touch", "b2_cloud_residency", "b2_voxelmap_offload", "b2_voxelmap_reload", "b2_voxelmap_touch",
              "b2_voxelmap_residency", "b2_access_time_current", "b2_factor_set_enable_offloading", "b2_factor_device_bytes"):
        assert s in syms, s


def homogeneous(p, c):
    xyz1 = np.concatenate([p, np.ones((len(p), 1))], 1)
    c4 = np.zeros((len(p), 4, 4))
    c4[:, :3, :3] = c
    return xyz1, c4


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_offload_driver(mock_gtsam):
    exe = native.adapter_driver("test_offload", mock_gtsam)
    tp, tc = syn.make_cloud(30000, stream=41, scale=0.3)
    sp, sc = syn.make_cloud(7001, stream=42, scale=0.3)
    rng = np.random.default_rng(4)
    Ts, Ts2 = syn.random_pose(rng, 0.03, 0.2), syn.random_pose(rng, 0.03, 0.2)
    native.run_driver(exe, [*homogeneous(tp, tc), *homogeneous(sp, sc), np.eye(4), Ts, Ts2], timeout=180)
