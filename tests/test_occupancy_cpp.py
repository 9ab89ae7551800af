"""The C++ adapters' FastOccupancyGridGPU and raycast_gpu compile against the C ABI -- standalone and against the header mocks
(tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_occupancy.cpp) is checked against the CPU oracle."""
import os
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_occupancy_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_occupancy", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_occgrid_create", "b2_occgrid_insert", "b2_occgrid_overlap", "b2_occgrid_free_rays", "b2_occgrid_download", "b2_raycast"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_occupancy_driver(mock_gtsam):
    import occupancy_oracle as oo
    from gtsam_points_b200 import synthetic as syn

    exe = native.adapter_driver("test_occupancy", mock_gtsam)
    k00 = np.load(os.path.join(native.ROOT, "tests", "golden", "kitti00_pair.npz"))
    tgt, src = k00["frame0"].astype(np.float64), k00["frame1"].astype(np.float64)
    res = 0.5
    rng = np.random.default_rng(5)
    poses = np.stack([np.eye(4), k00["T_final"]] + [syn.random_pose(rng, 0.05, 0.5) for _ in range(6)])
    orc = oo.Grid(res)
    orc.insert(tgt, poses[0])
    counts = [orc.overlaps(src, T)[0] for T in poses]
    flags = orc.overlaps(src, poses[0])[1]
    orc.free_rays(src, poses[1])
    rays = rng.uniform(-20, 20, (200, 6))
    off, coords = oo.raycast(rays[:, :3], rays[:, 3:], res)
    xyz1 = lambda p: np.concatenate([p, np.ones((len(p), 1))], 1)  # noqa: E731
    native.run_driver(exe, [xyz1(tgt), xyz1(src), [res], poses.reshape(-1), counts, flags, orc.cells(), rays, off, coords], timeout=180)
