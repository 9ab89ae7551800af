"""Multi-pose optimization through the C++ adapters (optimize_poses_gpu and NonlinearFactorSetGPU::optimize_poses in
gtsam_points_b200.hpp) compiles against the C ABI -- standalone and against the header mocks (tests/cpp/mock_gtsam).  On a GPU box
the driver (tests/cpp/test_optimize_graph.cpp) optimizes three frames linked by binary VGICP and GICP factors with a prior on frame
0, and must return the poses the Python package returns for the same data, bit for bit."""
import subprocess

import numpy as np
import pytest

import native
from gtsam_points_b200 import synthetic as syn


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_optimize_graph_adapter_compiles(mock_gtsam):
    exe = native.adapter_driver("test_optimize_graph", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_factor_set_optimize_poses", "b2_lm_params_default"):
        assert s in syms, s


def homogeneous(p, c):
    xyz1 = np.concatenate([p, np.ones((len(p), 1))], 1)
    c4 = np.zeros((len(p), 4, 4))
    c4[:, :3, :3] = c
    return xyz1, c4


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_optimize_graph_driver(mock_gtsam):
    import gtsam_points_b200 as g

    exe = native.adapter_driver("test_optimize_graph", mock_gtsam)
    pts, covs = syn.make_cloud(20000, stream=61, scale=0.3)
    rng = np.random.default_rng(8)
    gt = [np.eye(4), syn.random_pose(rng, 0.05, 0.5), syn.random_pose(rng, 0.05, 0.5)]
    frames = []
    for T in gt:
        R, t = T[:3, :3], T[:3, 3]
        frames.append(((pts - t) @ R, R.T @ covs @ R))
    init = [gt[0]] + [T @ syn.random_pose(rng, 0.02, 0.1) for T in gt[1:]]
    # the same objects through the Python package: the adapters store the points in the same way (homogeneous rows, 4x4 covariances)
    clouds = [g.PointCloud(p, c) for p, c in frames]
    maps = []
    for c in clouds:
        vm = g.GaussianVoxelMapGPU(0.5)
        vm.insert(c)
        maps.append(vm)
    fs = [g.IntegratedVGICPFactor(0, 1, maps[0], clouds[1]), g.IntegratedVGICPFactor(1, 2, maps[1], clouds[2]),
          g.IntegratedGICPFactor(0, 2, clouds[0], clouds[2], g.KdTree(clouds[0]))]
    res = g.optimize_graph_gpu(fs, {k: init[k] for k in range(3)}, [g.PriorFactorPose3(0, gt[0], 1e6)])
    arrays = [a for p, c in frames for a in homogeneous(p, c)]
    native.run_driver(exe, arrays + [np.stack(init), gt[0], np.stack([res.values[k] for k in range(3)]), np.array([res.iterations, res.inner_iterations], dtype=np.float64)],
                      timeout=180)
