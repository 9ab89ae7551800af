"""Pose optimization through the C++ adapters (optimize_pose_gpu in gtsam_points_b200.hpp) compiles against the C ABI -- standalone
and against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_optimize.cpp) optimizes a unary VGICP
and a unary GICP factor on one key and must return the pose the Python package returns for the same data, bit for bit."""
import subprocess

import numpy as np
import pytest

import native
from gtsam_points_b200 import synthetic as syn


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_optimize_adapter_compiles(mock_gtsam):
    exe = native.adapter_driver("test_optimize", mock_gtsam)
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
def test_optimize_driver(mock_gtsam):
    import gtsam_points_b200 as g

    exe = native.adapter_driver("test_optimize", mock_gtsam)
    tp, tc = syn.make_cloud(30000, stream=51, scale=0.3)
    sp, sc = syn.make_cloud(7001, stream=52, scale=0.3)
    rng = np.random.default_rng(6)
    Tt = syn.random_pose(rng, 0.1, 1.0)
    T0 = Tt @ syn.random_pose(rng, 0.03, 0.2)
    # the same objects through the Python package: the adapters store the points in the same way (homogeneous rows, 4x4 covariances)
    target, source = g.PointCloud(tp, tc), g.PointCloud(sp, sc)
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(target)
    fs = [g.IntegratedVGICPFactor(Tt, 1, vm, source), g.IntegratedGICPFactor(Tt, 1, target, source, g.KdTree(target))]
    res = g.optimize_pose_gpu(fs, T0)
    native.run_driver(exe, [*homogeneous(tp, tc), *homogeneous(sp, sc), Tt, T0, res.pose, np.array([res.iterations, res.inner_iterations], dtype=np.float64)],
                      timeout=180)
