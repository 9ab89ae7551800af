"""The C++ adapters' region growing (region_growing_init_gpu, region_growing_update_gpu) compiles against the C ABI -- standalone and
against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_segmentation.cpp) is checked against the
CPU oracle's trace."""
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_segmentation_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_segmentation", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_region_growing_create", "b2_region_growing_update", "b2_region_growing_get", "b2_region_growing_destroy", "b2_min_cut"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_segmentation_driver(mock_gtsam):
    import segmentation_oracle as so

    exe = native.adapter_driver("test_segmentation", mock_gtsam)
    rng = np.random.default_rng(3)
    n = 3000
    p = np.c_[rng.uniform(-5, 5, (n, 2)), rng.normal(0, 0.01, n)]
    nr = np.tile([0.0, 0.0, 1.0], (n, 1)) + rng.normal(0, 0.1, (n, 3))
    nr /= np.linalg.norm(nr, axis=1, keepdims=True)
    seed_point, dist, angle, dil, maxc = np.array([0.5, -0.5, 0.0]), 0.4, 0.2, 0.3, 1500
    steps = [1, 40, 0, 1000, 10**6, 1]
    trace = so.trace(p, nr, so.nearest(p, seed_point), steps, distance_threshold=dist, angle_threshold=angle, dilation_radius=dil, max_cluster_size=maxc)
    flags = [float(c) for c, _ in trace]
    sizes = [len(cl) for _, cl in trace]
    clusters = np.concatenate([cl for _, cl in trace]).astype(np.float64)
    prm = np.r_[seed_point, dist, angle, dil, maxc]
    import gtsam_points_b200 as g

    cut = g.min_cut(g.PointCloud(p, normals=nr), 17, g.MinCutParams(background_mask_radius=2.0))
    mc = np.r_[17, cut.cluster_indices].astype(np.float64)
    native.run_driver(exe, [np.c_[p, np.ones(n)], np.c_[nr, np.zeros(n)], prm, steps, flags, sizes, clusters, mc], timeout=180)
