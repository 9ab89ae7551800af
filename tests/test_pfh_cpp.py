"""The C++ adapters' PFH and keypoint feature path (estimate_pfh_gpu, the indices overloads, PFHEstimationParams) compiles against
the C ABI -- standalone and against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_pfh.cpp) is
checked against the CPU registration oracle."""
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_pfh_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_pfh", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    for s in ("b2_features_create_pfh", "b2_features_create_fpfh_at", "b2_features_create_fpfh", "b2_features_download"):
        assert s in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_pfh_driver(mock_gtsam):
    import registration_cases as rc
    import registration_oracle as ro

    exe = native.adapter_driver("test_pfh", mock_gtsam)
    P, N = rc.small_scene(700, seed=8, extent=8.0)
    idx = np.array([699, 3, 41, 3, 0, 512])
    radius = 1.5
    pf, pe, _ = ro.pfh(P, N, radius, 10000, indices=idx)
    ff, fe, _ = ro.fpfh_at(P, N, idx, radius, 10000)

    def pad(a, w):
        return np.concatenate([a, np.full((len(a), 1), w)], 1)

    native.run_driver(exe, [pad(P, 1.0), pad(N, 0.0), idx, pf, pe, ff, fe, [radius]], timeout=300)
