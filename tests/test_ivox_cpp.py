"""The C++ adapters of the iVox (iVoxGPU, IntegratedGICPFactor over it, gtsam_points_b200/cpp) compile against the C ABI --
standalone and in their GTSAM-typed form against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver
(tests/cpp/test_ivox.cpp) runs in the optimizer's call order and is checked against the Python restatement of the iVox
(tests/ivox_np.py) with np_ref's GICP algebra."""
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_ivox_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_ivox", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    assert "gtsam_points_b200::iVoxGPU" in syms
    if mock_gtsam:
        assert "gtsam::HessianFactor" in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_ivox_driver_in_optimizer_call_order(mock_gtsam):
    import ivox_np
    from gtsam_points_b200 import synthetic as syn
    from test_ivox_cpu import trajectory_frames

    exe = native.adapter_driver("test_ivox", mock_gtsam)
    frames = trajectory_frames(num_frames=3)
    ref = ivox_np.IvoxNp(1.0)
    ref.lru_horizon, ref.lru_clear_cycle = 10, 10
    for p, c in frames[:2]:
        ref.insert(p, c)
    sp, sc = syn.make_cloud(3000, stream=77, scale=1.0)
    rng = np.random.default_rng(6)
    Ts = syn.random_pose(rng, 0.05, 0.3)
    Ts2 = Ts @ syn.se3_exp(np.full(6, 0.01))
    rf = ivox_np.GicpIvoxNp(ref, sp, sc)
    lin = rf.linearize(Ts)
    err = rf.error(Ts2)
    corr = rf.corr.copy()
    ex = ref.export()
    q = ex["points"][rng.integers(0, len(ex["points"]), 64)] + rng.normal(scale=0.3, size=(64, 3))
    knn = np.array([ref.knn(x, 5, 1.5)[1] for x in q])
    ref.insert(*frames[2])
    lin2 = ivox_np.GicpIvoxNp(ref, sp, sc).linearize(Ts)

    def record(l):
        r = np.zeros(128)
        r[0:36], r[36:72], r[72:108] = l["H_target"].ravel(), l["H_source"].ravel(), l["H_target_source"].ravel()
        r[108:114], r[114:120], r[120], r[121] = l["b_target"], l["b_source"], l["error"], l["num_inliers"]
        return r

    def pad4(p):
        return np.concatenate([p, np.ones((len(p), 1))], 1)

    def pad44(c):
        m = np.zeros((len(c), 4, 4))
        m[:, :3, :3] = c
        return m

    arrays = [frames[0][0], frames[0][1], frames[1][0], frames[1][1], frames[2][0], frames[2][1], pad4(sp), pad44(sc), Ts, Ts2]
    arrays += [record(lin), np.array([err]), corr.astype(np.float64), q, knn, record(lin2)]
    native.run_driver(exe, arrays, timeout=180)
