"""The C++ adapters of ICP on iVox targets (IntegratedICPFactor over an iVoxGPU, IntegratedPointToPlaneICPFactor over an
iVoxCovarianceEstimationGPU, gtsam_points_b200/cpp) compile against the C ABI -- standalone and in their GTSAM-typed form against
the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_ivox_icp.cpp) runs in the optimizer's call order
and is checked against the restatement (ivox_icp_np.IcpIvoxNp)."""
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_ivox_icp_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_ivox_icp", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    assert "gtsam_points_b200::IntegratedPointToPlaneICPFactor" in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_ivox_icp_driver_in_optimizer_call_order(mock_gtsam):
    import ivox_cov_np
    import ivox_icp_np
    import ivox_np
    from gtsam_points_b200 import synthetic as syn
    from test_ivox_cov_cpu import reduced, scene_frames

    exe = native.adapter_driver("test_ivox_icp", mock_gtsam)
    frames = scene_frames(3)
    plain, est = ivox_np.IvoxNp(1.0), reduced(ivox_cov_np.IvoxCovNp(1.0))
    for p in frames[:2]:
        plain.insert(p)
        est.insert(p)
    rng = np.random.default_rng(6)
    n = 1200
    sp = frames[2][rng.choice(len(frames[2]), n, replace=False)] + rng.normal(scale=0.05, size=(n, 3))
    Ts = syn.random_pose(rng, 0.02, 0.1)
    Ts2 = Ts @ syn.se3_exp(np.full(6, 0.01))
    rp, rq = ivox_icp_np.IcpIvoxNp(plain, sp), ivox_icp_np.IcpIvoxNp(est, sp, point_to_plane=True)
    lin = [rp.linearize(Ts), rq.linearize(Ts)]
    corr = [rp.corr, rq.corr]
    err = [rp.error(Ts2), rq.error(Ts2)]
    assert min(l["num_inliers"] for l in lin) > 100
    plain.insert(frames[2])
    est.insert(frames[2])
    lin2 = [rp.linearize(Ts), rq.linearize(Ts)]

    def record(l):
        r = np.zeros(128)
        r[0:36], r[36:72], r[72:108] = l["H_target"].ravel(), l["H_source"].ravel(), l["H_target_source"].ravel()
        r[108:114], r[114:120], r[120], r[121] = l["b_target"], l["b_source"], l["error"], l["num_inliers"]
        return r

    arrays = [frames[0], frames[1], frames[2], np.concatenate([sp, np.ones((n, 1))], 1), Ts, Ts2, record(lin[0]), record(lin[1]), np.array(err)]
    arrays += [corr[0].astype(np.float64), corr[1].astype(np.float64), record(lin2[0]), record(lin2[1])]
    native.run_driver(exe, arrays, timeout=180)
