"""The C++ adapter of iVoxCovarianceEstimation (iVoxCovarianceEstimationGPU, and IntegratedGICPFactor over it,
gtsam_points_b200/cpp) compiles against the C ABI -- standalone and in its GTSAM-typed form against the header mocks
(tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_ivox_cov.cpp) runs in the optimizer's call order and is checked
against the restatement (tests/ivox_cov_np.py) with np_ref's GICP algebra."""
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_ivox_cov_adapter_compiles(mock_gtsam):
    exe = native.adapter_driver("test_ivox_cov", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    assert "gtsam_points_b200::iVoxCovarianceEstimationGPU" in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_ivox_cov_driver_in_optimizer_call_order(mock_gtsam):
    import ivox_cov_np
    import ivox_np
    import np_ref
    from gtsam_points_b200 import synthetic as syn
    from test_ivox_cov_cpu import reduced, scene_frames

    exe = native.adapter_driver("test_ivox_cov", mock_gtsam)
    frames = scene_frames(3)
    ref = reduced(ivox_cov_np.IvoxCovNp(1.0))
    for p in frames[:2]:
        ref.insert(p)
    ex = ref.export()
    valid = ref.valid_mask()
    vidx = np.array(sorted(ref.flat_index(), key=lambda c: ref.flat_index()[c]), dtype=np.int64)[valid]
    rng = np.random.default_rng(6)
    q = ex["points"][rng.integers(0, len(ex["points"]), 64)] + rng.normal(scale=0.3, size=(64, 3))
    force = ref.knn_batch(q, 5, 1.5, False)[1]
    n = 1200
    sp = frames[2][rng.choice(len(frames[2]), n, replace=False)] + rng.normal(scale=0.05, size=(n, 3))
    A = rng.normal(size=(n, 3, 3)) * 0.05
    sc = A @ A.transpose(0, 2, 1) + 1e-3 * np.eye(3)
    Ts = syn.random_pose(rng, 0.02, 0.1)
    Ts2 = Ts @ syn.se3_exp(np.full(6, 0.01))

    def lin_at(delta, eval_delta=None):
        corr = ref.knn_batch(ivox_np.transform(delta, sp), 1, 1.0, True)[0][:, 0]
        fi, e = ref.flat_index(), ref.export()
        flat = np.array([fi[int(c)] if c >= 0 else -1 for c in corr], dtype=np.int64)
        return corr, np_ref.linearize(delta, sp, sc, e["points"], e["covs"], flat, eval_delta if eval_delta is not None else delta)

    corr, lin = lin_at(Ts)
    err = lin_at(Ts, Ts2)[1]["error"]
    ref.insert(frames[2])
    lin2 = lin_at(Ts)[1]

    def record(l):
        r = np.zeros(128)
        r[0:36], r[36:72], r[72:108] = l["H_target"].ravel(), l["H_source"].ravel(), l["H_target_source"].ravel()
        r[108:114], r[114:120], r[120], r[121] = l["b_target"], l["b_source"], l["error"], l["num_inliers"]
        return r

    pad44 = np.zeros((n, 4, 4))
    pad44[:, :3, :3] = sc
    arrays = [frames[0], frames[1], frames[2], np.concatenate([sp, np.ones((n, 1))], 1), pad44, Ts, Ts2]
    arrays += [vidx.astype(np.float64), ex["points"][valid], ex["normals"][valid], ex["covs"][valid], q, force, record(lin), np.array([err]), corr.astype(np.float64), record(lin2)]
    native.run_driver(exe, arrays, timeout=180)
