"""The header-only C++ adapters (gtsam_points_b200/cpp) compile against the C ABI -- standalone AND in their GTSAM-typed
form against header mocks of GTSAM / Eigen / gtsam_points' linearization hook (tests/cpp/mock_gtsam; there is no GTSAM in this
image).  On a GPU box both drivers are run against oracle results in the reference optimizer's call order."""
import os
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_adapters_compile_against_c_abi(mock_gtsam):
    exe = native.adapter_driver("test_adapters", mock_gtsam)
    assert os.path.exists(exe)
    if mock_gtsam:  # the GTSAM branch really was compiled: its symbols are in the binary
        syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
        assert "gtsam::HessianFactor" in syms and "gtsam_points::NonlinearFactorSet" in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_adapters_match_oracle_in_reference_call_order(mock_gtsam):
    import oracle_lib as orc
    from gtsam_points_b200 import synthetic as syn

    exe = native.adapter_driver("test_adapters", mock_gtsam)
    tp, tc = syn.make_cloud(30000, stream=1, scale=0.25)
    sp, sc = syn.make_cloud(12000, stream=2, scale=0.25)
    rng = np.random.default_rng(2)
    Tt = syn.random_pose(rng, 0.4, 3.0)
    Ts = Tt @ syn.random_pose(rng, 0.01, 0.1)
    Ts2 = Tt @ syn.random_pose(rng, 0.01, 0.1)

    def pad4(p):
        return np.concatenate([p, np.ones((len(p), 1))], 1)

    def pad44(c):  # the reference's column-major Matrix4d with zero row/col 3 (symmetric => layout-agnostic)
        m = np.zeros((len(c), 4, 4))
        m[:, :3, :3] = c
        return m

    otgt, osrc = orc.Cloud(tp, tc), orc.Cloud(sp, sc)
    vm = orc.VoxelMap(0.5)
    vm.insert(otgt)
    fv = orc.Factor(vm, osrc, num_threads=4)
    fg = orc.Factor(otgt, osrc, tree=orc.KdTree(otgt, 4), num_threads=4)
    d, d2 = orc.calc_delta(Tt, Ts), orc.calc_delta(Tt, Ts2)
    ev, eg = fv.linearize_raw(d), fg.linearize_raw(d)
    errs = np.array([fv.error(d2), fg.error(d2)])
    overlap = np.array([vm.overlap(osrc, d)])
    eicp = orc.Factor(otgt, osrc, tree=orc.KdTree(otgt, 4), num_threads=4, icp="point").linearize_raw(d)
    merged_xyz, _ = orc.merge_frames(np.stack([Tt, Ts]), [otgt, osrc], 0.5)
    cov_head = orc.estimate_covariances(tp, 10, num_threads=4)[:256]
    native.run_driver(exe, (pad4(tp), pad44(tc), pad4(sp), pad44(sc), Tt, Ts, Ts2, ev, eg, errs, np.array([0.5]), ev, overlap, eicp, np.array([len(merged_xyz)]), cov_head), timeout=180)
