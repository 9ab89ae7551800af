"""The C++ adapters' normals paths (PointCloudGPU with normals and from_frame picking them up, IntegratedVGICPFactor::
set_enable_surface_validation, point-to-plane IntegratedICPFactor over a target cloud with normals) compile against the C ABI --
standalone and against the header mocks (tests/cpp/mock_gtsam).  On a GPU box the driver (tests/cpp/test_normals.cpp) is
checked against the host restatement of surface validation (tests/normals_ref.py)."""
import subprocess

import numpy as np
import pytest

import native


@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_normals_adapters_compile(mock_gtsam):
    exe = native.adapter_driver("test_normals", mock_gtsam)
    syms = subprocess.run(["nm", "-C", exe], capture_output=True, text=True).stdout
    assert "b2_factor_set_enable_surface_validation" in syms and "b2_cloud_create_with_normals" in syms


@pytest.mark.gpu
@pytest.mark.parametrize("mock_gtsam", [False, True])
def test_normals_driver(mock_gtsam):
    import normals_ref as nref
    import oracle_lib as orc
    from gtsam_points_b200 import synthetic as syn

    exe = native.adapter_driver("test_normals", mock_gtsam)
    tp, tc = syn.make_cloud(8000, stream=1, scale=0.25)
    sp, sc = syn.make_cloud(5000, stream=2, scale=0.25)
    nrm = nref.normals_from_covs(sp, sc)
    nrm[::3] *= -1.0
    rng = np.random.default_rng(4)
    tn = rng.normal(size=(len(tp), 3))
    tn /= np.linalg.norm(tn, axis=1, keepdims=True)
    T = syn.random_pose(rng, 0.02, 0.2)
    ovm = orc.VoxelMap(0.5)
    ovm.insert(orc.Cloud(tp, tc))
    plain = orc.Factor(ovm, orc.Cloud(sp, sc), num_threads=2)
    val = nref.ValidatedVGICP(ovm, sp, sc, nrm)
    inliers = [plain.linearize(T)["num_inliers"], val.linearize(T)["num_inliers"]]
    assert inliers[1] < inliers[0]

    def pad4(p, w):
        return np.concatenate([p, np.full((len(p), 1), w)], 1)

    def pad44(c):
        m = np.zeros((len(c), 4, 4))
        m[:, :3, :3] = c
        return m

    native.run_driver(exe, [pad4(tp, 1.0), pad44(tc), pad4(sp, 1.0), pad44(sc), pad4(nrm, 0.0), tn, T, np.array(inliers), val.correspondences()], timeout=180)
