"""The device's alignment step -- RANSAC's 3- and 2-point hypotheses and GNC's first, unweighted solve -- against the
extended-precision SVD reference (alignment_ref.py) on the case families of alignment_cases.py: random rotations and rotations within
1e-6 of pi, noisy correspondences, thin triangles and rods (s2 / s1 down to 1e-8), exactly collinear sets, mirrored sources, sets
1e3 - 1e6 m from the origin, 4-DoF pairs with no preferred rotation, and N from 2 to 4000.  The solvers are reached only through
estimate_pose_ransac and estimate_pose_gnc; the reference is computed from the clouds' stored points."""
import numpy as np
import pytest

import alignment_cases as ac
import gtsam_points_b200 as g
from gtsam_points_b200 import capi

pytestmark = pytest.mark.gpu


def _stored(cloud):
    out = np.zeros((len(cloud), 3))
    capi.check(capi.lib().b2_cloud_download(cloud.h, capi.dptr(out), None, None))
    return out


def _run_all(cases, solve, what):
    """solve(case) -> (T, target, source) for each case; every case's bound is checked and every failure reported."""
    ratios, failures = {}, []
    for case in cases:
        try:
            T, tgt, src = solve(case)
            r = ac.check(case, T, tgt, src)
            ratios.setdefault(case.family, []).append(r)
        except AssertionError as e:
            failures.append(f"{case.family}/{case.name} (dof {case.dof}): {e}")
    for fam, r in sorted(ratios.items()):
        print(f"{what} {fam}: max |R - R_ref|_max = {max(r):.3g} eps kappa over {len(r)} cases (bound {ac.C_R:g})")
    assert not failures, "\n".join(failures)


def test_ransac_single_hypothesis_alignment():
    """One hypothesis over the whole 3-point (dof 6) or 2-point (dof 4) set: one-hot features match point i to point i, the polygon
    test and the voxel count accept any finite pose, so the hypothesis wins iff its pose is finite (a NaN pose counts 0)."""

    def solve(case):
        n = len(case.source)
        tgt, src = g.PointCloud(case.target), g.PointCloud(case.source)
        F = g.Features.from_array(np.eye(n))
        params = g.RANSACParams(max_iterations=1, dof=case.dof, poly_error_thresh=1e9, inlier_voxel_resolution=1e7)
        res = g.estimate_pose_ransac(tgt, src, F, F, params, hypothesis_inliers=True)
        assert res.hypothesis == 0 and res.hypothesis_inliers[0] > 0, f"hypothesis {res.hypothesis}, count {res.hypothesis_inliers[0]}, T {res.T_target_source[:3]}"
        return res.T_target_source, _stored(tgt), _stored(src)

    _run_all(ac.ransac_cases(), solve, "RANSAC")


def test_gnc_single_unweighted_solve():
    """max_iterations = inner_iterations = 1 without the tuple check, identical distinct feature rows on both sides: C is (k, k) for
    every k, and T_target_source is the device's unweighted alignment of all N pairs."""

    def solve(case):
        n = len(case.source)
        tgt, src = g.PointCloud(case.target), g.PointCloud(case.source)
        F = g.Features.from_array(np.random.default_rng(n).standard_normal((n, 4)))
        params = g.GNCParams(max_init_samples=n, tuple_check=False, max_iterations=1, inner_iterations=1, dof=case.dof)
        res, C = g.estimate_pose_gnc(tgt, src, F, F, params, correspondences=True)
        assert np.array_equal(C, np.repeat(np.arange(n), 2).reshape(n, 2)), C[:5]
        return res.T_target_source, _stored(tgt), _stored(src)

    _run_all(ac.gnc_cases(), solve, "GNC")


@pytest.mark.parametrize("dof", [6, 4])
def test_ransac_rejects_coincident_target_samples(dof):
    """Two sampled target points coincide: d_t = 0 against d_s > 0 is a polygon error of 1, so the hypothesis is rejected (-2) and
    the result is the identity."""
    S = np.array([[0.0, 0.0, 0.0], [4.0, 1.0, 0.5], [1.0, 5.0, -2.0]])[: 3 if dof == 6 else 2]
    T = np.array([[3.0, 3.0, 3.0], [3.0, 3.0, 3.0], [7.0, 2.0, 1.0]])[: len(S)]
    F = g.Features.from_array(np.eye(len(S)))
    res = g.estimate_pose_ransac(g.PointCloud(T), g.PointCloud(S), F, F, g.RANSACParams(max_iterations=1, dof=dof), hypothesis_inliers=True)
    assert res.hypothesis_inliers[0] == -2 and res.hypothesis == -1
    assert np.array_equal(res.T_target_source, np.eye(4)) and res.num_inliers == 0
