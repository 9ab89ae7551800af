"""The extended-precision alignment reference (alignment_ref.py) against known answers and numpy, and the CPU oracle's restatement of
the device's alignment (registration_oracle.cpp: Horn's quaternion, the planar closed form) against the reference on every case
family of alignment_cases.py."""
import mpmath as mp
import numpy as np
import pytest

import alignment_cases as ac
import alignment_ref as ar
import registration_oracle as ro


def _exact_pose(R, t, S):
    """Target rows R s + t kept in extended precision (no float64 rounding), so the alignment is exactly (R, t)."""
    return ar.apply(R, t, S)


@pytest.mark.parametrize("angle", [0.0, 0.3, 2.0, mp.pi - mp.mpf("1e-6"), mp.pi - mp.mpf("1e-12")])
@pytest.mark.parametrize("n", [3, 20])
def test_reference_recovers_known_rotations(angle, n):
    rng = np.random.default_rng(n)
    S = rng.uniform(-10.0, 10.0, (n, 3))
    R = ar.rotation(rng.standard_normal(3), angle)
    t = [1.5, -2.0, 1e3]
    ref = ar.align(_exact_pose(R, t, S), S)
    assert ar.max_abs(ref.R, R) <= 1e-30
    assert ar.max_abs(ref.t, mp.matrix(t)) <= 1e-27
    assert ref.kappa < 1e3 and (n == 3 or ref.d == 1)  # a 3-point H has s3 = 0, so the sign of det U det V is arbitrary
    with mp.workdps(ar.DPS):
        assert abs(mp.det(ref.R) - 1) <= 1e-30


def test_reference_recovers_planar_rotations():
    rng = np.random.default_rng(4)
    for n in (2, 30):
        S = rng.uniform(-10.0, 10.0, (n, 3))
        for angle in (0.0, 1.0, -2.5, mp.pi - mp.mpf("1e-9")):
            R = ar.rotation([0.0, 0.0, 1.0], angle)
            ref = ar.align(_exact_pose(R, [3.0, 4.0, 5.0], S), S, dof=4)
            assert ar.max_abs(ref.R, R) <= 1e-30 and ar.max_abs(ref.t, mp.matrix([3.0, 4.0, 5.0])) <= 1e-28


@pytest.mark.parametrize("mirror", [[1.0, 1.0, -1.0], [-1.0, -1.0, -1.0], [1.0, -1.0, 1.0]])
def test_reference_is_proper_on_mirrored_sets(mirror):
    rng = np.random.default_rng(11)
    T = rng.uniform(-10.0, 10.0, (50, 3)) * [3.0, 2.0, 1.0]
    ref = ar.align(T, T * mirror)
    assert ref.d == -1
    with mp.workdps(ar.DPS):
        assert abs(mp.det(ref.R) - 1) <= 1e-30
        assert mp.mnorm(ref.R.T * ref.R - mp.eye(3), 1) <= 1e-30
    # numpy's Kabsch with the same reflection fix
    U, _, Vt = np.linalg.svd((T - T.mean(0)).T @ (T * mirror - (T * mirror).mean(0)))
    R = U @ np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))]) @ Vt
    assert np.abs(ref.R64() - R).max() <= 1e-13


def test_reference_agrees_with_numpy_svd():
    rng = np.random.default_rng(3)
    for n in (3, 10, 200):
        T, S = rng.standard_normal((n, 3)) * 5.0, rng.standard_normal((n, 3)) * 5.0
        ref = ar.align(T, S)
        H = (T - T.mean(0)).T @ (S - S.mean(0))
        U, sv, Vt = np.linalg.svd(H)
        R = U @ np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))]) @ Vt
        assert np.abs(np.array([float(s) for s in ref.sigma]) - sv).max() <= 1e-13 * sv[0]
        assert np.abs(ref.R64() - R).max() <= 1e-12 * ref.kappa
        assert np.abs(ref.t64() - (T.mean(0) - R @ S.mean(0))).max() <= 1e-11 * ref.kappa


def test_weighted_reference():
    rng = np.random.default_rng(8)
    T, S = rng.standard_normal((12, 3)), rng.standard_normal((12, 3))
    w = rng.integers(1, 4, 12)
    ref_w = ar.align(T, S, weights=w)
    ref_rep = ar.align(np.repeat(T, w, axis=0), np.repeat(S, w, axis=0))
    assert ar.max_abs(ref_w.R, ref_rep.R) <= 1e-60 and ar.max_abs(ref_w.t, ref_rep.t) <= 1e-60
    ref_1 = ar.align(T, S, weights=np.full(12, 0.5))
    ref_0 = ar.align(T, S)
    assert ar.max_abs(ref_1.R, ref_0.R) <= 1e-60 and ar.max_abs(ref_1.t, ref_0.t) <= 1e-60


def test_reference_on_degenerate_sets():
    # rank-1 H: kappa is infinite; the reference still maps the source line onto the target line
    lam = np.array([[-1.0], [0.0], [2.0]])
    ref = ar.align(lam * [0.0, 1.0, 0.0], lam * [1.0, 0.0, 0.0])
    assert ref.kappa == float("inf") and ar.max_abs(ref.R * mp.matrix([1, 0, 0]), mp.matrix([0, 1, 0])) <= 1e-60
    # H = 0: the identity, as Eigen's JacobiSVD of a zero matrix gives
    ref = ar.align(np.array([[1.0, 2.0, 3.0], [1.0, 2.0, 7.0]]), np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 1.0]]), dof=4)
    assert ar.max_abs(ref.R, mp.eye(3)) == 0.0 and ref.kappa == float("inf")


def _report(ratios, what):
    for fam, r in sorted(ratios.items()):
        print(f"{what} {fam}: max |R - R_ref| = {max(r):.3g} eps kappa over {len(r)} cases")


def test_oracle_restatement_meets_the_bounds_ransac():
    """orc_align -- the device's 3- and 2-point alignment, operation for operation -- on every RANSAC case family."""
    ratios = {}
    for case in ac.ransac_cases():
        T, _ = ro.align(case.target, case.source)
        ratios.setdefault(case.family, []).append(ac.check(case, T))
    _report(ratios, "oracle RANSAC")


def test_oracle_restatement_meets_the_bounds_gnc():
    """orc_gnc's first, unweighted alignment (one outer and one inner iteration over the pairs (k, k)) on every GNC case family."""
    ratios = {}
    for case in ac.gnc_cases():
        n = len(case.target)
        F = np.random.default_rng(n).standard_normal((n, 4))
        want = ro.gnc(case.target, case.source, F, F, max_init_samples=n, tuple_check=False, max_iterations=1, inner_iterations=1, dof=case.dof)
        assert np.array_equal(want["C"], np.repeat(np.arange(n), 2).reshape(n, 2))
        ratios.setdefault(case.family, []).append(ac.check(case, want["T_target_source"]))
    _report(ratios, "oracle GNC")


def test_oracle_degenerate_flag():
    """The oracle flags a 3-point hypothesis as ill-determined when s2 / s1 falls below about 1e-4."""
    rng = np.random.default_rng(1)
    for e in (1, 2, 3, 5, 6, 7):
        base = np.array([[0.0, 0.0, 0.0], [10.0, 0.0, 0.0], [3.0, 10.0 ** (1 - e / 2), 0.0]])
        T = ac._posed(ar.rotation(rng.standard_normal(3), 1.0), [1.0, 2.0, 3.0], base)
        kappa = ar.align(T, base).kappa
        assert 10.0 ** (e - 1) < kappa < 10.0 ** (e + 1)
        assert ro.align(T, base)[1] == (e > 4), (e, kappa)
