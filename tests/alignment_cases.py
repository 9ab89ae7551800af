"""Point sets for testing RANSAC's and GNC's alignment step against the extended-precision reference (alignment_ref.py), and the
bounds a float64 solver must meet on them.  TEST INFRASTRUCTURE ONLY.

A case is a target / source pair list (pair i = (target[i], source[i])) and how well R is determined:
  "full"  the alignment is unique (kappa finite): |R - R_ref|_max <= C_R eps kappa, |t - t_ref|_max <= C_R eps kappa scale;
  "line"  every pair lies on one line per side (H has rank 1): only the line is determined, so R must be a finite proper rotation
          that maps the source direction onto the target direction, with t = mt - R ms;
  "free"  H = 0 (dof 4: H00 + H11 = H10 - H01 = 0): every rotation is optimal; R must be the identity.
with kappa = max(1, s1 / g) (alignment_ref.Alignment.kappa) and scale = |mt| + |ms| + the largest |s_i - ms| (2-norms).
"""
from __future__ import annotations

from dataclasses import dataclass

import mpmath as mp
import numpy as np

import alignment_ref as ar

EPS = np.finfo(np.float64).eps
C_R = 16.0  # fixed once, from the well-conditioned cases: their largest |R - R_ref|_max is about 3 eps kappa (printed by the tests)


@dataclass
class Case:
    family: str
    name: str
    target: np.ndarray  # n x 3 float64
    source: np.ndarray
    dof: int
    kind: str = "full"  # "full", "line" or "free"


def _posed(R, t, S):
    """float64 rows of R s + t (each the nearest double of the exact value)."""
    return np.array([[float(v) for v in row] for row in ar.apply(R, t, S)])


def _random_rotation(rng, angle=None):
    axis = rng.standard_normal(3)
    return ar.rotation(axis, rng.uniform(0.0, np.pi) if angle is None else angle)


def _yaw(angle):
    return ar.rotation([0.0, 0.0, 1.0], angle)


def ransac_cases() -> list[Case]:
    """3-point sets (dof 6) and 2-point sets (dof 4)."""
    rng = np.random.default_rng(20261018)
    out = []
    for k in range(6):
        S = rng.uniform(-10.0, 10.0, (3, 3))
        R = ar.rotation([0.0, 0.0, 1.0], 0.0) if k == 0 else _random_rotation(rng)
        out.append(Case("random", f"r{k}", _posed(R, rng.uniform(-20, 20, 3), S), S, 6))
    for k, da in enumerate([1e-6, 1e-7, 3e-10]):
        S = rng.uniform(-10.0, 10.0, (3, 3))
        out.append(Case("near_pi", f"pi-{da:g}", _posed(_random_rotation(rng, mp.pi - da), rng.uniform(-5, 5, 3), S), S, 6))
    for k in range(3):
        S = rng.uniform(-10.0, 10.0, (3, 3))
        out.append(Case("noisy", f"n{k}", _posed(_random_rotation(rng), rng.uniform(-5, 5, 3), S) + rng.normal(0.0, 0.05, (3, 3)), S, 6))
    for e in range(1, 9):
        h = 10.0 ** (-e / 2)  # s2 / s1 of the triangle is about h^2 = 10^-e
        base = np.array([[0.0, 0.0, 0.0], [10.0, 0.0, 0.0], [3.0, 10.0 * h, 0.0]])
        S = _posed(_random_rotation(rng), rng.uniform(-5, 5, 3), base)
        out.append(Case("thin", f"1e-{e}", _posed(_random_rotation(rng), rng.uniform(-5, 5, 3), S), S, 6))
    # exactly collinear in float64: integer steps along small-integer directions, and along the axes
    lam = np.array([[-1.0], [0.0], [2.0]])
    out.append(Case("collinear", "general", np.array([1.0, -2.0, 3.0]) + lam * [2.0, 1.0, -2.0], np.array([4.0, 0.5, -1.0]) + lam * [1.0, 2.0, 2.0], 6, "line"))
    out.append(Case("collinear", "x_to_y", np.array([0.0, 5.0, 0.0]) + lam * [0.0, 1.0, 0.0], lam * [1.0, 0.0, 0.0], 6, "line"))
    out.append(Case("collinear", "x_to_x", lam * [3.0, 0.0, 0.0], np.array([0.0, 1.0, 1.0]) + lam * [3.0, 0.0, 0.0], 6, "line"))
    for k in range(3):
        T = rng.uniform(-10.0, 10.0, (3, 3))
        out.append(Case("mirrored", f"m{k}", T, T * [1.0, 1.0, -1.0] if k < 2 else -T, 6))
    for e in (3, 4, 5, 6):
        S = rng.uniform(-10.0, 10.0, (3, 3)) + rng.choice([-1.0, 1.0], 3) * 10.0**e
        out.append(Case("offset", f"1e{e}", _posed(_random_rotation(rng), rng.choice([-1.0, 1.0], 3) * 10.0**e, S), S, 6))
    for k in range(4):
        S = rng.uniform(-10.0, 10.0, (2, 3))
        R = _yaw(0.0 if k == 0 else (np.pi - 1e-7 if k == 1 else rng.uniform(-np.pi, np.pi)))
        out.append(Case("dof4", f"yaw{k}", _posed(R, rng.uniform(-20, 20, 3), S), S, 4))
    for e in (3, 6):
        S = rng.uniform(-10.0, 10.0, (2, 3)) + 10.0**e
        out.append(Case("dof4_offset", f"1e{e}", _posed(_yaw(rng.uniform(-np.pi, np.pi)), [10.0**e, -(10.0**e), 7.0], S), S, 4))
    # vertical pairs: H's top-left 2 x 2 is 0
    out.append(Case("dof4_vertical", "source", np.array([[1.0, 2.0, 3.0], [4.0, -1.0, 5.0]]), np.array([[7.0, 7.0, 0.0], [7.0, 7.0, 4.0]]), 4, "free"))
    out.append(Case("dof4_vertical", "both", np.array([[1.0, 2.0, 3.0], [1.0, 2.0, -5.0]]), np.array([[7.0, 7.0, 0.0], [7.0, 7.0, 8.0]]), 4, "free"))
    return out


def gnc_cases() -> list[Case]:
    """N-pair sets for GNC's first (unweighted) alignment."""
    rng = np.random.default_rng(5489)
    out = []
    for n in (3, 10, 100, 1000, 4000):
        S = rng.uniform(-20.0, 20.0, (n, 3))
        out.append(Case("random", f"N{n}", _posed(_random_rotation(rng), rng.uniform(-20, 20, 3), S), S, 6))
        out.append(Case("noisy", f"N{n}", _posed(_random_rotation(rng), rng.uniform(-20, 20, 3), S) + rng.normal(0.0, 0.1, (n, 3)), S, 6))
    S = rng.uniform(-20.0, 20.0, (200, 3))
    out.append(Case("random", "identity", S.copy(), S, 6))
    out.append(Case("near_pi", "pi-1e-7", _posed(_random_rotation(rng, mp.pi - 1e-7), rng.uniform(-5, 5, 3), S), S, 6))
    for e in (2, 4, 6, 8):
        h = 10.0 ** (-e / 2)  # a thin rod: s2 / s1 about h^2 = 10^-e
        base = rng.uniform(-1.0, 1.0, (500, 3)) * [20.0, 20.0 * h, 20.0 * h]
        Sr = _posed(_random_rotation(rng), rng.uniform(-5, 5, 3), base)
        out.append(Case("thin", f"1e-{e}", _posed(_random_rotation(rng), rng.uniform(-5, 5, 3), Sr), Sr, 6))
    base = rng.uniform(-10.0, 10.0, (300, 3)) * [1.0, 1.0, 0.0]  # planar: s3 = 0
    Sp = _posed(_random_rotation(rng), [1.0, 2.0, 3.0], base)
    out.append(Case("planar", "N300", _posed(_random_rotation(rng), rng.uniform(-5, 5, 3), Sp), Sp, 6))
    lam = np.arange(-50.0, 51.0)[:, None]
    out.append(Case("collinear", "general", np.array([1.0, -2.0, 3.0]) + lam * [2.0, 1.0, -2.0], np.array([4.0, 0.5, -1.0]) + lam * [1.0, 2.0, 2.0], 6, "line"))
    out.append(Case("collinear", "x_to_y", lam * [0.0, 1.0, 0.0], lam * [1.0, 0.0, 0.0], 6, "line"))
    T = rng.uniform(-10.0, 10.0, (400, 3)) * [3.0, 2.0, 1.0]
    out.append(Case("mirrored", "z", T, T * [1.0, 1.0, -1.0], 6))
    out.append(Case("mirrored", "point", T, -T, 6))
    for e in (3, 4, 5, 6):
        S = rng.uniform(-10.0, 10.0, (500, 3)) + rng.choice([-1.0, 1.0], 3) * 10.0**e
        out.append(Case("offset", f"1e{e}", _posed(_random_rotation(rng), rng.choice([-1.0, 1.0], 3) * 10.0**e, S), S, 6))
    for n in (2, 50, 3000):
        S = rng.uniform(-20.0, 20.0, (n, 3))
        out.append(Case("dof4", f"N{n}", _posed(_yaw(rng.uniform(-np.pi, np.pi)), rng.uniform(-20, 20, 3), S) + rng.normal(0.0, 0.05, (n, 3)), S, 4))
    S = rng.uniform(-10.0, 10.0, (500, 3)) + 1e6
    out.append(Case("dof4_offset", "1e6", _posed(_yaw(2.0), [1e6, 3e5, -2e5], S), S, 4))
    # H's top-left 2 x 2 = diag(2, -2): a mirrored square, H00 + H11 = H10 - H01 = 0
    sq = np.array([[1.0, 0.0, 0.5], [-1.0, 0.0, 1.5], [0.0, 1.0, -2.0], [0.0, -1.0, 3.0]])
    out.append(Case("dof4_mirrored", "square", sq, sq * [1.0, -1.0, 2.0], 4, "free"))
    return out


def check(case: Case, T: np.ndarray, target=None, source=None) -> float:
    """Assert that T (4 x 4 or 3 x 4) meets the case's bound against the reference computed from `target` / `source` (default: the
    case's points).  Returns |R - R_ref|_max / (eps kappa) for a "full" case, else 0."""
    target = case.target if target is None else target
    source = case.source if source is None else source
    ref = ar.align(target, source, dof=case.dof)
    T = np.asarray(T, dtype=np.float64)
    R, t = T[:3, :3], T[:3, 3]
    where = f"{case.family}/{case.name} (dof {case.dof})"
    assert np.isfinite(T[:3]).all(), (where, T)
    if case.dof == 4:
        assert np.array_equal(R[2], [0.0, 0.0, 1.0]) and np.array_equal(R[:2, 2], [0.0, 0.0]), (where, R)
    with mp.workdps(ar.DPS):
        mt, ms = ref.mt, ref.ms
        extent = max(mp.norm(mp.matrix([mp.mpf(v) for v in s[:3]]) - ms) for s in source)
        scale = float(mp.norm(mt) + mp.norm(ms) + extent)
        Rm = mp.matrix(R.tolist())
        t_means = mt - Rm * ms  # t as the means and this R determine it
    if case.kind == "free":
        assert np.array_equal(R, np.eye(3)), (where, R)
        assert ar.max_abs(t.reshape(3, 1), t_means) <= C_R * EPS * scale, where
        return 0.0
    if case.kind == "line":
        assert case.dof == 6
        assert np.abs(R.T @ R - np.eye(3)).max() <= C_R * EPS and abs(np.linalg.det(R) - 1.0) <= C_R * EPS, (where, R)
        with mp.workdps(ar.DPS):
            err = ar.max_abs(Rm * ref.Vt[0, :].T, ref.U[:, 0])  # R v1 = u1
        assert err <= C_R * EPS, (where, err)
        assert ar.max_abs(t.reshape(3, 1), t_means) <= C_R * EPS * scale, where
        return 0.0
    kappa = max(1.0, ref.kappa)
    eR = ar.max_abs(R, ref.R)
    et = ar.max_abs(t.reshape(3, 1), ref.t)
    assert eR <= C_R * EPS * kappa, f"{where}: |R - R_ref|_max = {eR:.3g} > {C_R:g} eps kappa = {C_R * EPS * kappa:.3g} (kappa {kappa:.3g})"
    assert et <= C_R * EPS * kappa * scale, f"{where}: |t - t_ref|_max = {et:.3g} > {C_R:g} eps kappa scale = {C_R * EPS * kappa * scale:.3g}"
    return eR / (EPS * kappa)
