"""Extended-precision reference of the point-set alignment that RANSAC and GNC end in (the reference's align_points_se3 /
align_points_4dof, src/gtsam_points/registration/alignment.cpp): the rotation R maximising sum w_i t_i . R s_i about the weighted
centroids, from the SVD H = U S V^T of H = sum w_i (t_i - mt)(s_i - ms)^T, with the reflection fix S(last) = -1 when
det U det V < 0, and t = mt - R ms.  TEST INFRASTRUCTURE ONLY.

Every input value is taken exactly (float64 values are exact in mpmath) and the means, H, its SVD and the pose are computed with
DPS decimal digits, so the result is the exact alignment of the given numbers to far below float64 rounding.

Accuracy of a float64 solver: a perturbation dH of H moves the optimal rotation by at most about |dH| / g, where g is the smallest
sum of two signed singular values (s1, s2, d s3), d = sign(det U det V): g = s2 + d s3 in 3-D, s1 + d s2 in the plane.  A solver
whose error comes from rounding H and working on it backward-stably therefore errs by O(eps * kappa) with kappa = s1 / g.  kappa
is infinite when R is not determined (collinear sets, or a planar H with r = 0).
"""
from __future__ import annotations

from dataclasses import dataclass

import mpmath as mp
import numpy as np

DPS = 80


@dataclass
class Alignment:
    R: mp.matrix  # 3 x 3 (dof 4: the planar rotation about z, row and column 2 exactly e_z)
    t: mp.matrix  # 3 x 1
    mt: mp.matrix  # weighted means of the target / source points
    ms: mp.matrix
    sigma: list  # singular values of H, descending (3 of them, or 2 for dof 4)
    d: int  # sign(det U det V): -1 when the reflection fix applied
    H: mp.matrix  # the exact cross-covariance (3 x 3, or its top-left 2 x 2 for dof 4)
    U: mp.matrix  # H = U diag(sigma) Vt
    Vt: mp.matrix

    @property
    def kappa(self) -> float:
        """s1 / g (see the module docstring); inf when R is not determined."""
        s = self.sigma
        g = s[1] + self.d * s[2] if len(s) == 3 else s[0] + self.d * s[1]
        return float("inf") if g <= 0 else float(s[0] / g)

    def R64(self) -> np.ndarray:
        return mat64(self.R)

    def t64(self) -> np.ndarray:
        return mat64(self.t).reshape(3)

    def T64(self) -> np.ndarray:
        """4 x 4 float64 T_target_source (each entry the nearest double)."""
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = self.R64(), self.t64()
        return T


def mat64(M) -> np.ndarray:
    return np.array([[float(M[i, j]) for j in range(M.cols)] for i in range(M.rows)])


def _rows(P):
    """n x 3 rows of exact mpf values (float64, int or mpf input; a 4th column is ignored)."""
    if isinstance(P, np.ndarray):
        P = P.tolist()
    return [[mp.mpf(v) for v in row[:3]] for row in P]


def align(target, source, weights=None, dof: int = 6, dps: int = DPS) -> Alignment:
    """The alignment of source onto target (n x 3 each, pair i = (target[i], source[i])), weights w_i (None: all 1), dof 6 or 4."""
    assert dof in (6, 4)
    with mp.workdps(dps):
        T, S = _rows(target), _rows(source)
        n = len(T)
        assert n == len(S) and n >= 1
        w = [mp.mpf(1)] * n if weights is None else [mp.mpf(v) for v in np.asarray(weights, dtype=object).tolist()]
        W = mp.fsum(w)
        mt = mp.matrix([mp.fsum(w[i] * T[i][a] for i in range(n)) / W for a in range(3)])
        ms = mp.matrix([mp.fsum(w[i] * S[i][a] for i in range(n)) / W for a in range(3)])
        k = 3 if dof == 6 else 2
        H = mp.matrix(k, k)
        for a in range(k):
            for b in range(k):
                H[a, b] = mp.fsum(w[i] * (T[i][a] - mt[a]) * (S[i][b] - ms[b]) for i in range(n))
        if all(H[a, b] == 0 for a in range(k) for b in range(k)):
            # Eigen's JacobiSVD of a zero matrix leaves U = V = I, so the reference returns R = I
            U, sig, Vt = mp.eye(k), [mp.mpf(0)] * k, mp.eye(k)
        else:
            U, sv, Vt = mp.svd_r(H, full_matrices=True, compute_uv=True)
            sig = [sv[i] for i in range(k)]
            assert all(sig[i] >= sig[i + 1] for i in range(k - 1))
        d = -1 if mp.det(U) * mp.det(Vt) < 0 else 1
        D = mp.diag([1] * (k - 1) + [d])
        Rk = U * D * Vt
        R = mp.eye(3)
        for a in range(k):
            for b in range(k):
                R[a, b] = Rk[a, b]
        t = mt - R * ms
        return Alignment(R, t, mt, ms, sig, d, H, U, Vt)


def max_abs(A, B) -> float:
    """max |A - B| over entries of two equally shaped matrices (mp or numpy), evaluated in extended precision."""
    with mp.workdps(DPS):
        A = A.tolist() if isinstance(A, np.ndarray) else [[A[i, j] for j in range(A.cols)] for i in range(A.rows)]
        B = B.tolist() if isinstance(B, np.ndarray) else [[B[i, j] for j in range(B.cols)] for i in range(B.rows)]
        return float(max(abs(mp.mpf(a) - mp.mpf(b)) for ra, rb in zip(A, B) for a, b in zip(ra, rb)))


def rotation(axis, angle, dps: int = DPS) -> mp.matrix:
    """The rotation about `axis` by `angle` (Rodrigues), in extended precision; angle may be an mpf (e.g. pi - 1e-7)."""
    with mp.workdps(dps):
        a = [mp.mpf(v) for v in axis]
        nrm = mp.sqrt(mp.fsum(v * v for v in a))
        x, y, z = (v / nrm for v in a)
        c, s = mp.cos(angle), mp.sin(angle)
        C = 1 - c
        return mp.matrix([[c + x * x * C, x * y * C - z * s, x * z * C + y * s],
                          [y * x * C + z * s, c + y * y * C, y * z * C - x * s],
                          [z * x * C - y * s, z * y * C + x * s, c + z * z * C]])


def apply(R, t, P, dps: int = DPS) -> list:
    """Rows R p + t of the n x 3 points P, in extended precision (mpf rows)."""
    with mp.workdps(dps):
        return [[mp.fsum(R[a, b] * p[b] for b in range(3)) + mp.mpf(t[a]) for a in range(3)] for p in _rows(P)]
