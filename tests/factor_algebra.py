"""Two restatements of a factor's linearization (tests/ only), for problems placed far from the origin.

* `extended_linearize`: the formula card (np_ref.linearize) in extended precision.  Its inputs are the float64 transformed
  point q = ((R0 x + R1 y) + R2 z) + t and the residual r = mean - q as the oracle rounds them; everything after that -- M from
  cofactors over the determinant, the Jacobians J_target = [-hat(q) | I], J_source = [R hat(p) | -R] and the sums -- runs in
  np.longdouble.  It covers the three weight metrics of the factor kernel: GICP / VGICP (M = (C_B + RL C_A RL^T)^-1),
  point-to-point ICP (M = I) and point-to-plane ICP (M = diag(n_x^2, n_y^2, n_z^2) of the target normal n).
* `kernel_linearize`: the factor kernel's algebra in float64 -- the 29 accumulators of accumulate_point_f about an expansion
  point c, and epilogue_build / epilogue_store: H_t = X^T A' X, H_s = D^T A' D, H_ts = -X^T A' D, b_t = X^T c',
  b_s = -D^T c' with X = [[I, 0], [-hat(t + c), I]] and D = [[R, 0], [-hat(c) R, R]].  c = 0 is the expansion about the
  origin; `expansion_point` is the kernel's c = R centre.
"""
import numpy as np

L = np.longdouble
assert np.finfo(L).nmant >= 63, "the extended-precision reference needs an x87 80-bit (or wider) long double"

BLOCKS = ("H_target", "H_source", "H_target_source", "b_target", "b_source")
METRICS = {"gicp": 0, "icp": 1, "plane": 2}


def hat(v):
    z = np.zeros(v.shape[:-1], dtype=v.dtype)
    return np.stack([np.stack([z, -v[..., 2], v[..., 1]], -1), np.stack([v[..., 2], z, -v[..., 0]], -1), np.stack([-v[..., 1], v[..., 0], z], -1)], -2)


def rotate(R, p):
    """((R0 x + R1 y) + R2 z), every float64 operation rounded on its own (numpy does not contract)."""
    return np.stack([(R[r, 0] * p[:, 0] + R[r, 1] * p[:, 1]) + R[r, 2] * p[:, 2] for r in range(3)], 1)


def transform(T, p):
    return rotate(T[:3, :3], p) + T[:3, 3]


def _weights(metric, RL, CA, CB, dtype):
    """Per-correspondence M (n x 3 x 3) in `dtype`; CB holds the target covariances (GICP) or the target normals (plane)."""
    n = len(CA) if CA is not None else len(CB)
    if metric == 1:
        return np.broadcast_to(np.eye(3, dtype=dtype), (n, 3, 3))
    if metric == 2:
        nb = CB.astype(dtype)
        M = np.zeros((n, 3, 3), dtype=dtype)
        for k in range(3):
            M[:, k, k] = nb[:, k] * nb[:, k]
        return M
    RLx = RL.astype(dtype)
    S = CB.astype(dtype) + RLx @ CA.astype(dtype) @ RLx.T
    s00, s01, s02, s11, s12, s22 = S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]
    c00 = s11 * s22 - s12 * s12
    c01 = s02 * s12 - s01 * s22
    c02 = s01 * s12 - s02 * s11
    c11 = s00 * s22 - s02 * s02
    c12 = s01 * s02 - s00 * s12
    c22 = s00 * s11 - s01 * s01
    det = s00 * c00 + s01 * c01 + s02 * c02
    inv = np.ones_like(det) / det if dtype is L else 1.0 / det
    return np.stack([np.stack([c00, c01, c02], -1), np.stack([c01, c11, c12], -1), np.stack([c02, c12, c22], -1)], -2) * inv[:, None, None]


def _gather(src_pts, src_covs, mean_B, cov_B, corr):
    valid = np.asarray(corr) >= 0
    idx = np.asarray(corr)[valid]
    p = np.asarray(src_pts, dtype=np.float64)[valid]
    CA = None if src_covs is None else np.asarray(src_covs, dtype=np.float64).reshape(-1, 3, 3)[valid]
    CB = None if cov_B is None else np.asarray(cov_B, dtype=np.float64)[idx]
    return valid, p, CA, np.asarray(mean_B, dtype=np.float64)[idx], CB


def extended_linearize(delta, src_pts, src_covs, mean_B, cov_B, corr, metric=0, delta_eval=None):
    """Formula card in np.longdouble from the float64 q and r.  cov_B: target covariances (n x 3 x 3, metric 0), target
    normals (n x 3, metric 2) or None (metric 1).  M is built at `delta`, residuals and Jacobians at `delta_eval`."""
    delta_eval = delta if delta_eval is None else delta_eval
    valid, p, CA, mB, CB = _gather(src_pts, src_covs, mean_B, cov_B, corr)
    R, t = delta_eval[:3, :3], delta_eval[:3, 3]
    q = transform(delta_eval, p)  # float64, the oracle's rounding
    r = (mB - q).astype(L)
    M = _weights(metric, delta[:3, :3], CA, CB, L)
    n = len(p)
    I = np.broadcast_to(np.eye(3, dtype=L), (n, 3, 3))
    Jt = np.concatenate([-hat(q.astype(L)), I], 2)
    RL_ = R.astype(L)
    Js = np.concatenate([RL_ @ hat(p.astype(L)), np.broadcast_to(-RL_, (n, 3, 3))], 2)
    JtM = np.einsum("nij,nik->njk", Jt, M)
    JsM = np.einsum("nij,nik->njk", Js, M)
    return dict(
        H_target=np.einsum("nij,njk->ik", JtM, Jt),
        H_source=np.einsum("nij,njk->ik", JsM, Js),
        H_target_source=np.einsum("nij,njk->ik", JtM, Js),
        b_target=np.einsum("nij,nj->i", JtM, r),
        b_source=np.einsum("nij,nj->i", JsM, r),
        error=np.einsum("ni,nij,nj->", r, M, r),
        num_inliers=int(valid.sum()),
    )


def expansion_point(R, centre):
    """The kernel's c = R centre: ((R0 cx + R1 cy) + R2 cz), every operation rounded."""
    return rotate(np.asarray(R, dtype=np.float64), np.asarray(centre, dtype=np.float64)[None])[0]


def kernel_linearize(delta, src_pts, src_covs, mean_B, cov_B, corr, c, metric=0):
    """The factor kernel's float64 algebra (linearize mode) about the expansion point c (3-vector)."""
    valid, p, CA, mB, CB = _gather(src_pts, src_covs, mean_B, cov_B, corr)
    R, t = delta[:3, :3], delta[:3, 3]
    c = np.asarray(c, dtype=np.float64)
    u = rotate(R, p)
    e = mB - (u + t)
    M = np.ascontiguousarray(_weights(metric, R, CA, CB, np.float64))
    Me = np.einsum("nij,nj->ni", M, e)
    w = u - c
    K = hat(w) @ M  # hat(w) M
    acc = dict(
        A_rr=np.einsum("nij,nkj->ik", K, hat(w)),  # K hat(w)^T
        A_rt=K.sum(0),
        A_tt=M.sum(0),
        c_r=np.cross(w, Me).sum(0),
        c_t=Me.sum(0),
        error=float(np.einsum("ni,ni->", e, Me)),
    )
    A = np.zeros((6, 6))
    A[:3, :3], A[:3, 3:], A[3:, :3], A[3:, 3:] = acc["A_rr"], acc["A_rt"], acc["A_rt"].T, acc["A_tt"]
    cp = np.concatenate([acc["c_r"], acc["c_t"]])
    X = np.eye(6)
    X[3:, :3] = -hat(t + c)
    D = np.zeros((6, 6))
    D[:3, :3], D[3:, 3:], D[3:, :3] = R, R, -hat(c) @ R
    return dict(H_target=X.T @ A @ X, H_source=D.T @ A @ D, H_target_source=-X.T @ A @ D, b_target=X.T @ cp, b_source=-D.T @ cp,
                error=acc["error"], num_inliers=int(valid.sum()))


def block_errors(got, ref, keys=BLOCKS):
    """Per block: max |got - ref| / max |ref|, evaluated in extended precision."""
    out = {}
    for k in keys:
        r = np.asarray(ref[k], dtype=L)
        d = np.abs(np.asarray(got[k], dtype=L) - r).max()
        out[k] = float(d / max(np.abs(r).max(), L(1e-300)))
    return out


def error_relerr(got, ref):
    return float(abs(L(got) - L(ref)) / max(abs(L(ref)), L(1e-300)))
