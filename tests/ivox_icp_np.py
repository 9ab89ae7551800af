"""Python / numpy float64 restatement of ICP and point-to-plane ICP on iVox targets (tests/ only).

IntegratedICPFactor_<iVox, PointCloud> and <iVoxCovarianceEstimation, PointCloud> (src/gtsam_points/factors/integrated_icp_factor.cpp:9-10,
impl/integrated_icp_factor_impl.hpp:131-248) on top of the map restatements: the iVox 1-NN of ivox_np.IvoxNp (GicpIvoxNp's search)
or, on an ivox_cov_np.IvoxCovNp, over its valid points only; then the ICP evaluate with M = I, or M = diag(n^2) of the map's
estimated normal (point-to-plane).
"""
import numpy as np

import ivox_cov_np
import ivox_np
import np_ref


def icp_linearize(delta, src_pts, mean_B, corr, normals_B=None, delta_eval=None):
    """np_ref.linearize's Jacobians and sums for ICP: M = I (point-to-point) or, with target normals, M = diag(n_x^2, n_y^2, n_z^2)
    (point-to-plane: residual and Jacobian rows scaled by n, integrated_icp_factor_impl.hpp:205-248).  The residual is taken at
    `delta_eval` (default `delta`)."""
    if delta_eval is None:
        delta_eval = delta
    valid = corr >= 0
    p = src_pts[valid]
    mB = mean_B[corr[valid]]
    if normals_B is None:
        M = np.broadcast_to(np.eye(3), (len(p), 3, 3))
    else:
        n = normals_B[corr[valid]]
        M = np.zeros((len(p), 3, 3))
        for a in range(3):
            M[:, a, a] = n[:, a] * n[:, a]
    R, t = delta_eval[:3, :3], delta_eval[:3, 3]
    q = p @ R.T + t
    r = mB - q
    Jt = np.concatenate([-np_ref._hat_batch(q), np.broadcast_to(np.eye(3), (len(p), 3, 3))], 2)
    Js = np.concatenate([R @ np_ref._hat_batch(p), np.broadcast_to(-R, (len(p), 3, 3))], 2)
    JtM = np.einsum("nij,nik->njk", Jt, M)
    JsM = np.einsum("nij,nik->njk", Js, M)
    return dict(
        H_target=np.einsum("nij,njk->ik", JtM, Jt),
        H_source=np.einsum("nij,njk->ik", JsM, Js),
        H_target_source=np.einsum("nij,njk->ik", JtM, Js),
        b_target=np.einsum("nij,nj->i", JtM, r),
        b_source=np.einsum("nij,nj->i", JsM, r),
        error=float(np.einsum("ni,nij,nj->", r, M, r)),
        num_inliers=int(valid.sum()),
    )


class IcpIvoxNp:
    """IntegratedICPFactor_<iVox, PointCloud> / <iVoxCovarianceEstimation, PointCloud> as a unary factor against the map frame: the
    iVox 1-NN at linearize (GicpIvoxNp's search on an IvoxNp; the valid points of an IvoxCovNp), then the ICP evaluate with M = I
    or, point_to_plane, diag(n^2) of the map's estimated normals.  error() re-uses the correspondences of the last linearize.
    Point-to-plane needs an IvoxCovNp: a plain iVox keeps no normals."""

    def __init__(self, ivox, src_pts, point_to_plane=False, max_corr_sq=1.0):
        if point_to_plane and not hasattr(ivox, "knn_batch"):
            raise ValueError("error: target frame doesn't have required attributes for icp")
        self.ivox, self.src_pts, self.point_to_plane, self.max_corr_sq = ivox, np.asarray(src_pts, dtype=np.float64), point_to_plane, max_corr_sq
        self.corr, self.delta_lin = None, None

    def associate(self, delta):
        if hasattr(self.ivox, "knn_batch"):  # iVoxCovarianceEstimation: valid points only
            return self.ivox.knn_batch(ivox_np.transform(delta, self.src_pts), 1, self.max_corr_sq, True)[0][:, 0]
        return ivox_np.correspondences(self.ivox, delta, self.src_pts, self.max_corr_sq)

    def linearize(self, delta):
        self.corr = self.associate(delta)
        self.delta_lin = np.array(delta)
        return self._eval(delta)

    def _eval(self, delta_eval):
        ex, fi = self.ivox.export(), self.ivox.flat_index()
        flat = np.array([fi[int(c)] if c >= 0 else -1 for c in self.corr], dtype=np.int64)
        return icp_linearize(self.delta_lin, self.src_pts, ex["points"], flat, ex["normals"] if self.point_to_plane else None, delta_eval)

    def error(self, delta):
        if self.corr is None:
            self.linearize(delta)
        return self._eval(delta)["error"]


def valid_cloud(m):
    """The valid points and normals of the IvoxCovNp `m` (valid_indices() order) and, for every voxel << 32 | slot of a valid
    point, its position there: the target cloud of an oracle factor over the same points."""
    ex, fi = m.export(), m.flat_index()
    valid = (ex["flags"] & np.uint64(ivox_cov_np.VALID_BIT)) != 0
    pos = np.cumsum(valid) - 1
    to_valid = {k: int(pos[o]) for k, o in fi.items() if valid[o]}
    return ex["points"][valid], ex["normals"][valid], to_valid
