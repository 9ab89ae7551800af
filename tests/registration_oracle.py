"""ctypes binding of tests/registration_oracle.cpp, the CPU restatement of FPFH, feature 1-NN, the single-threaded RANSAC loop, GNC
(b2_estimate_pose_gnc), PFH (b2_features_create_pfh) and FPFH at chosen points (b2_features_create_fpfh_at) -- TEST INFRASTRUCTURE
ONLY.  The library is compiled on first use by tests/native.py with the CPU oracles' flags.
"""
import ctypes as C
import functools
import os

import numpy as np

import native

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "registration_oracle.cpp")

_dp, _lp, _ip, _bp = C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_ubyte)


@functools.cache
def lib():
    L = native.shared_library([SRC], native.ORACLE_FLAGS)
    L.orc_reg_max_threads.restype = C.c_int
    L.orc_fpfh.restype = None
    L.orc_fpfh.argtypes = [_dp, _dp, C.c_size_t, C.c_double, C.c_size_t, C.c_int, _dp, _bp, _lp]
    L.orc_feature_nn.restype = None
    L.orc_feature_nn.argtypes = [_dp, C.c_size_t, _dp, C.c_size_t, C.c_int, C.c_int, _lp, _dp]
    L.orc_ransac.restype = None
    L.orc_ransac.argtypes = [_dp, C.c_size_t, _dp, C.c_size_t, _dp, _dp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_uint64, C.c_double,
                             C.c_double, _dp, C.c_size_t, C.c_int, _ip, _ip, _ip, _dp, _ip, _bp, _dp]
    L.orc_gnc.restype = None
    L.orc_gnc.argtypes = [_dp, C.c_size_t, _dp, C.c_size_t, _dp, _dp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int,
                          C.c_int, C.c_int, C.c_uint64, C.c_int, _lp, _lp, _lp, _lp, _ip, _ip, _lp, _lp, _bp, _dp]
    L.orc_align.restype = None
    L.orc_align.argtypes = [C.c_int, _dp, _dp, _dp, _bp]
    for fn in (L.orc_pfh, L.orc_fpfh_at):
        fn.restype = None
        fn.argtypes = [_dp, _dp, C.c_size_t, _lp, C.c_size_t, C.c_double, C.c_size_t, C.c_int, _dp, _bp, _lp]
    return L


def max_threads():
    return lib().orc_reg_max_threads()


def _f64(a, cols):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)[:, :cols])


def fpfh(points, normals, search_radius=5.0, max_num_neighbors=10000, num_threads=None):
    """-> (features n x 33, edge n bool, num_neighbors n): FPFH over brute-force radius neighbours; edge flags rows that a pair at a bin
    edge (nf * 11 within 1e-9 of an integer) enters."""
    p, nr = _f64(points, 3), _f64(normals, 3)
    n = len(p)
    out = np.zeros((max(n, 1), 33))
    edge = np.zeros(max(n, 1), dtype=np.uint8)
    nn = np.zeros(max(n, 1), dtype=np.int64)
    lib().orc_fpfh(p.ctypes.data_as(_dp), nr.ctypes.data_as(_dp), n, float(search_radius), int(max_num_neighbors), int(num_threads or max_threads()),
                   out.ctypes.data_as(_dp), edge.ctypes.data_as(_bp), nn.ctypes.data_as(_lp))
    return out[:n], edge[:n].astype(bool), nn[:n]


def feature_nearest(queries, targets, num_threads=None):
    """-> (index int64, squared distance): exact 1-NN, distances summed in dimension order, ties to the smallest index."""
    q = np.ascontiguousarray(queries, dtype=np.float64)
    t = np.ascontiguousarray(targets, dtype=np.float64)
    idx = np.zeros(max(len(q), 1), dtype=np.int64)
    sq = np.zeros(max(len(q), 1))
    lib().orc_feature_nn(q.ctypes.data_as(_dp), len(q), t.ctypes.data_as(_dp), len(t), q.shape[1], int(num_threads or max_threads()), idx.ctypes.data_as(_lp),
                         sq.ctypes.data_as(_dp))
    return idx[: len(q)], sq[: len(q)]


def ransac(target, source, target_features, source_features, max_iterations=5000, early_stop_inlier_rate=0.8, poly_error_thresh=0.5,
           inlier_voxel_resolution=1.0, dof=6, seed=5489, taboo_thresh_rot=0.5 * np.pi / 180.0, taboo_thresh_trans=0.25, taboo_list=(), num_threads=None):
    """The single-threaded RANSAC loop with every hypothesis evaluated.  Returns a dict: samples / targets (K x ns), status (the count
    or -1 / -2 / -3), T (K x 3 x 4), slack, degenerate (K bool), and the result: T_target_source (4 x 4), inlier_rate, num_inliers,
    hypothesis."""
    tp, sp = _f64(target, 3), _f64(source, 3)
    tf = np.ascontiguousarray(target_features, dtype=np.float64)
    sf = np.ascontiguousarray(source_features, dtype=np.float64)
    K, ns = int(max_iterations), (3 if dof == 6 else 2)
    tab = np.ascontiguousarray(np.asarray(taboo_list, dtype=np.float64).reshape(-1, 16)) if len(taboo_list) else np.zeros((1, 16))
    samples = np.zeros((max(K, 1), ns), dtype=np.int32)
    targets = np.zeros((max(K, 1), ns), dtype=np.int32)
    status = np.zeros(max(K, 1), dtype=np.int32)
    T = np.zeros((max(K, 1), 12))
    slack = np.zeros(max(K, 1), dtype=np.int32)
    deg = np.zeros(max(K, 1), dtype=np.uint8)
    res = np.zeros(19)
    lib().orc_ransac(tp.ctypes.data_as(_dp), len(tp), sp.ctypes.data_as(_dp), len(sp), tf.ctypes.data_as(_dp), sf.ctypes.data_as(_dp), tf.shape[1], K, int(dof),
                     float(early_stop_inlier_rate), float(poly_error_thresh), float(inlier_voxel_resolution), int(seed), float(taboo_thresh_rot), float(taboo_thresh_trans),
                     tab.ctypes.data_as(_dp), len(taboo_list), int(num_threads or max_threads()), samples.ctypes.data_as(_ip), targets.ctypes.data_as(_ip),
                     status.ctypes.data_as(_ip), T.ctypes.data_as(_dp), slack.ctypes.data_as(_ip), deg.ctypes.data_as(_bp), res.ctypes.data_as(_dp))
    return dict(samples=samples[:K], targets=targets[:K], status=status[:K], T=T[:K].reshape(K, 3, 4), slack=slack[:K], degenerate=deg[:K].astype(bool),
                T_target_source=res[:16].reshape(4, 4), inlier_rate=res[16], num_inliers=int(res[17]), hypothesis=int(res[18]))


def align(target, source):
    """One RANSAC hypothesis' alignment of 3 (dof 6) or 2 (dof 4) source points onto their target points, as
    b2_estimate_pose_ransac's step 4 computes it -> (T 3 x 4, degenerate)."""
    tp, sp = _f64(target, 3), _f64(source, 3)
    ns = len(tp)
    assert ns in (2, 3) and len(sp) == ns
    T = np.zeros(12)
    deg = np.zeros(1, dtype=np.uint8)
    lib().orc_align(ns, tp.ctypes.data_as(_dp), sp.ctypes.data_as(_dp), T.ctypes.data_as(_dp), deg.ctypes.data_as(_bp))
    return T.reshape(3, 4), bool(deg[0])


def gnc(target, source, target_features, source_features, max_init_samples=5000, reciprocal_check=True, tuple_check=False, max_num_tuples=1000,
        tuple_thresh=0.9, div_factor=1.4, max_corr_dist=0.25, inner_iterations=3, max_iterations=64, dof=6, seed=5489, num_threads=None):
    """GNC as b2_estimate_pose_gnc states it.  Returns a dict: samples (the sampled side's indices), swapped (the target is the
    sampled side), matched ((m0, 2) int64 (target, source) pairs before the tuple check), draws ((max_num_tuples, 3) tuple indices into
    matched, or None when the tuple check did not run), C ((m, 2) the final pairs), slack (m bool: the pair's last counted error lies
    within 1e-9 of the inlier threshold), and the result: T_target_source (4 x 4), inlier_rate, num_inliers."""
    tp, sp = _f64(target, 3), _f64(source, 3)
    tf = np.ascontiguousarray(target_features, dtype=np.float64)
    sf = np.ascontiguousarray(source_features, dtype=np.float64)
    nS = max(len(tp), len(sp))
    samples = np.zeros(max(nS, 1), dtype=np.int64)
    C0 = np.zeros((max(nS, 1), 2), dtype=np.int64)
    C1 = np.zeros((max(nS, 1), 2), dtype=np.int64)
    draws = np.zeros((max(int(max_num_tuples), 1), 3), dtype=np.int32)
    slack = np.zeros(max(nS, 1), dtype=np.uint8)
    ns, n0, nc, ran = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
    res = np.zeros(18)
    lib().orc_gnc(tp.ctypes.data_as(_dp), len(tp), sp.ctypes.data_as(_dp), len(sp), tf.ctypes.data_as(_dp), sf.ctypes.data_as(_dp), tf.shape[1], int(max_init_samples),
                  int(bool(reciprocal_check)), int(bool(tuple_check)), int(max_num_tuples), float(tuple_thresh), float(div_factor), float(max_corr_dist),
                  int(inner_iterations), int(max_iterations), int(dof), int(seed), int(num_threads or max_threads()), samples.ctypes.data_as(_lp), C.byref(ns),
                  C0.ctypes.data_as(_lp), C.byref(n0), draws.ctypes.data_as(_ip), C.byref(ran), C1.ctypes.data_as(_lp), C.byref(nc), slack.ctypes.data_as(_bp),
                  res.ctypes.data_as(_dp))
    return dict(samples=samples[: ns.value], swapped=not len(sp) < len(tp), matched=C0[: n0.value], draws=draws[: int(max_num_tuples)] if ran.value else None,
                C=C1[: nc.value], slack=slack[: nc.value].astype(bool), T_target_source=res[:16].reshape(4, 4), inlier_rate=res[16], num_inliers=int(res[17]))


def _rows(fn, dim, points, normals, search_radius, max_num_neighbors, num_threads, indices):
    p, nr = _f64(points, 3), _f64(normals, 3)
    idx = None if indices is None else np.ascontiguousarray(np.asarray(indices, dtype=np.int64).reshape(-1))
    nk = len(p) if idx is None else len(idx)
    out = np.zeros((max(nk, 1), dim))
    edge = np.zeros(max(nk, 1), dtype=np.uint8)
    nn = np.zeros(max(nk, 1), dtype=np.int64)
    fn(p.ctypes.data_as(_dp), nr.ctypes.data_as(_dp), len(p), None if idx is None else idx.ctypes.data_as(_lp), nk, float(search_radius), int(max_num_neighbors),
       int(num_threads or max_threads()), out.ctypes.data_as(_dp), edge.ctypes.data_as(_bp), nn.ctypes.data_as(_lp))
    return out[:nk], edge[:nk].astype(bool), nn[:nk]


def pfh(points, normals, search_radius=5.0, max_num_neighbors=10000, num_threads=None, indices=None):
    """-> (features nk x 125, edge nk bool, num_neighbors nk): PFH over brute-force radius neighbours at the points `indices` (None:
    every point); edge flags rows with a pair whose nf_theta * 5 lies within 1e-9 of an integer."""
    return _rows(lib().orc_pfh, 125, points, normals, search_radius, max_num_neighbors, num_threads, indices)


def fpfh_at(points, normals, indices, search_radius=5.0, max_num_neighbors=10000, num_threads=None):
    """-> (features nk x 33, edge nk bool, num_neighbors nk): the FPFH rows of the points `indices` (SPFH over every point), with
    the registration oracle's edge flags and neighbour counts of those points."""
    return _rows(lib().orc_fpfh_at, 33, points, normals, search_radius, max_num_neighbors, num_threads, indices)
