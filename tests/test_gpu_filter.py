"""Frame filtering on the device (b2_cloud_create_sampled / _random_sampled / _randomgrid / _inliers): the selected caller indices,
mean neighbour distances and threshold equal the CPU oracle (tests/filter_oracle.cpp) bit for bit, and every new cloud is the cloud
b2_cloud_create makes of the downloaded rows it selects -- stored bits and info."""
import ctypes as C

import numpy as np
import pytest

import filter_oracle as fo
import preprocess_cases as pc
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
SCANS = pc.scans()
INFO = ("num_points", "point_bytes", "cov_bytes", "normal_bytes", "reordered", "device_bytes")


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def download(cloud):
    """The stored values in caller order: points, covs (n x 3 x 3) or None, normals or None."""
    info = cloud.info()
    n = int(info.num_points)
    p = np.zeros((n, 3))
    c = np.zeros((n, 3, 3)) if info.cov_bytes else None
    nr = np.zeros((n, 3)) if info.normal_bytes else None
    capi.check(capi.lib().b2_cloud_download(cloud.h, capi.dptr(p), None if c is None else capi.dptr(c), None if nr is None else capi.dptr(nr)))
    return p, c, nr


def assert_is_rows(g, got, rows, K, flags):
    """got == b2_cloud_create_with_normals of rows[K] under flags: stored bits and info."""
    p, c, nr = rows
    want = g.PointCloud(p[K], None if c is None else c[K], flags=flags, normals=None if nr is None else nr[K])
    a, b = download(got), download(want)
    for x, y in zip(a, b):
        assert pc.same_bits(x, y)
    gi, wi = got.info(), want.info()
    assert all(getattr(gi, f) == getattr(wi, f) for f in INFO)
    assert pc.same_bits(a[0], fo.gather(p, K))


def make(g, pts, seed, with_covs=True, with_normals=True, flags=capi.B2_CLOUD_DEFAULT):
    covs, nrm = pc.attributes(pts, seed)
    return g.PointCloud(pts, covs if with_covs else None, normals=nrm if with_normals else None, flags=flags)


def run_all(g, cloud, res, rate, seed, k, flags=capi.B2_CLOUD_DEFAULT):
    """Every filter on `cloud` against the oracle over its stored values (outlier removal with k neighbours unless k is None); returns
    the outputs for comparisons between calls."""
    rows = download(cloud)
    n = len(rows[0])
    out = {}
    got, K = g.types._random_sampled(cloud, rate, seed, flags)
    assert np.array_equal(K, fo.random_sampling(n, rate, seed))
    assert_is_rows(g, got, rows, K, flags)
    out["random"] = (K, download(got))
    got, K = g.types._randomgrid(cloud, res, rate, seed, flags)
    assert np.array_equal(K, fo.randomgrid_sampling(rows[0], res, rate, seed))
    assert_is_rows(g, got, rows, K, flags)
    out["grid"] = (K, download(got))
    if k is not None:
        got, K, d, th = g.types._inliers(cloud, k, 1.0, None, flags)
        want_K, want_d, want_th = fo.inliers(rows[0], k, 1.0)
        assert np.array_equal(K, want_K) and pc.same_bits(d, want_d) and pc.same_bits(th, want_th)
        assert_is_rows(g, got, rows, K, flags)
        out["inliers"] = (K, d, th, download(got))
    idx = np.random.default_rng(seed).integers(0, max(n, 1), size=min(n, 777)) if n else np.zeros(0, np.int64)
    got = g.sample(cloud, idx, flags=flags)
    assert_is_rows(g, got, rows, idx, flags)
    out["sample"] = download(got)
    return out


def same_outputs(a, b):
    def flat(x):
        if isinstance(x, (tuple, list)):
            return [y for z in x for y in flat(z)]
        return [x]

    fa, fb = flat([a[k] for k in sorted(a)]), flat([b[k] for k in sorted(b)])
    return len(fa) == len(fb) and all((x is None and y is None) or pc.same_bits(x, y) for x, y in zip(fa, fb))


@pytest.mark.parametrize("name", sorted(SCANS))
def test_filters_match_oracle_on_scans(g, name):
    pts = SCANS[name].astype(np.float64)
    for j, res in enumerate(pc.RESOLUTIONS):
        layout = [(True, True, capi.B2_CLOUD_DEFAULT), (False, False, capi.B2_CLOUD_DEFAULT), (True, False, capi.B2_CLOUD_COMPACT_F32),
                  (False, True, capi.B2_CLOUD_FORCE_F64)][j]
        cloud = make(g, pts, j, *layout)
        k = (1, 10, 64, 10)[j]
        rate, seed = (0.5, 0.1, 0.3, 0.75)[j], 5489 + j
        run_all(g, cloud, res, rate, seed, k, flags=(capi.B2_CLOUD_DEFAULT, capi.B2_CLOUD_FORCE_F64, capi.B2_CLOUD_COMPACT_F32, capi.B2_CLOUD_NO_REORDER)[j])


def test_storage_order_and_repeat_independence(g):
    pts = SCANS["kitti00_0"].astype(np.float64)
    a = run_all(g, make(g, pts, 1), 0.5, 0.4, 77, 10)
    b = run_all(g, make(g, pts, 1, flags=capi.B2_CLOUD_NO_REORDER), 0.5, 0.4, 77, 10)
    c = run_all(g, make(g, pts, 1), 0.5, 0.4, 77, 10)
    assert same_outputs(a, b) and same_outputs(a, c)
    # float64 storage: the f64 tree records and distances
    f64 = pts + 1e-7 * np.random.default_rng(3).normal(size=pts.shape)
    cloud = make(g, f64, 2)
    assert cloud.info().point_bytes == 8
    run_all(g, cloud, 0.25, 0.5, 5, 10)


@pytest.mark.parametrize("name", sorted(pc.edge_cases()))
def test_edge_cases(g, name):
    pts, res = pc.edge_cases()[name]
    pts = pts[np.all(np.isfinite(pts), axis=1)]  # what a device cloud can hold
    cloud = make(g, pts, 4)
    finite_sq = np.all(np.abs(pts) < 1e150)  # squared distances that do not overflow
    run_all(g, cloud, res, 0.25, 11, 10 if finite_sq and len(pts) >= 10 else None)
    if name in ("big_voxel", "run_across_1024"):
        # one voxel's run is sampled as one group: the oracle's whole-voxel rule, matched above; its share is at most ppv
        K = g.types._randomgrid(cloud, 1.0, 0.25, 11, 0)[1]
        voxels = {}
        for i, p in enumerate(pts):
            voxels.setdefault(tuple(np.floor(p).astype(int)), []).append(i)
        ppv = int(np.ceil(0.25 * len(pts) / len(voxels)))
        big = max(voxels.values(), key=len)
        assert len(big) > ppv and np.isin(K, big).sum() <= ppv


def test_million_points(g):
    pts = syn.make_cloud(1_000_000, stream=21, scale=2.0)[0]
    run_all(g, make(g, pts, 6, with_normals=False), 0.5, 0.5, 123, 10)


def test_rate_edges_and_one_voxel(g):
    rng = np.random.default_rng(4)
    cloud = make(g, rng.uniform(0.1, 0.9, size=(500, 3)), 1)
    assert len(g.types._randomgrid(cloud, 1.0, 0.3, 1, 0)[1]) == 150
    for rate in (0.0, 0.99, 1.7):
        run_all(g, cloud, 1.0, rate, 1, 10)
    empty = make(g, np.zeros((0, 3)), 1)
    for got in (g.random_sampling(empty, 0.5), g.randomgrid_sampling(empty, 0.5, 0.5), g.remove_outliers(empty), g.sample(empty, [])):
        assert len(got) == 0 and got.info().cov_bytes > 0 and got.info().normal_bytes > 0
    assert np.isnan(g.types._inliers(empty, 10, 1.0, None, 0)[3])
    lattice = np.stack(np.meshgrid(*[np.arange(8.0)] * 3), -1).reshape(-1, 3)
    got, K, d, th = g.types._inliers(make(g, lattice, 2), 1, 1.0, None, 0)
    assert len(K) == 0 and th == 0.0 and np.all(d == 0.0)


def test_with_tree(g):
    cloud = make(g, SCANS["kitti07_0"].astype(np.float64), 3)
    tree = g.KdTree.from_cloud(cloud)
    a = g.types._inliers(cloud, 20, 0.5, tree, 0)
    b = g.types._inliers(cloud, 20, 0.5, None, 0)
    assert np.array_equal(a[1], b[1]) and pc.same_bits(a[2], b[2]) and pc.same_bits(a[3], b[3])
    assert np.array_equal(g.find_inlier_points(cloud, 20, 0.5, tree), a[1])


def test_argument_errors(g):
    cloud = make(g, SCANS["kitti07_3"].astype(np.float64), 5)
    other = make(g, SCANS["kitti07_0"].astype(np.float64), 5)
    bad = [
        lambda: g.random_sampling(cloud, np.nan), lambda: g.random_sampling(cloud, -0.1), lambda: g.random_sampling(cloud, np.inf),
        lambda: g.randomgrid_sampling(cloud, 0.0, 0.5), lambda: g.randomgrid_sampling(cloud, np.inf, 0.5), lambda: g.randomgrid_sampling(cloud, -1.0, 0.5),
        lambda: g.randomgrid_sampling(cloud, 0.5, np.nan), lambda: g.randomgrid_sampling(cloud, 0.5, -1.0),
        lambda: g.remove_outliers(cloud, 0), lambda: g.remove_outliers(cloud, 65), lambda: g.remove_outliers(cloud, 10, np.nan),
        lambda: g.remove_outliers(cloud, 10, tree=g.KdTree.from_cloud(other)), lambda: g.remove_outliers(cloud, 10, tree=g.KdTree(cloud.points)),
        lambda: g.remove_outliers(make(g, np.random.default_rng(1).normal(size=(9, 3)), 1), 10),
        lambda: g.sample(cloud, [0, -1]), lambda: g.sample(cloud, [len(cloud)]),
    ]
    for f in bad:
        with pytest.raises(capi.B2Error) as e:
            f()
        assert e.value.status == 1  # B2_ERR_INVALID_ARGUMENT
    L = capi.lib()
    h = C.c_void_p(1)
    assert L.b2_cloud_create_sampled(None, None, 0, 0, C.byref(h)) == 1 and not h.value
    assert L.b2_cloud_create_inliers(cloud.h, None, 10, 1.0, 0, None, None, None, None) == 1
    # the failures left the cloud usable
    run_all(g, cloud, 0.5, 0.5, 1, 10)


def records(f, deltas):
    out = []
    for d in deltas:
        buf = np.zeros(capi.B2_LINEARIZED_DOUBLES)
        capi.check(capi.lib().b2_factor_linearize(f.h, capi.dptr(np.ascontiguousarray(d)), capi.dptr(buf)))
        out.append(buf)
    return np.array(out)


def test_outliers_then_estimation_then_gicp(g):
    """remove_outliers -> covariance estimation -> kd-tree from the new cloud -> GICP factor, all on the device, linearizes to the bits
    of the same chain built from host arrays."""
    tgt_raw = g.voxelgrid_sampling(SCANS["kitti00_0"], 0.25)
    src = g.voxelgrid_sampling(SCANS["kitti00_1"], 0.25).estimated(10)
    tgt = g.remove_outliers(tgt_raw, 10, 1.0).estimated(10)
    tree = g.KdTree.from_cloud(tgt)
    K = fo.inliers(download(tgt_raw)[0], 10, 1.0)[0]
    host_tgt = g.PointCloud(download(tgt_raw)[0][K]).estimated(10)
    host_tgt = g.PointCloud(download(host_tgt)[0], download(host_tgt)[1])
    host_src = g.PointCloud(download(src)[0], download(src)[1])
    rng = np.random.default_rng(12)
    deltas = [syn.random_pose(rng, 0.02, 0.3) for _ in range(3)]
    a = records(g.IntegratedGICPFactor(0, 1, tgt, src, target_tree=tree), deltas)
    b = records(g.IntegratedGICPFactor(0, 1, host_tgt, host_src, target_tree=g.KdTree(host_tgt.points)), deltas)
    assert pc.same_bits(a, b) and a[0, 121] > 0.5 * len(src)
