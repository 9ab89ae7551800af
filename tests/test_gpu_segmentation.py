"""Region growing on the device (b2_region_growing_*) against the CPU oracle (tests/segmentation_oracle.cpp), bit for bit: the
cluster and the converged flag after every update, the visit order, the size cap and the dilation set."""
import ctypes as C
import os

import numpy as np
import pytest

import segmentation_oracle as so
from gtsam_points_b200 import capi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def stored(cloud):
    """The cloud's stored points and normals in caller order."""
    n = int(cloud.info().num_points)
    p, nr = np.zeros((n, 3)), np.zeros((n, 3))
    capi.check(capi.lib().b2_cloud_download(cloud.h, capi.dptr(p), None, capi.dptr(nr)))
    return p, nr


def planes_and_box(seed, n=20000):
    """A ground plane, a wall and a box on the ground, with exact face normals and a little noise on the points."""
    rng = np.random.default_rng(seed)
    k = n // 4
    ground = np.c_[rng.uniform(-10, 10, (k, 2)), rng.normal(0, 0.005, k)]
    wall = np.c_[rng.uniform(-10, 10, k), np.full(k, 8.0) + rng.normal(0, 0.005, k), rng.uniform(0, 4, k)]
    faces, normals = [], []
    for a in range(3):
        for sgn in (0.0, 1.0):
            m = (n - 2 * k) // 6
            f = rng.uniform(0, 1, (m, 3))
            f[:, a] = sgn
            faces.append(f * np.array([2.0, 2.0, 1.5]) + np.array([-1.0, -1.0, 0.0]))
            nv = np.zeros((m, 3))
            nv[:, a] = 1.0 if sgn else -1.0
            normals.append(nv)
    p = np.vstack([ground, wall] + faces)
    nr = np.vstack([np.tile([0, 0, 1.0], (k, 1)), np.tile([0, -1.0, 0], (k, 1))] + normals)
    return p, nr


def kitti(name, key):
    return np.load(os.path.join(ROOT, "tests", "golden", name))[key].astype(np.float64)


def check(g, cloud, seed_point, steps, dist=0.5, angle=np.deg2rad(10.0), dil=0.5, maxc=1000000, tree=None):
    """Every update's flag and cluster equal the oracle's over the cloud's stored values; returns the device trace."""
    p, nr = stored(cloud)
    seed = so.nearest(p, seed_point) if len(p) else -1
    want = so.trace(p, nr, seed, steps, distance_threshold=dist, angle_threshold=angle, dilation_radius=dil, max_cluster_size=maxc)
    prm = g.RegionGrowingParams(dist, angle, dil, maxc)
    rg = g.RegionGrowing.init(cloud, seed_point, prm, tree)
    got = []
    for s, (conv, cl) in zip(steps, want):
        c = rg.update(s)
        idx = rg.cluster_indices
        got.append((c, idx))
        assert c == conv
        assert np.array_equal(idx, cl)
    return got


@pytest.mark.parametrize("flags", [capi.B2_CLOUD_DEFAULT, capi.B2_CLOUD_NO_REORDER])
@pytest.mark.parametrize("scene", [0, 1])
def test_planes_and_box(g, flags, scene):
    p, nr = planes_and_box(scene)
    cloud = g.PointCloud(p, normals=nr, flags=flags)
    for seed_point in ([0.0, 0.0, 0.0], [0.0, 0.0, 1.5], [3.0, 8.0, 2.0]):
        check(g, cloud, seed_point, [10**6])
        check(g, cloud, seed_point, [1, 5, 0, 300, 2, 10**6, 1], dist=0.3, dil=0.2)
    check(g, cloud, [0.0, 0.0, 0.0], [1, 1, 1000], dil=0.0)  # dilation 0: the cluster stays in visit order
    check(g, cloud, [0.0, 0.0, 0.0], [10**6], angle=0.0)
    check(g, cloud, [0.0, 0.0, 0.0], [10**6], angle=np.pi, dist=0.4)
    check(g, cloud, [0.0, 0.0, 1.5], [50, 10**6, 3], maxc=100)  # the cap: max_cluster_size + 1 points, then one step clears


@pytest.mark.parametrize("name,key", [("kitti00_pair.npz", "frame0"), ("kitti07_pair.npz", "source_points")])
def test_kitti_with_device_normals(g, name, key):
    pts = kitti(name, key)[:, :3]
    cloud = g.PointCloud(pts).estimated(10, normals=True)
    tree = g.KdTree.from_cloud(cloud)
    p, nr = stored(cloud)
    for seed_point in (p[0], p[len(p) // 2], [0.0, 0.0, -1.7]):
        check(g, cloud, seed_point, [10**6], tree=tree)
        check(g, cloud, seed_point, [7, 0, 200, 1, 10**6, 1], dist=1.0, angle=0.3, dil=0.3)


def test_stale_entries_delay_the_flag(g):
    """Scenes whose last visit leaves stale entries: converged comes one update later, with the dilation."""
    rng = np.random.default_rng(5)
    seen = 0
    for s in range(12):
        p = rng.uniform(-3, 3, (400, 3)) * np.array([1, 1, 0.3])
        nr = np.tile([0, 0, 1.0], (400, 1)) + rng.normal(0, 0.3, (400, 3))
        nr /= np.linalg.norm(nr, axis=1, keepdims=True)
        cloud = g.PointCloud(p, normals=nr)
        q, qn = stored(cloud)
        seed = so.nearest(q, q[s])
        full = so.RegionGrowing(q, qn, seed, 0.8, 0.4, 0.0)
        full.update()
        V = len(full.cluster_indices)
        got = check(g, cloud, q[s], [V, 1], dist=0.8, angle=0.4, dil=0.3)
        seen += not got[0][0]
    assert seen >= 1


def test_seeds_far_and_isolated(g):
    p, nr = planes_and_box(2, 4000)
    p = np.vstack([p, [[50.0, 50.0, 50.0]]])
    nr = np.vstack([nr, [[0.0, 0.0, 1.0]]])
    cloud = g.PointCloud(p, normals=nr)
    check(g, cloud, [1e6, -1e6, 3e5], [10**6, 1])
    got = check(g, cloud, [49.0, 50.0, 50.0], [1, 1], dil=0.0)
    assert len(got[0][1]) == 1 and got[0][0]


def test_one_million_points_past_the_default_cap(g):
    """A dense plane of 1.2M points: with the defaults the cluster reaches 1000001 points and one more step clears the queue."""
    rng = np.random.default_rng(9)
    n = 1_200_000
    p = np.c_[rng.uniform(0, 60, (n, 2)), rng.normal(0, 0.002, n)]
    nr = np.tile([0.0, 0.0, 1.0], (n, 1))
    cloud = g.PointCloud(p, normals=nr)
    got = check(g, cloud, [30.0, 30.0, 0.0], [10**6, 10**6], dist=0.1, dil=0.0)
    assert len(got[0][1]) == 1000000 and not got[0][0]
    assert len(got[1][1]) == 1000001 and got[1][0]


def test_repeated_calls_identical(g):
    p, nr = planes_and_box(3)
    cloud = g.PointCloud(p, normals=nr)
    runs = []
    for _ in range(3):
        rg = g.RegionGrowing.init(cloud, [0.0, 0.0, 0.0], g.RegionGrowingParams(0.3, 0.2, 0.2, 5000))
        runs.append([(rg.update(s), rg.cluster_indices) for s in (100, 10**6, 1)])
    for r in runs[1:]:
        assert all(a[0] == b[0] and np.array_equal(a[1], b[1]) for a, b in zip(runs[0], r))


def test_empty_cloud_and_errors(g):
    empty = g.PointCloud(np.zeros((0, 3)), normals=np.zeros((0, 3)))
    rg = g.RegionGrowing.init(empty, [0.0, 0.0, 0.0])
    assert rg.update() and len(rg.cluster_indices) == 0
    p, nr = planes_and_box(4, 2000)
    cloud = g.PointCloud(p, normals=nr)
    bad = [
        (g.PointCloud(p), [0, 0, 0], g.RegionGrowingParams()),  # no normals
        (cloud, [np.nan, 0, 0], g.RegionGrowingParams()),
        (cloud, [0, 0, 0], g.RegionGrowingParams(distance_threshold=-1.0)),
        (cloud, [0, 0, 0], g.RegionGrowingParams(angle_threshold=np.inf)),
        (cloud, [0, 0, 0], g.RegionGrowingParams(dilation_radius=np.nan)),
        (cloud, [0, 0, 0], g.RegionGrowingParams(max_cluster_size=-1)),
    ]
    for c, sp, prm in bad:
        with pytest.raises(capi.B2Error) as e:
            g.RegionGrowing.init(c, sp, prm)
        assert e.value.status == 1
    other = g.KdTree.from_cloud(g.PointCloud(p, normals=nr))
    with pytest.raises(capi.B2Error):
        g.RegionGrowing.init(cloud, [0, 0, 0], tree=other)
    rg = g.RegionGrowing.init(cloud, [0, 0, 0])
    with pytest.raises(capi.B2Error):
        rg.update(g.RegionGrowingParams(distance_threshold=0.7))
    assert isinstance(rg.update(g.RegionGrowingParams(max_steps=3)), bool)
    out = C.c_void_p()
    assert capi.lib().b2_region_growing_create(cloud.h, None, None, 0.5, 0.1, 0.5, 10, C.byref(out)) == 1 and not out.value
