"""FastOccupancyGrid and VoxelRaycaster on the device (b2_occgrid_*, b2_raycast) against the CPU oracle (tests/occupancy_oracle.cpp),
bit for bit: overlap counts and per-point flags in caller order, the occupied cells after every insert and free_rays, and raycast CSR
rows.  The oracle always runs on the values b2_cloud_download returns, so float32-compact and Morton-ordered clouds are checked in
caller order."""
import ctypes as C
import os

import numpy as np
import pytest

import occupancy_oracle as oo
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
K00 = np.load(os.path.join(GOLDEN, "kitti00_pair.npz"))
K07 = np.load(os.path.join(GOLDEN, "kitti07_frames.npz"))
STORAGE = {"morton": capi.B2_CLOUD_DEFAULT, "caller": capi.B2_CLOUD_NO_REORDER, "f32": capi.B2_CLOUD_COMPACT_F32}


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def download(cloud):
    p = np.zeros((cloud.size(), 3))
    if len(p):
        capi.check(capi.lib().b2_cloud_download(cloud.h, capi.dptr(p), None, None))
    return p


def poses(rng, m, rot, trans):
    return np.stack([syn.random_pose(rng, rot, trans) for _ in range(m)])


def assert_same_grid(grid, orc):
    assert grid.num_occupied_cells() == orc.num_occupied_cells()
    assert np.array_equal(grid.occupied_cells(), orc.cells())


def check_overlaps(grid, orc, cloud, Ts):
    rows = download(cloud)
    counts, flags = grid.calc_overlaps(cloud, Ts, flags=True)
    for j, T in enumerate(Ts):
        c, f = orc.overlaps(rows, T)
        assert int(counts[j]) == c, j
        assert np.array_equal(flags[j], f), j
    return counts


@pytest.mark.parametrize("storage", sorted(STORAGE))
@pytest.mark.parametrize("res", [0.25, 0.5, 1.0])
def test_kitti00_overlap(g, storage, res):
    tgt = g.PointCloud(K00["frame0"], flags=STORAGE[storage])
    src = g.PointCloud(K00["frame1"], flags=STORAGE[storage])
    grid, orc = g.FastOccupancyGrid(res), oo.Grid(res)
    grid.insert(tgt)
    orc.insert(download(tgt))
    assert_same_grid(grid, orc)
    rng = np.random.default_rng(7)
    Ts = np.concatenate([K00["T_final"][None], poses(rng, 63, 0.05, 0.5)])
    counts = check_overlaps(grid, orc, src, Ts)
    assert counts[0] > 0.3 * src.size()  # the registered pose overlaps
    one = check_overlaps(grid, orc, src, Ts[:1])
    assert one[0] == counts[0]
    assert grid.calc_overlap(src, Ts[0]) == counts[0]
    assert grid.calc_overlap_rate(src, Ts[0]) == counts[0] / float(src.size())
    assert np.array_equal(grid.get_overlaps(src, Ts[0]), orc.overlaps(download(src), Ts[0])[1])
    assert grid.calc_overlap(src) == orc.overlaps(download(src))[0]


@pytest.mark.parametrize("storage", ["morton", "f32"])
def test_kitti07_incremental(g, storage):
    """insert -> free_rays -> insert over the KITTI-07 frames at their poses; the cells after every call."""
    res = 0.5
    grid, orc = g.FastOccupancyGrid(res), oo.Grid(res)
    for k in range(5):
        cloud = g.PointCloud(K07[f"points{k}"], flags=STORAGE[storage])
        T = K07["poses"][k]
        rows = download(cloud)
        if k > 0:
            grid.free_rays(cloud, T)
            orc.free_rays(rows, T)
            assert_same_grid(grid, orc)
        grid.insert(cloud, T)
        orc.insert(rows, T)
        assert_same_grid(grid, orc)
    cloud = g.PointCloud(K07["points0"])
    check_overlaps(grid, orc, cloud, K07["poses"])


@pytest.mark.parametrize("res", [0.25, 0.5])
def test_kitti00_free_rays(g, res):
    grid, orc = g.FastOccupancyGrid(res), oo.Grid(res)
    a, b = g.PointCloud(K00["frame0"]), g.PointCloud(K00["frame1"])
    grid.insert(a)
    orc.insert(download(a))
    before = grid.num_occupied_cells()
    grid.free_rays(b, K00["T_final"])
    orc.free_rays(download(b), K00["T_final"])
    assert_same_grid(grid, orc)
    assert grid.num_occupied_cells() < before
    grid.free_rays(b, K00["T_final"])  # idempotent
    assert_same_grid(grid, orc)


def test_synthetic_1m(g):
    """A ~1M-point scene inserted under random poses in three batches (the table grows), overlaps under 16 poses, then free_rays."""
    pts = syn.make_cloud(1_000_000, stream=21, scale=2.0)[0]
    rng = np.random.default_rng(3)
    grid, orc = g.FastOccupancyGrid(0.2), oo.Grid(0.2)
    for part, T in zip(np.array_split(pts, 3), poses(rng, 3, 0.1, 2.0)):
        cloud = g.PointCloud(part)
        grid.insert(cloud, T)
        orc.insert(download(cloud), T)
    assert_same_grid(grid, orc)
    assert grid.info().num_blocks > 512
    src = g.PointCloud(pts[::7])
    check_overlaps(grid, orc, src, poses(rng, 16, 0.1, 2.0))
    T = syn.random_pose(rng, 0.1, 2.0)
    grid.free_rays(src, T)
    orc.free_rays(download(src), T)
    assert_same_grid(grid, orc)


def test_edge_points(g):
    """Empty clouds, points outside the key range (dropped), poses that overflow to infinity, points on cell faces and negative
    coordinates."""
    res = 0.5
    grid, orc = g.FastOccupancyGrid(res), oo.Grid(res)
    empty = g.PointCloud(np.zeros((0, 3)))
    grid.insert(empty)
    grid.free_rays(empty)
    assert grid.calc_overlap(empty) == 0 and grid.calc_overlap_rate(empty) == 0.0
    assert grid.calc_overlaps(empty, np.stack([np.eye(4)] * 3)).tolist() == [0, 0, 0]
    assert grid.num_occupied_cells() == 0 and grid.occupied_cells().shape == (0, 3)
    lim = 2.0**20 * res
    pts = np.array([[0, 0, 0], [-0.0, 0.5, -0.5], [lim - 0.25, 0, 0], [lim, 0, 0], [-lim, 1, 1], [-lim - 1e-6, 1, 1], [4.0, -4.0, 3.5], [-4.0, 4.0, -3.5],
                    [3.9999999999999996, 0, 0], [1e9, 0, 0], [0, -1e9, 0]], dtype=np.float64)
    cloud = g.PointCloud(pts, flags=capi.B2_CLOUD_NO_REORDER)
    grid.insert(cloud)
    orc.insert(pts)
    assert_same_grid(grid, orc)
    c, f = orc.overlaps(pts)
    assert f[3] == 0 and f[5] == 0 and f[9] == 0 and f[10] == 0 and f[2] == 1 and f[4] == 1
    check_overlaps(grid, orc, cloud, np.stack([np.eye(4)]))
    huge = np.eye(4)
    huge[:3, :3] *= 1e308
    check_overlaps(grid, orc, cloud, np.stack([huge, np.eye(4)]))
    grid.insert(cloud, huge)  # every posed coordinate but the zeros overflows or leaves the key range
    orc.insert(pts, huge)
    assert_same_grid(grid, orc)


def rays_rows(off, coords, i):
    return coords[int(off[i]):int(off[i + 1])]


def check_raycast(g, s, e, vs):
    off, coords = g.raycast(s, e, vs)
    woff, wcoords = oo.raycast(s, e, vs)
    assert np.array_equal(off, woff)
    assert np.array_equal(coords, wcoords)
    return off, coords


def test_raycast_random(g):
    rng = np.random.default_rng(11)
    for vs in (0.1, 0.25, 0.5, 1.0, 2.5):
        s = rng.uniform(-50, 50, (3000, 3))
        e = rng.uniform(-50, 50, (3000, 3))
        check_raycast(g, s, e, vs)


def test_raycast_edges(g):
    """Axis-aligned rays, rays through cell edges and corners (ties in the minimum-axis rule), zero-length and sub-eps rays, negative
    directions, one ray of at least 1e5 voxels."""
    rows = [
        ([0.5, 0.5, 0.5], [10.5, 0.5, 0.5]), ([0.5, 0.5, 0.5], [0.5, -10.5, 0.5]), ([0.5, 0.5, 0.5], [0.5, 0.5, 7.25]),
        ([0.0, 0.0, 0.0], [5.0, 5.0, 5.0]), ([0.0, 0.0, 0.0], [5.0, 5.0, 0.0]), ([0.0, 0.0, 0.0], [-5.0, -5.0, -5.0]), ([1.0, 1.0, 1.0], [-3.0, 2.0, -3.0]),
        ([0.25, 0.25, 0.25], [0.25, 0.25, 0.25]), ([0.25, 0.25, 0.25], [0.25 + 1e-10, 0.25, 0.25]), ([0.9999999999, 0.2, 0.2], [1.0000000001, 0.2, 0.2]),
        ([0.5, 0.5, 0.5], [0.5 + 5e-10, 3.5, 0.5 - 5e-10]), ([-0.5, -0.5, -0.5], [-10.0, -0.5, -3.0]), ([-1e-300, 0, 0], [1e-300, 0, 0]),
        ([2.0, 3.0, 4.0], [2.0, 3.0, 5.0]), ([0.1, 0.2, 0.3], [0.1, 0.2, 0.3 - 2.0]), ([0.0, 0.0, 0.0], [1.0, 2.0, 3.0]),
    ]
    s = np.array([r[0] for r in rows], dtype=np.float64)
    e = np.array([r[1] for r in rows], dtype=np.float64)
    for vs in (1.0, 0.5, 0.1):
        off, coords = check_raycast(g, s, e, vs)
        assert off[8] == off[7]  # start voxel == end voxel
    long_s, long_e = np.array([[0.05, 0.05, 0.05]]), np.array([[12345.67, -23.4, 4567.8]])
    off, coords = check_raycast(g, long_s, long_e, 0.1)
    assert off[1] >= 100_000
    off, coords = check_raycast(g, np.zeros((0, 3)), np.zeros((0, 3)), 0.5)
    assert off.tolist() == [0]


def test_argument_errors(g):
    for bad in (0.0, -1.0, np.nan, np.inf):
        with pytest.raises(capi.B2Error):
            g.FastOccupancyGrid(bad)
    grid = g.FastOccupancyGrid(0.5)
    cloud = g.PointCloud(K07["points0"])
    grid.insert(cloud)
    before = grid.occupied_cells()
    T = np.eye(4)
    T[1, 3] = np.nan
    for call in (grid.insert, grid.free_rays):
        with pytest.raises(capi.B2Error):
            call(cloud, T)
    with pytest.raises(capi.B2Error):
        grid.calc_overlaps(cloud, np.stack([np.eye(4), T]))
    far = np.eye(4)
    far[0, 3] = 1e12  # the sensor origin's voxel coordinate leaves int32
    with pytest.raises(capi.B2Error):
        grid.free_rays(cloud, far)
    assert np.array_equal(grid.occupied_cells(), before)
    L = capi.lib()
    s = np.zeros((2, 3))
    e = np.array([[3.0, 0, 0], [0, 4.0, 0]])
    off = np.zeros(3, dtype=np.uint64)
    coords = np.zeros((1, 3), dtype=np.int32)
    st = L.b2_raycast(g.default_context().h, capi.dptr(s), capi.dptr(e), 2, 1.0, off.ctypes.data_as(C.POINTER(C.c_uint64)), 1, coords.ctypes.data_as(C.POINTER(C.c_int32)))
    assert st == 1
    assert off.tolist() == [0, 3, 7]
    for bad_e in ([np.nan, 0, 0], [np.inf, 0, 0], [3e9, 0, 0]):
        with pytest.raises(capi.B2Error):
            g.raycast(s[:1], np.array([bad_e]), 1.0)
    with pytest.raises(capi.B2Error):
        g.raycast(s, e, 0.0)


def test_cloud_on_another_device(g):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device: no second device to place the cloud on")
    other = g.Context(1)
    cloud = g.PointCloud(K07["points0"], ctx=other)
    grid = g.FastOccupancyGrid(0.5)
    for call in (grid.insert, grid.free_rays, grid.calc_overlap):
        with pytest.raises(capi.B2Error):
            call(cloud)


def test_cloud_of_another_context(g):
    """A cloud of another context on the grid's device: the work runs on the grid's stream."""
    ctx = g.Context(0)
    cloud = g.PointCloud(K07["points1"], ctx=ctx)
    grid, orc = g.FastOccupancyGrid(0.25), oo.Grid(0.25)
    grid.insert(cloud, K07["poses"][1])
    orc.insert(download(cloud), K07["poses"][1])
    assert_same_grid(grid, orc)
