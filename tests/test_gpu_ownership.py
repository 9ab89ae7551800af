"""Device-memory ownership of the handles (pytest -m gpu).

`device_bytes` of clouds, voxel maps and iVoxes equals the sizes of the arrays each handle owns, computed here from the
allocation rules (plane strides, bucket-table size, capacity growth, the iVox slot layout).  A create that fails leaves the
out-pointer NULL with the documented status and message; an iVox insert that fails leaves the map as it was; and the same
context goes on building valid objects that give the results of a fresh context."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from gtsam_points_b200 import capi

B2_ERR_INVALID_ARGUMENT = 1
BUCKET_BYTES = 16  # VoxelBucket
RECORD_BYTES = 80  # 10 doubles: mean, covariance upper triangle, count
SENTINEL = 0x1234  # out-pointer value before a call: a failed create must overwrite it with NULL


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def n_pad(n):
    return (max(n, 1) + 31) // 32 * 32


def bucket_count(num_voxels):
    return 1 << (max(64, 4 * num_voxels) - 1).bit_length()


def map_bytes(num_voxels, capacity, slot_records=1, counts=False):
    """Bucket table + per-voxel records (slot_records records each), coordinates, LRU and, for an iVox, point counts."""
    return bucket_count(num_voxels) * BUCKET_BYTES + capacity * (slot_records * RECORD_BYTES + 12 + 4 + (4 if counts else 0))


class VoxelModel:
    """Voxel set, LRU and capacity of IncrementalVoxelMap-style inserts of points at voxel centres."""

    def __init__(self, horizon=10, cycle=10):
        self.lru = {}  # voxel -> lru counter of the last insert that touched it (dict keeps first-touch order)
        self.counter, self.capacity, self.horizon, self.cycle = 0, 1, horizon, cycle

    def insert(self, voxels):
        new = [v for v in dict.fromkeys(voxels) if v not in self.lru]
        want = len(self.lru) + len(new)
        if want > self.capacity:
            self.capacity = max(want, 2 * self.capacity)
        for v in voxels:
            self.lru[v] = self.counter
        self.counter += 1
        if self.counter % self.cycle == 0:
            self.lru = {v: c for v, c in self.lru.items() if c + self.horizon >= self.counter}


def centre_points(voxels, per_voxel, res, rng):
    """`per_voxel` points inside each voxel (well away from its faces), voxels in the given order."""
    v = np.repeat(np.asarray(voxels, dtype=np.float64), per_voxel, axis=0)
    return (v + 0.5 + rng.uniform(-0.3, 0.3, v.shape)) * res


def identity_covs(n):
    return np.ascontiguousarray(np.broadcast_to(np.eye(3), (n, 3, 3)))


def voxel_block(x0, count):
    """Voxels x0 .. x0 + count - 1 of one fixed staircase: blocks with overlapping x ranges share those voxels."""
    return [(x, (x * 7) % 5, -(x % 3)) for x in range(x0, x0 + count)]


# ---- device_bytes ----------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("n", [0, 1, 37, 1000])
@pytest.mark.parametrize("precision", ["f32", "f64"])
@pytest.mark.parametrize("with_covs", [True, False])
@pytest.mark.parametrize("reorder", [True, False])
def test_cloud_device_bytes(g, n, precision, with_covs, reorder):
    rng = np.random.default_rng(n + 7)
    pts = rng.normal(size=(n, 3)).astype(np.float32).astype(np.float64)
    covs = identity_covs(n) * 0.5 if with_covs else None
    if precision == "f64":
        pts = pts + 1e-9  # not float32-representable
        if with_covs:
            covs = covs + 1e-9
    flags = capi.B2_CLOUD_DEFAULT if reorder else capi.B2_CLOUD_NO_REORDER
    info = g.PointCloud(pts, covs, flags=flags).info()
    pb = 8 if precision == "f64" and n > 0 else 4
    cb = 0 if not with_covs else (8 if precision == "f64" and n > 0 else 4)
    reordered = reorder and n > 1
    assert (info.point_bytes, info.cov_bytes, bool(info.reordered)) == (pb, cb, reordered)
    assert info.device_bytes == 3 * n_pad(n) * pb + 6 * n_pad(n) * cb + (4 * n if reordered else 0)


def voxelmap_info(h):
    info = capi.VoxelMapInfo()
    capi.check(capi.lib().b2_voxelmap_get_info(h, C.byref(info)))
    return info


def test_voxelmap_device_bytes_across_inserts_and_eviction(g):
    L = capi.lib()
    res = 0.5
    h = C.c_void_p()
    capi.check(L.b2_voxelmap_create(g.default_context().h, res, C.byref(h)))
    try:
        model = VoxelModel(horizon=1, cycle=4)
        capi.check(L.b2_voxelmap_set_lru(h, model.horizon, model.cycle))
        info = voxelmap_info(h)
        assert (info.num_voxels, info.num_buckets, info.device_bytes) == (0, 64, map_bytes(0, 1))
        rng = np.random.default_rng(3)
        batches = [
            voxel_block(0, 10),  # capacity 1 -> 10
            voxel_block(5, 35),  # 5 voxels exist already; capacity -> 40, table 64 -> 256 buckets
            voxel_block(38, 3),  # one new voxel: capacity 40 -> 80 (doubling)
            voxel_block(39, 4),  # 4th insert: keeps only the voxels it touched, the table shrinks again
        ]
        sizes = []
        for voxels in batches:
            pts = centre_points(voxels, 3, res, rng)
            covs = identity_covs(len(pts))
            capi.check(L.b2_voxelmap_insert(h, capi.dptr(pts), 3, capi.dptr(covs), 9, len(pts)))
            model.insert(voxels)
            info = voxelmap_info(h)
            V = len(model.lru)
            sizes.append(V)
            assert (info.num_voxels, info.num_buckets) == (V, bucket_count(V))
            assert info.device_bytes == map_bytes(V, model.capacity)
        assert sizes == [10, 40, 41, 4] and model.capacity == 80
    finally:
        L.b2_voxelmap_destroy(h)


@pytest.mark.parametrize("V", [1, 17, 100])
def test_voxelmap_device_bytes_from_voxels_and_load(g, V, tmp_path):
    rng = np.random.default_rng(V)
    coords = np.array(voxel_block(-50, V), dtype=np.int32)
    means = (coords + 0.5) * 0.25
    covs = identity_covs(V)
    vm = g.GaussianVoxelMapGPU.from_voxels(0.25, coords, means, covs, num_points=rng.integers(1, 9, V))
    info = vm.info()
    assert (info.num_voxels, info.num_buckets, info.device_bytes) == (V, bucket_count(V), map_bytes(V, V))
    path = tmp_path / "map.bin"
    vm.save_compact(path)
    info = g.GaussianVoxelMapGPU.load(path).info()
    assert (info.num_voxels, info.num_buckets, info.device_bytes) == (V, bucket_count(V), map_bytes(V, V))


def test_ivox_device_bytes_layout_growth_clear(g):
    res, stride = 0.5, 4
    iv = g.iVox(res)
    iv.set_max_num_points_in_cell(stride)
    info = iv.info()
    assert (info.num_voxels, info.device_bytes) == (0, map_bytes(0, 1))  # Gaussian-voxel layout until the first insert
    model = VoxelModel()
    rng = np.random.default_rng(5)
    for voxels in (voxel_block(0, 6), voxel_block(3, 20), voxel_block(23, 10)):
        pts = centre_points(voxels, 2, res, rng)
        iv.insert(pts, identity_covs(len(pts)))
        model.insert(voxels)
        info = iv.info()
        V = len(model.lru)
        assert info.num_voxels == V
        assert info.device_bytes == map_bytes(V, model.capacity, slot_records=stride, counts=True)
    assert model.capacity == 46  # the first insert lays out 6 voxels, then 6 -> 23 -> 46 (doubling)
    iv.clear()  # the slot layout and the capacity stay, the table goes back to its minimum
    info = iv.info()
    assert (info.num_voxels, info.device_bytes) == (0, map_bytes(0, model.capacity, slot_records=stride, counts=True))


# ---- failed creates / inserts ----------------------------------------------------------------------------------------


def last_error():
    return capi.lib().b2_last_error().decode()


def test_cloud_create_nan_then_same_results(g):
    L = capi.lib()
    ctx = g.Context(0)
    rng = np.random.default_rng(11)
    pts = rng.normal(size=(500, 3))
    covs = identity_covs(len(pts))
    bad = pts.copy()
    bad[123, 1] = np.nan
    h = C.c_void_p(SENTINEL)
    st = L.b2_cloud_create(ctx.h, capi.dptr(bad), 3, capi.dptr(covs), 9, len(bad), capi.B2_CLOUD_DEFAULT, C.byref(h))
    assert (st, last_error(), h.value) == (B2_ERR_INVALID_ARGUMENT, "b2_cloud_create: non-finite coordinate or covariance entry", None)
    got = g.merge_frames_gpu(np.eye(4)[None], [g.PointCloud(pts, covs, ctx=ctx)], 0.3)
    ref = g.merge_frames_gpu(np.eye(4)[None], [g.PointCloud(pts, covs, ctx=g.Context(0))], 0.3)
    assert len(got.points) > 0
    assert np.array_equal(got.points, ref.points) and np.array_equal(got.covs, ref.covs)


def test_kdtree_create_nan_then_same_results(g):
    L = capi.lib()
    ctx = g.Context(0)
    rng = np.random.default_rng(12)
    pts = rng.normal(size=(3000, 3))
    bad = pts.copy()
    bad[2999, 2] = np.nan  # found by the device scan, after the tree's buffers exist
    h = C.c_void_p(SENTINEL)
    st = L.b2_kdtree_create(ctx.h, capi.dptr(bad), 3, len(bad), C.byref(h))
    assert (st, last_error(), h.value) == (B2_ERR_INVALID_ARGUMENT, "b2_kdtree_create: non-finite coordinate", None)
    q = rng.normal(size=(400, 3))
    for k in (1, 5):
        idx, sq = g.KdTree(pts, ctx=ctx).knn_search(q, k)
        ref_idx, ref_sq = g.KdTree(pts, ctx=g.Context(0)).knn_search(q, k)
        assert np.array_equal(idx, ref_idx) and np.array_equal(sq, ref_sq)


def test_voxelmap_from_voxels_duplicate_then_same_results(g):
    L = capi.lib()
    ctx = g.Context(0)
    coords = np.array(voxel_block(0, 30), dtype=np.int32)
    means = (coords + 0.5) * 0.5
    covs = identity_covs(len(coords)).reshape(-1, 9)
    dup = coords.copy()
    dup[20] = dup[7]
    ip = C.POINTER(C.c_int32)
    h = C.c_void_p(SENTINEL)
    st = L.b2_voxelmap_create_from_voxels(ctx.h, 0.5, dup.ctypes.data_as(ip), capi.dptr(means), capi.dptr(covs), None, len(dup), C.byref(h))
    x, y, z = (int(c) for c in coords[7])
    msg = f"b2_voxelmap_create_from_voxels: duplicate voxel coordinate ({x}, {y}, {z}) at ids 7 and 20"
    assert (st, last_error(), h.value) == (B2_ERR_INVALID_ARGUMENT, msg, None)
    q = np.concatenate([means, means + 0.6])
    got = g.GaussianVoxelMapGPU.from_voxels(0.5, coords, means, covs, ctx=ctx).lookup_voxel_index(q)
    ref = g.GaussianVoxelMapGPU.from_voxels(0.5, coords, means, covs, ctx=g.Context(0)).lookup_voxel_index(q)
    assert np.array_equal(got, ref) and np.array_equal(got[: len(coords)], np.arange(len(coords)))


def test_ivox_mixed_covariance_insert_leaves_map_unchanged(g):
    L = capi.lib()
    ctx, fresh = g.Context(0), g.Context(0)
    res = 0.5
    rng = np.random.default_rng(13)
    first = centre_points(voxel_block(0, 25), 3, res, rng)
    second = centre_points(voxel_block(10, 25), 3, res, rng)
    iv = g.iVox(res, ctx=ctx)
    iv.insert(first, identity_covs(len(first)))
    before, info_before = iv.download(), iv.info()
    st = L.b2_ivox_insert(iv.h, capi.dptr(second), 3, None, 0, len(second))
    assert (st, last_error()) == (B2_ERR_INVALID_ARGUMENT, "b2_ivox_insert: the map holds points with covariances; inserts cannot mix both")
    after, info_after = iv.download(), iv.info()
    for key in ("coords", "counts", "points", "covs"):
        assert np.array_equal(before[key], after[key]), key
    assert (info_after.num_voxels, info_after.num_points, info_after.device_bytes) == (info_before.num_voxels, info_before.num_points, info_before.device_bytes)
    # the map takes the valid insert and answers like a map that never saw the failed one
    iv.insert(second, identity_covs(len(second)))
    ref = g.iVox(res, ctx=fresh)
    ref.insert(first, identity_covs(len(first)))
    ref.insert(second, identity_covs(len(second)))
    q = centre_points(voxel_block(5, 30), 1, res, rng)
    for k in (1, 4):
        idx, sq = iv.knn_search(q, k)
        ref_idx, ref_sq = ref.knn_search(q, k)
        assert np.array_equal(idx, ref_idx) and np.array_equal(sq, ref_sq)
