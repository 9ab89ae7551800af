"""Per-point intensities on the device (-m gpu): device clouds and every producer, the Gaussian voxel map's per-voxel maximum, the
iVox's per-slot intensities and the compact map file, bit for bit against the CPU oracle (tests/intensity_oracle.cpp) at both
storages and with and without Morton reorder; and the factors, which must compute the same bits with and without intensities."""
import ctypes as C

import numpy as np
import pytest

import intensity_oracle as io
from test_intensities_cpu import awkward_intensities, batches, same_bits

pytestmark = pytest.mark.gpu

FLAGS = [0, 1, 2, 4]  # default, B2_CLOUD_NO_REORDER, B2_CLOUD_COMPACT_F32, B2_CLOUD_FORCE_F64


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def stored(x, flags):
    """The values a cloud made under `flags` stores: float32 when every value is float32-exact (NaN is not) or with COMPACT_F32,
    float64 otherwise or with FORCE_F64."""
    x = np.asarray(x, dtype=np.float64)
    exact = np.all(np.float32(x).astype(np.float64) == x)
    f32 = not (flags & 4) and (bool(flags & 2) or exact)
    return (np.float32(x).astype(np.float64) if f32 else x.copy()), (4 if f32 else 8)


def stored_points(g, cloud):
    """b2_cloud_download's points: the stored values, after any float32 rounding."""
    out = np.zeros((len(cloud), 3))
    g.capi.check(g.capi.lib().b2_cloud_download(cloud.h, g.capi.dptr(out), None, None))
    return out


def stored_arrays(g, cloud):
    """b2_cloud_download's points, covariances and normals of a cloud that has all three."""
    n = len(cloud)
    p, c, nr = np.zeros((n, 3)), np.zeros((n, 3, 3)), np.zeros((n, 3))
    g.capi.check(g.capi.lib().b2_cloud_download(cloud.h, g.capi.dptr(p), g.capi.dptr(c), g.capi.dptr(nr)))
    return p, c, nr


def cloud_with(g, rng, n, flags, exact=False, covs=True):
    pts = rng.uniform(-4.0, 4.0, (n, 3))
    ints = np.float32(rng.uniform(0.0, 100.0, n)).astype(np.float64) if exact else awkward_intensities(rng, n)
    cov = np.tile(np.eye(3) * 0.01, (n, 1, 1)) if covs else None
    return g.PointCloud(pts, cov, flags=flags, intensities=ints), ints


@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("exact", [False, True])
def test_cloud_roundtrip(g, flags, exact):
    rng = np.random.default_rng(flags + 10 * exact)
    cloud, ints = cloud_with(g, rng, 3001, flags, exact)
    want, nbytes = stored(ints, flags)
    assert cloud.intensity_bytes() == nbytes
    assert same_bits(cloud.intensities_gpu(), want)
    assert bool(cloud.info().reordered) == (not flags & 1)
    plain = g.PointCloud(cloud.points, cloud.covs, flags=flags)
    assert plain.intensity_bytes() == 0
    assert cloud.info().device_bytes - plain.info().device_bytes == 3008 * nbytes  # n_pad = 3008: one plane of their own
    with pytest.raises(g.B2Error) as e:
        plain.intensities_gpu()
    assert e.value.status == 4
    empty = g.PointCloud(np.zeros((0, 3)), intensities=np.zeros(0), flags=flags)
    assert empty.intensity_bytes() in (4, 8) and len(empty.intensities_gpu()) == 0


@pytest.mark.parametrize("flags", FLAGS)
def test_producers(g, flags):
    from gtsam_points_b200 import types as t

    rng = np.random.default_rng(100 + flags)
    cloud, ints = cloud_with(g, rng, 4000, flags)
    src = cloud.intensities_gpu()  # caller order, as stored
    T = np.eye(4)
    T[:3, :3] = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    T[:3, 3] = [1.5, -2.25, 0.1]
    moved = t.transform_gpu(cloud, T, flags=flags)
    assert same_bits(moved.intensities_gpu(), stored(src, flags)[0])  # unchanged by the pose
    idx = rng.integers(0, len(cloud), 777)
    assert same_bits(t.sample(cloud, idx, flags=flags).intensities_gpu(), stored(src[idx], flags)[0])
    for res, K in (t._random_sampled(cloud, 0.3, 7, flags), t._randomgrid(cloud, 0.5, 0.4, 7, flags), t._inliers(cloud, 8, 1.0, None, flags)[:2]):
        assert len(K) > 0
        assert same_bits(res.intensities_gpu(), stored(src[K], flags)[0])
        assert same_bits(res.intensities, res.intensities_gpu())
    assert t.sample(g.PointCloud(cloud.points), idx).intensity_bytes() == 0  # no intensities in, none out


@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("est_flags", [0, 2, 4])
def test_estimated_keeps_intensities(g, flags, est_flags):
    """estimate_covariances leaves a frame's intensities in place: the estimated cloud keeps the stored ones, under its own flags."""
    rng = np.random.default_rng(150 + flags + 10 * est_flags)
    cloud, _ = cloud_with(g, rng, 5000, flags, covs=False)
    est = cloud.estimated(k_neighbors=10, normals=True, flags=est_flags)
    want, nbytes = stored(cloud.intensities_gpu(), est_flags)
    assert est.intensity_bytes() == nbytes and est.has_covs()
    assert same_bits(est.intensities_gpu(), want)
    assert g.PointCloud(cloud.points, flags=flags).estimated(flags=est_flags).intensity_bytes() == 0


def added_intensities(g, cloud, ints, flags):
    h = C.c_void_p()
    x = np.ascontiguousarray(ints, dtype=np.float64)
    g.capi.check(g.capi.lib().b2_cloud_create_with_added_intensities(cloud.h, g.capi.dptr(x), int(flags), C.byref(h)))
    return g.PointCloud._from_handle(h, cloud.ctx)


@pytest.mark.parametrize("flags", FLAGS)
def test_added_intensities_keep_the_cloud(g, flags):
    """b2_cloud_create_with_added_intensities: the same stored arrays, order and centre (a factor computes the same bits), also for
    COMPACT_F32 points that are not float32-exact, whose re-upload would move the centre and the Morton order."""
    rng = np.random.default_rng(170 + flags)
    pts = rng.uniform(-4.0, 4.0, (6000, 3)) + 1e-3 / 3.0
    cloud = g.PointCloud(pts, g.estimate_covariances(pts, 10), flags=flags, normals=rng.normal(0.0, 1.0, (6000, 3)))
    ints = awkward_intensities(rng, len(pts))
    more = added_intensities(g, cloud, ints, flags)
    a, b = cloud.info(), more.info()
    assert (a.point_bytes, a.cov_bytes, a.normal_bytes, a.reordered) == (b.point_bytes, b.cov_bytes, b.normal_bytes, b.reordered)
    for x, y in zip(stored_arrays(g, more), stored_arrays(g, cloud)):
        assert same_bits(x, y)
    assert same_bits(more.intensities_gpu(), stored(ints, flags)[0])
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert_cloud(cloud)
    delta = np.eye(4)
    delta[:3, 3] = [0.02, -0.01, 0.03]
    fa, fb = g.IntegratedVGICPFactor(np.eye(4), 1, vm, cloud), g.IntegratedVGICPFactor(np.eye(4), 1, vm, more)
    ra, rb = factor_record(fa, {1: delta}), factor_record(fb, {1: delta})
    assert same_bits(ra[0], rb[0]) and same_bits([ra[1]], [rb[1]])


@pytest.mark.parametrize("flags", FLAGS)
def test_voxelgrid(g, flags):
    rng = np.random.default_rng(200 + flags)
    pts = rng.uniform(-5.0, 5.0, (20000, 3))
    pts[7] = np.nan
    ints = rng.normal(20.0, 10.0, len(pts)) / 3.0
    ints[::9] = -0.0
    out = g.voxelgrid_sampling(pts, 0.4, intensities=ints, flags=flags)
    want, nbytes = stored(io.voxelgrid(pts, ints, 0.4), flags)
    assert out.intensity_bytes() == nbytes
    assert same_bits(out.intensities_gpu(), want)
    assert g.voxelgrid_sampling(pts, 0.4, flags=flags).intensity_bytes() == 0


def merge_to_cloud(g, frames, poses, res, flags):
    P = np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(len(frames), 16))
    arr = (C.c_void_p * len(frames))(*[f.h for f in frames])
    h = C.c_void_p()
    g.capi.check(g.capi.lib().b2_merge_frames_to_cloud(frames[0].ctx.h, g.capi.dptr(P), arr, len(frames), float(res), int(flags), C.byref(h)))
    return g.PointCloud._from_handle(h, frames[0].ctx)


@pytest.mark.parametrize("flags", FLAGS)
def test_merge_frames_to_cloud(g, flags):
    rng = np.random.default_rng(300 + flags)
    frames, poses, keys, vals = [], [], [], []
    for f in range(4):
        cloud, _ = cloud_with(g, rng, 2500, flags)
        t = np.eye(4)
        if f:
            t[:3, 3] = rng.integers(-4, 5, 3) * 0.5  # the first pose is the identity: the key frame is the world
        frames.append(cloud)
        poses.append(t)
        keys.append(stored_points(g, cloud) + t[:3, 3])  # the posed points, each sum rounded once, as on the device
        vals.append(cloud.intensities_gpu())
    out = merge_to_cloud(g, frames, poses, 0.3, flags)
    want, nbytes = stored(io.merge_frames(np.concatenate(keys), np.concatenate(vals), 0.3), flags)
    assert len(out) == len(want) and out.intensity_bytes() == nbytes
    assert same_bits(out.intensities_gpu(), want)
    assert np.all(out.intensities_gpu() >= 0.0)
    # one frame without intensities: the merged cloud has none; its points and covariances are as before
    plain = g.PointCloud(frames[1].points, frames[1].covs, flags=flags)
    mixed = merge_to_cloud(g, [frames[0], plain] + frames[2:], poses, 0.3, flags)
    assert mixed.intensity_bytes() == 0
    assert same_bits(mixed.points, out.points) and same_bits(mixed.covs, out.covs)


@pytest.mark.parametrize("flags", [0, 2])
@pytest.mark.parametrize("path", ["host", "cloud", "posed"])
@pytest.mark.parametrize("lead", [0, 2])
def test_voxelmap_insert(g, flags, path, lead):
    """lead: inserts without intensities before the first with them, so the map's intensity array starts from voxels it holds."""
    from gtsam_points_b200 import types as t

    rng = np.random.default_rng(400 + flags)
    vm, orc = g.GaussianVoxelMapGPU(0.5), io.Map(0.5, lru_horizon=2, lru_clear_cycle=3)
    vm.set_lru(2, 3)
    T = np.eye(4)
    T[:3, 3] = [0.25, -0.5, 1.0]
    for b, pts in enumerate(batches(rng, 10, 3000, 3.0)):
        ints = None if b < lead or b % 4 == 3 else awkward_intensities(rng, len(pts))
        cloud = g.PointCloud(pts, np.tile(np.eye(3) * 0.02, (len(pts), 1, 1)), flags=flags, intensities=ints)
        v = None if ints is None else cloud.intensities_gpu()
        if path == "host":
            vm.insert(cloud)  # the PointCloud's host arrays: the caller's intensities
            orc.insert(pts, ints)
        elif path == "cloud":
            vm.insert_cloud(cloud)
            orc.insert(stored_points(g, cloud), v)
        else:
            vm.insert_cloud(cloud, T)
            orc.insert(t.transform_gpu(cloud, T).points, v)
        coords, want = orc.export()
        d = vm.download()
        assert np.array_equal(d["coords"], coords)
        assert same_bits(vm.voxel_intensities(), want)
    assert vm.num_voxels > 0 and np.all(vm.voxel_intensities() >= 0.0)


def test_voxelmap_without_intensities(g):
    rng = np.random.default_rng(450)
    pts = rng.uniform(-2.0, 2.0, (5000, 3))
    cov = np.tile(np.eye(3) * 0.02, (len(pts), 1, 1))
    a, b = g.GaussianVoxelMapGPU(0.5), g.GaussianVoxelMapGPU(0.5)
    a.insert(g.PointCloud(pts, cov))
    b.insert(g.PointCloud(pts, cov, intensities=rng.uniform(1.0, 2.0, len(pts))))
    assert np.all(a.voxel_intensities() == 0.0)
    da, db = a.download(), b.download()
    for k in ("coords", "means", "covs", "n"):
        assert same_bits(da[k], db[k]) if da[k].dtype == np.float64 else np.array_equal(da[k], db[k])
    assert b.info().device_bytes > a.info().device_bytes


@pytest.mark.parametrize("path", ["host", "cloud"])
def test_ivox_slots(g, path):
    rng = np.random.default_rng(500)
    iv, orc = g.iVox(0.5), io.Map(0.5, lru_horizon=3, lru_clear_cycle=2, max_points_in_cell=20, min_dist_in_cell=0.1)
    iv.set_lru(3, 2)
    for pts in batches(rng, 8, 4000, 2.0):
        cloud = g.PointCloud(pts, intensities=awkward_intensities(rng, len(pts)))
        if path == "host":
            iv.insert(pts, intensities=cloud.intensities)
            orc.insert(pts, cloud.intensities)
        else:
            iv.insert_cloud(cloud)
            orc.insert(stored_points(g, cloud), cloud.intensities_gpu())
        coords, counts, p, want = orc.export()
        d = iv.download()
        assert np.array_equal(d["counts"], counts) and same_bits(d["points"], p)
        assert same_bits(iv.voxel_intensities(), want)
    # a frame without intensities into a map with them: rejected before the map changes
    size = iv.size()
    with pytest.raises(g.B2Error) as e:
        iv.insert(pts)
    assert e.value.status == 1 and iv.size() == size
    with pytest.raises(g.B2Error):
        iv.insert_cloud(g.PointCloud(pts))
    iv.clear()  # the next insert decides again
    iv.insert(pts)
    with pytest.raises(g.B2Error) as e:
        iv.voxel_intensities()
    assert e.value.status == 4
    # and after another clear, with intensities again: the slots of the kept layout get them afresh
    iv.clear()
    orc = io.Map(0.5, lru_horizon=3, lru_clear_cycle=2, max_points_in_cell=20, min_dist_in_cell=0.1)
    for pts in batches(rng, 3, 4000, 2.0):
        x = awkward_intensities(rng, len(pts))
        iv.insert(pts, intensities=x)
        orc.insert(pts, x)
    coords, counts, p, want = orc.export()
    assert np.array_equal(iv.download()["counts"], counts)
    assert same_bits(iv.voxel_intensities(), want)


def test_ivox_covariance_estimation_has_none(g):
    rng = np.random.default_rng(550)
    iv = g.iVoxCovarianceEstimation(0.5)
    pts = rng.uniform(-2.0, 2.0, (3000, 3))
    iv.insert_cloud(g.PointCloud(pts, intensities=rng.uniform(0.0, 1.0, len(pts))))
    iv.insert(pts)  # intensities are ignored, so frames with and without them mix
    with pytest.raises(g.B2Error) as e:
        iv.voxel_intensities()
    assert e.value.status == 4


HEADER = b"compact 1\nresolution 0.5\nlru_count 7\nlru_cycle 10\nlru_thresh 10\nvoxel_bytes 56\nnum_voxels %d\n"
RECORD = np.dtype([("coord", "<i4", 3), ("num_points", "<i4"), ("mean", "<f4", 3), ("cov", "<f4", 6), ("intensity", "<f4")])


def test_compact_file_roundtrip(g, tmp_path):
    rng = np.random.default_rng(600)
    V = 5000
    rec = np.zeros(V, dtype=RECORD)
    rec["coord"] = np.stack(np.unravel_index(rng.choice(64**3, V, replace=False), (64, 64, 64)), 1) - 32
    rec["num_points"] = rng.integers(1, 50, V)
    rec["mean"] = rng.normal(0.0, 10.0, (V, 3))
    rec["cov"] = rng.normal(0.0, 1.0, (V, 6))
    rec["intensity"] = rng.normal(0.0, 100.0, V)
    rec["intensity"][::13] = -0.0
    rec["intensity"][::17] = 0.0
    src, out = tmp_path / "ref.bin", tmp_path / "out.bin"
    src.write_bytes(HEADER % V + rec.tobytes())
    vm = g.GaussianVoxelMapGPU.load(src)
    assert same_bits(vm.voxel_intensities(), rec["intensity"].astype(np.float64))
    vm.save_compact(out)
    assert out.read_bytes()[-V * 56 :] == rec.tobytes()
    # a file of zero intensities: a map without them, written back as it was read
    rec["intensity"] = 0.0
    src.write_bytes(HEADER % V + rec.tobytes())
    vm = g.GaussianVoxelMapGPU.load(src)
    vm.save_compact(out)
    assert out.read_bytes()[-V * 56 :] == rec.tobytes()
    # a map built on the device writes (float)v
    pts = rng.uniform(-3.0, 3.0, (8000, 3))
    ints = awkward_intensities(rng, len(pts))
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(g.PointCloud(pts, np.tile(np.eye(3) * 0.02, (len(pts), 1, 1)), intensities=ints))
    vm.save_compact(out)
    got = np.frombuffer(out.read_bytes()[-vm.num_voxels * 56 :], dtype=RECORD)
    assert same_bits(got["intensity"].astype(np.float64), np.float32(vm.voxel_intensities()).astype(np.float64))


def test_from_voxels(g):
    rng = np.random.default_rng(650)
    V = 300
    coords = np.stack([np.arange(V), np.zeros(V), np.zeros(V)], 1).astype(np.int32)
    means = coords * 0.5 + 0.25
    covs = np.tile(np.eye(3) * 0.01, (V, 1, 1))
    ints = rng.normal(0.0, 5.0, V)
    vm = g.GaussianVoxelMapGPU.from_voxels(0.5, coords, means, covs, ints * 0 + 3, intensities=ints)
    assert same_bits(vm.voxel_intensities(), ints)  # stored as given
    x = rng.normal(0.0, 5.0, V)
    vm.insert(g.PointCloud(means, covs, intensities=x))  # one point per voxel: v = (v < x) ? x : v
    assert same_bits(vm.voxel_intensities(), np.where(ints < x, x, ints))


def factor_record(f, values):
    f.linearize(values)
    rec = np.concatenate([np.ravel(v) for v in f._last.values()]).astype(np.float64)
    return rec, f.error(values)


@pytest.mark.parametrize("flags", [0, 1, 2])
def test_factors_ignore_intensities(g, flags):
    rng = np.random.default_rng(700 + flags)
    tgt = rng.uniform(-5.0, 5.0, (20000, 3))
    src = tgt[::3] + rng.normal(0.0, 0.02, (len(tgt[::3]), 3))
    tcov = g.estimate_covariances(tgt, 10)
    scov = g.estimate_covariances(src, 10)
    ti, si = awkward_intensities(rng, len(tgt)), awkward_intensities(rng, len(src))
    delta = np.eye(4)
    delta[:3, 3] = [0.03, -0.02, 0.01]
    values = {1: delta}
    results = []
    for with_ints in (False, True):
        T = g.PointCloud(tgt, tcov, flags=flags, intensities=ti if with_ints else None)
        S = g.PointCloud(src, scov, flags=flags, intensities=si if with_ints else None)
        vm = g.GaussianVoxelMapGPU(0.5)
        vm.insert_cloud(T)
        iv = g.iVox(0.5)
        iv.insert_cloud(T)
        recs = [factor_record(g.IntegratedVGICPFactor(np.eye(4), 1, vm, S), values), factor_record(g.IntegratedGICPFactor(np.eye(4), 1, T, S), values),
                factor_record(g.IntegratedGICPFactor(np.eye(4), 1, iv, S), values)]
        results.append(recs)
    for (ra, ea), (rb, eb) in zip(*results):
        assert same_bits(ra, rb) and same_bits([ea], [eb])
