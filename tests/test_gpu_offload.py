"""GPU memory offloading (-m gpu): offload, reload and touch of device clouds and Gaussian voxel maps, and factors that touch what
they read (b2_factor_set_enable_offloading).

Every result after an offload and a reload -- downloads, the compact map file, lookups, factor records, errors and
correspondences -- must be bit-identical to the result before it, as must a factor launch that reloads what it reads itself.
Entry points that read an offloaded object without touching it fail with B2_ERR_INVALID_STATE and change nothing."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn
from test_gpu_entry_points import FactorSet
from test_gpu_exchange_one_rank import Exchange

B2_ERR_INVALID_STATE = 4
FLAGS = [0, 1, 2, 4]  # default, B2_CLOUD_NO_REORDER, B2_CLOUD_COMPACT_F32, B2_CLOUD_FORCE_F64
KINDS = ("vgicp", "vgicp_validated", "gicp", "icp", "icp_plane", "gicp_ivox", "icp_ivox")


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def unit_normals(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


@pytest.fixture(scope="module")
def scene(g):
    rng = np.random.default_rng(7)
    tp, tc = syn.make_cloud(40000, stream=21, scale=0.3)
    sp, sc = syn.make_cloud(9001, stream=22, scale=0.3)
    return dict(tp=tp, tc=tc, tn=unit_normals(rng, len(tp)), sp=sp, sc=sc, sn=unit_normals(rng, len(sp)), si=rng.uniform(0.0, 100.0, len(sp)) / 3.0)


def changed_of(fn, h):
    ch = C.c_int32(-1)
    capi.check(fn(h, C.byref(ch)))
    return ch.value


def cloud_state(g, c):
    """Every array a cloud stores, as b2_cloud_download / _download_intensities return them."""
    info = c.info()
    n = int(info.num_points)
    p = np.zeros((n, 3))
    cv = np.zeros((n, 3, 3)) if info.cov_bytes else None
    nr = np.zeros((n, 3)) if info.normal_bytes else None
    capi.check(capi.lib().b2_cloud_download(c.h, capi.dptr(p), None if cv is None else capi.dptr(cv), None if nr is None else capi.dptr(nr)))
    out = [p, cv, nr]
    if c.intensity_bytes():
        out.append(c.intensities_gpu())
    return [a for a in out if a is not None]


def same_bits(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(a, b))


# ---- clouds ----------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("normals", [False, True])
@pytest.mark.parametrize("intensities", [False, True])
@pytest.mark.parametrize("n", [0, 3001])
def test_cloud_roundtrip(g, scene, flags, normals, intensities, n):
    L = capi.lib()
    c = g.PointCloud(scene["sp"][:n], scene["sc"][:n], flags=flags, normals=scene["sn"][:n] if normals else None, intensities=scene["si"][:n] if intensities else None)
    before = cloud_state(g, c)
    dev = c.memory_usage_gpu()
    assert dev == c.info().device_bytes > 0 and c.loaded_on_gpu()
    last = c.last_accessed_time()
    for rnd in range(2):  # the second offload reuses the host copy the cloud keeps
        assert changed_of(L.b2_cloud_offload, c.h) == 1
        assert changed_of(L.b2_cloud_offload, c.h) == 0
        r = c.residency()
        assert r.loaded_on_gpu == 0 and r.device_bytes == 0 and c.info().device_bytes == 0 and r.host_bytes == dev
        assert c.info().num_points == n
        assert changed_of(L.b2_cloud_reload, c.h) == 1
        assert changed_of(L.b2_cloud_reload, c.h) == 0
        assert c.loaded_on_gpu() and c.memory_usage_gpu() == dev and c.residency().host_bytes == dev
        assert same_bits(cloud_state(g, c), before)
    assert c.last_accessed_time() == last  # offload and reload are not accesses


def test_cloud_touch_and_clock(g, scene):
    t0 = g.current_access_time()
    c = g.PointCloud(scene["sp"][:100], scene["sc"][:100])
    assert c.last_accessed_time() == t0  # the clock's value at creation
    assert c.touch() is False and c.last_accessed_time() == t0 and g.current_access_time() == t0 + 1
    assert c.offload_gpu() is True and c.touch() is True
    assert c.loaded_on_gpu() and c.last_accessed_time() == t0 + 1 and g.current_access_time() == t0 + 2
    c.offload_gpu()
    del c  # destroy works offloaded


# ---- Gaussian voxel maps -----------------------------------------------------------------------------------------------------


def map_state(g, vm, tmp_path):
    d = vm.download()
    path = tmp_path / "map.bin"
    vm.save_compact(path)
    return [d["coords"], d["means"], d["covs"], d["n"], vm.voxel_intensities(), np.frombuffer(path.read_bytes(), dtype=np.uint8)]


@pytest.mark.parametrize("intensities", [False, True])
@pytest.mark.parametrize("empty", [False, True])
def test_map_roundtrip(g, scene, tmp_path, intensities, empty):
    L = capi.lib()
    vm = g.GaussianVoxelMapGPU(0.5)
    n = 0 if empty else len(scene["tp"])
    vm.insert(g.PointCloud(scene["tp"][:n], scene["tc"][:n], intensities=scene["tn"][:n, 0] * 50.0 if intensities else None))
    probe = np.concatenate([scene["sp"], scene["tp"][:2000]])
    before, look = map_state(g, vm, tmp_path), vm.lookup_voxel_index(probe)
    info = vm.info()
    for _ in range(2):
        assert changed_of(L.b2_voxelmap_offload, vm.h) == 1 and changed_of(L.b2_voxelmap_offload, vm.h) == 0
        r = vm.residency()
        assert r.loaded_on_gpu == 0 and r.device_bytes == 0 and vm.info().device_bytes == 0 and (r.host_bytes > 0) == (not empty)
        assert vm.info().num_voxels == info.num_voxels
        assert changed_of(L.b2_voxelmap_reload, vm.h) == 1 and changed_of(L.b2_voxelmap_reload, vm.h) == 0
        after = vm.info()
        assert after.device_bytes == info.device_bytes and after.num_buckets == info.num_buckets
        assert same_bits(map_state(g, vm, tmp_path), before)
        assert np.array_equal(vm.lookup_voxel_index(probe), look)


def test_map_inserts_with_offload(g, scene):
    """The same inserts (with LRU sweeps) into two maps, one offloaded and reloaded around every insert, give the same map after
    every insert; an insert drops the host copy, so the next offload copies the new contents."""
    rng = np.random.default_rng(3)
    a, b = g.GaussianVoxelMapGPU(0.4), g.GaussianVoxelMapGPU(0.4)
    for m in (a, b):
        m.set_lru(3, 2)
    tp, tc = scene["tp"], scene["tc"]
    for step in range(8):
        sel = rng.choice(len(tp), 6000, replace=False)
        shift = np.array([0.5 * step, 0.0, 0.0])
        frame = g.PointCloud(tp[sel] + shift, tc[sel], intensities=rng.uniform(0, 10, len(sel)) if step % 2 else None)
        if step % 3 == 2:  # insert_cloud reads the frame on the device
            a.insert_cloud(frame)
            b.insert_cloud(frame)
        else:
            a.insert(frame)
            b.insert(frame)
        assert b.offload_gpu() and b.residency().host_bytes > 0
        assert b.reload_gpu()
        da, db = a.download(), b.download()
        for k in ("coords", "means", "covs", "n"):
            assert da[k].tobytes() == db[k].tobytes(), (step, k)
        assert a.voxel_intensities().tobytes() == b.voxel_intensities().tobytes()
        assert a.info().num_buckets == b.info().num_buckets


def test_unbuilt_map(g):
    """A map with nothing inserted has no device map yet: it reports the clock at its construction, moves nothing, and touch()
    makes the device map to record the access on."""
    t0 = g.current_access_time()
    vm = g.GaussianVoxelMapGPU(0.5)
    assert vm.h is None and vm.last_accessed_time() == t0 and vm.loaded_on_gpu() and vm.memory_usage_gpu() == 0
    assert not vm.offload_gpu() and not vm.reload_gpu() and vm.h is None
    assert not vm.touch() and vm.h is not None
    assert vm.last_accessed_time() == t0 and g.current_access_time() == t0 + 1


def test_overlap_touches_targets_then_source(g, scene):
    vm1, vm2 = g.GaussianVoxelMapGPU(0.5), g.GaussianVoxelMapGPU(0.5)
    vm1.insert(g.PointCloud(scene["tp"][:20000], scene["tc"][:20000]))
    vm2.insert(g.PointCloud(scene["tp"][20000:], scene["tc"][20000:]))
    src = g.PointCloud(scene["sp"], scene["sc"])
    Ts = [np.eye(4), np.eye(4)]
    want = g.overlap_gpu([vm1, vm2], src, Ts)
    for o in (vm1, vm2, src):
        o.offload_gpu()
    t0 = g.current_access_time()
    assert g.overlap_gpu([vm1, vm2], src, Ts) == want
    assert all(o.loaded_on_gpu() for o in (vm1, vm2, src))
    assert (vm1.last_accessed_time(), vm2.last_accessed_time(), src.last_accessed_time()) == (t0, t0 + 1, t0 + 2)


# ---- factors ---------------------------------------------------------------------------------------------------------------


class Objects:
    """Fresh clouds and maps for one factor of `kind`; `offloadable` lists what the factor reads that can be offloaded, and
    `target` the kd-tree factors' target cloud, which they do not read at launch."""

    def __init__(self, g, scene, kind, n=9001, flags=0):
        sn = scene["sn"][:n] if kind == "vgicp_validated" else None
        self.src = g.PointCloud(scene["sp"][:n], scene["sc"][:n], flags=flags, normals=sn, intensities=scene["si"][:n])
        self.target = None
        if kind.startswith("vgicp"):
            self.map = g.GaussianVoxelMapGPU(0.5)
            self.map.insert(g.PointCloud(scene["tp"], scene["tc"]))
            self.offloadable = [self.map, self.src]
        elif kind.endswith("ivox"):
            self.ivox = g.iVox(0.5)
            self.ivox.insert(scene["tp"], scene["tc"])
            self.offloadable = [self.src]
        else:
            self.target = g.PointCloud(scene["tp"], scene["tc"], normals=scene["tn"])
            self.tree = g.KdTree(self.target)
            self.offloadable = [self.src]

    def factor(self, g, kind):
        if kind.startswith("vgicp"):
            f = g.IntegratedVGICPFactor(0, 1, self.map, self.src)
            if kind == "vgicp_validated":
                f.set_enable_surface_validation(True)
            return f
        if kind == "gicp":
            return g.IntegratedGICPFactor(0, 1, self.target, self.src, target_tree=self.tree)
        if kind in ("icp", "icp_plane"):
            return g.IntegratedICPFactor(0, 1, self.target, self.src, target_tree=self.tree, use_point_to_plane=kind == "icp_plane")
        if kind == "gicp_ivox":
            return g.IntegratedGICPFactor(0, 1, self.ivox, self.src)
        return g.IntegratedICPFactor(0, 1, self.ivox, self.src)

    def everything(self):
        return self.offloadable + ([self.target] if self.target is not None else [])


def lin(f, delta):
    buf = np.zeros(capi.B2_LINEARIZED_DOUBLES)
    capi.check(capi.lib().b2_factor_linearize(f.h, capi.dptr(np.ascontiguousarray(delta)), capi.dptr(buf)))
    return buf


def err(f, delta):
    e = np.zeros(1)
    capi.check(capi.lib().b2_factor_error(f.h, capi.dptr(np.ascontiguousarray(delta)), capi.dptr(e)))
    return e


def poses(seed, F):
    rng = np.random.default_rng(seed)
    return np.stack([syn.random_pose(rng, 0.03, 0.2) for _ in range(F)])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("flags", [0, 2])
def test_single_factor(g, scene, kind, flags):
    objs = Objects(g, scene, kind, flags=flags)
    f = objs.factor(g, kind)
    d0, d1 = poses(5, 2)
    r0, e0, c0 = lin(f, d0), err(f, d1), f.correspondences()
    assert r0[121] > 0  # inliers
    # error() after offload and reload, with no linearize in between, uses the stored correspondences
    for o in objs.everything():
        assert o.offload_gpu()
    for o in objs.everything():
        assert o.reload_gpu()
    assert err(f, d1).tobytes() == e0.tobytes()
    assert lin(f, d0).tobytes() == r0.tobytes() and np.array_equal(f.correspondences(), c0)
    # offloaded at the call with offloading on: the launch reloads what it reads, and only that
    f.set_enable_offloading(True)
    for o in objs.everything():
        o.offload_gpu()
    assert err(f, d1).tobytes() == e0.tobytes()
    assert all(o.loaded_on_gpu() for o in objs.offloadable)
    for o in objs.offloadable:
        o.offload_gpu()
    assert lin(f, d0).tobytes() == r0.tobytes()
    assert all(o.loaded_on_gpu() for o in objs.offloadable)
    if objs.target is not None:  # a kd-tree factor reads its gathered target records, not its target cloud
        assert not objs.target.loaded_on_gpu()
    assert np.array_equal(f.correspondences(), c0)
    # clone() carries the setting over (making a factor reads its objects: they are resident then)
    for o in objs.everything():
        o.reload_gpu()
    h = f.clone()
    for o in objs.offloadable:
        o.offload_gpu()
    assert lin(h, d0).tobytes() == r0.tobytes()


@pytest.mark.parametrize("path", ["host", "issue", "device"])
def test_mixed_set(g, scene, path):
    """A set where some members' objects are offloaded and some are not, with one map shared by several VGICP factors: records,
    errors and correspondences equal the all-resident set's, and the touches follow the set order."""
    shared = Objects(g, scene, "vgicp", n=7001)
    others = [Objects(g, scene, k, n=n) for k, n in (("gicp", 5000), ("vgicp_validated", 6001), ("icp_plane", 3000), ("gicp_ivox", 4097))]
    src2 = g.PointCloud(scene["sp"][:8000], scene["sc"][:8000])
    factors = [shared.factor(g, "vgicp"), others[0].factor(g, "gicp"), g.IntegratedVGICPFactor(0, 1, shared.map, src2), others[1].factor(g, "vgicp_validated"),
               others[2].factor(g, "icp_plane"), others[3].factor(g, "gicp_ivox")]
    fs = FactorSet(factors)
    run = {"host": fs.lin_host, "issue": fs.lin_issue, "device": fs.lin_device}[path]
    D, E = poses(11, len(factors)), poses(12, len(factors))
    r0 = run(D)
    e0, c0 = fs.err_host(E), fs.correspondences()
    for f in factors:
        f.set_enable_offloading(True)
    for o in (shared.map, src2, others[1].map, others[1].src, others[2].target, others[3].src):  # the rest stays resident
        o.offload_gpu()
    t0 = g.current_access_time()
    r1 = run(D)
    assert r1.tobytes() == r0.tobytes()
    # touch order: (map, source) of each member in set order; the shared map keeps the later touch
    objs = [(shared.map, shared.src), (None, others[0].src), (shared.map, src2), (others[1].map, others[1].src), (None, others[2].src), (None, others[3].src)]
    t, want = t0, {}
    for vm, src in objs:
        if vm is not None:
            want[id(vm)] = (vm, t)
            t += 1
        want[id(src)] = (src, t)
        t += 1
    assert g.current_access_time() == t
    for o, w in want.values():
        assert o.last_accessed_time() == w and o.loaded_on_gpu()
    assert not others[2].target.loaded_on_gpu()
    for o in (shared.map, others[0].src):
        o.offload_gpu()
    assert fs.err_host(E).tobytes() == e0.tobytes()
    assert all(np.array_equal(a, b) for a, b in zip(fs.correspondences(), c0))


def test_exchange_one_rank(g, scene):
    objs = [Objects(g, scene, k, n=n) for k, n in (("vgicp", 6001), ("gicp", 4000), ("icp_ivox", 3001))]
    factors = [o.factor(g, k) for o, k in zip(objs, ("vgicp", "gicp", "icp_ivox"))]
    fs = FactorSet(factors)
    D = poses(21, len(factors))
    r0 = fs.lin_host(D)
    ex = Exchange(g, len(factors))
    for f in factors:
        f.set_enable_offloading(True)
    for o in objs:
        for x in o.everything():
            x.offload_gpu()
    out = ex.linearize_host(fs, D, 0, 1)
    assert out.tobytes() == r0.tobytes()
    assert all(x.loaded_on_gpu() for o in objs for x in o.offloadable)


@pytest.mark.parametrize("single", [False, True])
def test_offloading_off_rejects(g, scene, single):
    objs = Objects(g, scene, "vgicp")
    f = objs.factor(g, "vgicp")
    other = Objects(g, scene, "gicp").factor(g, "gicp")
    D = poses(31, 2)
    fs = FactorSet([other, f])
    r0 = fs.lin_host(D)
    for o in objs.offloadable:
        o.offload_gpu()
        L = capi.lib()
        n0 = fs.launches()
        lasts = [x.last_accessed_time() for x in objs.offloadable]
        buf = np.zeros((2, capi.B2_LINEARIZED_DOUBLES))
        st = L.b2_factor_linearize(f.h, capi.dptr(D[1]), capi.dptr(buf[1])) if single else L.b2_factor_set_linearize(fs.h, capi.dptr(D), capi.dptr(buf))
        assert st == B2_ERR_INVALID_STATE
        msg = L.b2_last_error().decode()
        assert "member" in msg and ("map" if o is objs.map else "source cloud") in msg, msg
        assert fs.launches() == n0 and not o.loaded_on_gpu()
        assert [x.last_accessed_time() for x in objs.offloadable] == lasts
        o.reload_gpu()
    assert fs.lin_host(D).tobytes() == r0.tobytes()


def test_offloading_off_is_checked_before_any_touch(g, scene):
    """A member with offloading off that reads a map another member (offloading on, earlier in the set) would reload: the call
    fails as the header says, before anything is touched."""
    objs = Objects(g, scene, "vgicp")
    on, off = objs.factor(g, "vgicp"), g.IntegratedVGICPFactor(0, 1, objs.map, g.PointCloud(scene["sp"][:5000], scene["sc"][:5000]))
    on.set_enable_offloading(True)
    fs = FactorSet([on, off])
    D = poses(41, 2)
    r0 = fs.lin_host(D)
    objs.map.offload_gpu()
    n0, last = fs.launches(), objs.map.last_accessed_time()
    out = np.zeros((2, capi.B2_LINEARIZED_DOUBLES))
    assert capi.lib().b2_factor_set_linearize(fs.h, capi.dptr(D), capi.dptr(out)) == B2_ERR_INVALID_STATE
    assert "member 1" in capi.lib().b2_last_error().decode()
    assert fs.launches() == n0 and not objs.map.loaded_on_gpu() and objs.map.last_accessed_time() == last
    off.set_enable_offloading(True)
    assert fs.lin_host(D).tobytes() == r0.tobytes()


# ---- the rejection table ---------------------------------------------------------------------------------------------------


def rejection_calls(g, scene, tmp_path):
    """(name, call, object it must reject) for every entry point that reads a cloud or a map.  Each call returns a status."""
    L = capi.lib()
    ctx = g.default_context()
    n = 2000
    cloud = g.PointCloud(scene["sp"][:n], scene["sc"][:n], normals=scene["sn"][:n], intensities=scene["si"][:n])
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(g.PointCloud(scene["tp"][:n], scene["tc"][:n]))
    resident = g.PointCloud(scene["tp"][:n], scene["tc"][:n], normals=scene["tn"][:n])
    tree = g.KdTree(resident)
    ivox = g.iVox(0.5)
    ivox.insert(scene["tp"][:n], scene["tc"][:n])
    occ = C.c_void_p()
    capi.check(L.b2_occgrid_create(ctx.h, 0.5, C.byref(occ)))
    out = C.c_void_p()
    I = np.eye(4).ravel().copy()
    P, CV, NR, IN = np.zeros((n, 3)), np.zeros((n, 9)), np.zeros((n, 3)), np.zeros(n)
    idx = np.arange(10, dtype=np.int64)
    lp = idx.ctypes.data_as(C.POINTER(C.c_int64))
    ev = np.array([1e-3, 1.0, 1.0])
    seed = np.ascontiguousarray(scene["sp"][0])
    ip = np.zeros(n, dtype=np.int32).ctypes.data_as(C.POINTER(C.c_int32))
    counts, flags8 = np.zeros(1, dtype=np.uint64), np.zeros(n, dtype=np.uint8)
    frames = (C.c_void_p * 1)(cloud.h.value)
    msz = C.c_size_t()
    prm = capi.MinCutParamsC(0.25, 0.2, 0.1, 0.5, 0.5, 0.5, 10, 0)
    res = capi.MinCutResultC()
    rp, gp, rr = capi.RansacParams(), capi.GncParams(), capi.RegistrationResultC()
    rg_out = C.c_void_p()
    f_out = C.c_void_p()
    corr = np.zeros(n, dtype=np.int64)
    vgicp = C.c_void_p()
    capi.check(L.b2_vgicp_factor_create(ctx.h, vm.h, cloud.h, C.byref(vgicp)))
    path = str(tmp_path / "m.bin").encode()
    c = cloud.h
    calls = [
        ("b2_cloud_download", lambda: L.b2_cloud_download(c, capi.dptr(P), capi.dptr(CV), capi.dptr(NR)), cloud),
        ("b2_cloud_download_normals", lambda: L.b2_cloud_download_normals(c, capi.dptr(NR)), cloud),
        ("b2_cloud_download_intensities", lambda: L.b2_cloud_download_intensities(c, capi.dptr(IN)), cloud),
        ("b2_cloud_create_with_added_intensities", lambda: L.b2_cloud_create_with_added_intensities(c, capi.dptr(IN), 0, C.byref(out)), cloud),
        ("b2_cloud_create_transformed", lambda: L.b2_cloud_create_transformed(c, capi.dptr(I), 0, C.byref(out)), cloud),
        ("b2_cloud_create_estimated", lambda: L.b2_cloud_create_estimated(c, None, 10, capi.dptr(ev), 0, 0, C.byref(out)), cloud),
        ("b2_cloud_create_sampled", lambda: L.b2_cloud_create_sampled(c, lp, len(idx), 0, C.byref(out)), cloud),
        ("b2_cloud_create_random_sampled", lambda: L.b2_cloud_create_random_sampled(c, 0.5, 1, 0, None, C.byref(out)), cloud),
        ("b2_cloud_create_randomgrid", lambda: L.b2_cloud_create_randomgrid(c, 0.5, 0.5, 1, 0, None, C.byref(out)), cloud),
        ("b2_cloud_create_inliers", lambda: L.b2_cloud_create_inliers(c, None, 10, 1.0, 0, None, None, None, C.byref(out)), cloud),
        ("b2_merge_frames", lambda: L.b2_merge_frames(ctx.h, capi.dptr(I), frames, 1, 0.5, capi.dptr(P), capi.dptr(CV), C.byref(msz)), cloud),
        ("b2_merge_frames_to_cloud", lambda: L.b2_merge_frames_to_cloud(ctx.h, capi.dptr(I), frames, 1, 0.5, 0, C.byref(out)), cloud),
        ("b2_kdtree_create_from_cloud", lambda: L.b2_kdtree_create_from_cloud(c, C.byref(out)), cloud),
        ("b2_features_create_fpfh", lambda: L.b2_features_create_fpfh(c, None, 0.5, 30, C.byref(out)), cloud),
        ("b2_features_create_fpfh_at", lambda: L.b2_features_create_fpfh_at(c, None, 0.5, 30, lp, len(idx), C.byref(out)), cloud),
        ("b2_features_create_pfh", lambda: L.b2_features_create_pfh(c, None, 0.5, 30, lp, len(idx), C.byref(out)), cloud),
        ("b2_estimate_pose_ransac(target)", lambda: L.b2_estimate_pose_ransac(c, resident.h, None, None, C.byref(rp), C.byref(rr), None), cloud),
        ("b2_estimate_pose_ransac(source)", lambda: L.b2_estimate_pose_ransac(resident.h, c, None, None, C.byref(rp), C.byref(rr), None), cloud),
        ("b2_estimate_pose_gnc", lambda: L.b2_estimate_pose_gnc(resident.h, c, None, None, C.byref(gp), C.byref(rr), None, 0, None), cloud),
        ("b2_region_growing_create", lambda: L.b2_region_growing_create(c, None, capi.dptr(seed), 0.5, 0.5, 0.0, 100, C.byref(rg_out)), cloud),
        ("b2_min_cut", lambda: L.b2_min_cut(c, None, 0, None, C.byref(prm), C.byref(res), None, None), cloud),
        ("b2_occgrid_insert", lambda: L.b2_occgrid_insert(occ, c, capi.dptr(I)), cloud),
        ("b2_occgrid_overlap", lambda: L.b2_occgrid_overlap(occ, c, capi.dptr(I), 1, counts.ctypes.data_as(C.POINTER(C.c_uint64)), flags8.ctypes.data_as(C.POINTER(C.c_uint8))), cloud),
        ("b2_occgrid_free_rays", lambda: L.b2_occgrid_free_rays(occ, c, capi.dptr(I)), cloud),
        ("b2_voxelmap_insert_cloud(frame)", lambda: L.b2_voxelmap_insert_cloud(vm.h, c, None), cloud),
        ("b2_ivox_insert_cloud", lambda: L.b2_ivox_insert_cloud(ivox.h, c, None), cloud),
        ("b2_vgicp_factor_create(source)", lambda: L.b2_vgicp_factor_create(ctx.h, vm.h, c, C.byref(f_out)), cloud),
        ("b2_gicp_factor_create(source)", lambda: L.b2_gicp_factor_create(ctx.h, resident.h, tree.h, c, C.byref(f_out)), cloud),
        ("b2_icp_factor_create(source)", lambda: L.b2_icp_factor_create(ctx.h, resident.h, tree.h, c, 0, None, C.byref(f_out)), cloud),
        ("b2_gicp_ivox_factor_create", lambda: L.b2_gicp_ivox_factor_create(ctx.h, ivox.h, c, C.byref(f_out)), cloud),
        ("b2_icp_ivox_factor_create", lambda: L.b2_icp_ivox_factor_create(ctx.h, ivox.h, c, 0, C.byref(f_out)), cloud),
        ("b2_factor_correspondences", lambda: L.b2_factor_correspondences(vgicp, corr.ctypes.data_as(C.POINTER(C.c_int64))), cloud),
        ("b2_gicp_factor_create(target)", lambda: L.b2_gicp_factor_create(ctx.h, resident.h, tree.h, c, C.byref(f_out)), resident),
        ("b2_icp_factor_create(target)", lambda: L.b2_icp_factor_create(ctx.h, resident.h, tree.h, c, 1, None, C.byref(f_out)), resident),
        ("b2_voxelmap_insert", lambda: L.b2_voxelmap_insert(vm.h, capi.dptr(P), 3, capi.dptr(CV), 9, n), vm),
        ("b2_voxelmap_insert_with_intensities", lambda: L.b2_voxelmap_insert_with_intensities(vm.h, capi.dptr(P), 3, capi.dptr(CV), 9, capi.dptr(IN), n), vm),
        ("b2_voxelmap_insert_cloud(map)", lambda: L.b2_voxelmap_insert_cloud(vm.h, resident.h, None), vm),
        ("b2_voxelmap_download", lambda: L.b2_voxelmap_download(vm.h, ip, capi.dptr(P), capi.dptr(CV), ip), vm),
        ("b2_voxelmap_download_intensities", lambda: L.b2_voxelmap_download_intensities(vm.h, capi.dptr(np.zeros(vm.num_voxels))), vm),
        ("b2_voxelmap_save_compact", lambda: L.b2_voxelmap_save_compact(vm.h, path), vm),
        ("b2_voxelmap_lookup", lambda: L.b2_voxelmap_lookup(vm.h, capi.dptr(P), 3, n, ip), vm),
        ("b2_vgicp_factor_create(map)", lambda: L.b2_vgicp_factor_create(ctx.h, vm.h, resident.h, C.byref(f_out)), vm),
    ]
    made = (out, f_out, rg_out)
    keep = (cloud, vm, resident, tree, ivox)
    return calls, made, keep, lambda: (L.b2_occgrid_destroy(occ), L.b2_factor_destroy(vgicp))


def test_rejection_table(g, scene, tmp_path):
    """Each entry point returns B2_ERR_INVALID_STATE on an offloaded handle, creates nothing, touches nothing and leaves the object
    offloaded; a map keeps its voxels."""
    calls, made, keep, cleanup = rejection_calls(g, scene, tmp_path)
    L = capi.lib()
    try:
        assert len(calls) >= 40
        for name, call, obj in calls:
            before = obj.info().num_voxels if isinstance(obj, g.GaussianVoxelMapGPU) else None
            assert obj.offload_gpu(), name
            last = obj.last_accessed_time()
            st = call()
            assert st == B2_ERR_INVALID_STATE, (name, st, L.b2_last_error().decode())
            assert "offloaded" in L.b2_last_error().decode(), name
            assert not obj.loaded_on_gpu() and obj.last_accessed_time() == last, name
            assert not any(h.value for h in made), name
            assert obj.reload_gpu(), name
            if before is not None:
                assert obj.info().num_voxels == before, name
    finally:
        cleanup()
