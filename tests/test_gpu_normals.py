"""Normals on the device: the cloud attribute, their estimation, VGICP surface validation and point-to-plane ICP from cloud
normals, against the host restatements in tests/normals_ref.py (which stand on the CPU oracle)."""
import ctypes as C
import os

import numpy as np
import pytest

import normals_ref as nref
import oracle_lib as orc
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


@pytest.fixture(scope="module")
def scene(g):
    tp, tc = syn.make_cloud(30000, stream=1, scale=0.3)
    sp, sc = syn.make_cloud(20011, stream=2, scale=0.3)  # a partial last warp and a partial last tile
    nrm = nref.normals_from_covs(sp, sc)
    nrm[::3] *= -1.0  # back faces
    nrm[::7] = 0.0
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(g.PointCloud(tp, tc))
    ovm = orc.VoxelMap(0.5)
    ovm.insert(orc.Cloud(tp, tc))
    poses = [syn.random_pose(np.random.default_rng(40 + i), 0.03, 0.3) for i in range(8)]
    return dict(tp=tp, tc=tc, sp=sp, sc=sc, nrm=nrm, vm=vm, ovm=ovm, poses=poses)


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


# ---- cloud attribute ----------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("stride", [3, 4])
@pytest.mark.parametrize("exact", [True, False])
def test_cloud_normals_round_trip(g, scene, stride, exact):
    nrm = scene["nrm"].astype(np.float32).astype(np.float64) if exact else scene["nrm"]
    arr = nrm if stride == 3 else np.concatenate([nrm, np.zeros((len(nrm), 1))], 1)
    plain = g.PointCloud(scene["sp"], scene["sc"])
    cloud = g.PointCloud(scene["sp"], scene["sc"], normals=arr)
    info, pinfo = cloud.info(), plain.info()
    assert info.normal_bytes == (4 if exact else 8) and pinfo.normal_bytes == 0
    assert np.array_equal(cloud.normals_gpu(), nrm)
    assert info.device_bytes - pinfo.device_bytes == 3 * ((len(nrm) + 31) // 32 * 32) * info.normal_bytes
    assert g.PointCloud(scene["sp"], scene["sc"], normals=arr, flags=capi.B2_CLOUD_FORCE_F64).info().normal_bytes == 8
    compact = g.PointCloud(scene["sp"], scene["sc"], normals=arr, flags=capi.B2_CLOUD_COMPACT_F32)
    assert compact.info().normal_bytes == 4 and np.array_equal(compact.normals_gpu(), nrm.astype(np.float32).astype(np.float64))
    with pytest.raises(capi.B2Error):
        plain.normals_gpu()


# ---- estimation ---------------------------------------------------------------------------------------------------------


def kitti_points():
    d = np.load(os.path.join(HERE, "golden", "kitti07_frames.npz"))
    return np.ascontiguousarray(d["points0"], dtype=np.float64)


@pytest.mark.parametrize("k", [5, 10, 20])
@pytest.mark.parametrize("data", ["synthetic", "kitti07"])
def test_estimated_normals_match_the_host_restatement(g, scene, data, k):
    pts = scene["sp"][:6001] if data == "synthetic" else kitti_points()[:6001]
    tree = g.KdTree(pts)
    nrm, covs = tree.estimate_normals(k, with_covs=True)
    assert np.array_equal(covs, tree.estimate_covariances(k)), "the fused call's covariances are not bit-identical"
    assert np.array_equal(nrm, g.estimate_normals(pts, k))
    # from-covs form on the same covariances, 3x3 and Matrix4d layout
    c4 = np.zeros((len(pts), 4, 4))
    c4[:, :3, :3] = covs
    assert np.array_equal(g.estimate_normals(pts, covs), nrm) and np.array_equal(g.estimate_normals(np.c_[pts, np.ones(len(pts))], c4), nrm)
    ref_from_covs = nref.normals_from_covs(pts, covs)
    assert np.abs(nrm - ref_from_covs).max() < 1e-9
    # k-NN form against the oracle's covariances; points without a defined normal direction are set aside and counted
    ref, _ = nref.estimate_normals(pts, k)
    w = nref.raw_neighbourhood_eigenvalues(pts, k)
    undefined = (w[:, 1] - w[:, 0]) <= 1e-6 * np.maximum(np.abs(w[:, 1]), 1e-300)
    print(f"{data} k={k}: {int(undefined.sum())} of {len(pts)} points without a defined normal direction excluded")
    assert undefined.mean() < 0.01
    assert np.abs(nrm - ref)[~undefined].max() < 1e-9


def test_estimation_edges(g):
    rng = np.random.default_rng(1)
    few = rng.uniform(-3, 3, (4, 3))
    nrm, covs = g.KdTree(few).estimate_normals(5, with_covs=True)  # n < k: identity covariance and its normal
    assert np.array_equal(covs, np.tile(np.eye(3), (4, 1, 1)))
    assert np.array_equal(nrm, nref.normals_from_covs(few, covs))
    assert g.estimate_normals(np.zeros((0, 3)), 10).shape == (0, 3)
    assert g.estimate_normals(np.zeros((0, 3)), np.zeros((0, 3, 3))).shape == (0, 3)
    pts = rng.uniform(-5, 5, (32 * 9 + 5, 3))  # a partial last warp
    nrm = g.estimate_normals(pts, 10)
    ref, _ = nref.estimate_normals(pts, 10)
    assert np.abs(nrm - ref).max() < 1e-9


# ---- surface validation -------------------------------------------------------------------------------------------------


def check_against_oracle(f, ref, pose, out):
    rl = ref.linearize(pose)
    assert np.array_equal(f.correspondences(), ref.correspondences())
    for key in ("H_target", "H_source", "H_target_source", "b_target", "b_source", "error"):
        assert rel(out[key], rl[key]) < 1e-12, key
    assert out["num_inliers"] == rl["num_inliers"]


def test_validation_off_ignores_the_normals(g, scene):
    a = g.IntegratedVGICPFactor(0, 1, scene["vm"], g.PointCloud(scene["sp"], scene["sc"]))
    b = g.IntegratedVGICPFactor(0, 1, scene["vm"], g.PointCloud(scene["sp"], scene["sc"], normals=scene["nrm"]))
    v = {0: np.eye(4), 1: scene["poses"][0]}
    a.linearize(v), b.linearize(v)
    assert all(np.array_equal(a._last[k], b._last[k]) for k in a._last)
    assert np.array_equal(a.correspondences(), b.correspondences())


@pytest.mark.parametrize("pb", [4, 8])
def test_validated_single_factor(g, scene, pb):
    sp = scene["sp"] if pb == 4 else scene["sp"] + 1e-9
    src = g.PointCloud(sp, scene["sc"], normals=scene["nrm"])
    assert src.info().point_bytes == pb
    f = g.IntegratedVGICPFactor(0, 1, scene["vm"], src)
    f.set_enable_surface_validation(True)
    ref = nref.ValidatedVGICP(scene["ovm"], sp, scene["sc"], scene["nrm"])
    v = {0: np.eye(4), 1: scene["poses"][1]}
    f.linearize(v)
    first = {k: np.copy(f._last[k]) for k in f._last}
    check_against_oracle(f, ref, scene["poses"][1], f._last)
    rejected = nref.surface_rejected(sp, scene["nrm"], scene["poses"][1])
    assert 0.05 < rejected.mean() < 0.95 and (f.correspondences()[rejected] == -1).all()
    assert rel(f.error({0: np.eye(4), 1: scene["poses"][2]}), ref.error(scene["poses"][2])) < 1e-12
    f.linearize(v)
    assert all(np.array_equal(first[k], f._last[k]) for k in first), "not bit-reproducible"
    f.set_enable_surface_validation(False)  # back to the plain instantiation
    f.linearize(v)
    plain = orc.Factor(scene["ovm"], orc.Cloud(sp, scene["sc"]), num_threads=2)
    plain.linearize(scene["poses"][1])
    assert np.array_equal(f.correspondences(), plain.correspondences())


def test_validated_error_before_linearize_unary(g, scene):
    src = g.PointCloud(scene["sp"], scene["sc"], normals=scene["nrm"])
    f = g.IntegratedVGICPFactor(np.eye(4), 1, scene["vm"], src)
    f.set_enable_surface_validation(True)
    ref = nref.ValidatedVGICP(scene["ovm"], scene["sp"], scene["sc"], scene["nrm"])
    e = f.error({1: scene["poses"][3]})  # the first evaluation associates at its own pose
    assert rel(e, ref.error(scene["poses"][3])) < 1e-12
    assert np.array_equal(f.correspondences(), ref.correspondences())


def test_set_of_mixed_validated_and_plain_factors(g, scene):
    n = [20011, 5000, 64, 12345, 1, 9000, 700, 15000]
    factors, refs = [], []
    for i in range(8):
        sp, sc, nr = scene["sp"][: n[i]], scene["sc"][: n[i]], scene["nrm"][: n[i]]
        f = g.IntegratedVGICPFactor(0, i + 1, scene["vm"], g.PointCloud(sp, sc, normals=nr))
        if i % 2 == 0:
            f.set_enable_surface_validation(True)
            refs.append(nref.ValidatedVGICP(scene["ovm"], sp, sc, nr))
        else:
            refs.append(orc.Factor(scene["ovm"], orc.Cloud(sp, sc), num_threads=2))
        factors.append(f)
    fs = g.NonlinearFactorSetGPU()
    fs.add(factors)
    values = {0: np.eye(4), **{i + 1: scene["poses"][i] for i in range(8)}}
    out = fs.linearize(values)
    assert fs.launch_count() == 2, "validated and plain VGICP factors are two launch groups"
    for i, f in enumerate(factors):
        check_against_oracle(f, refs[i], scene["poses"][i], capi.unpack_linearized(out[i]))
    assert np.array_equal(out, fs.linearize(values)), "not bit-reproducible"
    # switching one factor regroups the live set
    factors[1].set_enable_surface_validation(True)
    out2 = fs.linearize(values)
    r = nref.ValidatedVGICP(scene["ovm"], scene["sp"][: n[1]], scene["sc"][: n[1]], scene["nrm"][: n[1]])
    check_against_oracle(factors[1], r, scene["poses"][1], capi.unpack_linearized(out2[1]))
    assert np.array_equal(out2[[0, 2, 3, 4, 5, 6, 7]], out[[0, 2, 3, 4, 5, 6, 7]])


def adversarial_normals(points, pose, rng):
    """Unit-ish normals whose q . m - c |q| sits within a few ulp of zero, on both sides: the normal is built at the threshold
    angle to the transformed ray and one component is then stepped by -3 .. 3 ulp."""
    R = pose[:3, :3]
    q = points @ R.T + pose[:3, 3]
    qh = q / np.linalg.norm(q, axis=1, keepdims=True)
    perp = np.cross(qh, rng.normal(size=qh.shape))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    m = nref.THRESH * qh + np.sqrt(1 - nref.THRESH**2) * perp
    n = m @ R  # R^T m
    steps = rng.integers(-3, 4, len(n))
    ax = np.argmax(np.abs(q @ R), axis=1)  # the component the margin is most sensitive to
    col = n[np.arange(len(n)), ax]
    for _ in range(3):
        col = np.where(steps > 0, np.nextafter(col, np.inf), np.where(steps < 0, np.nextafter(col, -np.inf), col))
        steps = steps - np.sign(steps)
    n[np.arange(len(n)), ax] = col
    return n


def test_adversarial_threshold_scene(g, scene):
    rng = np.random.default_rng(9)
    pose = scene["poses"][4]
    sp, sc = scene["sp"][:8000], scene["sc"][:8000]
    nrm = adversarial_normals(sp, pose, rng)
    margin = nref.validation_margin(sp, nrm, pose)
    rejected = nref.surface_rejected(sp, nrm, pose)
    assert np.abs(margin).max() < 1e-12 and 0.2 < rejected.mean() < 0.8, "the scene must straddle the threshold"
    f = g.IntegratedVGICPFactor(0, 1, scene["vm"], g.PointCloud(sp, sc, normals=nrm))
    f.set_enable_surface_validation(True)
    f.linearize({0: np.eye(4), 1: pose})
    ref = nref.ValidatedVGICP(scene["ovm"], sp, sc, nrm)
    check_against_oracle(f, ref, pose, f._last)


def test_enabling_validation_where_it_cannot_apply(g, scene):
    src = g.PointCloud(scene["sp"], scene["sc"])
    f = g.IntegratedVGICPFactor(0, 1, scene["vm"], src)
    with pytest.raises(capi.B2Error) as e:
        f.set_enable_surface_validation(True)
    assert e.value.status == 4  # B2_ERR_INVALID_STATE: no normals
    tgt = g.PointCloud(scene["tp"], scene["tc"])
    fg = g.IntegratedGICPFactor(0, 1, tgt, g.PointCloud(scene["sp"], scene["sc"], normals=scene["nrm"]))
    assert capi.lib().b2_factor_set_enable_surface_validation(fg.h, 1) == 1  # B2_ERR_INVALID_ARGUMENT
    v = {0: np.eye(4), 1: scene["poses"][0]}
    f.linearize(v), fg.linearize(v)
    plain = orc.Factor(scene["ovm"], orc.Cloud(scene["sp"], scene["sc"]), num_threads=2)
    plain.linearize(scene["poses"][0])
    assert np.array_equal(f.correspondences(), plain.correspondences()) and fg.num_inliers() > 0


# ---- point-to-plane ICP -------------------------------------------------------------------------------------------------


def test_point_to_plane_icp_from_cloud_normals(g, scene):
    """The cloud's normal planes give the same factor, bit for bit, as the host normal array, for float64 normals and for
    float32-exact ones (stored as float32 planes)."""
    rng = np.random.default_rng(12)
    tn64 = rng.normal(size=(len(scene["tp"]), 3))
    tn64 /= np.linalg.norm(tn64, axis=1, keepdims=True)
    src = g.PointCloud(scene["sp"])
    delta = np.ascontiguousarray(scene["poses"][5])
    for normal_bytes, tn in ((8, tn64), (4, tn64.astype(np.float32).astype(np.float64))):
        tgt = g.PointCloud(scene["tp"], normals=tn)
        assert tgt.info().normal_bytes == normal_bytes
        tree = g.KdTree(tgt)
        from_cloud = g.IntegratedPointToPlaneICPFactor(0, 1, tgt, src, target_tree=tree)
        h = C.c_void_p()
        bare = g.PointCloud(scene["tp"])  # the same target without normals: they come as the host array
        capi.check(capi.lib().b2_icp_factor_create(tgt.ctx.h, bare.h, tree.h, src.h, 1, capi.dptr(np.ascontiguousarray(tn)), C.byref(h)))
        buf = np.zeros(capi.B2_LINEARIZED_DOUBLES)
        capi.check(capi.lib().b2_factor_linearize(h, capi.dptr(delta), capi.dptr(buf)))
        from_cloud.linearize({0: np.eye(4), 1: delta})
        host = capi.unpack_linearized(buf)
        assert all(np.array_equal(host[k], from_cloud._last[k]) for k in host), f"{normal_bytes}-byte normals"
        capi.lib().b2_factor_destroy(h)
    with pytest.raises((capi.B2Error, ValueError)):
        g.IntegratedPointToPlaneICPFactor(0, 1, g.PointCloud(scene["tp"]), src, target_tree=tree)
