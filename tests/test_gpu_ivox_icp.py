"""ICP and point-to-plane ICP on iVox targets (-m gpu) against the restatement (ivox_icp_np.IcpIvoxNp).

* parity in neighbour modes 1, 7, 19 and 27: point-to-point ICP on an iVox filled without covariances, from a source without
  covariances, and point-to-plane ICP on an iVoxCovarianceEstimation (its valid points and normals): correspondences bit-identical,
  H / b / error within 1e-9, error() at the linearization point equal to the linearized error, error() elsewhere on the frozen
  correspondences, a second linearize bit-identical;
* map changes: insert, clear and neighbour mode re-associate even under a freezing correspondence-update tolerance; on an
  iVoxCovarianceEstimation, points that turn valid or change their normal between inserts reach the next linearize through the
  plane view; a point-to-plane factor created on a populated map builds the view;
* preconditions: point-to-plane on a plain iVox, empty maps and handles on different devices fail before any device work;
* every ivox_icp_kernel instantiation (kind x point storage x mode x by-value pose) runs, against the restatement;
* one factor set holding every factor kind equals the one-factor calls, and a one-rank exchange over it equals the set;
* the KITTI-07 frame-to-map loop through the device map and factor follows the restatement's LM pose track iteration by
  iteration for both kinds, so it meets the reference's gates on the frames the restatement meets them (test_ivox_icp_cpu.py
  records the misses).
"""
import os
import re
import subprocess

import numpy as np
import pytest

import ivox_cov_np
import ivox_icp_np
import ivox_np
import mini_lm
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn
from test_ivox_cov_cpu import scene_frames
from test_ivox_cpu import UnaryAdapter, kitti07, odometry, trajectory_frames

B2_ERR_INVALID_ARGUMENT = 1
KIND_ID = {"point": 6, "plane": 7}  # b2_factor_kind: B2_FACTOR_ICP_IVOX, B2_FACTOR_ICP_PLANE_IVOX
ICP_MSG_TARGET = "error: target frame doesn't have required attributes for icp"


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def check_lin(dev_l, ref_l, tol=1e-9):
    for k in ("H_target", "H_source", "H_target_source", "b_target", "b_source"):
        scale = max(1.0, float(np.abs(ref_l[k]).max()))
        assert np.abs(dev_l[k] - ref_l[k]).max() <= tol * scale, k
    assert abs(dev_l["error"] - ref_l["error"]) <= tol * max(1.0, abs(ref_l["error"]))
    assert dev_l["num_inliers"] == ref_l["num_inliers"]


def plain_pair(g, frames, mode=7):
    """A plain iVox and its restatement filled with the frames' points only (no covariances)."""
    dev, ref = g.iVox(1.0), ivox_np.IvoxNp(1.0)
    dev.set_neighbor_voxel_mode(mode)
    ref.mode = mode
    for pts, _ in frames:
        dev.insert(pts)
        ref.insert(pts)
    return dev, ref


def cov_pair(g, num_frames=20, mode=7):
    """An iVoxCovarianceEstimation and its restatement (test_gpu_ivox_cov.py's settings) after `num_frames` scene frames."""
    from test_gpu_ivox_cov import make_pair

    dev, ref = make_pair(g, mode)
    for pts in scene_frames(24)[:num_frames]:
        dev.insert(pts)
        ref.insert(pts)
    return dev, ref


def plain_source(n=3000, stream=99):
    pts, _ = syn.make_cloud(n, stream=stream, scale=1.0)
    return np.asarray(pts, dtype=np.float64)


def cov_source(seed=3, n=1500):
    from test_gpu_ivox_cov import source_frame

    return source_frame(seed, n)[0]


def make_case(g, target, mode):
    """(device map, restatement, source points, point_to_plane) of a parity case."""
    if target == "plain":
        dev, ref = plain_pair(g, trajectory_frames(num_frames=3), mode)
        return dev, ref, plain_source(), False
    dev, ref = cov_pair(g, mode=mode)
    return dev, ref, cov_source(), target == "plane"


CASES = [pytest.param(t, m, id=f"{t}-{m}") for t in ("plain", "plane") for m in (1, 7, 19, 27)] + [pytest.param("cov-point", 7, id="cov-point-7")]


@pytest.mark.gpu
@pytest.mark.parametrize("target,mode", CASES)
def test_factor_matches_restatement(g, target, mode):
    dev, ref, src, plane = make_case(g, target, mode)
    cloud = g.PointCloud(src)  # no covariances: ICP reads none
    assert not cloud.has_covs()
    f = g.IntegratedICPFactor(np.eye(4), 1, dev, cloud, use_point_to_plane=plane)
    rf = ivox_icp_np.IcpIvoxNp(ref, src, point_to_plane=plane)
    delta = syn.random_pose(np.random.default_rng(mode), rot=0.02 if plane else 0.05, trans=0.1 if plane else 0.3)
    f.linearize({1: delta})
    dl = f._last
    rl = rf.linearize(delta)
    assert rl["num_inliers"] > 30
    assert np.array_equal(f.correspondences(), rf.corr)
    check_lin(dl, rl)
    assert abs(f.error({1: delta}) - dl["error"]) <= 1e-12 * max(1.0, abs(dl["error"]))
    delta2 = delta @ syn.se3_exp(np.full(6, 0.01))
    assert abs(f.error({1: delta2}) - rf.error(delta2)) <= 1e-9 * max(1.0, rf.error(delta2))
    f.linearize({1: delta})
    for k in dl:
        assert np.array_equal(np.asarray(dl[k]), np.asarray(f._last[k])), k
    c = f.clone()
    assert c.target is dev and c.use_point_to_plane == plane


@pytest.mark.gpu
def test_point_to_point_map_changes_reassociate(g):
    frames = trajectory_frames(num_frames=6)
    dev, ref = plain_pair(g, frames[:3])
    src = plain_source()
    f = g.IntegratedICPFactor(np.eye(4), 1, dev, g.PointCloud(src))
    f.set_correspondence_update_tolerance(10.0, 100.0)  # would freeze forever if the map change were ignored
    delta = syn.random_pose(np.random.default_rng(2), rot=0.05, trans=0.3)
    f.linearize({1: delta})
    corr0 = f.correspondences()
    for pts, _ in frames[3:]:
        dev.insert(pts)
        ref.insert(pts)
    rf = ivox_icp_np.IcpIvoxNp(ref, src)
    e_ref = rf.linearize(delta)["error"]
    assert abs(f.error({1: delta}) - e_ref) <= 1e-9 * max(1.0, abs(e_ref))  # error() before the next linearize associates
    f.linearize({1: delta})
    assert np.array_equal(f.correspondences(), rf.corr) and not np.array_equal(rf.corr, corr0)
    check_lin(f._last, rf.linearize(delta))
    dev.set_neighbor_voxel_mode(27)
    ref.mode = 27
    f.linearize({1: delta})
    rl = rf.linearize(delta)
    assert np.array_equal(f.correspondences(), rf.corr)
    check_lin(f._last, rl)
    dev.clear()
    ref.clear()
    dev.insert(frames[0][0])
    ref.insert(frames[0][0])
    f.linearize({1: delta})
    rl = rf.linearize(delta)
    assert np.array_equal(f.correspondences(), rf.corr)
    check_lin(f._last, rl)


def changed_targets(before, after, corr):
    """How many of `corr` (voxel << 32 | slot of `after`) name a point that was stored before but then had another validity or
    normal: the changes only the plane view's rewrite can carry to the factor."""
    ex0, fi0 = before
    ex1, fi1 = after
    key0 = {tuple(ex0["points"][o]): o for o in fi0.values()}
    n = 0
    for c in corr:
        if c < 0:
            continue
        o1 = fi1[int(c)]
        o0 = key0.get(tuple(ex1["points"][o1]))
        if o0 is None:
            continue
        v0, v1 = bool(ex0["flags"][o0] & np.uint64(ivox_cov_np.VALID_BIT)), bool(ex1["flags"][o1] & np.uint64(ivox_cov_np.VALID_BIT))
        if v0 != v1 or not np.array_equal(ex0["normals"][o0], ex1["normals"][o1]):
            n += 1
    return n


@pytest.mark.gpu
def test_point_to_plane_sees_map_updates(g):
    """Frames 20 and 21 make points valid and re-estimate normals: the next linearize, under a freezing tolerance, associates with
    and weights by the rewritten plane view."""
    frames = scene_frames(24)
    dev, ref = cov_pair(g, num_frames=18)
    src = cov_source()
    bytes0 = dev.info().device_bytes
    f = g.IntegratedPointToPlaneICPFactor(np.eye(4), 1, dev, g.PointCloud(src))
    assert dev.info().device_bytes > bytes0  # the view of the populated map was built at creation and is counted
    f.set_correspondence_update_tolerance(10.0, 100.0)
    rf = ivox_icp_np.IcpIvoxNp(ref, src, point_to_plane=True)
    delta = syn.random_pose(np.random.default_rng(1), rot=0.02, trans=0.1)
    f.linearize({1: delta})
    check_lin(f._last, rf.linearize(delta))
    before = (ref.export(), ref.flat_index())
    for pts in frames[18:21]:
        dev.insert(pts)
        ref.insert(pts)
    assert set(dev.insert_timings()) == {"base_insert", "estimation", "statistics", "removal"}
    f.linearize({1: delta})
    rl = rf.linearize(delta)
    assert changed_targets(before, (ref.export(), ref.flat_index()), rf.corr) > 0
    assert np.array_equal(f.correspondences(), rf.corr)
    check_lin(f._last, rl)
    # a second point-to-plane factor reuses the view; a clear and re-fill re-associates
    f2 = g.IntegratedPointToPlaneICPFactor(np.eye(4), 1, dev, g.PointCloud(src))
    f2.linearize({1: delta})
    assert np.array_equal(f2.correspondences(), rf.corr)
    dev.clear()
    ref.clear()
    for pts in frames[:4]:
        dev.insert(pts)
        ref.insert(pts)
    f.linearize({1: delta})
    rl = rf.linearize(delta)
    assert np.array_equal(f.correspondences(), rf.corr)
    check_lin(f._last, rl)


@pytest.mark.gpu
def test_preconditions(g):
    src = g.PointCloud(plain_source(100))
    plain, _ = plain_pair(g, trajectory_frames(num_frames=1))
    bytes0 = plain.info().device_bytes
    with pytest.raises(g.B2Error) as e:
        g.IntegratedPointToPlaneICPFactor(np.eye(4), 1, plain, src)
    assert e.value.status == B2_ERR_INVALID_ARGUMENT and ICP_MSG_TARGET in str(e.value)
    assert plain.info().device_bytes == bytes0
    for empty in (g.iVox(1.0), g.iVoxCovarianceEstimation(1.0)):
        for plane in (False, True):
            with pytest.raises(g.B2Error) as e:
                g.IntegratedICPFactor(np.eye(4), 1, empty, src, use_point_to_plane=plane)
            assert e.value.status == B2_ERR_INVALID_ARGUMENT and ICP_MSG_TARGET in str(e.value)
    cov, _ = cov_pair(g, num_frames=3)
    cov_bytes = cov.info().device_bytes
    with pytest.raises(ValueError, match="source frame doesn't have required attributes for icp"):
        g.IntegratedICPFactor(np.eye(4), 1, cov, None, use_point_to_plane=True)
    assert cov.info().device_bytes == cov_bytes  # no plane view for a factor that was never made


@pytest.mark.gpu
def test_handles_on_different_devices(g):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    dev, _ = cov_pair(g, num_frames=3)
    bytes0 = dev.info().device_bytes
    other = g.Context(1)
    src = g.PointCloud(cov_source(n=200), ctx=other)
    for plane in (False, True):
        with pytest.raises(g.B2Error) as e:
            g.IntegratedICPFactor(np.eye(4), 1, dev, src, use_point_to_plane=plane, ctx=g.default_context())
        assert e.value.status == B2_ERR_INVALID_ARGUMENT and "different devices" in str(e.value)
    assert dev.info().device_bytes == bytes0


# ---- every instantiation ---------------------------------------------------------------------------------------------------------


def expected_kernels():
    return {(KIND_ID[k], pt, "float", mode, single) for k in KIND_ID for pt in ("float", "double") for mode in (0, 1) for single in (False, True)}


def test_every_compiled_ivox_icp_kernel_is_covered():
    """The library's ivox_icp_kernel instantiations, read from its device code, are the 16 of kind x point storage x mode x
    by-value pose (CT is a dummy float), and the GPU tests below launch each of them."""
    from gtsam_points_b200 import build

    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    syms = subprocess.run([cuobjdump, "-symbols", build.LIB], capture_output=True, text=True, check=True).stdout
    names = set(re.findall(r"_ZN2b2\d*ws\w*ivox_icp_kernel\w*", syms))
    demangled = subprocess.run(["c++filt"], input="\n".join(sorted(names)), capture_output=True, text=True, check=True).stdout
    compiled = set()
    for m in re.finditer(r"ivox_icp_kernel<(float|double), (float|double), (\d+), (\d+), (true|false)>", demangled):
        compiled.add((int(m.group(3)), m.group(1), m.group(2), int(m.group(4)), m.group(5) == "true"))
    covered = {(KIND_ID[k], {4: "float", 8: "double"}[pb], "float", mode, single) for k, pb in STORAGE_CASES for mode in (0, 1) for single in (False, True)}
    assert len(expected_kernels()) == 16
    assert compiled == expected_kernels() == covered


STORAGE_CASES = [(k, pb) for k in KIND_ID for pb in (4, 8)]


@pytest.fixture(scope="module")
def maps(g):
    plain, rplain = plain_pair(g, trajectory_frames(num_frames=3))
    cov, rcov = cov_pair(g)
    return dict(point=(plain, rplain), plane=(cov, rcov))


def storage_source(kind, pb, n, offset):
    """float32-exact source points (pb 4) or the same offset by 2^-30 (pb 8), around the kind's map."""
    p = (plain_source(6000) if kind == "point" else cov_source(n=1500))[offset : offset + n]
    p = p.astype(np.float32).astype(np.float64)
    return np.ascontiguousarray(p + 2.0**-30 if pb == 8 else p)


def storage_factor(g, maps, kind, pb, n, offset):
    dev, ref = maps[kind]
    p = storage_source(kind, pb, n, offset)
    cloud = g.PointCloud(p)
    assert cloud.info().point_bytes == pb
    return g.IntegratedICPFactor(0, 1, dev, cloud, use_point_to_plane=kind == "plane"), ivox_icp_np.IcpIvoxNp(ref, p, point_to_plane=kind == "plane")


@pytest.mark.gpu
def test_all_storages_in_one_set(g, maps):
    """Device-pose instantiations: one set of the four (kind, point storage) groups, one launch per group and mode."""
    pairs = [storage_factor(g, maps, k, pb, 900 + 37 * i, 13 * i) for i, (k, pb) in enumerate(STORAGE_CASES)]
    fs = g.NonlinearFactorSetGPU()
    fs.add([f for f, _ in pairs])
    rng = np.random.default_rng(21)
    delta = syn.random_pose(rng, 0.02, 0.1)
    out = fs.linearize({0: np.eye(4), 1: delta})
    assert fs.launch_count() == 4
    for (f, rf), rec in zip(pairs, out):
        rl = rf.linearize(delta)
        assert rl["num_inliers"] > 50
        assert np.array_equal(f.correspondences(), rf.corr)
        check_lin(capi.unpack_linearized(rec), rl)
    d2 = delta @ syn.random_pose(rng, 0.01, 0.05)
    errs = fs.error({0: np.eye(4), 1: d2})
    assert fs.launch_count() == 8
    for (f, rf), e in zip(pairs, errs):
        assert abs(e - rf.error(d2)) <= 1e-9 * abs(rf.error(d2))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,pb", STORAGE_CASES, ids=[f"{k}-p{pb}" for k, pb in STORAGE_CASES])
def test_one_factor_by_value(g, maps, kind, pb):
    f, rf = storage_factor(g, maps, kind, pb, 1200, 101)
    fs = g.NonlinearFactorSetGPU()
    fs.add(f)
    rng = np.random.default_rng(7)
    delta = syn.random_pose(rng, 0.02, 0.1)
    out = fs.linearize({0: np.eye(4), 1: delta})
    assert fs.launch_count() == 1
    rl = rf.linearize(delta)
    assert np.array_equal(f.correspondences(), rf.corr)
    check_lin(capi.unpack_linearized(out[0]), rl)
    d2 = delta @ syn.random_pose(rng, 0.01, 0.05)
    e = fs.error({0: np.eye(4), 1: d2})[0]
    assert abs(e - rf.error(d2)) <= 1e-9 * abs(rf.error(d2))


# ---- every factor kind in one set ------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def mixed_scene(g):
    tp, tc = syn.make_cloud(30000, stream=1, scale=0.3)
    sp, sc = syn.make_cloud(16000, stream=2, scale=0.3)
    rng = np.random.default_rng(12)
    tn = rng.normal(size=(len(tp), 3))
    tn /= np.linalg.norm(tn, axis=1, keepdims=True)
    sn = rng.normal(size=(len(sp), 3))
    sn /= np.linalg.norm(sn, axis=1, keepdims=True)
    tgt = g.PointCloud(tp, tc, normals=tn)
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(tgt)
    plain = g.iVox(0.5)
    plain.insert(tp, tc)
    cov = g.iVoxCovarianceEstimation(0.5)
    cov.insert(tp)
    return dict(sp=sp, sc=sc, sn=sn, tgt=tgt, tree=g.KdTree(tgt), vm=vm, plain=plain, cov=cov)


MIXED = ("vgicp", "vgicp-validated", "gicp", "icp", "plane", "gicp-ivox", "icp-ivox", "plane-ivox")


def mixed_factors(g, s):
    out = []
    for i, kind in enumerate(MIXED):
        sl = slice(1500 * i, 1500 * i + 1200 + 97 * i)
        src = g.PointCloud(s["sp"][sl], s["sc"][sl], normals=s["sn"][sl], flags=capi.B2_CLOUD_FORCE_F64)
        if kind.startswith("vgicp"):
            f = g.IntegratedVGICPFactor(0, 1, s["vm"], src)
            if kind == "vgicp-validated":
                f.set_enable_surface_validation(True)
        elif kind == "gicp":
            f = g.IntegratedGICPFactor(0, 1, s["tgt"], src, target_tree=s["tree"])
        elif kind in ("icp", "plane"):
            f = g.IntegratedICPFactor(0, 1, s["tgt"], src, target_tree=s["tree"], use_point_to_plane=kind == "plane")
        elif kind == "gicp-ivox":
            f = g.IntegratedGICPFactor(0, 1, s["plain"], src)
        else:
            f = g.IntegratedICPFactor(0, 1, s["plain"] if kind == "icp-ivox" else s["cov"], src, use_point_to_plane=kind == "plane-ivox")
        out.append(f)
    return out


@pytest.mark.gpu
def test_mixed_factor_set_every_kind(g, mixed_scene):
    factors = mixed_factors(g, mixed_scene)
    rng = np.random.default_rng(4)
    values = {0: np.eye(4), 1: syn.random_pose(rng, 0.02, 0.1)}
    fs = g.NonlinearFactorSetGPU()
    fs.add(factors)
    out = fs.linearize(values)
    evals = {0: np.eye(4), 1: values[1] @ syn.random_pose(rng, 0.005, 0.02)}
    errs = fs.error(evals)
    for kind, f, rec, e in zip(MIXED, factors, out, errs):
        f.linearize(values)
        single = f._last
        assert single["num_inliers"] > 100, kind
        check_lin(capi.unpack_linearized(rec), single, 1e-12)
        assert abs(e - f.error(evals)) <= 1e-12 * max(1.0, abs(e)), kind


@pytest.mark.gpu
def test_one_rank_exchange_over_every_kind(g, mixed_scene):
    from test_gpu_entry_points import FactorSet, seeded_poses
    from test_gpu_exchange_error import ErrorExchange

    keep_a, keep_b = mixed_factors(g, mixed_scene), mixed_factors(g, mixed_scene)
    fs, twin = FactorSet(keep_a), FactorSet(keep_b)
    F = len(MIXED)
    ex = ErrorExchange(g, F)
    deltas, evals = seeded_poses(F, 77)
    ex.linearize(fs, deltas, 0, 1)
    assert np.array_equal(ex.records(1), twin.lin_host(deltas))
    for a, b in zip(fs.correspondences(), twin.correspondences()):
        assert np.array_equal(a, b)
    ex.error(fs, evals, 0, 2)
    assert np.array_equal(ex.errors(2), twin.err_host(evals))


# ---- KITTI-07 ------------------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("plane", [False, True], ids=["point", "plane"])
def test_kitti07_frame_to_map_odometry_device(g, plane):
    """Frames go in without covariances; the source needs none.  Point-to-point on a plain iVox (gates met on frames 1 and 3),
    point-to-plane on an iVoxCovarianceEstimation (frames 1-3; frame 4 misses the rotation gate by 3 %)."""
    pts, covs, poses_gt = kitti07()
    dev = g.iVoxCovarianceEstimation(1.0) if plane else g.iVox(1.0)
    keep = []

    def make_factor(src, scov):
        cloud = g.PointCloud(src)
        f = g.IntegratedICPFactor(np.eye(4), len(keep) + 1, dev, cloud, use_point_to_plane=plane)
        keep.append((cloud, f))
        return f

    est_dev, hist_dev = odometry(pts, covs, poses_gt, make_factor, lambda p, c: dev.insert(p))
    ref = ivox_cov_np.IvoxCovNp(1.0) if plane else ivox_np.IvoxNp(1.0)
    state = {}

    def make_ref(src, scov):
        f = ivox_icp_np.IcpIvoxNp(ref, src, point_to_plane=plane)
        state["key"] = state.get("key", 0) + 1
        return UnaryAdapter(state["key"], f.linearize, f.error)

    est_ref, hist_ref = odometry(pts, covs, poses_gt, make_ref, lambda p, c: ref.insert(p))
    for a, b in zip(hist_dev, hist_ref):  # the LM pose track, iteration by iteration
        assert len(a) == len(b)
        for Ta, Tb in zip(a, b):
            assert np.abs(Ta - Tb).max() < 1e-7
    # the gates, frame by frame: the restatement's misses (test_ivox_icp_cpu.py) are the device's
    for i in range(1, 5):
        dev_err, ref_err = mini_lm.pose_error(est_dev[i], poses_gt[i]), mini_lm.pose_error(est_ref[i], poses_gt[i])
        assert (dev_err[0] < 0.015 and dev_err[1] < 0.15) == (ref_err[0] < 0.015 and ref_err[1] < 0.15), (i, dev_err, ref_err)
    met = [i for i in range(1, 5) if (lambda e: e[0] < 0.015 and e[1] < 0.15)(mini_lm.pose_error(est_dev[i], poses_gt[i]))]
    assert met == ([1, 2, 3] if plane else [1, 3]), met
