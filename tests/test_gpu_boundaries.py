"""The device on inputs built to sit on rounding boundaries (tests/adversarial.py), against the oracle (pytest -m gpu).

* voxel faces at leaf 0.5, 0.3, 0.2 (and points where floor(q * inv_leaf) != floor(q / leaf)): VGICP correspondences in a
  one-factor set (pose by value) and a multi-factor set (device pose), lookup_voxel_index, overlap_gpu, insert, and the
  iVox in neighbour mode 1, where the floor alone picks the candidate voxel;
* bisectors of two targets: kd-tree k-NN (k = 1, 2) and GICP / ICP / point-to-plane correspondences, for float32-exact and
  float64 targets (both leaf-record kinds of the tree);
* the correspondence sphere: a query exactly at the maximum distance is excluded (strict '<'), one ulp inside is kept;
* merge_frames keys at the ends of the 21-bit range.
Indices are compared bit for bit; H / b / error within 1e-9 as in test_gpu_parity.py.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import adversarial as adv
import ivox_np
import oracle_lib as orc
from gtsam_points_b200 import capi
from test_gpu_parity import assert_linearized_close


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


FACES = [(leaf, False) for leaf in adv.LEAVES] + [(0.2, True)]


@pytest.fixture(scope="module", params=FACES, ids=[f"leaf{l}" + ("_div" if d else "") for l, d in FACES])
def face(request):
    leaf, divide = request.param
    s = adv.face_scene(leaf, divide=divide, count=300 if divide else adv.FACE_COUNT, seed=2 if divide else 1)
    ovm = orc.VoxelMap(leaf)
    ovm.insert(orc.Cloud(s["target"], s["target_covs"]))
    s["ovm"] = ovm
    return s


def test_face_vgicp_correspondences(g, face):
    s = face
    vm = g.GaussianVoxelMapGPU(s["leaf"])
    vm.insert(g.PointCloud(s["target"], s["target_covs"]))
    ref = orc.Factor(s["ovm"], orc.Cloud(s["p"], s["covs"])).linearize(s["T"])
    values = {0: np.eye(4), 1: s["T"]}
    # one-factor set: the pose travels by value
    f = g.IntegratedVGICPFactor(0, 1, vm, g.PointCloud(s["p"], s["covs"]))
    f.linearize(values)
    assert np.array_equal(f.correspondences(), s["expected"])
    assert_linearized_close(f._last, ref)
    # multi-factor set: the kernel reads the pose from device memory
    half = len(s["p"]) // 2
    parts = [(s["p"][:half], s["covs"][:half]), (s["p"][half:], s["covs"][half:])]
    fs = g.NonlinearFactorSetGPU()
    factors = [g.IntegratedVGICPFactor(0, 1, vm, g.PointCloud(pp, cc)) for pp, cc in parts]
    fs.add(factors)
    out = fs.linearize(values)
    got = np.concatenate([x.correspondences() for x in factors])
    assert np.array_equal(got, s["expected"])
    for (pp, cc), rec in zip(parts, out):
        assert_linearized_close(capi.unpack_linearized(rec), orc.Factor(s["ovm"], orc.Cloud(pp, cc)).linearize(s["T"]))


def test_face_lookup_overlap_insert(g, face):
    s = face
    vm = g.GaussianVoxelMapGPU(s["leaf"])
    vm.insert(g.PointCloud(s["target"], s["target_covs"]))
    assert np.array_equal(vm.lookup_voxel_index(s["qu"]), s["expected"])
    src = g.PointCloud(s["p"], s["covs"])
    osrc = orc.Cloud(s["p"], s["covs"])
    assert g.overlap_gpu(vm, src, s["T"]) == s["ovm"].overlap(osrc, s["T"]) == 1.0
    # half the voxels: the overlap counts exactly the points whose unfused voxel survived
    keep = s["coords"][: len(s["coords"]) // 2]
    vm2 = g.GaussianVoxelMapGPU(s["leaf"])
    vm2.insert(g.PointCloud((keep + 0.5) * s["leaf"], s["target_covs"][: len(keep)]))
    ovm2 = orc.VoxelMap(s["leaf"])
    ovm2.insert(orc.Cloud((keep + 0.5) * s["leaf"], s["target_covs"][: len(keep)]))
    assert g.overlap_gpu(vm2, src, s["T"]) == ovm2.overlap(osrc, s["T"]) == np.mean(s["expected"] < len(keep))
    # insert of points lying on faces: the device floors them like the CPU map
    vm3 = g.GaussianVoxelMapGPU(s["leaf"])
    vm3.insert(g.PointCloud(s["qu"], s["covs"]))
    ovm3 = orc.VoxelMap(s["leaf"])
    ovm3.insert(orc.Cloud(s["qu"], s["covs"]))
    got, ref = vm3.download(), ovm3.export()
    for k in ("coords", "n", "means", "covs"):
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(ref["coords"][vm3.lookup_voxel_index(s["qu"])], np.floor(s["qu"] * (1.0 / s["leaf"])).astype(np.int32))


def test_face_ivox_mode1(g, face):
    s = face
    dev = g.iVox(s["leaf"])
    dev.set_neighbor_voxel_mode(1)
    ref = ivox_np.IvoxNp(s["leaf"])
    ref.mode = 1
    for m in (dev, ref):
        m.insert(s["target"], s["target_covs"])
    assert np.array_equal(dev.download()["coords"], ref.export()["coords"])
    idx, sqd = dev.knn_search(s["qu"], 1, 1.0)
    want = np.array([ref.knn(q, 1, 1.0)[0][0] for q in s["qu"]])
    assert np.array_equal(idx[:, 0], want)
    assert np.array_equal(idx[:, 0] >> 32, s["expected"])  # one point per voxel: the voxel the unfused value floors to
    f = g.IntegratedGICPFactor(np.eye(4), 1, dev, g.PointCloud(s["p"], s["covs"]))
    rf = ivox_np.GicpIvoxNp(ref, s["p"], s["covs"])
    f.linearize({1: s["T"]})
    rl = rf.linearize(s["T"])
    assert np.array_equal(f.correspondences(), rf.corr)
    assert_linearized_close(f._last, rl)


@pytest.fixture(scope="module", params=[True, False], ids=["f32_targets", "f64_targets"])
def bis(request):
    s = adv.bisector_scene(request.param)
    s["ocl"] = orc.Cloud(s["targets"], s["target_covs"])
    s["ocl"].set_normals(s["normals"])
    s["otree"] = orc.KdTree(s["ocl"])
    return s


def test_bisector_knn(g, bis):
    s = bis
    tree = g.KdTree(s["targets"])
    for k in (1, 2):
        idx, sqd = tree.knn_search(s["qu"], k)
        oidx, osqd, _ = s["otree"].knn(s["qu"], k)
        if k == 1:
            idx, sqd = idx[:, None], sqd[:, None]
        assert np.array_equal(idx, oidx), k
        assert np.array_equal(sqd, osqd), k
    assert np.array_equal(idx[:, 0], s["nearest"])


@pytest.mark.parametrize("kind", ["gicp", "icp", "plane"])
def test_bisector_factors(g, bis, kind):
    s = bis
    src = g.PointCloud(s["p"], s["covs"])
    tgt = g.PointCloud(s["targets"], s["target_covs"], normals=s["normals"])
    tree = g.KdTree(tgt)
    if kind == "gicp":
        f = g.IntegratedGICPFactor(0, 1, tgt, src, target_tree=tree)
    else:
        f = g.IntegratedICPFactor(0, 1, tgt, src, target_tree=tree, use_point_to_plane=kind == "plane")
    of = orc.Factor(s["ocl"], orc.Cloud(s["p"], s["covs"]), tree=s["otree"], icp=None if kind == "gicp" else ("point" if kind == "icp" else "plane"))
    f.linearize({0: np.eye(4), 1: s["T"]})
    ref = of.linearize(s["T"])
    assert np.array_equal(f.correspondences(), s["nearest"])
    assert np.array_equal(f.correspondences(), of.correspondences())
    assert_linearized_close(f._last, ref)


@pytest.mark.parametrize("kind", ["gicp", "icp", "plane"])
def test_sphere_exclusive(g, kind):
    s = adv.sphere_scene()
    tgt = g.PointCloud(s["targets"], s["target_covs"], normals=s["normals"])
    src = g.PointCloud(s["q"], s["covs"])
    assert tgt.info().point_bytes == 4 and src.info().point_bytes == 4
    tree = g.KdTree(tgt)
    idx, _ = tree.knn_search(s["q"], 1, s["radius"] * s["radius"])
    assert np.array_equal(idx, s["expected"])
    if kind == "gicp":
        f = g.IntegratedGICPFactor(0, 1, tgt, src, target_tree=tree)
    else:
        f = g.IntegratedICPFactor(0, 1, tgt, src, target_tree=tree, use_point_to_plane=kind == "plane")
    f.set_max_correspondence_distance(s["radius"])
    ocl = orc.Cloud(s["targets"], s["target_covs"])
    ocl.set_normals(s["normals"])
    of = orc.Factor(ocl, orc.Cloud(s["q"], s["covs"]), tree=orc.KdTree(ocl), icp=None if kind == "gicp" else ("point" if kind == "icp" else "plane"))
    of.set_max_correspondence_distance(s["radius"])
    f.linearize({0: np.eye(4), 1: np.eye(4)})
    ref = of.linearize(np.eye(4))
    assert np.array_equal(of.correspondences(), s["expected"])
    assert np.array_equal(f.correspondences(), s["expected"])
    assert_linearized_close(f._last, ref)


def test_merge_frames_key_range(g):
    """Voxel coordinates -2^20 - 1 and 2^20 fall outside the reference's 21-bit keys; those points are not keyed and fold into
    the voxel of the smallest key.  -2^20 and 2^20 - 1 are the ends of the range."""
    res = 0.5
    rng = np.random.default_rng(17)
    ends = np.array([-(2**20) - 1, -(2**20), 2**20 - 1, 2**20])
    first = []
    for axis in range(3):
        for c in ends:
            p = rng.uniform(-3, 3, 3)
            p[axis] = (c + 0.5) * res
            first.append(p)
    first = np.concatenate([np.array(first), rng.uniform(-5, 5, (200, 3))]) + 2.0**-30  # not float32-exact
    covs0 = adv.spd(len(first), 1)
    second = rng.uniform(-5, 5, (300, 3))
    covs1 = adv.spd(len(second), 2)
    from gtsam_points_b200 import synthetic as syn

    poses = np.stack([np.eye(4), syn.random_pose(rng, 0.1, 1.0)])
    frames = [g.PointCloud(first, covs0, flags=capi.B2_CLOUD_FORCE_F64), g.PointCloud(second, covs1, flags=capi.B2_CLOUD_FORCE_F64)]
    assert frames[0].info().point_bytes == 8
    merged = g.merge_frames_gpu(poses, frames, res)
    xyz, cov = orc.merge_frames(poses, [orc.Cloud(first, covs0), orc.Cloud(second, covs1)], res)
    assert len(merged.points) == len(xyz)
    assert np.array_equal(merged.points, xyz)
    assert np.array_equal(merged.covs, cov.reshape(-1, 3, 3))
    # the in-range ends are voxels of their own (one point each: the mean is the point), except z = -2^20: that voxel has the
    # smallest key, and the six out-of-range points fold into it
    alone = [(xyz == first[i]).all(1).any() for i in range(12)]
    assert alone == [False, True, True, False, False, True, True, False, False, False, True, False]
