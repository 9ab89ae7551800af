"""The adversarial constructors of tests/adversarial.py (no GPU): each yields its floor of sensitive items for the committed
seeds, and the C++ oracle (built with -ffp-contract=off) agrees with the numpy unfused value on every item -- voxel lookup,
VGICP / GICP / ICP correspondences, overlap and kd-tree k-NN.  This pins the expected values the GPU tests compare against."""
import numpy as np
import pytest

import adversarial as adv
import oracle_lib as orc


@pytest.fixture(scope="module", params=adv.LEAVES)
def face(request):
    return adv.face_scene(request.param)


@pytest.fixture(scope="module")
def face_div():
    return adv.face_scene(0.2, divide=True, count=300, seed=2)


@pytest.fixture(scope="module", params=[True, False], ids=["f32_targets", "f64_targets"])
def bis(request):
    return adv.bisector_scene(request.param)


def oracle_face_checks(s):
    ovm = orc.VoxelMap(s["leaf"])
    ovm.insert(orc.Cloud(s["target"], s["target_covs"]))
    assert np.array_equal(ovm.export()["coords"], s["coords"])  # one voxel per target point, in first-touch order
    assert np.array_equal(ovm.lookup(s["qu"]), s["expected"])
    of = orc.Factor(ovm, orc.Cloud(s["p"], s["covs"]))
    assert of.linearize(s["T"])["num_inliers"] == len(s["p"])
    assert np.array_equal(of.correspondences(), s["expected"])
    assert ovm.overlap(orc.Cloud(s["p"], s["covs"]), s["T"]) == 1.0


def test_face_points(face):
    n = adv.sensitive_face_count(face["T"], face["leaf"], face["p"], face["axes"])
    print(f"leaf {face['leaf']}: {n} face points a contraction moves to another voxel")
    assert n == len(face["p"]) == adv.FACE_COUNT
    oracle_face_checks(face)


def test_face_points_division(face_div):
    s = face_div
    n = int(np.count_nonzero(np.floor(s["qu"] * (1.0 / 0.2)) != np.floor(s["qu"] / 0.2)))
    print(f"leaf 0.2: {n} face points where floor(q * inv_leaf) != floor(q / leaf)")
    assert n == len(s["p"]) == 300
    oracle_face_checks(s)


def test_contracted_variants_are_exact():
    """fma() rounds once: a * b + c where the product alone is not representable."""
    a, b, c = 1.0 + 2.0**-30, 1.0 + 2.0**-30, -1.0
    assert adv.fma(a, b, c) == 2.0**-29 + 2.0**-60 and a * b + c == 2.0**-29
    T = adv.pose()
    p = np.array([12.345, -6.789, 3.21])
    v = adv.contracted_variants(T, p)
    assert v.shape == (4, 3) and np.array_equal(v[0], adv.transform(T, p[None])[0])
    assert np.abs(v[1:] - v[0]).max() < 1e-13


def test_bisector_queries(bis):
    s = bis
    print(f"{len(s['p'])} bisector queries a contraction sends to the other target")
    assert len(s["p"]) >= 180
    assert np.all(adv.sq_dist(s["targets"][s["nearest"]], s["qu"]) < adv.sq_dist(s["targets"][s["other"]], s["qu"]))
    ocl = orc.Cloud(s["targets"], s["target_covs"])
    ocl.set_normals(s["normals"])
    tree = orc.KdTree(ocl)
    idx, sqd, found = tree.knn(s["qu"], 1)
    assert np.array_equal(idx[:, 0], s["nearest"])
    assert np.array_equal(sqd[:, 0], adv.sq_dist(s["targets"][s["nearest"]], s["qu"]))
    idx, sqd, found = tree.knn(s["qu"], 2)
    assert np.array_equal(idx, np.stack([s["nearest"], s["other"]], 1))
    for icp in (None, "point", "plane"):
        of = orc.Factor(ocl, orc.Cloud(s["p"], s["covs"]), tree=tree, icp=icp)
        of.linearize(s["T"])
        assert np.array_equal(of.correspondences(), s["nearest"]), icp


def test_sphere_points():
    s = adv.sphere_scene()
    r2 = s["radius"] * s["radius"]
    d = adv.sq_dist(s["targets"], s["q"])
    assert np.array_equal(d, np.where(s["tags"] < 0, np.nextafter(r2, 0.0), np.where(s["tags"] > 0, np.nextafter(r2, 2.0), r2)))
    assert np.all(s["q"].astype(np.float32) == s["q"]) and np.all(s["targets"].astype(np.float32) == s["targets"])
    ocl = orc.Cloud(s["targets"], s["target_covs"])
    ocl.set_normals(s["normals"])
    tree = orc.KdTree(ocl)
    idx, _, found = tree.knn(s["q"], 1, r2)
    assert np.array_equal(np.where(found > 0, idx[:, 0], -1), s["expected"])  # strict '<': on the sphere is outside
    for icp in (None, "point", "plane"):
        of = orc.Factor(ocl, orc.Cloud(s["q"], s["covs"]), tree=tree, icp=icp)
        of.set_max_correspondence_distance(s["radius"])
        of.linearize(np.eye(4))
        assert np.array_equal(of.correspondences(), s["expected"]), icp
