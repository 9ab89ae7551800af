"""Every factor kind far from the origin (pytest -m gpu): the scenes of far_scenes.py against the CPU oracle (bit-identical
correspondences, the 1e-9 bar on H, b and error) and against the extended-precision formula card (1e-11 on every H and b block,
built from the device's correspondences once they are shown to equal the oracle's).  Single factors take the by-value pose
path, factor sets the descriptor path, and the tolerance-frozen linearize re-uses stored correspondences."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import factor_algebra as fa
import far_scenes as fs
import ivox_np
import normals_ref as nref
import oracle_lib as orc
from gtsam_points_b200 import capi

TOL = 1e-9
TOL_EXT = 1e-11
KINDS = ("vgicp", "vgicp_validated", "gicp", "icp", "plane", "ivox")
IVOX_STRIDE = 3  # the iVox holds every third target point (its restatement is plain Python)


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


@pytest.fixture(scope="module")
def scenes():
    return fs.all_scenes()


class Problem:
    """Device targets of one scene and their references, built once."""

    def __init__(self, g, s):
        self.s = s
        self.vm = g.GaussianVoxelMapGPU(fs.VOXEL)
        self.vm.insert(g.PointCloud(s["tp"], s["tc"]))
        self.ovm = orc.VoxelMap(fs.VOXEL)
        self.ovm.insert(orc.Cloud(s["tp"], s["tc"]))
        self.vex = self.ovm.export()
        self.target = g.PointCloud(s["tp"], s["tc"], normals=s["tn"])
        self.tree = g.KdTree(self.target)
        self.otarget = orc.Cloud(s["tp"], s["tc"])
        self.otarget.set_normals(s["tn"])
        self.otree = orc.KdTree(self.otarget, 4)
        ip, ic = s["tp"][::IVOX_STRIDE], s["tc"][::IVOX_STRIDE]
        self.ivox = g.iVox(fs.IVOX_VOXEL)
        self.ivox.insert(ip, ic)
        self.rivox = ivox_np.IvoxNp(fs.IVOX_VOXEL)
        self.rivox.insert(ip, ic)
        self.iex, self.ifi = self.rivox.export(), self.rivox.flat_index()

    def source(self, g):
        return g.PointCloud(self.s["sp"], self.s["sc"], normals=self.s["sn"])

    def factor(self, g, kind, key=1, src=None):
        src = src or self.source(g)
        eye = np.eye(4)
        if kind.startswith("vgicp"):
            f = g.IntegratedVGICPFactor(eye, key, self.vm, src)
            if kind == "vgicp_validated":
                f.set_enable_surface_validation(True)
            return f
        if kind == "gicp":
            f = g.IntegratedGICPFactor(eye, key, self.target, src, target_tree=self.tree)
        elif kind == "icp":
            f = g.IntegratedICPFactor(eye, key, self.target, src, target_tree=self.tree)
        elif kind == "plane":
            f = g.IntegratedPointToPlaneICPFactor(eye, key, self.target, src, target_tree=self.tree)
        else:
            return g.IntegratedGICPFactor(eye, key, self.ivox, src)
        f.set_max_correspondence_distance(fs.MAX_CORR)
        return f

    def reference(self, kind):
        s = self.s
        if kind == "vgicp":
            return orc.Factor(self.ovm, orc.Cloud(s["sp"], s["sc"]), num_threads=4)
        if kind == "vgicp_validated":
            return nref.ValidatedVGICP(self.ovm, s["sp"], s["sc"], s["sn"], num_threads=4)
        if kind == "ivox":
            return ivox_np.GicpIvoxNp(self.rivox, s["sp"], s["sc"], fs.MAX_CORR**2)
        f = orc.Factor(self.otarget, orc.Cloud(s["sp"], s["sc"]), tree=self.otree, num_threads=4, icp={"gicp": None, "icp": "point", "plane": "plane"}[kind])
        f.set_max_correspondence_distance(fs.MAX_CORR)
        return f

    def ref_correspondences(self, kind, ref):
        return ref.corr if kind == "ivox" else ref.correspondences()

    def records(self, kind, corr):
        """(target means, covariances / normals / None, metric, correspondences as record indices)."""
        s = self.s
        if kind.startswith("vgicp"):
            return self.vex["means"], self.vex["covs"], 0, corr
        if kind == "ivox":
            flat = np.array([self.ifi[int(c)] if c >= 0 else -1 for c in corr], dtype=np.int64)
            return self.iex["points"], self.iex["covs"], 0, flat
        return s["tp"], {"gicp": s["tc"], "icp": None, "plane": s["tn"]}[kind], fa.METRICS[kind], corr

    def extended(self, kind, corr, delta):
        mean_B, cov_B, metric, idx = self.records(kind, corr)
        return fa.extended_linearize(delta, self.s["sp"], self.s["sc"], mean_B, cov_B, idx, metric)


_PROBLEMS = {}


def problem(g, scenes, name):
    if name not in _PROBLEMS:
        if len(_PROBLEMS) >= 2:  # at most two scenes' device targets at a time
            _PROBLEMS.pop(next(iter(_PROBLEMS)))
        _PROBLEMS[name] = Problem(g, scenes[name])
    return _PROBLEMS[name]


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def check(P, kind, got, ref_lin, corr, delta):
    """got: a linearized record; ref_lin: the reference's at the same pose; corr: the device correspondences (== the reference's)."""
    for k in fa.BLOCKS:
        assert rel(got[k], ref_lin[k]) < TOL, (kind, k, rel(got[k], ref_lin[k]))
    assert abs(got["error"] - ref_lin["error"]) <= TOL * abs(ref_lin["error"])
    assert got["num_inliers"] == ref_lin["num_inliers"]
    errs = fa.block_errors(got, P.extended(kind, corr, delta))
    assert max(errs.values()) < TOL_EXT, (kind, errs)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", fs.SCENES)
def test_single_factor_linearize_and_error(g, scenes, name, kind):
    P = problem(g, scenes, name)
    s = P.s
    src = P.source(g)
    assert src.info().point_bytes == (4 if name in ("S0", "S2", "S4") else 8)
    f, ref = P.factor(g, kind, src=src), P.reference(kind)
    d0, d1 = s["deltas"][0], s["deltas"][1]
    f.linearize({1: d0})
    ref_lin = ref.linearize(d0)
    corr = f.correspondences()
    assert np.array_equal(corr, P.ref_correspondences(kind, ref)), "correspondences differ from the reference"
    assert ref_lin["num_inliers"] > len(s["sp"]) // 10
    check(P, kind, f._last, ref_lin, corr, d0)
    e, eref = f.error({1: d1}), ref.error(d1)
    assert abs(e - eref) <= TOL * abs(eref)
    first = {k: np.copy(f._last[k]) for k in f._last}
    f.linearize({1: d0})
    assert all(np.array_equal(first[k], f._last[k]) for k in first), "not bit-reproducible"


@pytest.mark.parametrize("name", fs.SCENES)
def test_factor_set_of_every_kind(g, scenes, name):
    P = problem(g, scenes, name)
    s = P.s
    src = P.source(g)
    factors = [P.factor(g, kind, key=i + 1, src=src) for i, kind in enumerate(KINDS)]
    refs = [P.reference(kind) for kind in KINDS]
    d0, d1 = s["deltas"][0], s["deltas"][2]
    fset = g.NonlinearFactorSetGPU()
    fset.add(factors)
    out = fset.linearize({i + 1: d0 for i in range(len(KINDS))})
    for i, kind in enumerate(KINDS):
        ref_lin = refs[i].linearize(d0)
        corr = factors[i].correspondences()
        assert np.array_equal(corr, P.ref_correspondences(kind, refs[i])), kind
        check(P, kind, capi.unpack_linearized(out[i]), ref_lin, corr, d0)
    errs = fset.error({i + 1: d1 for i in range(len(KINDS))})
    for i, kind in enumerate(KINDS):
        eref = refs[i].error(d1)
        assert abs(errs[i] - eref) <= TOL * abs(eref), kind
    assert np.array_equal(out, fset.linearize({i + 1: d0 for i in range(len(KINDS))})), "not bit-reproducible"


@pytest.mark.parametrize("name", fs.SCENES)
def test_tolerance_frozen_linearize(g, scenes, name):
    """A pure translation of the source frame stays inside the tolerance wherever the frame sits: the second linearize keeps
    the first correspondences and linearizes them at the new pose."""
    P = problem(g, scenes, name)
    s = P.s
    f = P.factor(g, "gicp")
    f.set_correspondence_update_tolerance(0.1, 0.5)
    d0 = s["deltas"][0]
    d2 = d0 @ fs.translation([0.05, -0.03, 0.02])
    f.linearize({1: d0})
    corr0 = f.correspondences()
    ref = P.reference("gicp")
    ref.linearize(d0)
    assert np.array_equal(corr0, ref.correspondences())
    f.linearize({1: d2})
    assert np.array_equal(f.correspondences(), corr0), "the second linearize re-associated"
    ext = P.extended("gicp", corr0, d2)
    errs = fa.block_errors(f._last, ext)
    assert max(errs.values()) < TOL_EXT, errs
    assert fa.error_relerr(f._last["error"], ext["error"]) < TOL


@pytest.mark.parametrize("kind", KINDS)
def test_far_source_h_target_equals_origin_h_target(g, scenes, kind):
    """S1 is S0 with the source frame moved: where the correspondences agree, H_target must too (no oracle involved)."""
    got = {}
    for name in ("S0", "S1"):
        P = problem(g, scenes, name)
        f = P.factor(g, kind)
        f.linearize({1: scenes[name]["deltas"][0]})
        got[name] = (f.correspondences(), np.copy(f._last["H_target"]))
    if not np.array_equal(got["S0"][0], got["S1"][0]):
        pytest.skip("moving the source changed a correspondence")
    assert rel(got["S1"][1], got["S0"][1]) < 1e-10


@pytest.mark.parametrize("name", ("S2", "S3"))
def test_far_target_lookups(g, scenes, name):
    P = problem(g, scenes, name)
    s = P.s
    q = fa.transform(s["deltas"][0], s["sp"])
    assert np.array_equal(P.vm.lookup_voxel_index(q), P.ovm.lookup(q))
    ov = g.overlap_gpu(P.vm, P.source(g), s["deltas"][0])
    assert ov == P.ovm.overlap(orc.Cloud(s["sp"], s["sc"]), s["deltas"][0])
    assert 0.2 < ov <= 1.0
    idx, sqd = P.ivox.knn_search(q[:2000], 1, fs.MAX_CORR**2)
    for i in range(2000):
        ri, rd = P.rivox.knn(q[i], 1, fs.MAX_CORR**2)
        assert idx[i, 0] == ri[0] and sqd[i, 0] == rd[0], i

