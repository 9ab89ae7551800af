"""Every factor_kernel instantiation against the float64 references.

b2_factors.cu instantiates the factor kernel per (kind, source point type PT, source covariance type CT, mode, by-value pose):
VGICP, GICP and iVox-GICP for the 4 (PT, CT) storages x {linearize, error} x {device pose, by-value pose}, and ICP /
point-to-plane ICP for the 2 PT storages x {linearize, error} with device poses only (their CT is a dummy): 56 kernels.  The
storages used here are all lossless -- float32-exact or not points, float32-rounded or not covariances -- so every kernel is
held to the 1e-9 bar with bit-identical correspondences:

* one set holding all 16 (kind, PT, CT) groups: one launch per group, every factor against its oracle, then again with a
  correspondence-update tolerance that freezes the GICP / ICP / iVox factors on the second call;
* one-factor sets of the 12 kinds with a by-value instantiation, through the host-pose path;
* the 4 GICP target storages (gather_leaf_records_kernel<PT, CT>) and the 2 ICP ones;
* COMPACT_F32 storage of every kind with source covariances, against the oracle fed the float32-rounded inputs.
A CPU test reads the kernels compiled into the library and checks that the parametrisation covers every one of them.
"""
import os
import re
import subprocess

import numpy as np
import pytest

import ivox_np
import np_ref
import oracle_lib as orc
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn
from test_gpu_parity import assert_linearized_close

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE_COV_KINDS = ("vgicp", "gicp", "ivox")
ICP_KINDS = ("icp", "plane")
KIND_ID = {"vgicp": 0, "gicp": 1, "icp": 2, "plane": 3, "ivox": 4}  # b2_factor_kind
STORAGES = [(4, 4), (4, 8), (8, 4), (8, 8)]  # (point bytes, covariance bytes)
TYPE = {4: "float", 8: "double"}
MODES = (0, 1)  # linearize, error


def expected_kernels():
    """(kind, PT, CT, mode, by_value) of every instantiation, from KernelConfig's rules: kinds with source covariances have all
    four (PT, CT) and a by-value form; ICP kinds have CT = float (a dummy) and no by-value form."""
    out = set()
    for kind in SOURCE_COV_KINDS:
        for pb, cb in STORAGES:
            for mode in MODES:
                for single in (False, True):
                    out.add((KIND_ID[kind], TYPE[pb], TYPE[cb], mode, single))
    for kind in ICP_KINDS:
        for pb in (4, 8):
            for mode in MODES:
                out.add((KIND_ID[kind], TYPE[pb], "float", mode, False))
    return out


def covered_kernels():
    """The instantiations the GPU tests of this module launch: the all-groups set (device pose) and the one-factor sets."""
    out = set()
    for kind, pb, cb in SET_GROUPS:
        for mode in MODES:
            out.add((KIND_ID[kind], TYPE[pb], TYPE[cb] if kind in SOURCE_COV_KINDS else "float", mode, False))
    for kind, (pb, cb) in SINGLES:
        for mode in MODES:
            out.add((KIND_ID[kind], TYPE[pb], TYPE[cb], mode, True))
    return out


SET_GROUPS = [(k, pb, cb) for k in SOURCE_COV_KINDS for pb, cb in STORAGES] + [(k, pb, 0) for k in ICP_KINDS for pb in (4, 8)]
SINGLES = [(k, st) for k in SOURCE_COV_KINDS for st in STORAGES]


def test_parametrisation_covers_every_compiled_kernel():
    """The library's factor kernels, read from its device code, are exactly the 56 the rules give, and this module covers
    them all; a new storage type or kind fails here until it is tested."""
    from gtsam_points_b200 import build

    lib = build.LIB
    assert os.path.exists(lib)
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    syms = subprocess.run([cuobjdump, "-symbols", lib], capture_output=True, text=True, check=True).stdout
    names = set(re.findall(r"_ZN2b2\d*ws\w*factor_kernel\w*", syms))
    demangled = subprocess.run(["c++filt"], input="\n".join(sorted(names)), capture_output=True, text=True, check=True).stdout
    compiled = set()
    for m in re.finditer(r"factor_kernel<(float|double), (float|double), (\d+), (\d+), (true|false)>", demangled):
        compiled.add((int(m.group(3)), m.group(1), m.group(2), int(m.group(4)), m.group(5) == "true"))
    assert len(expected_kernels()) == 56
    assert compiled == expected_kernels()
    assert covered_kernels() == expected_kernels()
    assert len(SET_GROUPS) == 16 and len(SINGLES) == 12


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


@pytest.fixture(scope="module")
def scene(g):
    tp, tc = syn.make_cloud(30000, stream=1, scale=0.3)
    sp, sc = syn.make_cloud(20000, stream=2, scale=0.3)
    rng = np.random.default_rng(12)
    normals = rng.normal(size=(len(tp), 3))
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    tgt = g.PointCloud(tp, tc, normals=normals)
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(tgt)
    ovm = orc.VoxelMap(0.5)
    ovm.insert(orc.Cloud(tp, tc))
    itp, itc = tp[:8000], tc[:8000]
    ivox = g.iVox(0.5)
    ivox.insert(itp, itc)
    rivox = ivox_np.IvoxNp(0.5)
    rivox.insert(itp, itc)
    otgt = orc.Cloud(tp, tc)
    otgt.set_normals(normals)
    return dict(tp=tp, tc=tc, sp=sp, sc=sc, normals=normals, tgt=tgt, tree=g.KdTree(tgt), vm=vm, ovm=ovm, ivox=ivox, rivox=rivox, otgt=otgt, otree=orc.KdTree(otgt, 4))


def source_arrays(scene, pb, cb, offset, n):
    """Lossless storage variants: float32-exact points (pb 4) or offset by 2^-30 (pb 8); covariances rounded through float32
    (cb 4) or as they are (cb 8)."""
    p = scene["sp"][offset : offset + n]
    c = scene["sc"][offset : offset + n]
    if pb == 8:
        p = p + 2.0**-30
    if cb == 4:
        c = c.astype(np.float32).astype(np.float64)
    return np.ascontiguousarray(p), np.ascontiguousarray(c)


class Ref:
    """One factor and its float64 reference."""

    def __init__(self, g, scene, kind, pb, cb, offset, n, flags=capi.B2_CLOUD_DEFAULT):
        self.kind = kind
        p, c = source_arrays(scene, pb, cb if cb else 8, offset, n)
        if flags == capi.B2_CLOUD_COMPACT_F32:  # compact storage holds the float32-rounded values exactly
            p, c = p.astype(np.float32).astype(np.float64), c.astype(np.float32).astype(np.float64)
            cloud = g.PointCloud(source_arrays(scene, pb, 8, offset, n)[0], source_arrays(scene, pb, 8, offset, n)[1], flags=flags)
        else:
            cloud = g.PointCloud(p, None if kind in ICP_KINDS else c, flags=flags)
        self.p, self.c, self.cloud = p, c, cloud
        info = cloud.info()
        if flags == capi.B2_CLOUD_DEFAULT:
            assert (info.point_bytes, info.cov_bytes) == (pb, cb), (kind, pb, cb)
        if kind == "vgicp":
            self.f = g.IntegratedVGICPFactor(0, 1, scene["vm"], cloud)
            self.of = orc.Factor(scene["ovm"], orc.Cloud(p, c))
        elif kind == "gicp":
            self.f = g.IntegratedGICPFactor(0, 1, scene["tgt"], cloud, target_tree=scene["tree"])
            self.of = orc.Factor(scene["otgt"], orc.Cloud(p, c), tree=scene["otree"], num_threads=2)
        elif kind in ICP_KINDS:
            self.f = g.IntegratedICPFactor(0, 1, scene["tgt"], cloud, target_tree=scene["tree"], use_point_to_plane=kind == "plane")
            self.of = orc.Factor(scene["otgt"], orc.Cloud(p), tree=scene["otree"], num_threads=2, icp="point" if kind == "icp" else "plane")
        else:
            self.f = g.IntegratedGICPFactor(0, 1, scene["ivox"], cloud)
            self.of = ivox_np.GicpIvoxNp(scene["rivox"], p, c)
            self.rivox = scene["rivox"]
        self.frozen = None

    def set_tolerance(self, angle, trans):
        self.f.set_correspondence_update_tolerance(angle, trans)
        if self.kind != "ivox":
            self.of.set_correspondence_update_tolerance(angle, trans)

    def linearize(self, delta):
        if self.kind == "ivox" and self.frozen is not None:  # the restatement of the tolerance path: kept indices, new pose
            ex, fi = self.rivox.export(), self.rivox.flat_index()
            flat = np.array([fi[c] if c >= 0 else -1 for c in self.frozen], dtype=np.int64)
            return np_ref.linearize(delta, self.p, self.c, ex["points"], ex["covs"], flat), self.frozen
        l = self.of.linearize(delta)
        corr = self.of.corr if self.kind == "ivox" else self.of.correspondences()
        return l, corr

    def error(self, delta):
        return self.of.error(delta)


def check(ref, rec, delta, tol=1e-9):
    l, corr = ref.linearize(delta)
    assert np.array_equal(ref.f.correspondences(), corr), ref.kind
    assert_linearized_close(capi.unpack_linearized(rec) if not isinstance(rec, dict) else rec, l, tol)
    return corr


@pytest.mark.gpu
def test_all_groups_in_one_set(g, scene):
    rng = np.random.default_rng(5)
    sizes = rng.integers(700, 2600, len(SET_GROUPS))
    sizes[::5] = [1, 33, 1025, 257][: len(sizes[::5])]
    refs = [Ref(g, scene, k, pb, cb, 37 * i, int(n)) for i, ((k, pb, cb), n) in enumerate(zip(SET_GROUPS, sizes))]
    fs = g.NonlinearFactorSetGPU()
    fs.add([r.f for r in refs])
    deltas = {0: np.eye(4), 1: syn.random_pose(rng, 0.02, 0.2)}
    out = fs.linearize(deltas)
    n_lin = fs.launch_count()
    assert n_lin == 16
    for r, rec in zip(refs, out):
        check(r, rec, deltas[1])
    d2 = deltas[1] @ syn.random_pose(rng, 0.01, 0.05)
    errs = fs.error({0: np.eye(4), 1: d2})
    assert fs.launch_count() == n_lin + 16
    for r, e in zip(refs, errs):
        eref = r.error(d2)
        assert abs(e - eref) <= 1e-9 * abs(eref) + 1e-300, r.kind


@pytest.mark.gpu
def test_all_groups_tolerance_frozen(g, scene):
    """Second linearize inside the correspondence-update tolerance: the set kernels take the frozen-flags path for the GICP,
    ICP and iVox factors (VGICP has no tolerance and re-associates)."""
    rng = np.random.default_rng(6)
    refs = [Ref(g, scene, k, pb, cb, 53 * i, 900 + 61 * i) for i, (k, pb, cb) in enumerate(SET_GROUPS)]
    for r in refs:
        if r.kind != "vgicp":
            r.set_tolerance(0.05, 0.5)
    fs = g.NonlinearFactorSetGPU()
    fs.add([r.f for r in refs])
    d0 = syn.random_pose(rng, 0.01, 0.1)
    d1 = d0 @ syn.se3_exp(np.array([0.01, -0.01, 0.005, 0.05, -0.05, 0.02]))
    out0 = fs.linearize({0: np.eye(4), 1: d0})
    first = [check(r, rec, d0) for r, rec in zip(refs, out0)]
    for r, c in zip(refs, first):
        if r.kind == "ivox":
            r.frozen = c
    out1 = fs.linearize({0: np.eye(4), 1: d1})
    assert fs.launch_count() == 32
    for r, rec, c in zip(refs, out1, first):
        corr = check(r, rec, d1)
        if r.kind != "vgicp":
            assert np.array_equal(corr, c), r.kind  # frozen
    fresh = Ref(g, scene, "gicp", 4, 8, 0, 900)
    fresh.f.linearize({0: np.eye(4), 1: d1})
    assert not np.array_equal(fresh.f.correspondences(), first[SET_GROUPS.index(("gicp", 4, 8))])  # the freeze is visible


@pytest.mark.gpu
@pytest.mark.parametrize("kind,storage", SINGLES, ids=[f"{k}-p{pb}c{cb}" for k, (pb, cb) in SINGLES])
def test_one_factor_by_value(g, scene, kind, storage):
    pb, cb = storage
    r = Ref(g, scene, kind, pb, cb, 101, 5003)
    fs = g.NonlinearFactorSetGPU()
    fs.add(r.f)
    rng = np.random.default_rng(7)
    delta = syn.random_pose(rng, 0.02, 0.2)
    out = fs.linearize({0: np.eye(4), 1: delta})
    assert fs.launch_count() == 1
    check(r, out[0], delta)
    d2 = delta @ syn.random_pose(rng, 0.01, 0.05)
    e = fs.error({0: np.eye(4), 1: d2})[0]
    eref = r.error(d2)
    assert abs(e - eref) <= 1e-9 * abs(eref)


TARGET_STORAGES = [(pb, cb) for pb in (4, 8) for cb in (4, 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("storage", TARGET_STORAGES, ids=[f"p{pb}c{cb}" for pb, cb in TARGET_STORAGES])
def test_gicp_target_storages(g, scene, storage):
    """Each target storage builds its records with its own gather_leaf_records_kernel<PT, CT>; the kd-tree's leaf records
    follow the target points (float32 for float32-exact points)."""
    pb, cb = storage
    tp, tc = scene["tp"][:15000], scene["tc"][:15000]
    if pb == 8:
        tp = tp + 2.0**-30
    if cb == 4:
        tc = tc.astype(np.float32).astype(np.float64)
    tgt = g.PointCloud(tp, tc)
    assert (tgt.info().point_bytes, tgt.info().cov_bytes) == (pb, cb)
    sp, sc = scene["sp"][:6000], scene["sc"][:6000]
    f = g.IntegratedGICPFactor(0, 1, tgt, g.PointCloud(sp, sc))
    otgt = orc.Cloud(tp, tc)
    of = orc.Factor(otgt, orc.Cloud(sp, sc), tree=orc.KdTree(otgt, 4), num_threads=4)
    delta = syn.random_pose(np.random.default_rng(8), 0.02, 0.2)
    f.linearize({0: np.eye(4), 1: delta})
    ref = of.linearize(delta)
    assert ref["num_inliers"] > 3000
    assert np.array_equal(f.correspondences(), of.correspondences())
    assert_linearized_close(f._last, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("pb", [4, 8])
@pytest.mark.parametrize("plane", [False, True])
def test_icp_target_storages(g, scene, pb, plane):
    tp = scene["tp"][:15000] + (2.0**-30 if pb == 8 else 0.0)
    normals = scene["normals"][:15000]
    tgt = g.PointCloud(tp, normals=normals)
    assert tgt.info().point_bytes == pb
    sp = scene["sp"][:6000]
    f = g.IntegratedICPFactor(0, 1, tgt, g.PointCloud(sp), use_point_to_plane=plane)
    otgt = orc.Cloud(tp)
    otgt.set_normals(normals)
    of = orc.Factor(otgt, orc.Cloud(sp), tree=orc.KdTree(otgt, 4), num_threads=4, icp="plane" if plane else "point")
    delta = syn.random_pose(np.random.default_rng(9), 0.02, 0.2)
    f.linearize({0: np.eye(4), 1: delta})
    ref = of.linearize(delta)
    assert np.array_equal(f.correspondences(), of.correspondences())
    assert_linearized_close(f._last, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", SOURCE_COV_KINDS)
def test_compact_f32_is_exact_on_rounded_inputs(g, scene, kind):
    """COMPACT_F32 stores the float32-rounded points and covariances; against the oracle fed those rounded values it is
    exact to the 1e-9 bar with identical correspondences (test_gpu_parity.py keeps the 1e-4 check against unrounded inputs)."""
    r = Ref(g, scene, kind, 8, 8, 11, 6001, flags=capi.B2_CLOUD_COMPACT_F32)
    info = r.cloud.info()
    assert (info.point_bytes, info.cov_bytes) == (4, 4)
    delta = syn.random_pose(np.random.default_rng(10), 0.02, 0.2)
    r.f.linearize({0: np.eye(4), 1: delta})
    check(r, r.f._last, delta)
    d2 = delta @ syn.random_pose(np.random.default_rng(11), 0.01, 0.05)
    e, eref = r.f.error({0: np.eye(4), 1: d2}), r.error(d2)
    assert abs(e - eref) <= 1e-9 * abs(eref)
