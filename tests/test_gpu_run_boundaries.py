"""Factor-run boundaries of the factor kernel in every warp shape, and every instantiation and normal storage of
surface-validated VGICP.

The factor kernel is persistent: CTA c of a launch owns the tiles [c T / G, (c + 1) T / G) of all the factors of its launch
group (T tiles, G = min(T, SM count) CTAs), so a CTA often ends one factor run and starts the next.  At such a boundary the
probe warps reload the descriptor, the pose and the frozen flag, the ring hand-shake closes the run, the accumulate warps
flush into slot blockIdx.x - cta_first, and the last CTA of a factor reduces the factor's num_slots partials, 24 kC slots per
round.  The tiles of the three warp shapes (b2_factor_kernel_ws.cuh):

  VGICP                                  8 probe / 8 accumulate warps, 2 points per lane   512 points
  VGICP with surface validation          8 / 8, 1 point per lane                           256 points
  GICP, ICP, point-to-plane ICP, iVox    28 / 4, 1 point per lane                          896 points

(test_gpu_parity.py covers the plain VGICP shape.)  Every factor here is held to its float64 reference: correspondences
bit-identical, each H / b block within 1e-9 of its own largest entry, error within 1e-9, num_inliers exact, and exact zeros
where the reference has no inliers.

* Tree shape: per kind one launch of 200 factors over one shared target, sizes on and around the warp tile and the CTA tile,
  each with its own pose.  Every other factor has a correspondence-update tolerance, and the second linearize moves half of
  those within it and half beyond it, so frozen and re-associating runs follow each other inside CTAs.  Also a kd-tree factor
  that spans more than 96 CTA slots between one-tile factors (a second epilogue round at a nonzero cta_first), and a set of all
  four kinds in interleaved order (non-contiguous out_index values within a group, frozen flags indexed across groups).
* Surface-validated VGICP: all 16 validated_vgicp_kernel<PT, CT, MODE, SINGLE> instantiations with float32 and float64
  normals, COMPACT_F32 storage, and one launch of 150 factors around the 256-point tile whose normals alternate between
  float32 and float64 storage.  A CPU test reads the instantiations compiled into the library and checks that this module
  covers them all.
* A CPU test shows that the per-factor check rejects a result that lacks one point's contribution, at tile-edge sizes.

The layout the tests assert on is the host's (build_groups), restated in cta_layout() at the SM count of the device; other
SM counts move the boundaries elsewhere.  Run with -s to print where each tile-edge factor landed.
"""
import os
import re
import subprocess

import numpy as np
import pytest

import ivox_np
import normals_ref as nref
import np_ref
import oracle_lib as orc
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn
from test_gpu_parity import TOL, assert_linearized_close

TREE_KINDS = ("gicp", "icp", "plane", "ivox")
TREE_TILE, VALIDATED_TILE = 896, 256  # source points per CTA tile (kP * 32 * kPPL)
TREE_EPILOGUE_ROUND = 24 * 4  # slots one round of the last CTA's partial-sum loads covers (kInFlight * kC, kC = 4)
TREE_EDGES = [0, 1, 31, 32, 33, 895, 896, 897, 1791, 1792, 1793, 2687, 2689]
VALIDATED_EDGES = [0, 1, 31, 32, 33, 255, 256, 257, 511, 512, 513, 767, 768, 769]
TOL_ANGLE, TOL_TRANS = 0.05, 0.5
STEP_IN = syn.se3_exp(np.array([0.01, -0.01, 0.005, 0.05, -0.05, 0.02]))  # 0.015 rad, 0.07 m: within the tolerance
STEP_OUT = syn.se3_exp(np.array([0.01, 0.0, -0.01, 0.6, -0.3, 0.1]))  # 0.68 m: beyond it
N_SOURCE = 200000
TYPE = {4: "float", 8: "double"}


def round32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


# ---- the host's tile and slot layout ------------------------------------------------------------------------------------


def num_tiles(n, tile):
    return max(1, -(-n // tile))


def cta_layout(sizes, tile, sm_count):
    """build_groups restated for one launch group: G and, per factor, (tile_begin, num_tiles, cta_first, num_slots)."""
    tiles = [num_tiles(n, tile) for n in sizes]
    T = sum(tiles)
    G = min(T, sm_count)
    begin = lambda c: c * T // G  # cta_tile_begin
    out, c, tb = [], 0, 0
    for nt in tiles:
        while begin(c + 1) <= tb:
            c += 1
        last = c
        while begin(last + 1) < tb + nt:
            last += 1
        out.append((tb, nt, c, last - c + 1))
        tb += nt
    return G, out


def runs_per_cta(layout, G):
    """Factor indices each CTA works on, in run order."""
    runs = [[] for _ in range(G)]
    for k, (_, _, c0, ns) in enumerate(layout):
        for c in range(c0, c0 + ns):
            runs[c].append(k)
    return runs


def report(name, sizes, layout, G, labels, edges, index=None):
    """Prints where the tile-edge factors (and any factor over more than one epilogue round of CTAs) landed: their tiles, their
    CTAs, and whether their first / last CTA also works on another factor."""
    T = sum(nt for _, nt, _, _ in layout)
    shared = sum(len(r) >= 2 for r in runs_per_cta(layout, G))
    print(f"\n{name}: {T} tiles on {G} CTAs, {shared} of which work on more than one factor")
    for k, (n, (tb, nt, c0, ns)) in enumerate(zip(sizes, layout)):
        if n in edges or ns > TREE_EPILOGUE_ROUND:
            shared = [w for w, s in (("first", c0 * T // G < tb), ("last", (c0 + ns) * T // G > tb + nt)) if s]
            where = f"{' and '.join(shared)} CTA shared" if shared else "CTAs not shared"
            i = k if index is None else index[k]
            print(f"  factor {i:3d} {labels[k]:<24s} n={n:<6d} tiles {tb}..{tb + nt - 1}  CTAs {c0}..{c0 + ns - 1}  {where}")


# ---- references ---------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def host_scene():
    tp, tc = syn.make_cloud(30000, stream=1, scale=0.3)
    sp, sc = syn.make_cloud(N_SOURCE, stream=2, scale=0.3)
    rng = np.random.default_rng(12)
    tn = rng.normal(size=(len(tp), 3))
    tn /= np.linalg.norm(tn, axis=1, keepdims=True)
    otgt = orc.Cloud(tp, tc)
    otgt.set_normals(tn)
    return dict(tp=tp, tc=tc, tn=tn, sp=sp, sc=sc, sc32=round32(sc), otgt=otgt, otree=orc.KdTree(otgt, 4))


class TreeCase:
    """One tree-shape factor and its float64 reference: the CPU oracle for the kd-tree kinds (which applies the tolerance
    itself), the numpy iVox restatement for iVox (told which linearizations keep their correspondences).  Source points are
    float32-exact and covariances rounded through float32, so every factor of a kind, the empty one included, has the same
    storage and the same launch group."""

    def __init__(self, g, scene, kind, n, offset, key):
        self.kind, self.n = kind, n
        self.p = np.ascontiguousarray(scene["sp"][offset : offset + n])
        self.c = np.ascontiguousarray(scene["sc32"][offset : offset + n])
        covs = None if kind in ("icp", "plane") else self.c
        cloud = g.PointCloud(self.p, covs)
        assert (cloud.info().point_bytes, cloud.info().cov_bytes) == (4, 4 if covs is not None else 0)
        if kind == "gicp":
            self.f = g.IntegratedGICPFactor(0, key, scene["tgt"], cloud, target_tree=scene["tree"])
            self.of = orc.Factor(scene["otgt"], orc.Cloud(self.p, self.c), tree=scene["otree"], num_threads=2)
        elif kind in ("icp", "plane"):
            self.f = g.IntegratedICPFactor(0, key, scene["tgt"], cloud, target_tree=scene["tree"], use_point_to_plane=kind == "plane")
            self.of = orc.Factor(scene["otgt"], orc.Cloud(self.p), tree=scene["otree"], num_threads=2, icp="point" if kind == "icp" else "plane")
        else:
            self.f = g.IntegratedGICPFactor(0, key, scene["ivox"], cloud)
            self.rivox, self.ivox_export, self.ivox_flat = scene["rivox"], scene["ivox_export"], scene["ivox_flat"]
            self.corr = self.lin = None
        self.tolerance = False

    def set_tolerance(self):
        self.f.set_correspondence_update_tolerance(TOL_ANGLE, TOL_TRANS)
        if self.kind != "ivox":
            self.of.set_correspondence_update_tolerance(TOL_ANGLE, TOL_TRANS)
        self.tolerance = True

    def _ivox_eval(self, delta_eval):
        flat = np.array([self.ivox_flat[c] if c >= 0 else -1 for c in self.corr], dtype=np.int64)
        ex = self.ivox_export
        return np_ref.linearize(self.lin, self.p, self.c, ex["points"], ex["covs"], flat, delta_eval)

    def linearize(self, delta, frozen):
        """(reference record, reference correspondences) of a linearize at `delta`."""
        if self.kind != "ivox":
            return self.of.linearize(delta), self.of.correspondences()
        if not frozen:
            self.corr = ivox_np.correspondences(self.rivox, delta, self.p)
        self.lin = np.array(delta)
        return self._ivox_eval(delta), self.corr

    def error(self, delta):
        return self._ivox_eval(delta)["error"] if self.kind == "ivox" else self.of.error(delta)


def check_factor(rec, corr, ref, ref_corr, what):
    """The per-factor bar: bit-identical correspondences, each block within 1e-9 of its largest entry, error within 1e-9,
    num_inliers exact, and all zeros where the reference has no inliers."""
    assert np.array_equal(corr, ref_corr), what
    got = rec if isinstance(rec, dict) else capi.unpack_linearized(rec)
    try:
        assert_linearized_close(got, ref)
    except AssertionError as e:
        raise AssertionError(what) from e
    if ref["num_inliers"] == 0 and not isinstance(rec, dict):
        assert not np.any(rec[: orc.LINEARIZED_DOUBLES]), what


def check_error(e, eref, what):
    assert abs(e - eref) <= TOL * abs(eref), (what, e, eref)  # exact zero when the reference is zero


def values_of(deltas):
    return {0: np.eye(4), **{i + 1: d for i, d in enumerate(deltas)}}


def set_sizes(n_factors, edges, lo, hi, seed, n_source=N_SOURCE):
    """Random sizes in [lo, hi) with the edge sizes spread over the set, away from its ends, at an odd stride so that they
    meet every freeze pattern; and a source slice for each."""
    rng = np.random.default_rng(seed)
    sizes = [int(x) for x in rng.integers(lo, hi, n_factors)]
    stride = ((n_factors - 8) // len(edges) - 1) | 1
    for j, n in enumerate(edges):
        sizes[3 + j * stride] = n
    offsets = [int(rng.integers(0, n_source - n + 1)) for n in sizes]
    return sizes, offsets


def tree_set_sizes(kind):
    """Sizes and source offsets of the one-kind tree-shape set: 200 factors, about 210 tiles."""
    return set_sizes(200, TREE_EDGES, 100, 700, seed=100 + TREE_KINDS.index(kind))


def freeze_pattern(i):
    """(has a tolerance, step of the second linearize): every other factor has a tolerance; of those, half move within it and
    keep their correspondences, half move beyond it and re-associate; the factors without one re-associate either way."""
    return i % 2 == 0, STEP_IN if i % 4 < 2 else STEP_OUT


def run_tree_set(g, cases, launches, seed, name):
    """Linearize at per-factor poses, error() at second poses, linearize again at the first poses (byte-identical), then
    linearize with mixed frozen state and evaluate the error once more; every factor against its reference at every step."""
    rng = np.random.default_rng(seed)
    for i, c in enumerate(cases):
        if freeze_pattern(i)[0]:
            c.set_tolerance()
    frozen = [freeze_pattern(i)[0] and freeze_pattern(i)[1] is STEP_IN for i in range(len(cases))]
    fs = g.NonlinearFactorSetGPU()
    fs.add([c.f for c in cases])
    d0 = [syn.random_pose(rng, 0.02, 0.2) for _ in cases]
    out0 = fs.linearize(values_of(d0)).copy()
    assert fs.launch_count() == launches, "one launch per kind"
    first = []
    for i, (c, rec, d) in enumerate(zip(cases, out0, d0)):
        ref, ref_corr = c.linearize(d, frozen=False)
        check_factor(rec, c.f.correspondences(), ref, ref_corr, (name, "linearize", i, c.kind, c.n))
        first.append(np.copy(ref_corr))
    assert sum(capi.unpack_linearized(r)["num_inliers"] for r in out0) > 0.5 * sum(c.n for c in cases)

    de = [d @ syn.random_pose(rng, 0.01, 0.05) for d in d0]
    errs = fs.error(values_of(de))
    assert fs.launch_count() == 2 * launches
    for i, (c, e, d) in enumerate(zip(cases, errs, de)):
        check_error(e, c.error(d), (name, "error", i, c.kind, c.n))

    # the tolerance factors take the frozen path now (no pose change since their association), the others re-associate
    again = fs.linearize(values_of(d0))
    assert again.tobytes() == out0.tobytes(), "not bit-reproducible"

    d1 = [d @ freeze_pattern(i)[1] for i, d in enumerate(d0)]
    out1 = fs.linearize(values_of(d1))
    for i, (c, rec, d) in enumerate(zip(cases, out1, d1)):
        ref, ref_corr = c.linearize(d, frozen=frozen[i])
        corr = c.f.correspondences()
        check_factor(rec, corr, ref, ref_corr, (name, "mixed frozen", i, c.kind, c.n, frozen[i]))
        if frozen[i]:
            assert np.array_equal(corr, first[i]), (name, i, "should have kept its correspondences")
        elif c.tolerance and c.n >= 32:
            assert not np.array_equal(corr, first[i]), (name, i, "should have re-associated")
    de2 = [d @ syn.random_pose(rng, 0.01, 0.05) for d in d1]
    errs = fs.error(values_of(de2))
    for i, (c, e, d) in enumerate(zip(cases, errs, de2)):
        check_error(e, c.error(d), (name, "error after mixed frozen", i, c.kind, c.n))
    return frozen


def assert_boundaries_crossed(layout, G, frozen, min_shared=20):
    """Many CTAs work on more than one factor run, and some go from a frozen run to a re-associating one."""
    runs = runs_per_cta(layout, G)
    assert sum(len(r) >= 2 for r in runs) >= min_shared
    assert any(frozen[a] and not frozen[b] for r in runs for a, b in zip(r, r[1:])), "no CTA meets a frozen -> re-associating transition"


def labels_of(cases, frozen):
    state = lambda i, c: "frozen" if frozen[i] else ("re-associated" if c.tolerance else "no tolerance")
    return [f"{c.kind} {state(i, c)}" for i, c in enumerate(cases)]


# ---- tree shape ---------------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


@pytest.fixture(scope="module")
def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def scene(g, host_scene):
    s = dict(host_scene)
    s["tgt"] = g.PointCloud(s["tp"], s["tc"], normals=s["tn"])
    s["tree"] = g.KdTree(s["tgt"])
    itp, itc = s["tp"][:8000], s["tc"][:8000]
    s["ivox"] = g.iVox(0.5)
    s["ivox"].insert(itp, itc)
    s["rivox"] = ivox_np.IvoxNp(0.5)
    s["rivox"].insert(itp, itc)
    s["ivox_export"], s["ivox_flat"] = s["rivox"].export(), s["rivox"].flat_index()
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("kind", TREE_KINDS)
def test_tree_shape_run_boundaries(g, scene, sm_count, kind):
    sizes, offsets = tree_set_sizes(kind)
    cases = [TreeCase(g, scene, kind, n, o, i + 1) for i, (n, o) in enumerate(zip(sizes, offsets))]
    G, layout = cta_layout(sizes, TREE_TILE, sm_count)
    frozen = run_tree_set(g, cases, 1, 200 + TREE_KINDS.index(kind), kind)
    report(kind, sizes, layout, G, labels_of(cases, frozen), TREE_EDGES)
    assert_boundaries_crossed(layout, G, frozen)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["gicp", "icp"])
def test_large_tree_factor_between_small_ones(g, scene, sm_count, kind):
    """A factor of 181000 points (203 tiles) between 16 small factors of one or two tiles: it covers more than 96 CTA slots,
    so its last CTA reduces them in two rounds, and its first and last CTAs also work on its neighbours."""
    rng = np.random.default_rng(7)
    sizes = [int(x) for x in rng.integers(1, TREE_TILE + 1, 17)]
    sizes[3], sizes[5], sizes[12], sizes[8] = 1, TREE_TILE + 1, TREE_TILE, 181000
    offsets = [int(rng.integers(0, N_SOURCE - n + 1)) for n in sizes]
    G, layout = cta_layout(sizes, TREE_TILE, sm_count)
    tb, nt, c0, ns = layout[8]
    T = sum(x[1] for x in layout)
    assert ns > TREE_EPILOGUE_ROUND and c0 > 0
    assert c0 * T // G < tb and (c0 + ns) * T // G > tb + nt, "its first and last CTAs must be shared with its neighbours"
    cases = [TreeCase(g, scene, kind, n, o, i + 1) for i, (n, o) in enumerate(zip(sizes, offsets))]
    frozen = run_tree_set(g, cases, 1, 300, f"large {kind}")
    assert frozen[8], "the large factor takes both the re-associating and the frozen path"
    report(f"large {kind}", sizes, layout, G, labels_of(cases, frozen), [1, TREE_TILE, TREE_TILE + 1])


@pytest.mark.gpu
def test_tree_kinds_interleaved(g, scene, sm_count):
    """All four tree kinds in one set, added in interleaved order: one launch group per kind, so a group's factors have
    non-contiguous out_index values and its frozen flags sit among the other groups'."""
    sizes, offsets = set_sizes(128, TREE_EDGES, 3000, 12000, seed=400)  # a few tiles each: more tiles than CTAs per group
    kinds = [TREE_KINDS[(i + i // 4) % 4] for i in range(len(sizes))]  # every kind meets every freeze pattern
    cases = [TreeCase(g, scene, k, n, o, i + 1) for i, (k, n, o) in enumerate(zip(kinds, sizes, offsets))]
    frozen = run_tree_set(g, cases, 4, 500, "interleaved")
    for kind in TREE_KINDS:
        idx = [i for i, k in enumerate(kinds) if k == kind]
        assert any(frozen[i] for i in idx) and not all(frozen[i] for i in idx)
        G, layout = cta_layout([sizes[i] for i in idx], TREE_TILE, sm_count)
        assert_boundaries_crossed(layout, G, [frozen[i] for i in idx], min_shared=8)
        report(f"interleaved {kind}", [sizes[i] for i in idx], layout, G, [labels_of(cases, frozen)[i] for i in idx], TREE_EDGES, idx)


# ---- surface-validated VGICP --------------------------------------------------------------------------------------------

VALIDATED_STORAGES = [(pb, cb, nb) for pb in (4, 8) for cb in (4, 8) for nb in (4, 8)]  # point, covariance, normal bytes
N_VALIDATED_SOURCE = 60000


def covered_validated_kernels():
    """(PT, CT, MODE, SINGLE) of the validated_vgicp_kernel instantiations this module launches."""
    out = set()
    for pb, cb, _ in VALIDATED_STORAGES:
        for mode in (0, 1):
            out.add((TYPE[pb], TYPE[cb], mode, True))  # test_validated_one_factor
            out.add((TYPE[pb], TYPE[cb], mode, False))  # test_validated_storages_in_one_set
    return out


def test_validated_parametrisation_covers_every_compiled_kernel():
    """The library's validated_vgicp_kernel instantiations, read from its device code, are exactly the 16 of (PT, CT) x mode x
    by-value pose, and this module launches them all with both normal storages; a new storage or mode fails here until it is
    tested."""
    from gtsam_points_b200 import build

    assert os.path.exists(build.LIB)
    cuobjdump = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")
    syms = subprocess.run([cuobjdump, "-symbols", build.LIB], capture_output=True, text=True, check=True).stdout
    names = set(re.findall(r"_ZN2b2\d*ws\w*validated_vgicp_kernel\w*", syms))
    demangled = subprocess.run(["c++filt"], input="\n".join(sorted(names)), capture_output=True, text=True, check=True).stdout
    compiled = set()
    for m in re.finditer(r"validated_vgicp_kernel<(float|double), (float|double), (\d+), (true|false)>", demangled):
        compiled.add((m.group(1), m.group(2), int(m.group(3)), m.group(4) == "true"))
    expected = {(TYPE[pb], TYPE[cb], mode, single) for pb in (4, 8) for cb in (4, 8) for mode in (0, 1) for single in (False, True)}
    assert len(expected) == 16
    assert compiled == expected
    assert covered_validated_kernels() == expected
    for pb in (4, 8):
        for cb in (4, 8):
            assert {nb for p, c, nb in VALIDATED_STORAGES if (p, c) == (pb, cb)} == {4, 8}


@pytest.fixture(scope="module")
def vscene(g, host_scene):
    tp, tc = host_scene["tp"], host_scene["tc"]
    sp, sc = host_scene["sp"][:N_VALIDATED_SOURCE], host_scene["sc"][:N_VALIDATED_SOURCE]
    nrm = nref.normals_from_covs(sp, sc)
    nrm[::3] *= -1.0  # back faces
    nrm[::7] = 0.0  # no normal: never rejected
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(g.PointCloud(tp, tc))
    ovm = orc.VoxelMap(0.5)
    ovm.insert(orc.Cloud(tp, tc))
    return dict(sp=sp, sc=sc, nrm=nrm, vm=vm, ovm=ovm)


class ValidatedCase:
    """A surface-validated VGICP factor over lossless storage (pb 8: points offset by 2^-30; cb / nb 4: covariances / normals
    rounded through float32), or COMPACT_F32 storage against the reference fed the float32-rounded inputs."""

    def __init__(self, g, vs, pb, cb, nb, offset, n, key, compact=False):
        p, c, nr = (vs[k][offset : offset + n] for k in ("sp", "sc", "nrm"))
        if pb == 8:
            p = p + 2.0**-30
        c = round32(c) if cb == 4 else c
        nr = round32(nr) if nb == 4 else nr
        p, c, nr = (np.ascontiguousarray(a) for a in (p, c, nr))
        cloud = g.PointCloud(p, c, normals=nr, flags=capi.B2_CLOUD_COMPACT_F32 if compact else capi.B2_CLOUD_DEFAULT)
        info = cloud.info()
        if compact:
            p, c, nr = round32(p), round32(c), round32(nr)
            assert (info.point_bytes, info.cov_bytes, info.normal_bytes) == (4, 4, 4)
        else:
            assert (info.point_bytes, info.cov_bytes, info.normal_bytes) == (pb, cb, nb), (pb, cb, nb, n)
        self.n, self.nb, self.p, self.nrm = n, nb, p, nr
        self.f = g.IntegratedVGICPFactor(0, key, vs["vm"], cloud)
        self.f.set_enable_surface_validation(True)
        self.ref = nref.ValidatedVGICP(vs["ovm"], p, c, nr)


def run_validated_set(g, cases, launches, seed, name):
    """Linearize, error() at second poses, linearize again (byte-identical); returns the poses and the rejection mask."""
    rng = np.random.default_rng(seed)
    fs = g.NonlinearFactorSetGPU()
    fs.add([c.f for c in cases])
    d0 = [syn.random_pose(rng, 0.03, 0.3) for _ in cases]
    out = fs.linearize(values_of(d0)).copy()
    assert fs.launch_count() == launches
    for i, (c, rec, d) in enumerate(zip(cases, out, d0)):
        ref = c.ref.linearize(d)
        check_factor(rec, c.f.correspondences(), ref, c.ref.correspondences(), (name, "linearize", i, c.n, c.nb))
    de = [d @ syn.random_pose(rng, 0.01, 0.05) for d in d0]
    errs = fs.error(values_of(de))
    assert fs.launch_count() == 2 * launches
    for i, (c, e, d) in enumerate(zip(cases, errs, de)):
        check_error(e, c.ref.error(d), (name, "error", i, c.n, c.nb))
    assert fs.linearize(values_of(d0)).tobytes() == out.tobytes(), "not bit-reproducible"
    rejected = np.concatenate([nref.surface_rejected(c.p, c.nrm, d) for c, d in zip(cases, d0)] + [np.zeros(0, bool)])
    return rejected


@pytest.mark.gpu
@pytest.mark.parametrize("storage", VALIDATED_STORAGES, ids=[f"p{pb}c{cb}n{nb}" for pb, cb, nb in VALIDATED_STORAGES])
def test_validated_one_factor(g, vscene, storage):
    """One-factor sets: the by-value-pose instantiation of each (PT, CT), with float32 and with float64 normals."""
    pb, cb, nb = storage
    case = ValidatedCase(g, vscene, pb, cb, nb, 101 + 977 * VALIDATED_STORAGES.index(storage), 5003, 1)
    rejected = run_validated_set(g, [case], 1, 600 + VALIDATED_STORAGES.index(storage), "one factor")
    assert 0.05 < rejected.mean() < 0.95


@pytest.mark.gpu
def test_validated_storages_in_one_set(g, vscene):
    """All eight storages in one set, two factors each: one launch per (PT, CT), float32 and float64 normals side by side."""
    cases = []
    for k, (pb, cb, nb) in enumerate(VALIDATED_STORAGES):
        for j, n in enumerate((VALIDATED_TILE + 1, 3001 + 37 * k)):
            cases.append(ValidatedCase(g, vscene, pb, cb, nb, 4000 * k + 2000 * j, n, len(cases) + 1))
    rejected = run_validated_set(g, cases, 4, 700, "storages")
    assert 0.05 < rejected.mean() < 0.95


@pytest.mark.gpu
def test_validated_compact_f32(g, vscene):
    """COMPACT_F32 storage with validation: points, covariances and normals in float32, exact against the reference fed the
    float32-rounded values."""
    cases = [ValidatedCase(g, vscene, 8, 8, 8, 11, 6001, 1, compact=True)]
    rejected = run_validated_set(g, cases, 1, 800, "compact one factor")
    assert 0.05 < rejected.mean() < 0.95
    cases = [ValidatedCase(g, vscene, 8, 8, 8, 7000 * k, n, k + 1, compact=True) for k, n in enumerate((1, 257, 4000, 33, 6001))]
    run_validated_set(g, cases, 1, 801, "compact set")


@pytest.mark.gpu
def test_validated_run_boundaries(g, vscene, sm_count):
    """150 validated factors in one launch, sizes around the 32-point warp tile and the 256-point CTA tile; the normals of
    every other factor are float32 (the probe warps' nrm_f32 branch), so CTAs move between float32- and float64-normal runs."""
    sizes, offsets = set_sizes(150, VALIDATED_EDGES, 1, 400, seed=900, n_source=N_VALIDATED_SOURCE)
    nrm = vscene["nrm"]
    # float64 normals for every other factor, unless its slice has only float32-exact ones (the empty and the tiny factors)
    nb = [8 if i % 2 and not np.array_equal(round32(nrm[o : o + n]), nrm[o : o + n]) else 4 for i, (n, o) in enumerate(zip(sizes, offsets))]
    assert sum(x == 8 for x in nb) > 60
    cases = [ValidatedCase(g, vscene, 4, 4, nb[i], o, n, i + 1) for i, (n, o) in enumerate(zip(sizes, offsets))]
    rejected = run_validated_set(g, cases, 1, 901, "validated boundaries")
    assert 0.05 < rejected.mean() < 0.95
    G, layout = cta_layout(sizes, VALIDATED_TILE, sm_count)
    runs = runs_per_cta(layout, G)
    assert sum(len(r) >= 2 for r in runs) >= 20
    assert any(cases[a].nb != cases[b].nb for r in runs for a, b in zip(r, r[1:])), "no CTA moves between normal storages"
    report("validated", sizes, layout, G, [f"normals float{8 * c.nb}" for c in cases], VALIDATED_EDGES)


# ---- sensitivity of the per-factor check --------------------------------------------------------------------------------


@pytest.mark.parametrize("n", [1, 33, 897, 1793, 2689])
def test_check_sees_one_missing_point(host_scene, n):
    """The kd-tree GICP set of test_tree_shape_run_boundaries, on the CPU: a factor's reference without the last point of its
    last tile -- what a run that ends one tile or one warp too early would deliver -- fails the per-factor check, and fails
    the 1e-9 block comparison on its own, while the same factor summed in another order (more oracle threads) passes."""
    sizes, offsets = tree_set_sizes("gicp")
    k = sizes.index(n)
    assert 0 < k < len(sizes) - 1
    p = host_scene["sp"][offsets[k] : offsets[k] + n]
    c = host_scene["sc32"][offsets[k] : offsets[k] + n]
    delta = syn.random_pose(np.random.default_rng(3), 0.02, 0.2)
    full = orc.Factor(host_scene["otgt"], orc.Cloud(p, c), tree=host_scene["otree"], num_threads=1)
    ref, ref_corr = full.linearize(delta), full.correspondences()
    assert ref_corr[n - 1] >= 0, "the dropped point must be an inlier"
    reordered = orc.Factor(host_scene["otgt"], orc.Cloud(p, c), tree=host_scene["otree"], num_threads=4)
    check_factor(reordered.linearize(delta), reordered.correspondences(), ref, ref_corr, "another summation order")

    short = orc.Factor(host_scene["otgt"], orc.Cloud(p[:-1], c[:-1]), tree=host_scene["otree"], num_threads=1)
    got = short.linearize(delta)
    got_corr = np.append(short.correspondences(), -1)  # the dropped point: no correspondence
    with pytest.raises(AssertionError):
        check_factor(got, got_corr, ref, ref_corr, "one point missing")
    with pytest.raises(AssertionError):
        check_factor(got, ref_corr, ref, ref_corr, "one point missing, correspondences intact")
    blocks_only = dict(got, num_inliers=ref["num_inliers"], error=ref["error"])
    with pytest.raises(AssertionError):
        assert_linearized_close(blocks_only, ref)
