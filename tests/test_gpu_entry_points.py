"""Every host entry point of a factor set computes the same thing (pytest -m gpu), through the C ABI.

A set can be linearized three ways -- b2_factor_set_linearize, issue_linearize + sync + store_linearized, linearize_device --
and evaluated three ways -- b2_factor_set_error, issue_error + sync + store_errors, error_device.  With the same seeded poses
all of them return identical correspondences.  Paths that run the same kernel instantiation return bit-identical results:
every path of a multi-factor set, and of a one-factor ICP set (ICP has no by-value-pose instantiation).  A one-factor set of
the other kinds passes its pose by value on the host-pose paths; that instantiation is held to the parity tolerance against
the device-pose path.  Each call launches once per (kind, storage) group of the set.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle_lib as orc
from gtsam_points_b200 import capi
from gtsam_points_b200 import synthetic as syn
from test_gpu_parity import assert_linearized_close, relerr

KINDS = ("vgicp", "gicp", "icp", "ivox")
B2_ERR_INVALID_STATE = 4
TOL = 1e-9  # test_gpu_parity.py


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


@pytest.fixture(scope="module")
def scene(g):
    tp, tc = syn.make_cloud(60000, stream=1, scale=0.3)
    sp, sc = syn.make_cloud(25001, stream=2, scale=0.3)
    tgt = g.PointCloud(tp, tc)
    vm = g.GaussianVoxelMapGPU(0.5)
    vm.insert(tgt)
    ivox = g.iVox(0.5)
    ivox.insert(tp, tc)
    return dict(tp=tp, tc=tc, sp=sp, sc=sc, tgt=tgt, tree=g.KdTree(tgt), vm=vm, ivox=ivox)


def make_factor(g, scene, kind, n, flags=capi.B2_CLOUD_FORCE_F64):
    # FORCE_F64: every source has the same storage, so a set has one group per factor kind
    src = g.PointCloud(scene["sp"][:n], scene["sc"][:n], flags=flags)
    if kind == "vgicp":
        return g.IntegratedVGICPFactor(0, 1, scene["vm"], src)
    if kind == "gicp":
        return g.IntegratedGICPFactor(0, 1, scene["tgt"], src, target_tree=scene["tree"])
    if kind == "icp":
        return g.IntegratedICPFactor(0, 1, scene["tgt"], src, target_tree=scene["tree"])
    return g.IntegratedGICPFactor(0, 1, scene["ivox"], src)


class FactorSet:
    def __init__(self, factors):
        self.L = capi.lib()
        self.factors = factors
        arr = (C.c_void_p * len(factors))(*[f.h for f in factors])
        self.h = C.c_void_p()
        capi.check(self.L.b2_factor_set_create(factors[0].ctx.h, arr, len(factors), C.byref(self.h)))

    def __del__(self):
        self.L.b2_factor_set_destroy(self.h)

    def launches(self):
        return self.L.b2_factor_set_launch_count(self.h)

    def sync(self):
        capi.check(self.L.b2_factor_set_sync(self.h))

    def correspondences(self):
        return [f.correspondences() for f in self.factors]

    # -- linearize: (F, 16) poses -> (F, 128) records
    def lin_host(self, deltas):
        out = np.zeros((len(self.factors), capi.B2_LINEARIZED_DOUBLES))
        capi.check(self.L.b2_factor_set_linearize(self.h, capi.dptr(deltas), capi.dptr(out)))
        return out

    def lin_issue(self, deltas):
        out = np.zeros((len(self.factors), capi.B2_LINEARIZED_DOUBLES))
        capi.check(self.L.b2_factor_set_issue_linearize(self.h, capi.dptr(deltas), None))
        self.sync()
        capi.check(self.L.b2_factor_set_store_linearized(self.h, capi.dptr(out)))
        return out

    def lin_device(self, deltas):
        import torch

        d_in = torch.from_numpy(deltas).cuda()
        d_out = torch.zeros((len(self.factors), capi.B2_LINEARIZED_DOUBLES), dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()  # the library works on its own stream
        capi.check(self.L.b2_factor_set_linearize_device(self.h, d_in.data_ptr(), d_out.data_ptr()))
        self.sync()
        return d_out.cpu().numpy()

    # -- error: (F, 16) poses -> (F,) errors
    def err_host(self, evals):
        out = np.zeros(len(self.factors))
        capi.check(self.L.b2_factor_set_error(self.h, capi.dptr(evals), capi.dptr(out)))
        return out

    def err_issue(self, evals):
        out = np.zeros(len(self.factors))
        capi.check(self.L.b2_factor_set_issue_error(self.h, capi.dptr(evals), None))
        self.sync()
        capi.check(self.L.b2_factor_set_store_errors(self.h, capi.dptr(out)))
        return out

    def err_device(self, evals):
        import torch

        d_in = torch.from_numpy(evals).cuda()
        d_out = torch.zeros(len(self.factors), dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        capi.check(self.L.b2_factor_set_error_device(self.h, d_in.data_ptr(), d_out.data_ptr()))
        self.sync()
        return d_out.cpu().numpy()


PATHS = ("host", "issue", "device")


def run_paths(fs, deltas, evals):
    """Per path: records, correspondences, errors, and the launches its linearize and its error call added."""
    res = {}
    for p in PATHS:
        n0 = fs.launches()
        rec = getattr(fs, "lin_" + p)(deltas)
        n1 = fs.launches()
        corr = fs.correspondences()
        err = getattr(fs, "err_" + p)(evals)
        res[p] = dict(rec=rec, corr=corr, err=err, lin_launches=n1 - n0, err_launches=fs.launches() - n1)
    return res


def seeded_poses(F, seed):
    rng = np.random.default_rng(seed)
    deltas = np.stack([syn.random_pose(rng, 0.01, 0.15) for _ in range(F)])
    evals = np.stack([d @ syn.random_pose(rng, 0.01, 0.1) for d in deltas])
    return np.ascontiguousarray(deltas), np.ascontiguousarray(evals)


def assert_records_close(a, b, tol):
    blocks = capi.unpack_linearized(a), capi.unpack_linearized(b)
    assert blocks[0]["num_inliers"] == blocks[1]["num_inliers"]
    for k in ("H_target", "H_source", "H_target_source", "b_target", "b_source"):
        assert relerr(blocks[0][k], blocks[1][k]) < tol, k
    assert abs(blocks[0]["error"] - blocks[1]["error"]) <= tol * abs(blocks[1]["error"])


def test_mixed_set_paths_agree(g, scene):
    sizes = [1, 513, 4096, 25001, 300, 7000, 2049, 12345]
    factors = [make_factor(g, scene, KINDS[i % len(KINDS)], n) for i, n in enumerate(sizes)]
    fs = FactorSet(factors)
    deltas, evals = seeded_poses(len(factors), 21)
    res = run_paths(fs, deltas, evals)
    ref = res["host"]
    assert all(capi.unpack_linearized(ref["rec"][i])["num_inliers"] > 100 for i, n in enumerate(sizes) if n >= 4096)
    for p in PATHS:
        r = res[p]
        for a, b in zip(r["corr"], ref["corr"]):
            assert np.array_equal(a, b), p
        assert np.array_equal(r["rec"], ref["rec"]), p  # one instantiation per group on every path
        assert np.array_equal(r["err"], ref["err"]), p
        assert r["lin_launches"] == len(KINDS) and r["err_launches"] == len(KINDS), p


@pytest.mark.parametrize("kind", KINDS)
def test_one_factor_set_paths_agree(g, scene, kind):
    fs = FactorSet([make_factor(g, scene, kind, 25001)])
    deltas, evals = seeded_poses(1, 22)
    res = run_paths(fs, deltas, evals)
    host, issue, dev = res["host"], res["issue"], res["device"]
    assert capi.unpack_linearized(host["rec"][0])["num_inliers"] > 1000
    for p in PATHS:
        assert np.array_equal(res[p]["corr"][0], host["corr"][0]), p
        assert res[p]["lin_launches"] == 1 and res[p]["err_launches"] == 1, p
    # host and issue both pass the pose by value (the ICP kinds have no such instantiation and take the staged path)
    assert np.array_equal(issue["rec"], host["rec"])
    assert np.array_equal(issue["err"], host["err"])
    if kind == "icp":
        assert np.array_equal(dev["rec"], host["rec"])
        assert np.array_equal(dev["err"], host["err"])
    else:
        assert_records_close(dev["rec"][0], host["rec"][0], TOL)
        assert abs(dev["err"][0] - host["err"][0]) <= TOL * abs(host["err"][0])


def test_error_before_linearize(g, scene):
    """issue_error / error_device need stored correspondences; b2_factor_set_error establishes them at the evaluation pose."""
    sizes = [700, 5000, 3000, 9000]
    fs = FactorSet([make_factor(g, scene, k, n) for k, n in zip(KINDS, sizes)])
    twin = FactorSet([make_factor(g, scene, k, n) for k, n in zip(KINDS, sizes)])
    _, evals = seeded_poses(len(sizes), 23)
    L = capi.lib()
    assert L.b2_factor_set_issue_error(fs.h, capi.dptr(evals), None) == B2_ERR_INVALID_STATE
    import torch

    d_in = torch.from_numpy(evals).cuda()
    d_out = torch.zeros(len(sizes), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    assert L.b2_factor_set_error_device(fs.h, d_in.data_ptr(), d_out.data_ptr()) == B2_ERR_INVALID_STATE
    assert fs.launches() == 0
    err = fs.err_host(evals)
    assert fs.launches() == len(KINDS)
    twin.lin_host(evals)
    for a, b in zip(fs.correspondences(), twin.correspondences()):
        assert np.array_equal(a, b)
    assert np.array_equal(err, twin.err_host(evals))


@pytest.mark.parametrize("kind", ["gicp", "ivox"])
def test_issue_linearize_honours_tolerance(g, scene, kind):
    """b2_factor_issue_linearize of a one-factor set (by-value pose) keeps the correspondences inside the correspondence-update
    tolerance, like b2_factor_linearize on a twin factor and, for GICP, like the oracle with the same setting."""
    import torch

    L = capi.lib()
    f, twin, fresh = (make_factor(g, scene, kind, 25001, flags=capi.B2_CLOUD_DEFAULT) for _ in range(3))
    for x in (f, twin):
        x.set_correspondence_update_tolerance(0.05, 0.5)
    rng = np.random.default_rng(8)
    d0 = syn.random_pose(rng, 0.01, 0.1)
    d1 = d0 @ syn.se3_exp(np.array([0.01, -0.01, 0.005, 0.05, -0.05, 0.02]))  # inside the tolerance of d0
    d_out = torch.zeros(capi.B2_LINEARIZED_DOUBLES, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    for d in (d0, d1):
        d = np.ascontiguousarray(d)
        capi.check(L.b2_factor_issue_linearize(f.h, capi.dptr(d), d_out.data_ptr()))
        capi.check(L.b2_factor_sync(f.h))
        twin.linearize({0: np.eye(4), 1: d})
    got = d_out.cpu().numpy()
    fresh.linearize({0: np.eye(4), 1: d1})
    corr = f.correspondences()
    assert np.array_equal(corr, twin.correspondences())
    assert not np.array_equal(corr, fresh.correspondences())  # re-associating at d1 would have changed them
    for k, v in capi.unpack_linearized(got).items():
        assert np.array_equal(v, twin._last[k]), k
    if kind == "gicp":
        otgt = orc.Cloud(scene["tp"], scene["tc"])
        of = orc.Factor(otgt, orc.Cloud(scene["sp"], scene["sc"]), tree=orc.KdTree(otgt, 4), num_threads=4)
        of.set_correspondence_update_tolerance(0.05, 0.5)
        of.linearize(d0)
        ref = of.linearize(d1)
        assert np.array_equal(corr, of.correspondences())
        assert_linearized_close(capi.unpack_linearized(got), ref)
