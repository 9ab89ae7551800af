"""Voxel maps whose bucket table has long probe chains, one of them wrapping from the last bucket group to group 0.

At load <= 0.25 about 95 % of lookups end in the home group, so the overflow walk -- in lookup_voxel, and written again inline
in the VGICP probe warps -- runs only by chance on random clouds, and its wrap-around probably never.  Here the voxel
coordinates are chosen through a numpy replica of voxel_hash (checked against the header itself on the CPU) so that about
40 voxels share the last group as home, and 40 more share a group in the middle.  Every map is sized by the library itself
(load <= 0.25), so every chain ends in a group with an empty slot.  Lookups (hits and misses), VGICP correspondences through
both kernel forms, overlap, re-insert, LRU rebuild, from_voxels, load(save_compact) and the iVox (mode 27) are compared
with the oracle / the iVox restatement bit for bit.
"""
import os
import subprocess

import numpy as np
import pytest

import ivox_np
import oracle_lib as orc
from gtsam_points_b200 import capi
from test_gpu_parity import assert_linearized_close

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEAF = 0.5
CHAIN = 40
NUM_ORDINARY = 3000


def voxel_hash(x, y, z):
    """numpy replica of b2::voxel_hash (gtsam_points_b200/csrc/b2_device.cuh): uint32 arithmetic, wrapping."""
    u = lambda v: np.asarray(v, dtype=np.int64).astype(np.uint32)
    with np.errstate(over="ignore"):
        h = (u(x) * np.uint32(0x8DA6B343)) ^ (u(y) * np.uint32(0xD8163841)) ^ (u(z) * np.uint32(0xCB1AB31F))
        h ^= h >> np.uint32(15)
        h *= np.uint32(0x2C1B3C6D)
        h ^= h >> np.uint32(12)
    return h


def groups_for(num_voxels):
    """Bucket groups of a table over num_voxels voxels: next_pow2(max(64, 4 V)) buckets of 16 bytes, 2 per group."""
    nb = 64
    while nb < 4 * num_voxels:
        nb *= 2
    return nb // 2


def test_voxel_hash_replica_matches_header(tmp_path):
    """Compiles a host-only stub around b2_device.cuh (no GPU needed) and compares its voxel_hash with the replica."""
    from gtsam_points_b200 import build

    stub = tmp_path / "hash_stub.cu"
    stub.write_text(
        '#include <cstdio>\n#include "b2_device.cuh"\n'
        "int main() { int x, y, z; while (std::scanf(\"%d %d %d\", &x, &y, &z) == 3) std::printf(\"%u\\n\", b2::voxel_hash(x, y, z)); return 0; }\n"
    )
    exe = tmp_path / "hash_stub"
    subprocess.run([build.NVCC, "-ccbin", build.HOST_CXX, "-std=c++17", "-I", build.CSRC, "-I", os.path.join(ROOT, "include"), str(stub), "-o", str(exe)],
                   check=True, capture_output=True)
    rng = np.random.default_rng(0)
    keys = np.concatenate([
        rng.integers(-(2**31), 2**31, (3000, 3)),
        rng.integers(-300, 300, (900, 3)),
        np.array([[-(2**31), 2**31 - 1, 0], [2**31 - 1, -(2**31), -1], [0, 0, 0], [-1, -1, -1]] * 25),
    ])
    out = subprocess.run([str(exe)], input="\n".join(" ".join(str(int(v)) for v in k) for k in keys), capture_output=True, text=True, check=True).stdout
    assert np.array_equal(np.array(out.split(), dtype=np.uint64), voxel_hash(keys[:, 0], keys[:, 1], keys[:, 2]).astype(np.uint64))
    assert len(keys) == 4000


def chained_coords(G, seed=0):
    """Ordinary voxels plus two chains: CHAIN voxels whose home group is the last one (the walk wraps to groups 0, 1, ...)
    and CHAIN whose home group is G / 2; also absent keys homed in those chains (misses that walk them)."""
    rng = np.random.default_rng(seed)
    cand = np.unique(rng.integers(-400, 400, (2_000_000, 3)), axis=0)
    cand = cand[rng.permutation(len(cand))]
    home = voxel_hash(cand[:, 0], cand[:, 1], cand[:, 2]) & np.uint32(G - 1)
    last = cand[home == G - 1]
    mid = cand[home == G // 2]
    wrapped = cand[home < 4]  # groups the last chain spills into
    assert len(last) >= CHAIN + 10 and len(mid) >= CHAIN + 10 and len(wrapped) >= 20
    chain = np.concatenate([last[:CHAIN], mid[:CHAIN]])
    used = {tuple(c) for c in chain}
    ordinary = [c for c in cand[: NUM_ORDINARY + 200] if tuple(c) not in used][:NUM_ORDINARY]
    used |= {tuple(c) for c in ordinary}
    misses = np.array([c for c in np.concatenate([last[CHAIN:], mid[CHAIN:], wrapped]) if tuple(c) not in used])
    return chain, np.array(ordinary), misses


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


@pytest.fixture(scope="module")
def scene():
    G = groups_for(2 * CHAIN + NUM_ORDINARY)
    chain, ordinary, misses = chained_coords(G)
    rng = np.random.default_rng(1)
    coords = np.concatenate([chain[:CHAIN], ordinary[: NUM_ORDINARY // 2], chain[CHAIN:], ordinary[NUM_ORDINARY // 2 :]])
    rng.shuffle(coords)
    centres = (coords + 0.5) * LEAF
    covs = np.tile(np.diag([0.01, 0.02, 0.015]), (len(coords), 1, 1)) + 0.004 * rng.uniform(0, 1, (len(coords), 1, 1)) * np.ones((3, 3))
    # source: near the centres of every chained voxel and of some ordinary ones, well inside (no face effects)
    from gtsam_points_b200 import synthetic as syn

    T = syn.random_pose(rng, 0.2, 2.0)
    src_voxels = np.concatenate([chain, ordinary[:1500]])
    near = np.concatenate([np.repeat((chain + 0.5) * LEAF, 8, axis=0), (ordinary[:1500] + 0.5) * LEAF])
    q = near + rng.uniform(-0.3, 0.3, near.shape) * LEAF
    p = (q - T[:3, 3]) @ T[:3, :3]
    scov = np.tile(np.diag([0.02, 0.01, 0.03]), (len(p), 1, 1))
    ovm = orc.VoxelMap(LEAF)
    ovm.insert(orc.Cloud(centres, covs))
    return dict(G=G, chain=chain, src_voxels=src_voxels, misses=misses, coords=coords, centres=centres, covs=covs, T=T, p=p, scov=scov, ovm=ovm)


def lookup_points(s):
    return np.concatenate([s["centres"], (s["misses"] + 0.5) * LEAF])


def check_map(g, vm, ovm, s):
    assert vm.info().num_buckets // 2 == s["G"]
    got, ref = vm.download(), ovm.export()
    for k in ("coords", "n", "means", "covs"):
        assert np.array_equal(got[k], ref[k]), k
    q = lookup_points(s)
    idx = vm.lookup_voxel_index(q)
    assert np.array_equal(idx, ovm.lookup(q))
    assert (idx[len(s["centres"]) :] == -1).all() and (idx[: len(s["centres"])] >= 0).all()


def check_vgicp(g, vm, ovm, s):
    values = {0: np.eye(4), 1: s["T"]}
    f = g.IntegratedVGICPFactor(0, 1, vm, g.PointCloud(s["p"], s["scov"]))
    of = orc.Factor(ovm, orc.Cloud(s["p"], s["scov"]))
    f.linearize(values)  # one-factor set: pose by value
    ref = of.linearize(s["T"])
    assert ref["num_inliers"] == len(s["p"])
    assert np.array_equal(f.correspondences(), of.correspondences())
    assert_linearized_close(f._last, ref)
    n = len(s["p"]) // 3
    parts = [(s["p"][:n], s["scov"][:n]), (s["p"][n:], s["scov"][n:])]
    factors = [g.IntegratedVGICPFactor(0, 1, vm, g.PointCloud(pp, cc)) for pp, cc in parts]
    fs = g.NonlinearFactorSetGPU()
    fs.add(factors)
    out = fs.linearize(values)  # multi-factor set: pose from device memory
    assert np.array_equal(np.concatenate([x.correspondences() for x in factors]), of.correspondences())
    for (pp, cc), rec in zip(parts, out):
        assert_linearized_close(capi.unpack_linearized(rec), orc.Factor(ovm, orc.Cloud(pp, cc)).linearize(s["T"]))
    src = g.PointCloud(s["p"], s["scov"])
    assert g.overlap_gpu(vm, src, s["T"]) == ovm.overlap(orc.Cloud(s["p"], s["scov"]), s["T"]) == 1.0


@pytest.mark.gpu
def test_chains_insert_lookup_vgicp(g, scene):
    s = scene
    vm = g.GaussianVoxelMapGPU(LEAF)
    vm.insert(g.PointCloud(s["centres"], s["covs"]))
    check_map(g, vm, s["ovm"], s)
    check_vgicp(g, vm, s["ovm"], s)
    # a second insert into the chained voxels: existing voxels are found through the walk, none is duplicated
    again = (np.repeat(s["chain"], 2, axis=0) + 0.5 + np.tile([[0.2, -0.2, 0.1], [-0.1, 0.15, -0.2]], (len(s["chain"]), 1))) * LEAF
    acov = np.tile(np.diag([0.03, 0.01, 0.02]), (len(again), 1, 1))
    ovm = orc.VoxelMap(LEAF)
    ovm.insert(orc.Cloud(s["centres"], s["covs"]))
    vm.insert(g.PointCloud(again, acov))
    ovm.insert(orc.Cloud(again, acov))
    assert vm.num_voxels == len(s["coords"])
    check_map(g, vm, ovm, s)
    check_vgicp(g, vm, ovm, s)


@pytest.mark.gpu
def test_chains_after_lru_rebuild(g, scene):
    """lru (1, 2): the second insert touches the chains, the voxels the source sees and some more; the sweep drops the rest
    and rebuilds the table at the same size, so the chains are rebuilt too."""
    s = scene
    vm = g.GaussianVoxelMapGPU(LEAF)
    vm.set_lru(1, 2)
    ovm = orc.VoxelMap(LEAF)
    ovm.set_lru(1, 2)
    keep = np.isin(np.arange(len(s["coords"])), np.random.default_rng(3).permutation(len(s["coords"]))[:2700])
    seen = {tuple(c) for c in s["src_voxels"]}
    keep |= np.array([tuple(c) in seen for c in s["coords"]])
    for pts, cv in ((s["centres"], s["covs"]), (s["centres"][keep], s["covs"][keep])):
        vm.insert(g.PointCloud(pts, cv))
        ovm.insert(orc.Cloud(pts, cv))
    assert vm.num_voxels == keep.sum() < len(s["coords"])
    got, ref = vm.download(), ovm.export()
    for k in ("coords", "n", "means", "covs"):
        assert np.array_equal(got[k], ref[k]), k
    assert vm.info().num_buckets // 2 == s["G"]
    q = lookup_points(s)
    assert np.array_equal(vm.lookup_voxel_index(q), ovm.lookup(q))
    check_vgicp(g, vm, ovm, s)


@pytest.mark.gpu
def test_chains_from_voxels_and_load(g, scene, tmp_path):
    s = scene
    ex = s["ovm"].export()
    vm = g.GaussianVoxelMapGPU.from_voxels(LEAF, ex["coords"], ex["means"], ex["covs"], ex["n"])
    check_map(g, vm, s["ovm"], s)
    check_vgicp(g, vm, s["ovm"], s)
    path = tmp_path / "chained.bin"
    s["ovm"].save_compact(path)
    loaded = g.GaussianVoxelMapGPU.load(path)
    oloaded = orc.VoxelMap.load(path)
    check_map(g, loaded, oloaded, s)
    check_vgicp(g, loaded, oloaded, s)


@pytest.mark.gpu
def test_chains_ivox(g, scene):
    s = scene
    dev = g.iVox(LEAF)
    dev.set_neighbor_voxel_mode(27)
    ref = ivox_np.IvoxNp(LEAF)
    ref.mode = 27
    for m in (dev, ref):
        m.insert(s["centres"], s["covs"])
    assert np.array_equal(dev.download()["coords"], ref.export()["coords"])
    q = np.concatenate([ivox_np.transform(s["T"], s["p"]), (s["misses"] + 0.5) * LEAF])
    idx, sqd = dev.knn_search(q, 1, 1.0)
    want = [ref.knn(x, 1, 1.0) for x in q]
    assert np.array_equal(idx[:, 0], np.array([w[0][0] for w in want]))
    assert np.array_equal(sqd[:, 0], np.array([w[1][0] for w in want]))
    f = g.IntegratedGICPFactor(np.eye(4), 1, dev, g.PointCloud(s["p"], s["scov"]))
    rf = ivox_np.GicpIvoxNp(ref, s["p"], s["scov"])
    f.linearize({1: s["T"]})
    rl = rf.linearize(s["T"])
    assert np.array_equal(f.correspondences(), rf.corr)
    assert (rf.corr >= 0).all()
    assert_linearized_close(f._last, rl)
