"""The min-cut oracle (tests/segmentation_oracle.cpp) pinned without a GPU: its integer Dinic flow and minimal source set against
scipy's maximum_flow on a coarser quantum and against a brute-force minimum cut on tiny networks; the foreground arcs change
nothing; NaN weights give capacity 0."""
import itertools

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import breadth_first_order, maximum_flow

import segmentation_oracle as so


def scene(seed, n=150):
    rng = np.random.default_rng(seed)
    p = rng.uniform(-2.5, 2.5, (n, 3)) * np.array([1.0, 1.0, 0.4])
    nr = np.tile([0.0, 0.0, 1.0], (n, 1)) + rng.normal(0, 0.4, (n, 3))
    nr /= np.linalg.norm(nr, axis=1, keepdims=True)
    return p, nr


def arcs(p, s, t, idx, q, br, qb):
    """Every arc (u, v, c) of the network with integer capacities, self arcs dropped, parallel arcs summed."""
    A = {}
    n, k = idx.shape
    d = np.sqrt(((p - p[s]) ** 2).sum(1))
    for i in range(n):
        for a in range(k):
            if q[i, a] >= 0 and idx[i, a] != i:
                A[(i, int(idx[i, a]))] = A.get((i, int(idx[i, a])), 0) + int(q[i, a])
        if i != t and d[i] > br:
            A[(i, t)] = A.get((i, t), 0) + qb
    return A


@pytest.mark.parametrize("seed", range(4))
def test_dinic_against_scipy_maximum_flow(seed):
    p, nr = scene(seed)
    t, idx, w, q = so.mc_network(p, nr, 0, k=8, distance_sigma=0.6, angle_sigma=0.5, background_mask_radius=1.5)
    assert t > 0
    qc = np.where(q < 0, -1, np.floor(np.nan_to_num(w) * 2**16 + 0.5)).astype(np.int64)  # a quantum of 2^-16 keeps scipy's int32 sums exact
    flow, S = so.mc_flow(p, 0, t, idx, qc, 1.5, 0.2, quantum=2.0**16)
    A = arcs(p, 0, t, idx, qc, 1.5, int(np.floor(0.2 * 2**16 + 0.5)))
    u, v = np.array([a[0] for a in A]), np.array([a[1] for a in A])
    G = csr_matrix((np.array(list(A.values()), dtype=np.int32), (u, v)), shape=(len(p), len(p)))
    r = maximum_flow(G, 0, t)
    assert r.flow_value == flow
    R = (G - r.flow).tocsr()  # residual: capacity - flow (flow is antisymmetric)
    R.data = (R.data > 0).astype(np.int32)
    R.eliminate_zeros()
    assert np.array_equal(np.sort(breadth_first_order(R, 0, directed=True, return_predecessors=False)), S)


def test_dinic_against_brute_force_on_tiny_networks():
    for seed in range(6):
        p, nr = scene(10 + seed, n=9)
        t, idx, w, q = so.mc_network(p, nr, 0, k=3, distance_sigma=1.0, angle_sigma=0.8, background_mask_radius=1.0)
        if t < 0:
            continue
        qb = 12345
        flow, S = so.mc_flow(p, 0, t, idx, q, 1.0, qb / 2**32)
        A = arcs(p, 0, t, idx, q, 1.0, qb)
        best, sets = None, []
        others = [i for i in range(9) if i not in (0, t)]
        for bits in itertools.product([0, 1], repeat=len(others)):
            X = {0} | {o for o, b in zip(others, bits) if b}
            c = sum(cap for (a, b), cap in A.items() if a in X and b not in X)
            if best is None or c < best:
                best, sets = c, [X]
            elif c == best:
                sets.append(X)
        assert flow == best
        assert set(S.tolist()) == set.intersection(*sets)  # the minimal minimum-cut source set


def test_foreground_arcs_change_nothing():
    for seed in range(4):
        p, nr = scene(seed)
        t, idx, w, q = so.mc_network(p, nr, 3, k=10, distance_sigma=0.5, angle_sigma=0.4, background_mask_radius=1.5)
        a = so.mc_flow(p, 3, t, idx, q, 1.5, 0.2)
        b = so.mc_flow(p, 3, t, idx, q, 1.5, 0.2, foreground_mask_radius=1.0, foreground_weight=5.0)
        assert a[0] == b[0] and np.array_equal(a[1], b[1])


def test_nan_weights_are_capacity_zero():
    """Exactly coplanar unit normals can round |n_i . n_j| above 1: acos gives NaN, the capacity is 0."""
    rng = np.random.default_rng(1)
    p = np.c_[rng.uniform(0, 2, (200, 2)), np.zeros(200)]
    v = rng.normal(0, 1, 3)
    v /= np.linalg.norm(v)
    nr = np.tile(v, (200, 1))
    t, idx, w, q = so.mc_network(p, nr, 0, k=6, background_mask_radius=1.0)
    dot = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
    if abs(dot) > 1.0:
        assert np.isnan(w).all() and (q == 0).all()
    else:
        assert not np.isnan(w).any()
    assert (q[np.isnan(w)] == 0).all()
