"""The region-growing oracle (tests/segmentation_oracle.cpp) pinned without a GPU: its radius search against a brute force, its
clusters against scipy's directed reachability, its visit order and update-by-update flags against a plain-Python deque, and
the level-synchronous BFS with push counts -- the way the device computes region growing -- against the oracle's step-by-step
trace, converged flag and dilation timing included."""
import collections

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import breadth_first_order

import segmentation_oracle as so


def scene(seed, n=300, spread=3.0, flips=0.3):
    """Points in a box with normals near +z, a share of them tilted or flipped, so the angle test cuts edges."""
    rng = np.random.default_rng(seed)
    p = rng.uniform(-spread, spread, (n, 3)) * np.array([1.0, 1.0, 0.3])
    nr = np.tile([0.0, 0.0, 1.0], (n, 1)) + rng.normal(0, 0.15, (n, 3))
    tilt = rng.random(n) < flips
    nr[tilt] = rng.normal(0, 1, (tilt.sum(), 3))
    nr /= np.linalg.norm(nr, axis=1, keepdims=True)
    return p, nr


def lists(p, r, max_nn):
    """b2_kdtree_radius_search's lists, brute force in numpy: d2 = (dx dx + dy dy) + dz dz < r^2, by (d2, index), first max_nn."""
    out = []
    for q in p:
        d = p - q
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        idx = np.nonzero(d2 < r * r)[0]
        idx = idx[np.lexsort((idx, d2[idx]))]
        out.append(idx[:max_nn])
    return out


def accept(nr, i, j, cos_t):
    return not ((nr[i, 0] * nr[j, 0] + nr[i, 1] * nr[j, 1]) + nr[i, 2] * nr[j, 2] < cos_t)


class PyRegionGrowing:
    """A plain-Python restatement of region_growing_step_ / _update_ / _dilation_."""

    def __init__(self, p, nr, seed, dist, angle, dil, maxc):
        self.L, self.D = lists(p, dist, maxc), lists(p, dil, len(p))
        self.nr, self.cos_t, self.dil, self.maxc = nr, np.cos(angle), dil, maxc
        self.q, self.visited, self.cluster = collections.deque([seed]), np.zeros(len(p), bool), []

    def step(self):
        while True:
            if not self.q:
                return
            if len(self.cluster) > self.maxc:
                self.q.clear()
                return
            i = self.q.popleft()
            if not self.visited[i]:
                break
        self.visited[i] = True
        self.cluster.append(i)
        self.q.extend(j for j in self.L[i] if not self.visited[j] and accept(self.nr, i, j, self.cos_t))

    def update(self, max_steps):
        if not self.q:
            return True
        for _ in range(max_steps):
            if not self.q:
                break
            self.step()
        if not self.q and self.dil > 0:
            self.cluster = sorted(set(int(j) for i in self.cluster for j in self.D[i]))
        return not self.q


def level_bfs(p, nr, seed, dist, angle, maxc):
    """The device's algorithm on the host: O level by level (new points sorted by (parent rank, list position)), the pushes of every
    visit (accepted neighbours ranked after it, or never ranked), V and T = V + [a push follows the last visit's first push]."""
    L, cos_t, cap = lists(p, dist, maxc), np.cos(angle), maxc + 1
    rank, key, O = {seed: 0}, {}, [seed]
    pushes, base, end = [], 0, 1
    while base < end and base < cap:
        found = {}
        for s in range(base, min(end, cap)):
            c = 0
            for q, j in enumerate(L[O[s]]):
                j = int(j)
                if not accept(nr, O[s], j, cos_t) or rank.get(j, 1 << 62) <= s:
                    continue
                c += 1
                if j not in rank:
                    found[j] = min(found.get(j, (1 << 62, 0)), (s, q))
            pushes.append(c)
        for j in sorted(found, key=found.get):
            rank[j], key[j] = len(O), found[j]
            O.append(j)
        base, end = end, len(O)
    V = min(len(O), cap)
    lo, extra = 0, False
    if V > 1:
        s0, q0 = key[O[V - 1]]
        lo = s0 + 1
        extra = any(accept(nr, O[s0], int(j), cos_t) and rank.get(int(j), 1 << 62) > s0 for j in L[O[s0]][q0 + 1:])
    extra = extra or any(c > 0 for c in pushes[lo:V])
    return O[:V], V + int(extra)


CASES = [(s, d, a, m) for s in range(4) for d, a, m in [(0.8, 0.35, 10**6), (1.2, 0.6, 10**6), (0.8, np.pi, 10**6), (0.8, 0.0, 10**6), (1.0, 0.5, 25), (1.5, 3.0, 7)]]


def test_radius_grid_matches_brute():
    p, _ = scene(7, 500)
    for r in (0.0, 0.3, 1.0, 50.0):
        for q in (p[3], p[77], np.array([40.0, 0, 0])):
            assert np.array_equal(so.radius(p, q, r), so.radius(p, q, r, brute=True))
            d = p - q
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            idx = np.nonzero(d2 < r * r)[0]
            assert np.array_equal(so.radius(p, q, r, 5), idx[np.lexsort((idx, d2[idx]))][:5])


def test_nearest_is_brute_force():
    p, _ = scene(3)
    for q in (p[10] + 1e-3, np.array([100.0, -4, 2])):
        d = ((p - q) ** 2).sum(1)
        assert so.nearest(p, q) == int(np.argmin(d))


@pytest.mark.parametrize("seed", range(3))
def test_cluster_is_directed_reachability(seed):
    p, nr = scene(seed)
    dist, angle = 0.9, 0.4
    L, cos_t = lists(p, dist, len(p)), np.cos(angle)
    rows, cols = [], []
    for i, l in enumerate(L):
        for j in l:
            if j != i and accept(nr, i, j, cos_t):
                rows.append(i), cols.append(j)
    G = csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(len(p), len(p)))
    want = np.sort(breadth_first_order(G, 11, directed=True, return_predecessors=False))
    rg = so.RegionGrowing(p, nr, 11, dist, angle, 0.0)
    assert rg.update()
    assert np.array_equal(np.sort(rg.cluster_indices), want)


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_python_deque(case):
    s, d, a, m = case
    p, nr = scene(s)
    for steps in ([10**6], [1] * 400, [3, 0, -2, 5, 17, 1, 1, 1000, 1]):
        py = PyRegionGrowing(p, nr, 5, d, a, 0.4, m)
        got = so.trace(p, nr, 5, steps, distance_threshold=d, angle_threshold=a, dilation_radius=0.4, max_cluster_size=m)
        for st, (conv, cl) in zip(steps, got):
            assert py.update(st) == conv
            assert np.array_equal(np.asarray(py.cluster, dtype=np.int64), cl)


@pytest.mark.parametrize("case", CASES)
def test_level_bfs_gives_the_step_trace(case):
    """One step at a time, the oracle visits O[t] at step t + 1, and converges exactly at step T, with the dilation then."""
    s, d, a, m = case
    p, nr = scene(s)
    O, T = level_bfs(p, nr, 5, d, a, m)
    rg = so.RegionGrowing(p, nr, 5, d, a, 0.0, m)
    for t in range(T):
        assert np.array_equal(rg.cluster_indices, np.asarray(O[:t], dtype=np.int64))
        assert rg.update(1) == (t + 1 == T)
    assert np.array_equal(rg.cluster_indices, np.asarray(O, dtype=np.int64))
    dil = so.RegionGrowing(p, nr, 5, d, a, 0.4, m)
    assert not dil.update(T - 1)
    assert np.array_equal(dil.cluster_indices, np.asarray(O[: T - 1], dtype=np.int64))
    assert dil.update(1)
    want = np.unique(np.concatenate([lists(p, 0.4, len(p))[i] for i in O]))
    assert np.array_equal(dil.cluster_indices, want)


def test_stale_duplicates_delay_the_flag_and_the_dilation():
    """Cases where the last visit leaves stale entries: the visits are done after V steps, but converged is False until one more
    step drains the queue, and only that call dilates."""
    seen = 0
    for s, d, a, m in CASES:
        p, nr = scene(s)
        O, T = level_bfs(p, nr, 5, d, a, m)
        if T == len(O):
            continue
        seen += 1
        rg = so.RegionGrowing(p, nr, 5, d, a, 0.4, m)
        assert not rg.update(len(O))
        assert np.array_equal(rg.cluster_indices, np.asarray(O, dtype=np.int64))
        assert rg.update(0) is False and rg.update(1)
        assert len(rg.cluster_indices) >= len(O) and np.all(np.diff(rg.cluster_indices) > 0)
    assert seen >= 3


def test_cap_and_edges():
    p, nr = scene(1)
    O, T = level_bfs(p, nr, 5, 1.5, 3.0, 7)
    assert len(O) == 8 and T == 9  # the cluster reaches max_cluster_size + 1, and one more step clears the queue
    empty = so.RegionGrowing(np.zeros((0, 3)), np.zeros((0, 3)), -1)
    assert empty.update(5) and len(empty.cluster_indices) == 0
    lone = np.vstack([p, [[100.0, 100.0, 100.0]]]), np.vstack([nr, [[0.0, 0.0, 1.0]]])
    rg = so.RegionGrowing(*lone, len(p), 0.8, 0.3, 0.0)
    assert rg.update(1) and np.array_equal(rg.cluster_indices, [len(p)])
