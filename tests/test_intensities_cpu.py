"""The intensity oracle (tests/intensity_oracle.cpp) against a plain numpy / Python restatement of the same rules: the Gaussian
voxel's running maximum under re-opening and LRU eviction, FlatContainer's per-slot intensities, voxelgrid_sampling's average and
merge_frames's maximum.  Inputs mix negative values, NaN, -0.0 and values that are not float32-exact."""
import math

import numpy as np
import pytest

import intensity_oracle as io


def same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def fast_floor(x):
    c = int(x)  # truncation, as the cast to int
    return c - (1 if x < float(c) else 0)


def std_max(a, b):
    return b if a < b else a


def awkward_intensities(rng, n):
    """Intensities that exercise every branch of the max rule: negatives, NaN, -0.0, +inf, non-float32-exact values."""
    x = rng.normal(0.0, 50.0, n)
    k = rng.integers(0, 6, n)
    x[k == 0] = np.nan
    x[k == 1] = -0.0
    x[k == 2] = -np.abs(x[k == 2])
    x[k == 3] = np.float32(x[k == 3]).astype(np.float64)
    x[rng.integers(0, n)] = np.inf
    return x


def batches(rng, num, n, extent):
    out = []
    for b in range(num):
        centre = rng.uniform(-extent, extent, 3) * (b % 3)  # later batches drift away, so old voxels age out
        out.append(centre + rng.uniform(-1.5, 1.5, (n, 3)))
    return out


class NpMap:
    """IncrementalVoxelMap in Python: first-touch ids, LRU eviction, GaussianVoxel / FlatContainer intensities."""

    def __init__(self, res, horizon, cycle, max_points=0, min_dist=0.1):
        self.inv, self.horizon, self.cycle, self.counter = 1.0 / res, horizon, cycle, 0
        self.max_points, self.min_sq = max_points, min_dist * min_dist
        self.voxels = []  # [coord, lru, intensity, points, ints]

    def insert(self, pts, ints):
        index = {tuple(v[0]): k for k, v in enumerate(self.voxels)}
        for i, p in enumerate(pts):
            c = tuple(fast_floor(float(p[a]) * self.inv) for a in range(3))
            if c not in index:
                index[c] = len(self.voxels)
                self.voxels.append([c, 0, 0.0, [], []])
            v = self.voxels[index[c]]
            v[1] = self.counter
            x = None if ints is None else float(ints[i])
            if not self.max_points:
                if x is not None:
                    v[2] = std_max(v[2], x)
            elif len(v[3]) < self.max_points:
                q = [float(t) for t in p[:3]]
                if all((((s[0] - q[0]) * (s[0] - q[0]) + (s[1] - q[1]) * (s[1] - q[1])) + (s[2] - q[2]) * (s[2] - q[2])) >= self.min_sq for s in v[3]):
                    v[3].append(q)
                    if x is not None:
                        v[4].append(x)
        self.counter += 1
        if self.counter % self.cycle == 0:
            self.voxels = [v for v in self.voxels if not v[1] + self.horizon < self.counter]


def key_of(p, inv):
    k = 0
    for r in range(3):
        x = float(p[r]) * inv
        if not math.isfinite(x):
            return None
        f = math.floor(x)
        if not (-1048576 <= f <= 1048575):
            return None
        k |= (f + (1 << 20)) << (21 * r)
    return k


@pytest.mark.parametrize("cycle", [1, 3, 10])
def test_gaussian_voxel_max_rule(cycle):
    rng = np.random.default_rng(cycle)
    orc, ref = io.Map(1.0, lru_horizon=2, lru_clear_cycle=cycle), NpMap(1.0, 2, cycle)
    for b, pts in enumerate(batches(rng, 9, 400, 4.0)):
        ints = None if b % 4 == 2 else awkward_intensities(rng, len(pts))  # a frame without intensities leaves every v as it is
        orc.insert(pts, ints)
        ref.insert(pts, ints)
        coords, v = orc.export()
        assert np.array_equal(coords, np.array([x[0] for x in ref.voxels], dtype=np.int32).reshape(-1, 3))
        assert same_bits(v, [x[2] for x in ref.voxels])
    assert np.all(v >= 0.0) and not np.any(np.isnan(v)) and not np.any(np.signbit(v))


def test_gaussian_voxel_reopen_and_order_independence():
    """A voxel re-opened by a later insert continues from its v; shuffling the points of a frame changes no v."""
    rng = np.random.default_rng(5)
    pts = rng.uniform(0.0, 2.0, (300, 3))
    ints = awkward_intensities(rng, 300)
    a, b = io.Map(1.0), io.Map(1.0)
    a.insert(pts[:150], ints[:150])
    a.insert(pts[150:], ints[150:])
    perm = rng.permutation(300)
    b.insert(pts[perm], ints[perm])
    ca, va = a.export()
    cb, vb = b.export()
    order = {tuple(c): k for k, c in enumerate(cb)}
    assert same_bits(va, vb[[order[tuple(c)] for c in ca]])
    # the max from 0 of the positive, non-NaN values of each voxel
    for c, v in zip(ca, va):
        sel = np.all(np.floor(pts).astype(int) == c, axis=1)
        xs = ints[sel]
        xs = xs[~np.isnan(xs)]
        assert v == max([0.0] + [x for x in xs if x > 0])


def test_flat_container_slots():
    rng = np.random.default_rng(7)
    orc, ref = io.Map(0.5, 3, 2, max_points_in_cell=5, min_dist_in_cell=0.05), NpMap(0.5, 3, 2, 5, 0.05)
    for pts in batches(rng, 7, 500, 2.0):
        ints = awkward_intensities(rng, len(pts))
        orc.insert(pts, ints)
        ref.insert(pts, ints)
        coords, counts, p, v = orc.export()
        assert np.array_equal(counts, [len(x[3]) for x in ref.voxels])
        assert same_bits(p, np.array([q for x in ref.voxels for q in x[3]]).reshape(-1, 3))
        assert same_bits(v, [q for x in ref.voxels for q in x[4]])
    assert counts.max() == 5


def test_voxelgrid_average():
    rng = np.random.default_rng(11)
    pts = rng.uniform(-3.0, 3.0, (2000, 3))
    pts[3] = np.nan  # dropped
    pts[4] = [1e7, 0.0, 0.0]  # outside the key range at resolution 0.5: dropped
    ints = rng.normal(0.0, 10.0, len(pts)) / 3.0  # not float32-exact
    ints[::7] = -0.0
    ints[::11] *= -1.0
    got = io.voxelgrid(pts, ints, 0.5)
    groups = {}
    for i, p in enumerate(pts):
        k = key_of(p, 1.0 / 0.5)
        if k is not None:
            groups.setdefault(k, []).append(i)
    want = []
    for k in sorted(groups):
        s = 0.0
        for i in groups[k]:
            s += float(ints[i])
        want.append(s / len(groups[k]))
    assert same_bits(got, want)


def test_merge_frames_max():
    rng = np.random.default_rng(13)
    pts = rng.uniform(-2.0, 2.0, (1500, 3))
    pts[0] = [1e9, 0.0, 0.0]  # cannot be keyed: keeps destination 0
    ints = awkward_intensities(rng, len(pts))
    ints[0] = 1e6  # and so raises voxel 0
    got = io.merge_frames(pts, ints, 0.25)
    keys = sorted({k for k in (key_of(p, 4.0) for p in pts) if k is not None})
    dest = {k: d for d, k in enumerate(keys)}
    want = [0.0] * len(keys)
    for p, x in zip(pts, ints):
        k = key_of(p, 4.0)
        d = 0 if k is None else dest[k]
        want[d] = std_max(want[d], float(x))
    assert same_bits(got, want)
    assert got[0] == 1e6
