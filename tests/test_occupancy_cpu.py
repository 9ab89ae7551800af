"""The CPU oracle of the occupancy grid and the voxel raycaster (tests/occupancy_oracle.cpp) pinned to plain models: the grid to a numpy
set of cell keys, the raycaster to a plain-Python restatement of VoxelRaycaster bit for bit, and both to the reference test's gates
(src/test/test_voxel_raycaster.cpp: RandomTest against naive_ray_traversal, CornerTest)."""
import math

import numpy as np
import pytest

import occupancy_oracle as oo

INF = float("inf")


def np_pose(points, T):
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    if T is None:
        return p.copy()
    T = np.asarray(T, dtype=np.float64)
    return np.stack([((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(3)], 1)


def np_cells(points, res, T=None):
    """The occupied cells of a grid holding `points` posed by T: the set of floor(q * (1 / res)) inside [-2^20, 2^20 - 1]."""
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor(np_pose(points, T) * (1.0 / res))
        keep = np.all((f >= -(2**20)) & (f <= 2**20 - 1), axis=1)
    return {tuple(int(v) for v in c) for c in f[keep]}


def key_order(cells):
    a = np.array(sorted(cells), dtype=np.int64).reshape(-1, 3)
    return a[np.lexsort((a[:, 0], a[:, 1], a[:, 2]))].astype(np.int32) if len(a) else a.astype(np.int32)


def py_ray(s, e, vs):
    """VoxelRaycaster, begin() up to end_voxel() excluded, in plain Python floats (each operation rounded on its own)."""
    eps = 1e-9
    inv = 1.0 / vs
    c = [math.floor(float(x) * inv) for x in s]
    ec = [math.floor(float(x) * inv) for x in e]
    d = [float(e[a]) - float(s[a]) for a in range(3)]
    step = [(x > 0) - (x < 0) for x in d]
    valid = [abs(x) > eps for x in d]
    td = [vs / abs(d[a]) if valid[a] else INF for a in range(3)]
    tm = [((float(c[a]) + (1.0 if step[a] > 0 else 0.0)) * vs - float(s[a])) / d[a] if valid[a] else INF for a in range(3)]
    out = []
    while c != ec:
        out.append(tuple(c))
        m = 0 if tm[0] < tm[1] and tm[0] < tm[2] else (1 if tm[1] < tm[2] else 2)
        if tm[m] > 1.0 + eps:
            break
        c[m] += step[m]
        tm[m] += td[m]
        if any((step[a] > 0 and c[a] > ec[a]) or (step[a] < 0 and c[a] < ec[a]) for a in range(3)):
            break
    return out


def oracle_rows(s, e, vs):
    off, coords = oo.raycast(s, e, vs)
    return [[tuple(int(v) for v in r) for r in coords[off[i]:off[i + 1]]] for i in range(len(s))]


def face_points(res, rng):
    """Points exactly on cell faces, on block boundaries (multiples of 8 cells), negative coordinates and small offsets around them."""
    k = np.arange(-40, 41, dtype=np.float64)
    on = k * res
    base = np.stack(np.meshgrid(on[::3], on[::4], on[::5], indexing="ij"), -1).reshape(-1, 3)
    near = base + rng.choice([-1e-12, 0.0, 1e-12, 0.5 * res], size=base.shape)
    return np.concatenate([base, near, rng.uniform(-30 * res, 30 * res, (3000, 3))])


@pytest.mark.parametrize("res", [0.1, 0.25, 0.3, 0.5, 1.0, 2.5])
def test_grid_is_a_set_of_keys(res):
    rng = np.random.default_rng(int(res * 1000))
    pts = face_points(res, rng)
    grid = oo.Grid(res)
    grid.insert(pts)
    want = np_cells(pts, res)
    assert grid.num_occupied_cells() == len(want)
    assert np.array_equal(grid.cells(), key_order(want))
    q = np.concatenate([pts[::3] + rng.normal(0, res, pts[::3].shape), pts[::5]])
    count, flags = grid.overlaps(q)
    member = np.array([tuple(int(v) for v in c) in want for c in np.floor(q * (1.0 / res))], dtype=np.uint8)
    assert np.array_equal(flags, member) and count == int(member.sum())


def test_grid_posed_incremental_and_rehash():
    """Incremental inserts under poses grow the reference's 512-entry table by rehash; the set stays the union of the keys."""
    rng = np.random.default_rng(2)
    res = 0.2
    grid, want = oo.Grid(res), set()
    for _ in range(4):
        th = rng.uniform(-np.pi, np.pi)
        T = np.eye(4)
        T[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
        T[:3, 3] = rng.uniform(-20, 20, 3)
        pts = rng.uniform(-15, 15, (20000, 3))
        grid.insert(pts, T)
        want |= np_cells(pts, res, T)
        assert np.array_equal(grid.cells(), key_order(want))
    assert grid.table_size() > 512


def test_grid_key_range_and_non_finite():
    res = 0.5
    lim = 2.0**20 * res
    pts = np.array([[lim - 0.25, 0, 0], [lim, 0, 0], [-lim, 0, 0], [-lim - 1e-6, 0, 0], [1e300, 0, 0], [0, 0, -1e300]])
    grid = oo.Grid(res)
    grid.insert(pts)
    assert np.array_equal(grid.cells(), key_order({(2**20 - 1, 0, 0), (-(2**20), 0, 0)}))
    T = np.eye(4)
    T[:3, :3] *= 1e308
    _, flags = grid.overlaps(pts, T)
    assert flags.tolist() == [0, 0, 0, 0, 0, 0]  # every posed coordinate overflows or leaves the range
    grid.insert(pts, T)
    assert grid.num_occupied_cells() == 2


def test_free_rays_is_set_free_along_the_raycaster():
    rng = np.random.default_rng(4)
    res = 0.5
    occ = rng.uniform(-10, 10, (4000, 3))
    scan = rng.uniform(-12, 12, (300, 3))
    T = np.eye(4)
    T[:3, 3] = [0.3, -0.7, 0.2]
    grid = oo.Grid(res)
    grid.insert(occ)
    grid.free_rays(scan, T)
    want = np_cells(occ, res)
    origin = T[:3, 3]
    for q in np_pose(scan, T):
        want -= set(py_ray(origin, q, res))
    assert np.array_equal(grid.cells(), key_order(want))
    # clearing never creates a block, and frees nothing where nothing is occupied
    empty = oo.Grid(res)
    empty.free_rays(scan, T)
    assert empty.num_occupied_cells() == 0 and empty.table_size() == 512


def random_rays(rng, n, lo, hi):
    return rng.uniform(lo, hi, (n, 3)), rng.uniform(lo, hi, (n, 3))


def edge_rays():
    rows = [
        ([0.5, 0.5, 0.5], [10.5, 0.5, 0.5]), ([0.5, 0.5, 0.5], [0.5, -10.5, 0.5]), ([0.0, 0.0, 0.0], [5.0, 5.0, 5.0]), ([0.0, 0.0, 0.0], [-5.0, -5.0, 0.0]),
        ([1.0, 1.0, 1.0], [-3.0, 2.0, -3.0]), ([0.25, 0.25, 0.25], [0.25, 0.25, 0.25]), ([0.25, 0.25, 0.25], [0.25 + 1e-10, 0.25, 0.25]),
        ([0.9999999999, 0.2, 0.2], [1.0000000001, 0.2, 0.2]), ([1 - 2e-10, 0.5, 0.5], [1 + 3e-10, 3.5, 0.5]), ([-0.5, -0.5, -0.5], [-10.0, -0.5, -3.0]),
        ([0.1, 0.2, 0.3], [0.1, 0.2, -1.7]), ([-1e-300, 0, 0], [1e-300, 0, 0]),
    ]
    return np.array([r[0] for r in rows]), np.array([r[1] for r in rows])


@pytest.mark.parametrize("vs", [0.1, 0.25, 0.5, 1.0, 2.5])
def test_raycaster_is_the_python_restatement(vs):
    rng = np.random.default_rng(int(vs * 100))
    s, e = random_rays(rng, 400, -25, 25)
    es, ee = edge_rays()
    s, e = np.concatenate([s, es]), np.concatenate([e, ee])
    got = oracle_rows(s, e, vs)
    for i in range(len(s)):
        assert got[i] == py_ray(s[i], e[i], vs), i


def test_random_gate():
    """RandomTest on the reference test's own rays: rows of up to 20 voxels equal naive_ray_traversal exactly, longer rows differ as
    sets by under 2.5 %."""
    rays, _ = oo.reference_test_rays()
    for k, res in enumerate(np.repeat([0.1, 0.5, 1.0, 2.5, 5.0], 25)):
        s, e = rays[k, :3], rays[k, 3:]
        ray = oracle_rows(s[None], e[None], res)[0]
        assert ray == py_ray(s, e, res)
        naive = [tuple(int(v) for v in c) for c in oo.naive_ray(s, e, res)]
        if len(ray) > 20:
            a, b = set(ray), set(naive)
            assert 1.0 - len(a & b) / max(len(a), len(b)) < 0.025, (res, len(a), len(b))
        else:
            assert ray == naive, (res, s, e)


def test_random_rays_near_the_naive_traversal():
    """Other random rays: the naive 1e-4 stepping can miss a voxel the segment only clips near an edge, so here every row, short or
    long, is held to the set gate (under 2.5 % disagreement, or one voxel for short rows)."""
    rng = np.random.default_rng(0)
    for res in (0.1, 0.5, 1.0, 2.5, 5.0):
        for _ in range(25):
            s, e = rng.uniform(-10, 10, 3), rng.uniform(-10, 10, 3)
            a = set(oracle_rows(s[None], e[None], res)[0])
            b = {tuple(int(v) for v in c) for c in oo.naive_ray(s, e, res)}
            assert len(a ^ b) <= max(2, 0.05 * max(len(a), len(b))), (res, len(a), len(b))


def test_corner_gate():
    """CornerTest on the reference test's rays: a ray from a point to itself, and rays inside one unit voxel, are empty."""
    _, rays = oo.reference_test_rays()
    off, _ = oo.raycast(rays[:100, :3], rays[:100, 3:], 0.25)
    assert np.all(off == 0)
    off, _ = oo.raycast(rays[100:, :3], rays[100:, 3:], 1.0)
    assert np.all(off == 0)


def test_quirks():
    # the end voxel is excluded: a ray over three unit voxels visits the first two
    assert oracle_rows(np.array([[0.5, 0.5, 0.5]]), np.array([[2.5, 0.5, 0.5]]), 1.0)[0] == [(0, 0, 0), (1, 0, 0)]
    # start voxel == end voxel gives an empty row, however long the segment inside it
    assert oracle_rows(np.array([[0.01, 0.01, 0.01]]), np.array([[0.99, 0.99, 0.99]]), 1.0)[0] == []
    # an axis with |d| <= 1e-9 never steps, even when its end coordinate differs: the walk ends on t_max > 1 + 1e-9
    row = oracle_rows(np.array([[1 - 2e-10, 0.5, 0.5]]), np.array([[1 + 3e-10, 3.5, 0.5]]), 1.0)[0]
    assert row == [(0, 0, 0), (0, 1, 0), (0, 2, 0), (0, 3, 0)]
    # ... while |d| just above 1e-9 is a valid axis and steps
    row = oracle_rows(np.array([[1 - 1e-9, 0.5, 0.5]]), np.array([[1 + 1e-9, 3.5, 0.5]]), 1.0)[0]
    assert row == [(0, 0, 0), (0, 1, 0), (1, 1, 0), (1, 2, 0)]
    # a tie in the minimum-axis rule picks the later axis (strict <): through a cell corner z steps before x and y
    row = oracle_rows(np.array([[0.5, 0.5, 0.5]]), np.array([[2.5, 2.5, 2.5]]), 1.0)[0]
    assert row[:2] == [(0, 0, 0), (0, 0, 1)]
