"""The CPU oracle of the frame filters (tests/filter_oracle.cpp) against plain-Python / numpy restatements of include/b2points.h's
rules, the priority stream's test vectors, the distribution of the random samplers, and the reference's quirks at the edges."""
import math

import numpy as np
import pytest

import filter_oracle as fo
import preprocess_cases as pc

SCANS = pc.scans()
M64 = 2**64 - 1


def py_priority(seed, i, s):
    z = (seed + (2 * i + s + 1) * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def py_smallest(idx, m, seed, s):
    return [i for _, i in sorted((py_priority(seed, i, s), i) for i in idx)[:m]]


def py_random_sampling(n, rate, seed):
    if rate >= 0.99:
        return list(range(n))
    return sorted(py_smallest(range(n), int(n * rate), seed, 0))


def py_key(p, inv):
    key = 0
    for a in range(3):
        q = float(p[a]) * inv
        if not math.isfinite(q):
            return None
        c = math.floor(q) + 2**20
        if c < 0 or c > 2**21 - 1:
            return None
        key |= c << (21 * a)
    return key


def py_voxels(points, resolution):
    inv = 1.0 / resolution
    voxels = {}
    for i, p in enumerate(points):
        key = py_key(p, inv)
        if key is not None:
            voxels.setdefault(key, []).append(i)
    return voxels


def py_randomgrid(points, resolution, rate, seed, apply_cap=True):
    n = len(points)
    if rate >= 0.99:
        return list(range(n))
    voxels = py_voxels(points, resolution)
    if not voxels:
        return []
    ppv = int(math.ceil((rate * n) / len(voxels)))
    kept = [i for key in sorted(voxels) for i in py_smallest(voxels[key], ppv, seed, 0)]
    cap = int((n * rate) * 1.2)
    if apply_cap and len(kept) > cap:
        kept = py_smallest(kept, cap, seed, 1)
    return sorted(kept)


def np_mean_knn_dists(points, k):
    """Brute force in numpy: every pair's ((dx dx + dy dy) + dz dz), the k smallest per row, sqrt summed in ascending order."""
    p = np.asarray(points, dtype=np.float64)[:, :3]
    d = [p[None, :, a] - p[:, None, a] for a in range(3)]
    sq = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
    sq.sort(axis=1)
    s = np.zeros(len(p))
    for j in range(k):
        s = s + np.sqrt(sq[:, j])
    return s / k


def py_find_inliers(d, std_thresh):
    n = len(d)
    S = Q = 0.0
    for c in range(0, n, 256):
        s = q = 0.0
        for x in d[c : c + 256]:
            s = s + float(x)
            q = q + float(x) * float(x)
        S, Q = S + s, Q + q
    mean = S / n
    var = Q / n - mean * mean
    thresh = mean + (math.sqrt(var) if var >= 0 else math.nan) * std_thresh
    return [i for i in range(n) if d[i] < thresh], thresh


def same_float(a, b):
    return np.array(a, dtype=np.float64).view(np.uint64) == np.array(b, dtype=np.float64).view(np.uint64)


def test_priority_test_vectors():
    assert fo.priority(0, 0, 0) == 0xE220A8397B1DCDAF and fo.priority(0, 0, 1) == 0x6E789E6AA1B965F4
    assert fo.priority(5489, 7, 0) == 0xF22DD99F91E8D40A and fo.priority(5489, 7, 1) == 0x6F93C0157C1B6D3C
    rng = np.random.default_rng(1)
    for seed, i, s in zip(rng.integers(0, 2**63, 200), rng.integers(0, 2**31, 200), rng.integers(0, 2, 200)):
        assert fo.priority(int(seed) * 2 + 1, int(i), int(s)) == py_priority(int(seed) * 2 + 1, int(i), int(s))
    assert fo.priority(M64, 3, 1) == py_priority(M64, 3, 1)


def test_gather():
    rows = np.random.default_rng(2).normal(size=(50, 3, 3))
    K = np.array([4, 4, 0, 49, 17])
    assert pc.same_bits(fo.gather(rows, K), rows[K])
    assert fo.gather(rows, np.zeros(0, np.int64)).shape == (0, 3, 3)


@pytest.mark.parametrize("rate", [0.0, 0.05, 0.3, 0.5, 0.9, 0.99, 1.5])
@pytest.mark.parametrize("seed", [0, 5489, 2**64 - 1])
def test_random_sampling_matches_python(rate, seed):
    for n in (0, 1, 7, 1000, 10781):
        got = fo.random_sampling(n, rate, seed)
        assert got.tolist() == py_random_sampling(n, rate, seed)
        assert len(got) == (n if rate >= 0.99 else int(n * rate))


@pytest.mark.parametrize("name", sorted(SCANS))
def test_randomgrid_matches_python_on_scans(name):
    pts = SCANS[name].astype(np.float64)
    for j, res in enumerate(pc.RESOLUTIONS):
        for rate in (0.1, 0.5):
            seed = 1000 * j + int(rate * 10)
            assert fo.randomgrid_sampling(pts, res, rate, seed).tolist() == py_randomgrid(pts, res, rate, seed)


@pytest.mark.parametrize("name", sorted(pc.edge_cases()))
def test_randomgrid_edge_cases(name):
    pts, res = pc.edge_cases()[name]
    for rate in (0.0, 0.25, 0.7):
        assert fo.randomgrid_sampling(pts, res, rate, 9).tolist() == py_randomgrid(pts, res, rate, 9)
    if name == "big_voxel" or name == "run_across_1024":
        # every voxel is sampled whole: the 3000 / 300 points of one voxel keep min(count, ppv) points before the cap
        voxels = py_voxels(pts, res)
        pre = set(fo.randomgrid_sampling(pts, res, 0.25, 9, apply_cap=False).tolist())
        ppv = math.ceil(0.25 * len(pts) / len(voxels))
        for idx in voxels.values():
            assert len(pre.intersection(idx)) == min(len(idx), ppv)


def test_random_sampling_is_uniform():
    n, rate, trials = 60, 0.3, 2000
    counts = np.zeros(n)
    for seed in range(trials):
        K = fo.random_sampling(n, rate, seed)
        assert len(K) == 18 and np.all(np.diff(K) > 0)
        counts[K] += 1
    p = int(n * rate) / n
    bound = 5.0 * math.sqrt(p * (1 - p) / trials)
    assert np.all(np.abs(counts / trials - p) < bound)


def test_randomgrid_per_voxel_counts():
    pts = SCANS["kitti07_3"].astype(np.float64)
    voxels = py_voxels(pts, 0.5)
    ppv = math.ceil(0.3 * len(pts) / len(voxels))
    counts = np.zeros(len(pts))
    for seed in range(40):
        pre = fo.randomgrid_sampling(pts, 0.5, 0.3, seed, apply_cap=False)
        mask = np.zeros(len(pts), bool)
        mask[pre] = True
        counts += mask
        for idx in voxels.values():
            assert mask[idx].sum() == min(len(idx), ppv)
        capped = fo.randomgrid_sampling(pts, 0.5, 0.3, seed)
        assert len(capped) == min(len(pre), int(len(pts) * 0.3 * 1.2)) and set(capped) <= set(pre)
    # inside a voxel with more points than ppv every point is drawn alike
    big = max(voxels.values(), key=len)
    assert len(big) > 3 * ppv
    assert np.ptp(counts[big]) < 40


def test_randomgrid_reference_quirks():
    rng = np.random.default_rng(4)
    one = rng.uniform(0.1, 0.9, size=(500, 3))  # one voxel: the reference divides by zero key transitions
    K = fo.randomgrid_sampling(one, 1.0, 0.3, 1)
    assert len(K) == min(math.ceil(0.3 * 500), int(500 * 0.3 * 1.2)) == 150
    assert K.tolist() == py_randomgrid(one, 1.0, 0.3, 1)
    assert len(fo.randomgrid_sampling(one, 1.0, 0.0, 1)) == 0 and len(fo.random_sampling(500, 0.0, 1)) == 0
    assert fo.randomgrid_sampling(one, 1.0, 0.99, 1).tolist() == list(range(500))
    assert fo.random_sampling(500, 0.99, 1).tolist() == list(range(500))
    assert len(fo.random_sampling(500, 0.989, 1)) == int(500 * 0.989)


@pytest.mark.parametrize("name", sorted(SCANS))
def test_mean_knn_dists_match_brute_force(name):
    pts = SCANS[name].astype(np.float64)
    sub = pts[np.random.default_rng(6).choice(len(pts), 2500, replace=False)]
    for k in (1, 10, 64):
        want = np_mean_knn_dists(sub, k)
        assert pc.same_bits(fo.mean_knn_dists(sub, k, brute=True), want)
        assert pc.same_bits(fo.mean_knn_dists(sub, k), want)


def test_mean_knn_dists_tree_equals_brute_force_on_full_scan():
    pts = SCANS["kitti07_3"].astype(np.float64)
    assert pc.same_bits(fo.mean_knn_dists(pts, 10), fo.mean_knn_dists(pts, 10, brute=True))


@pytest.mark.parametrize("std_thresh", [-0.5, 0.0, 1.0, 2.5])
def test_find_inliers_matches_python(std_thresh):
    pts = SCANS["kitti07_0"].astype(np.float64)
    d = fo.mean_knn_dists(pts, 10)
    K, th = fo.find_inliers(d, std_thresh)
    want_K, want_th = py_find_inliers(d.tolist(), std_thresh)
    assert K.tolist() == want_K and same_float(th, want_th)


def test_outlier_reference_quirks():
    # a lattice: every d_i is equal, the strict test keeps nothing
    g = np.arange(8, dtype=np.float64)
    lattice = np.stack(np.meshgrid(g, g, g), -1).reshape(-1, 3)
    d = fo.mean_knn_dists(lattice, 1)
    assert np.all(d == 0.0)
    K, th = fo.find_inliers(d, 1.0)
    assert len(K) == 0 and th == 0.0
    # n == k: every point's neighbours are all the points
    pts = np.random.default_rng(8).normal(size=(12, 3))
    assert pc.same_bits(fo.mean_knn_dists(pts, 12), np_mean_knn_dists(pts, 12))
    # a negative rounded variance gives a NaN threshold and no inliers
    d = np.full(1000, 0.1)
    d[::2] = np.nextafter(0.1, 1.0)
    K, th = fo.find_inliers(d, 1.0)
    want_K, want_th = py_find_inliers(d.tolist(), 1.0)
    assert math.isnan(th) and math.isnan(want_th) and len(K) == 0 and want_K == []


@pytest.mark.parametrize("name", ["kitti00_0", "kitti00_1", "kitti07_0", "kitti07_3"])
@pytest.mark.parametrize("k", [10, 20])
def test_chunked_and_sequential_thresholds_agree(name, k):
    """Deliberate difference (a): the reference's sequential sums move the threshold by rounding only (on these scans by 2 to 56
    ulps: the variance cancels), so the inlier sets are equal or differ only at points between the two thresholds."""
    d = fo.mean_knn_dists(SCANS[name].astype(np.float64), k)
    for std_thresh in (0.5, 1.0, 2.0):
        Kc, tc = fo.find_inliers(d, std_thresh)
        Ks, ts = fo.find_inliers(d, std_thresh, sequential=True)
        assert abs(tc - ts) <= 256 * np.spacing(tc)
        for i in set(Kc.tolist()) ^ set(Ks.tolist()):
            assert min(tc, ts) <= d[i] <= max(tc, ts)
