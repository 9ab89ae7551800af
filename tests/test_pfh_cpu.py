"""The registration oracle's PFH (orc_pfh) and FPFH at chosen points (orc_fpfh_at, tests/registration_oracle.cpp) against plain numpy restatements of the formulas
include/b2points.h states for b2_features_create_pfh and b2_features_create_fpfh_at, on small scenes."""
import math

import numpy as np
import pytest

import registration_cases as rc
import registration_oracle as ro
from test_registration_cpu import np_fpfh


def _dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)


def np_pair_features(p1, n1, p2, n2):
    """compute_pair_features of the pairs (p1, n1) -> (p2, n2), k x 3 each -> k x 3 (theta, phi, alpha), elementwise in the stated order."""
    e = p2 - p1
    d = np.sqrt(_dot(e, e))
    with np.errstate(invalid="ignore", divide="ignore"):
        e = e / d[:, None]
        a1, a2 = _dot(n1, e), _dot(n2, e)
        swap = np.abs(a1) < np.abs(a2)
        A = np.where(swap[:, None], n2, n1)
        B = np.where(swap[:, None], n1, n2)
        e = np.where(swap[:, None], -e, e)
        alpha = np.where(swap, -a2, a1)
        v = _cross(e, A)
        v = v / np.sqrt(_dot(v, v))[:, None]
        w = _cross(A, v)
        f = np.stack([np.arctan2(_dot(w, B), _dot(A, B)), _dot(v, B), alpha], axis=1)
    ok = (d != 0.0) & np.isfinite(v).all(axis=1)
    return np.where(ok[:, None], f, 0.0)


def np_neighbours(P, i, radius, max_nn):
    d = P - P[i]
    s = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    idx = np.nonzero(s < radius * radius)[0]
    return idx[np.lexsort((idx, s[idx]))][:max_nn]


def np_pfh(P, N, radius, max_nn, indices=None, reverse=False):
    """estimate_pfh at the points `indices` (None: every point); reverse=True takes each pair as (N[j], N[i]) instead."""
    indices = np.arange(len(P)) if indices is None else np.asarray(indices)
    pi = math.pi
    fmin = np.array([-pi, -1.0, -1.0])
    inv = np.array([1.0 / (pi - (-pi)), 1.0 / (1.0 - (-1.0)), 1.0 / (1.0 - (-1.0))])
    out = np.zeros((len(indices), 125))
    for k, p in enumerate(indices):
        nb = np_neighbours(P, p, radius, max_nn)
        m = len(nb)
        if m <= 1:
            continue
        ii, jj = np.tril_indices(m, -1)  # i > j, i-major: the reference's loop order (the order does not change the counts)
        a, b = (nb[jj], nb[ii]) if reverse else (nb[ii], nb[jj])
        f = np_pair_features(P[a], N[a], P[b], N[b])
        bins = np.clip(np.floor(((f - fmin) * inv) * 5.0), 0, 4).astype(np.int64)
        h = np.bincount(bins[:, 0] + 5 * bins[:, 1] + 25 * bins[:, 2], minlength=125)
        out[k] = h.astype(np.float64) * (100.0 / float(m * (m - 1) // 2))
    return out


ISOLATED, TIE = 161, 162


def scene(n=160, seed=3):
    """small_scene plus a point coincident with point 5 (their pair is the zero feature, bin 62), an isolated point (a zero row,
    index ISOLATED) and, far from the rest, two points with equal normals (indices TIE, TIE + 1).  The pair feature is symmetric to
    the bit except where |a_i| == |a_j|, which equal normals force: there (N[i], N[j]) and (N[j], N[i]) bin differently."""
    P, N = rc.small_scene(n, seed=seed)
    t = np.array([0.6, 0.0, 0.8])
    P = np.concatenate([P, [P[5], [50.0, 50.0, 50.0], [20.0, 20.0, 20.0], [20.3, 20.0, 20.2]]])
    N = np.concatenate([N, [N[7], [0.0, 0.0, 1.0], t, t]])
    return P, N


@pytest.mark.parametrize("max_nn", [10000, 12])
def test_oracle_pfh_matches_numpy(max_nn):
    P, N = scene()
    got, edge, nn = ro.pfh(P, N, 1.5, max_nn, num_threads=2)
    want = np_pfh(P, N, 1.5, max_nn)
    assert np.array_equal(got, want)
    assert not edge.any()
    assert not got[ISOLATED].any() and nn[ISOLATED] == 1
    assert got[5, 62] > 0.0 and got[160, 62] > 0.0  # the coincident pair
    assert np.allclose(got[nn > 1].sum(axis=1), 100.0)
    if max_nn == 12:
        assert nn.max() == 12
    else:
        assert nn.max() > 12


def test_oracle_pfh_follows_the_reference_pair_orientation():
    P, N = scene()
    got, _, _ = ro.pfh(P, N, 1.5, 10000, num_threads=2)
    rev = np_pfh(P, N, 1.5, 10000, reverse=True)
    differ = np.nonzero((got != rev).any(axis=1))[0]
    assert TIE in differ and TIE + 1 in differ  # so the oracle's rows are those of (N[i], N[j])
    assert np.array_equal(got, np_pfh(P, N, 1.5, 10000))


def test_oracle_pfh_at_indices():
    P, N = scene()
    idx = np.array([7, ISOLATED, 3, 7, 0, 160, TIE + 1, 159])  # unsorted, a duplicate, the isolated and a coincident point
    got, _, nn = ro.pfh(P, N, 1.5, 10000, num_threads=2, indices=idx)
    full, _, nn_full = ro.pfh(P, N, 1.5, 10000, num_threads=2)
    assert np.array_equal(got, full[idx]) and np.array_equal(nn, nn_full[idx])
    assert np.array_equal(got, np_pfh(P, N, 1.5, 10000, indices=idx))
    assert ro.pfh(P, N, 1.5, 10000, indices=np.zeros(0, dtype=np.int64))[0].shape == (0, 125)


@pytest.mark.parametrize("max_nn", [10000, 12])
def test_oracle_fpfh_at_indices(max_nn):
    P, N = scene()
    idx = np.array([9, 2, ISOLATED, 2, 5, TIE, 100])
    got, edge, nn = ro.fpfh_at(P, N, idx, 1.5, max_nn, num_threads=2)
    full, edge_full, nn_full = ro.fpfh(P, N, 1.5, max_nn, num_threads=2)
    assert np.array_equal(got, full[idx]) and np.array_equal(edge, edge_full[idx]) and np.array_equal(nn, nn_full[idx])
    want, want_nn = np_fpfh(P, N, 1.5, max_nn)
    assert np.array_equal(got, want[idx]) and np.array_equal(nn, want_nn[idx])
