"""The GNC oracle (orc_gnc in tests/registration_oracle.cpp) against plain numpy restatements of b2_estimate_pose_gnc's steps on small
clouds, and its end-to-end result on the KITTI-00 pair against the reference test's gates (src/test/test_global_registration.cpp)."""
import numpy as np
import pytest

import registration_cases as rc
import registration_oracle as ro


def _nn(Q, T):
    """Exact 1-NN, distances summed in dimension order, ties to the smallest index."""
    acc = np.zeros((len(Q), len(T)))
    for d in range(Q.shape[1]):
        diff = Q[:, None, d] - T[None, :, d]
        acc = acc + diff * diff
    return np.argmin(acc, axis=1)


@pytest.fixture(scope="module")
def scene():
    """240 target points with FPFH rows; the source is 200 of them in shuffled order, moved by the inverse of the reference test's
    offset, with their rows plus noise (so that some matches are not mutual)."""
    P, N = rc.small_scene(240, seed=5)
    F, _, _ = ro.fpfh(P, N, 2.0, 10000, num_threads=2)
    rng = np.random.default_rng(7)
    perm = rng.permutation(240)[:200]
    Ti = rc.pose_inverse(rc.offset_pose())
    src = (Ti[:3, :3] @ P[perm].T).T + Ti[:3, 3]
    return P, F, src, F[perm] + rng.normal(0.0, 4.0, (200, F.shape[1]))


def _align(t, s, w, dof):
    W = w.sum()
    mt, ms = (w[:, None] * t).sum(0) / W, (w[:, None] * s).sum(0) / W
    H = ((t - mt) * w[:, None]).T @ (s - ms)
    R = np.eye(3)
    if dof == 6:
        U, _, Vt = np.linalg.svd(H)
        R = U @ np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))]) @ Vt
    else:
        x, y = H[0, 0] + H[1, 1], H[1, 0] - H[0, 1]
        r = np.hypot(x, y)
        R[:2, :2] = [[x / r, -y / r], [y / r, x / r]]
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, mt - R @ ms
    return T


def np_gnc_loop(tgt, src, C, dof, max_iterations=64, inner_iterations=3, div_factor=1.4, max_corr_dist=0.25):
    t, s = tgt[C[:, 0]], src[C[:, 1]]
    mu = np.linalg.norm(tgt.max(0) - tgt.min(0))
    T, inl = np.eye(4), 0
    for i in range(max_iterations):
        for j in range(inner_iterations):
            e = (((T[:3, :3] @ s.T).T + T[:3, 3] - t) ** 2).sum(1)
            w = np.ones(len(e)) if i == 0 and j == 0 else (mu / (mu + e)) ** 2
            inl = int((e < (2 * max_corr_dist) ** 2).sum())
            T = _align(t, s, w, dof)
        mu /= div_factor
        if mu < max_corr_dist:
            break
    return T, inl


def test_samples_and_reciprocal_matching(scene):
    P, F, src, sf = scene
    r = ro.gnc(P, src, F, sf, max_init_samples=100, num_threads=2)
    smp = r["samples"]
    assert not r["swapped"] and len(smp) == 100 and len(np.unique(smp)) == 100 and np.all(np.diff(smp) > 0) and smp.max() < len(src)
    o = _nn(sf[smp], F)
    back = _nn(F[o], sf)
    mutual = back == smp
    assert np.array_equal(r["matched"], np.stack([o[mutual], smp[mutual]], 1))
    assert np.array_equal(r["C"], r["matched"]) and r["draws"] is None
    assert 0 < mutual.sum() < 100
    # without the reciprocal test every sample gives a pair
    r = ro.gnc(P, src, F, sf, max_init_samples=100, reciprocal_check=False, num_threads=2)
    assert np.array_equal(r["C"], np.stack([o, smp], 1))


def test_swapped_side(scene):
    P, F, src, sf = scene
    # the target (200 rows) is smaller than the source (240): the target is sampled, pairs still read (target, source)
    r = ro.gnc(src, P, sf, F, num_threads=2)
    assert r["swapped"] and np.array_equal(r["samples"], np.arange(200))
    o = _nn(sf, F)
    mutual = _nn(F[o], sf) == np.arange(200)
    assert np.array_equal(r["C"], np.stack([np.arange(200)[mutual], o[mutual]], 1))


def test_tuple_check(scene):
    P, F, src, sf = scene
    r = ro.gnc(P, src, F, sf, reciprocal_check=False, tuple_check=True, max_num_tuples=40, num_threads=2)
    m, C, draws = r["matched"], r["C"], r["draws"]
    assert len(m) == 200 and draws is not None and draws.shape == (40, 3) and draws.max() < 200
    want = []
    for k in range(40):
        c = m[draws[k]]
        ok = True
        for a in range(3):
            b = (a + 1) % 3
            with np.errstate(invalid="ignore"):
                ratio = np.linalg.norm(P[c[a, 0]] - P[c[b, 0]]) / np.linalg.norm(src[c[a, 1]] - src[c[b, 1]])
            ok = ok and not (ratio < 0.9 or ratio > 1.0 / 0.9)
        if ok:
            want += [tuple(x) for x in c]
    assert len(want) > 0
    first = {}
    for pair in want:
        first.setdefault(pair[1], pair)
    assert np.array_equal(C, np.array(sorted(first.values(), key=lambda p: p[1])))
    assert len(np.unique(C[:, 1])) == len(C) and np.all(np.diff(C[:, 1]) > 0)
    # under the branch's threshold (|C| <= 3 max_num_tuples) the check does not run
    assert ro.gnc(P, src, F, sf, reciprocal_check=False, tuple_check=True, max_num_tuples=67, num_threads=2)["draws"] is None


@pytest.mark.parametrize("dof", [6, 4])
def test_loop_matches_numpy(scene, dof):
    P, F, src, sf = scene
    r = ro.gnc(P, src, F, sf, reciprocal_check=False, dof=dof, num_threads=2)
    T, inl = np_gnc_loop(P, src, r["C"], dof)
    assert np.abs(r["T_target_source"] - T).max() <= 1e-9
    assert abs(r["num_inliers"] - inl) <= r["slack"].sum()
    assert r["inlier_rate"] == r["num_inliers"] / len(r["C"])
    if dof == 4:
        R = r["T_target_source"][:3, :3]
        assert np.array_equal(R[2], [0.0, 0.0, 1.0]) and np.array_equal(R[:, 2], [0.0, 0.0, 1.0])


def test_first_alignment_is_kabsch(scene):
    P, F, src, sf = scene
    r = ro.gnc(P, src, F, sf, reciprocal_check=False, max_iterations=1, inner_iterations=1, num_threads=2)
    C = r["C"]
    t, s = P[C[:, 0]], src[C[:, 1]]
    mt, ms = t.mean(0), s.mean(0)
    U, _, Vt = np.linalg.svd((t - mt).T @ (s - ms))
    R = U @ np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))]) @ Vt
    assert np.abs(r["T_target_source"][:3, :3] - R).max() <= 1e-9
    assert np.abs(r["T_target_source"][:3, 3] - (mt - R @ ms)).max() <= 1e-9


def test_empty_and_zero_iterations(scene):
    P, F, src, sf = scene
    for kw in (dict(max_iterations=0), dict(inner_iterations=0)):
        r = ro.gnc(P, src, F, sf, num_threads=2, **kw)
        assert np.array_equal(r["T_target_source"], np.eye(4)) and r["num_inliers"] == 0 and r["inlier_rate"] == 0.0
    # wrong matches never keep their edge ratios exactly: tuple_thresh = 1 empties C
    r = ro.gnc(P, src, F, np.roll(sf, 1, axis=0), reciprocal_check=False, tuple_check=True, max_num_tuples=10, tuple_thresh=1.0, num_threads=2)
    assert len(r["C"]) == 0 and np.array_equal(r["T_target_source"], np.eye(4)) and r["inlier_rate"] == 0.0


@pytest.mark.parametrize("dof", [6, 4])
def test_oracle_meets_the_reference_gate_on_kitti00(dof):
    import normals_ref
    import voxelgrid_oracle as vo

    d = rc.kitti00()
    tgt = vo.voxelgrid_sampling(d["frame0"], 0.5)[0]
    src = vo.voxelgrid_sampling(d["frame1"], 0.5)[0]
    tn = normals_ref.estimate_normals(tgt, 10)[0]
    sn = normals_ref.estimate_normals(src, 10)[0]
    T_off = rc.offset_pose()
    P = rc.pose_inverse(T_off) @ d["T_final"]
    src_p = (P[:3, :3] @ src.T).T + P[:3, 3]
    src_n = (P[:3, :3] @ sn.T).T
    tf, _, _ = ro.fpfh(tgt, tn, 5.0, 10000)
    sf, _, _ = ro.fpfh(src_p, src_n, 5.0, 10000)
    r = ro.gnc(tgt, src_p, tf, sf, dof=dof)
    et, er = rc.pose_error(r["T_target_source"], T_off)
    assert et <= 0.5 and er <= 0.1, (et, er, len(r["C"]), r["num_inliers"])
    if dof == 4:
        assert np.abs(r["T_target_source"][:3, 2] - [0.0, 0.0, 1.0]).max() <= 1e-6
