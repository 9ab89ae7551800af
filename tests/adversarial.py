"""Inputs built to sit where bit-parity with the CPU float64 path can break, plus an exact-rounding FMA emulator (tests/ only).

DESIGN.md section 2 fixes pose * point as ((R0 x + R1 y) + R2 z) + t with every operation rounded, the voxel floor as
floor(q * inv_leaf) and squared distances as (dx^2 + dy^2) + dz^2.  Random clouds almost never put a value within an ulp of a
voxel face or of the bisector of two targets, so a kernel that contracted the transform into FMAs, or floored q / leaf, would
still pass on them.  The constructors here keep only items that such a change would move:

* face_points: points whose transformed coordinate lies on a voxel face and floors differently under at least one FMA
  contraction of the transform (or, with divide=True, under floor(q / leaf));
* bisector_queries: queries on the bisector of two target points whose nearest target changes under a contraction;
* sphere_points: queries at squared distance exactly r^2, and one ulp either side, from their only target.

numpy's elementwise float64 operations are individually rounded (no contraction), so `transform` is the unfused value.
"""
from fractions import Fraction

import numpy as np


def fma(a, b, c):
    """a * b + c with one rounding (Fraction arithmetic is exact; float(Fraction) rounds to nearest even)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def transform(T, p):
    """((R0 x + R1 y) + R2 z) + t, every operation rounded: the unfused value, for an N x 3 array."""
    R, t = T[:3, :3], T[:3, 3]
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((R[r, 0] * x + R[r, 1] * y) + R[r, 2] * z) + t[r] for r in range(3)], 1)


def contracted_row(Tr, x, y, z):
    """The unfused value of one output row (Tr = row of T) and the three ways a compiler may contract it into FMAs."""
    r0, r1, r2, t = (float(v) for v in Tr[:4])
    x, y, z = float(x), float(y), float(z)
    a, b = r0 * x, r1 * y
    s = a + b
    return (
        ((s + r2 * z) + t),
        fma(r2, z, fma(r0, x, b)) + t,
        fma(r2, z, fma(r1, y, a)) + t,
        fma(r2, z, s) + t,
    )


def contracted_variants(T, p):
    """4 x 3 array for one point p: row 0 the unfused T p, rows 1..3 the contraction patterns."""
    return np.array([contracted_row(T[r], *p[:3]) for r in range(3)]).T


def _floor(v, inv):
    return int(np.floor(v * inv))


def face_points(T, leaf, count, seed, divide=False, extent=40.0):
    """Points p with (T p)[axis] on the voxel face k * leaf, for a random axis per point, kept when they are sensitive.

    Sensitive: some contracted variant of T p floors (times 1 / leaf) to another voxel than the unfused value; with
    divide=True instead: floor(q * (1 / leaf)) != floor(q / leaf) for the unfused q.  Returns (p, axis), p float64 N x 3."""
    rng = np.random.default_rng(seed)
    inv = 1.0 / leaf
    R, t = T[:3, :3], T[:3, 3]
    kmax = int(extent / leaf)
    out, axes = [], []
    while len(out) < count:
        n = 4096
        axis = rng.integers(0, 3, n)
        q = rng.uniform(-extent, extent, (n, 3))
        q[np.arange(n), axis] = rng.integers(-kmax, kmax, n) * leaf
        p = (q - t) @ R  # R^T (q - t)
        qu = transform(T, p)
        for i in range(n):
            a = axis[i]
            v = qu[i, a]
            if abs(v * inv - np.round(v * inv)) > 1e-9:
                continue
            if divide:
                keep = np.floor(v * inv) != np.floor(v / leaf)
            else:
                c0 = _floor(v, inv)
                keep = any(_floor(w, inv) != c0 for w in contracted_row(T[a], *p[i])[1:])
            if keep:
                out.append(p[i])
                axes.append(a)
                if len(out) == count:
                    break
    return np.array(out), np.array(axes)


def sensitive_face_count(T, leaf, p, axes):
    """How many of the points a contraction of the transform moves to another voxel (for the divide variant: how many the
    division does)."""
    inv = 1.0 / leaf
    n = 0
    for i in range(len(p)):
        v = contracted_row(T[axes[i]], *p[i])
        n += any(_floor(w, inv) != _floor(v[0], inv) for w in v[1:])
    return n


def sq_dist(a, q):
    d = np.asarray(q, dtype=np.float64) - np.asarray(a, dtype=np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def bisector_queries(T, num_pairs, seed, f32_targets=True, half_gap=0.1, spacing=2.5):
    """Target pairs (a, b) about 2 * half_gap apart, pair centres on a grid `spacing` apart (no other target nearby), and one
    query p per kept pair with T p on the bisector of a and b.  A query is kept when a contraction of the transform flips
    which of a and b is nearer; exact ties of the unfused distances are dropped (their index depends on visit order).
    f32_targets=False offsets the targets by 2^-30 so they are not float32-representable.

    Returns (targets (2M x 3), queries p (M x 3), nearest target index per query under the unfused transform)."""
    rng = np.random.default_rng(seed)
    R, t = T[:3, :3], T[:3, 3]
    g = np.arange(-8, 8) * spacing
    centres = np.stack(np.meshgrid(g, g, g[:6], indexing="ij"), -1).reshape(-1, 3)
    centres = centres[rng.permutation(len(centres))[:num_pairs]] + rng.uniform(-0.3, 0.3, (num_pairs, 3))
    u = rng.normal(size=(num_pairs, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    a = (centres + half_gap * u).astype(np.float32).astype(np.float64)
    b = (centres - half_gap * u).astype(np.float32).astype(np.float64)
    if not f32_targets:
        a, b = a + 2.0**-30, b + 2.0**-30
    m, d = 0.5 * (a + b), a - b
    v = rng.normal(size=(num_pairs, 3)) * 0.05
    v -= (np.einsum("ij,ij->i", v, d) / np.einsum("ij,ij->i", d, d))[:, None] * d  # in the bisector plane
    p = (m + v - t) @ R
    qu = transform(T, p)
    da, db = sq_dist(a, qu), sq_dist(b, qu)
    keep, nearest = [], []
    for i in range(num_pairs):
        if da[i] == db[i]:
            continue
        s0 = da[i] < db[i]
        var = contracted_variants(T, p[i])[1:]
        if any((sq_dist(a[i], w) < sq_dist(b[i], w)) != s0 or sq_dist(a[i], w) == sq_dist(b[i], w) for w in var):
            keep.append(i)
            nearest.append(0 if s0 else 1)
    keep = np.array(keep, dtype=np.int64)
    targets = np.stack([a[keep], b[keep]], 1).reshape(-1, 3)
    nearest = 2 * np.arange(len(keep)) + np.array(nearest, dtype=np.int64)
    return targets, p[keep], nearest


def sphere_points(count=2):
    """Targets a and queries q, all float32-representable, with the squared distance of q from a in the kernel's order,
    ((dx^2 + dy^2) + dz^2), equal to max_sq = radius * radius (tag 0), one ulp below (tag -1) or one ulp above (tag +1).
    Offsets (dx, dy, dz) are drawn from a float32 grid near 0.72 m; the radius is a double whose square rounds to a value that
    the grid reaches together with both its neighbours.  Targets sit 3 m apart on the y axis, so each query's only candidate
    within the radius is its own target.  Returns (targets, queries, tags, radius)."""
    dx = (np.float32(0.72) - np.arange(64, dtype=np.float32) * np.float32(2.0**-24)).astype(np.float64)
    dy = np.arange(64) * 2.0**-20
    dz = np.arange(64) * 2.0**-28
    s = (dx[:, None, None] * dx[:, None, None] + dy[None, :, None] * dy[None, :, None]) + dz[None, None, :] * dz[None, None, :]
    reach = set(s.ravel().tolist())
    radius = None
    for v in np.unique(s):
        r0 = np.sqrt(v)
        for r in (np.nextafter(r0, 0.0), r0, np.nextafter(r0, 2.0)):
            m = r * r
            if all(w in reach for w in (np.nextafter(m, 0.0), m, np.nextafter(m, 2.0))):
                radius = float(r)
                break
        if radius is not None:
            break
    max_sq = radius * radius
    want = {-1: np.nextafter(max_sq, 0.0), 0: max_sq, 1: np.nextafter(max_sq, 2.0)}
    targets, queries, tags = [], [], []
    for tag, w in want.items():
        i, j, k = np.argwhere(s == w)[0]
        for sign in (1.0, -1.0)[:count]:  # a mirrored copy has the same squared distance
            a = np.array([0.0, 3.0 * len(targets) - 9.0, 0.0])
            targets.append(a)
            queries.append(a + np.array([sign * dx[i], sign * dy[j], -sign * dz[k]]))
            tags.append(tag)
    return np.array(targets), np.array(queries), np.array(tags), radius


# ---- scenes shared by the CPU and GPU tests -----------------------------------------------------------------------------
POSE_SEED = 7
LEAVES = (0.5, 0.3, 0.2)
FACE_COUNT = 1000


def pose(seed=POSE_SEED):
    from gtsam_points_b200 import synthetic as syn

    return syn.random_pose(np.random.default_rng(seed), 0.3, 3.0)


def spd(n, seed):
    """n well-conditioned covariances (float64, symmetric)."""
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(n, 3, 3)) * 0.05
    C = A @ A.transpose(0, 2, 1) + 0.01 * np.eye(3)
    return 0.5 * (C + C.transpose(0, 2, 1))


def face_scene(leaf, divide=False, count=FACE_COUNT, seed=1):
    """Face points p under pose(), and a target of one point per voxel at the voxel centre: the voxel the unfused T p floors
    to, for every point, and the voxel the sensitive variant (a contraction, or floor(q / leaf)) picks instead, for every
    second point.  `expected` is each point's voxel id in first-touch order of the target."""
    T = pose()
    inv = 1.0 / leaf
    p, axes = face_points(T, leaf, count, seed, divide=divide)
    qu = transform(T, p)
    own = np.floor(qu * inv).astype(np.int64)
    other = own.copy()
    for i in range(len(p)):
        a = axes[i]
        if divide:
            other[i, a] = int(np.floor(qu[i, a] / leaf))
        else:
            other[i, a] = next(_floor(w, inv) for w in contracted_row(T[a], *p[i])[1:] if _floor(w, inv) != own[i, a])
    ids, coords = {}, []
    for i in range(len(p)):
        for c in ((own[i],) if i % 2 else (own[i], other[i])):
            key = tuple(int(v) for v in c)
            if key not in ids:
                ids[key] = len(coords)
                coords.append(key)
    coords = np.array(coords, dtype=np.int64)
    expected = np.array([ids[tuple(int(v) for v in c)] for c in own], dtype=np.int64)
    return dict(T=T, leaf=leaf, p=p, covs=spd(len(p), seed + 100), qu=qu, axes=axes, coords=coords,
                target=(coords + 0.5) * leaf, target_covs=spd(len(coords), seed + 200), expected=expected)


def bisector_scene(f32_targets=True, num_pairs=1500, seed=3):
    T = pose()
    targets, p, nearest = bisector_queries(T, num_pairs, seed, f32_targets=f32_targets)
    rng = np.random.default_rng(seed + 300)
    normals = rng.normal(size=(len(targets), 3))
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    return dict(T=T, p=p, covs=spd(len(p), seed + 100), qu=transform(T, p), targets=targets, target_covs=spd(len(targets), seed + 200),
                normals=normals, nearest=nearest, other=nearest ^ 1)


def sphere_scene():
    targets, q, tags, radius = sphere_points()
    normals = np.tile([0.0, 0.0, 1.0], (len(targets), 1))
    expected = np.where(tags < 0, np.arange(len(q)), -1)
    return dict(targets=targets, q=q, tags=tags, radius=radius, covs=spd(len(q), 5), target_covs=spd(len(targets), 6), normals=normals, expected=expected)
