"""Min-cut on the device (b2_min_cut) against the CPU oracle (tests/segmentation_oracle.cpp): the quantised capacities within one
quantum of the oracle's, and the oracle's Dinic flow over the device's own capacities equal to the device's maximum flow and
minimal source set exactly."""
import numpy as np
import pytest

import segmentation_oracle as so
from gtsam_points_b200 import capi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g():
    import gtsam_points_b200 as g

    return g


def stored(cloud):
    n = int(cloud.info().num_points)
    p, nr = np.zeros((n, 3)), np.zeros((n, 3))
    capi.check(capi.lib().b2_cloud_download(cloud.h, capi.dptr(p), None, capi.dptr(nr)))
    return p, nr


def object_on_ground(seed, n_ground=6000, n_box=1500):
    rng = np.random.default_rng(seed)
    ground = np.c_[rng.uniform(-6, 6, (n_ground, 2)), rng.normal(0, 0.003, n_ground)]
    f = rng.uniform(0, 1, (n_box, 3))
    ax = rng.integers(0, 3, n_box)
    f[np.arange(n_box), ax] = rng.integers(0, 2, n_box)
    box = f * np.array([0.8, 0.8, 1.0]) + np.array([-0.4, -0.4, 0.0])
    nb = np.zeros((n_box, 3))
    nb[np.arange(n_box), ax] = 1.0
    p = np.vstack([ground, box])
    nr = np.vstack([np.tile([0, 0, 1.0], (n_ground, 1)), nb])
    return p, nr


def check(g, cloud, source, prm):
    res = g.min_cut(cloud, source, prm, capacities=True)
    p, nr = stored(cloud)
    s = res.source_index
    if res.flags & capi.B2_MIN_CUT_NO_SINK:
        assert res.source_index == -1 and res.sink_index == -1 and res.max_flow == 0.0 and len(res.cluster_indices) == 0
        return res, 0
    t, idx, w, q = so.mc_network(p, nr, s, prm.k_neighbors, prm.distance_sigma, prm.angle_sigma, prm.background_mask_radius)
    assert t == res.sink_index
    diff = np.abs(res.capacities - q)
    assert diff.max() <= 1
    flow, S = so.mc_flow(p, s, t, idx, res.capacities, prm.background_mask_radius, prm.background_weight)
    assert flow == res.max_flow_q and res.max_flow == flow / 2.0**32
    assert np.array_equal(S, res.cluster_indices)
    return res, int((diff > 0).sum())


@pytest.mark.parametrize("flags", [capi.B2_CLOUD_DEFAULT, capi.B2_CLOUD_NO_REORDER])
def test_object_on_ground(g, flags):
    p, nr = object_on_ground(0)
    cloud = g.PointCloud(p, normals=nr, flags=flags)
    differing = 0
    for k, ds, br in ((20, 0.25, 3.0), (10, 0.5, 2.0), (40, 0.15, 4.0)):
        prm = g.MinCutParams(distance_sigma=ds, background_mask_radius=br, k_neighbors=k)
        res, d = check(g, cloud, [0.0, 0.0, 1.0], prm)
        differing += d
        assert res.flags == 0 and len(res.cluster_indices) > 0
        again = g.min_cut(cloud, [0.0, 0.0, 1.0], prm)
        assert again.max_flow_q == res.max_flow_q and np.array_equal(again.cluster_indices, res.cluster_indices)
    print(f"capacities differing from the oracle's by one quantum: {differing}")


def test_cropped_kitti_scene(g):
    import os

    pts = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti00_pair.npz"))["frame0"].astype(np.float64)[:, :3]
    full = g.PointCloud(pts).estimated(10, normals=True)
    p, _ = stored(full)
    centre = p[len(p) // 3]
    keep = np.nonzero(np.linalg.norm(p - centre, axis=1) < 8.0)[0]
    crop = g.types.sample(full, keep)  # b2_cloud_create_sampled, as in the reference demo
    res, d = check(g, crop, centre, g.MinCutParams(background_mask_radius=2.0))
    print(f"{len(keep)} points, cluster {len(res.cluster_indices)}, {d} capacities differ by one quantum")


def test_no_sink_few_neighbours_nan_arcs(g):
    p, nr = object_on_ground(1, 200, 50)
    res, _ = check(g, g.PointCloud(p, normals=nr), 0, g.MinCutParams(background_mask_radius=100.0))
    assert res.flags & capi.B2_MIN_CUT_NO_SINK
    tiny = g.PointCloud(p[:12] * 0.5, normals=nr[:12])
    res, _ = check(g, tiny, 0, g.MinCutParams(k_neighbors=20, background_mask_radius=0.5))
    assert res.flags & capi.B2_MIN_CUT_FEW_NEIGHBORS
    rng = np.random.default_rng(2)
    v = rng.normal(0, 1, 3)
    v /= np.linalg.norm(v)
    flat = np.c_[rng.uniform(0, 4, (500, 2)), np.zeros(500)]
    res, _ = check(g, g.PointCloud(flat, normals=np.tile(v, (500, 1))), 0, g.MinCutParams(background_mask_radius=2.0))


def test_argument_errors(g):
    p, nr = object_on_ground(3, 200, 50)
    cloud = g.PointCloud(p, normals=nr)
    for prm in (g.MinCutParams(distance_sigma=0.0), g.MinCutParams(angle_sigma=np.nan), g.MinCutParams(background_weight=-1.0),
                g.MinCutParams(foreground_weight=2.0**31), g.MinCutParams(k_neighbors=0), g.MinCutParams(k_neighbors=65), g.MinCutParams(background_mask_radius=-1.0)):
        with pytest.raises(capi.B2Error):
            g.min_cut(cloud, 0, prm)
    with pytest.raises(capi.B2Error):
        g.min_cut(g.PointCloud(p), 0)
    with pytest.raises(capi.B2Error):
        g.min_cut(cloud, len(p))
