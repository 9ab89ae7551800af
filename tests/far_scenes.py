"""One seeded factor problem placed far from the origin in several ways (tests/ only).

Every scene is the same problem moved as a whole, so that the target-side results do not change in exact arithmetic:
  S0 origin       the control;
  S1 far source   the source stored at +o, delta' = delta T(-o): the pose brings it back near the target's origin;
  S2 far target   the target cloud, voxel map and iVox at +o, delta' = T(o) delta: a unary frame-to-map factor in world
                  coordinates;
  S3 both far     delta' = T(o) delta T(-o);
  S4 far source, float32 storage: the source at +o4 = (3e4, 4e4, 50) rounded to float32, delta' = delta T(-o4).
o = kdtree_edges.UTM_OFFSET, which is not float32-exact.  Covariances are well conditioned (adversarial.spd); the clouds carry
unit normals for surface validation and point-to-plane ICP.
"""
import numpy as np

from adversarial import spd
from gtsam_points_b200 import synthetic as syn
from kdtree_edges import UTM_OFFSET

SCENES = ("S0", "S1", "S2", "S3", "S4")
F32_OFFSET = np.array([3e4, 4e4, 50.0])
N_TARGET = 60000
N_SOURCE = 20011  # ragged: not a multiple of any tile or warp size
VOXEL = 0.5
IVOX_VOXEL = 1.0
MAX_CORR = 1.0  # kd-tree / iVox correspondence distance (squared: 1.0)


def translation(o):
    T = np.eye(4)
    T[:3, 3] = o
    return T


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _base():
    tp, _ = syn.make_cloud(N_TARGET, stream=1, scale=0.3)
    sp, _ = syn.make_cloud(N_SOURCE, stream=2, scale=0.3)
    rng = np.random.default_rng(31)
    return dict(tp=np.asarray(tp, dtype=np.float64), sp=np.asarray(sp, dtype=np.float64), tc=spd(N_TARGET, 32), sc=spd(N_SOURCE, 33),
                tn=_unit(rng, N_TARGET), sn=_unit(rng, N_SOURCE),
                deltas=[syn.random_pose(np.random.default_rng(34 + i), 0.02, 0.2) for i in range(3)])


def bbox_centre(points):
    """The expansion point's centre as the device cloud computes it: 0.5 * (min + max) per axis of the stored points."""
    p = np.asarray(points, dtype=np.float64)
    return 0.5 * (p.min(0) + p.max(0)) if len(p) else np.zeros(3)


def scene(name, base=None):
    """dict(tp, tc, tn, sp, sc, sn, deltas, src_off, tgt_off): `deltas` are the scene's poses T_target_source (the first
    linearizes, the others are evaluation and re-linearization points)."""
    b = base or _base()
    src_off, tgt_off = np.zeros(3), np.zeros(3)
    if name in ("S1", "S3"):
        src_off = UTM_OFFSET
    if name in ("S2", "S3"):
        tgt_off = UTM_OFFSET
    sp = b["sp"] + src_off
    if name == "S4":
        src_off = F32_OFFSET
        sp = (b["sp"] + src_off).astype(np.float32).astype(np.float64)
    deltas = [translation(tgt_off) @ d @ translation(-src_off) for d in b["deltas"]]
    return dict(name=name, tp=b["tp"] + tgt_off, tc=b["tc"], tn=b["tn"], sp=sp, sc=b["sc"], sn=b["sn"], deltas=deltas, src_off=src_off, tgt_off=tgt_off)


def all_scenes():
    b = _base()
    return {n: scene(n, b) for n in SCENES}
