"""The camera-order kernels (ba2_pass_b, the camera-order linearisation, the Schur-Jacobi diagonal) on segments of
every length mod 32 and on the boundaries of the bucket split (seg_split in ba_kernels.cuh).

Pass B walks a segment in rounds of 32 observations, one per lane, with the point records of the next round and the
index of the round after it already loading; a segment's last round is partial, and the loads ahead stop at the
segment's end.  A (slice, camera) bucket of n observations is one segment below 384 and round(n / 256) equal segments
from there.  The scene here gives cameras exactly 1..33, 255, 256, 257, 383, 384 and 640 used observations, all of them
in the first of three point slices (B200SFM_PT_SLICES=3, 1024 points each), so the segments reach every residue mod
32, a single observation, one observation past a full round, the longest single segment (383), the first two-segment
bucket (2 x 192) and a three-segment one (213, 213, 214).  The first LM step of each path that runs pass B (NK = 0, 1,
2 and a known rig) is compared with the FP64 sparse reference through the operator-level probe and bounds of
test_ba_system_gpu.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_ba_system_gpu as TS  # noqa: E402
from glomap_b200 import geometry as G, synthetic as S  # noqa: E402

pytestmark = pytest.mark.gpu

C_ROUNDS, P_ROUNDS, SLICE = 300, 2600, 1024
ROUND_COUNTS = list(range(1, 34)) + [255, 256, 257, 383, 384, 640]
SPECIAL0 = 10                                 # cameras SPECIAL0 + i see ROUND_COUNTS[i] points of the first slice
SLICES = {"B200SFM_PT_SLICES": "3"}

PATHS = {
    "rounds_ell": (dict(K=1), {}, SLICES, dict(use_v2=1, use_ell=1, ext=0, kfast=0)),
    "rounds_kfast_nk1_K200": (dict(K=200), dict(optimize_intrinsics=True), SLICES, dict(use_ell=1, kfast=1, nk=1)),
    "rounds_kfast_nk2_simple_radial_K300": (dict(K=300, model=S.SIMPLE_RADIAL), dict(optimize_intrinsics=True), SLICES,
                                            dict(kfast=1, nk=2)),
    "rounds_rig_known": ("rig", {}, SLICES, dict(use_ell=1, ext=0)),
}


def make_rounds_scene(K=1, model=S.SIMPLE_PINHOLE, seed=11):
    rng = np.random.default_rng(seed)
    R, t = S.make_cameras(C_ROUNDS, seed, jitter_deg=2.0)
    cam_intr, intr_model, intr_params = S.make_intrinsics(C_ROUNDS, model, 1000.0, 1000, K)
    d = rng.normal(size=(P_ROUNDS, 3))
    pts = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0, 1, size=(P_ROUNDS, 1)) ** (1 / 3)
    special = SPECIAL0 + np.arange(len(ROUND_COUNTS))
    pool = np.setdiff1d(np.arange(C_ROUNDS), special)
    tracks = [list(rng.choice(pool, min(3 + rng.poisson(3), 10), replace=False)) for _ in range(P_ROUNDS)]
    for c, n in zip(special, ROUND_COUNTS):
        for p in rng.choice(SLICE, n, replace=False):
            tracks[p].append(int(c))
    obs_cam = np.concatenate([np.asarray(tr, np.int32) for tr in tracks])
    obs_pt = np.repeat(np.arange(P_ROUNDS), [len(tr) for tr in tracks])
    Xc = np.einsum("nij,nj->ni", R[obs_cam], pts[obs_pt]) + t[obs_cam]
    xy = np.empty((len(obs_cam), 2))
    for k in range(K):
        m = cam_intr[obs_cam] == k
        xy[m] = S.project(int(intr_model[k]), intr_params[k], Xc[m])
    xy += rng.normal(size=xy.shape) * 0.8
    ptb = np.zeros(P_ROUNDS + 1, np.int64)
    np.cumsum([len(tr) for tr in tracks], out=ptb[1:])
    sc = S.Scene(G.rotmat_to_quat_xyzw_fast(R), t, pts, ptb, obs_cam, xy, cam_intr, intr_model, intr_params)
    st = S.perturb_scene(sc, rot_deg=0.05, center_frac=0.001, point_frac=0.001, seed=seed)
    st.intr_params = sc.intr_params.copy()
    st.intr_params[:, 0] *= 1.002
    return st


@pytest.fixture(scope="module")
def scenes():
    cache = {}

    def get(spec):
        key = "rig" if spec == "rig" else tuple(sorted(spec.items()))
        if key not in cache:
            cache[key] = TS.make_rig() if spec == "rig" else make_rounds_scene(**spec)
        return cache[key]
    return get


def test_rounds_scene_reaches_every_residue(scenes):
    sc = scenes(dict(K=1))
    lens = np.diff(sc.pt_obs_begin)
    assert lens.min() >= TS.MIN_VIEWS and sc.P > 2 * SLICE
    obs_pt = np.repeat(np.arange(sc.P), lens)
    n = np.zeros((3, sc.C), int)
    np.add.at(n, (obs_pt // SLICE, sc.obs_cam), 1)
    special = SPECIAL0 + np.arange(len(ROUND_COUNTS))
    assert list(n[0, special]) == ROUND_COUNTS and not n[1:, special].any()
    assert all(c < sc.C // 2 for c in special)   # one camera half: the bucket is the camera's whole count
    assert set(np.unique(n[n > 0] % 32)) == set(range(32))


@pytest.mark.parametrize("name", list(PATHS))
def test_pass_b_rounds_match_the_fp64_reference(name, scenes, monkeypatch):
    monkeypatch.setitem(TS.PATHS, name, PATHS[name])
    TS.test_device_step_matches_the_fp64_reference(name, scenes, monkeypatch)
