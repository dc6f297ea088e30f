"""Reconstruction pruning on the GPU (b200sfm_prune_weakly_connected) against the CPU restatement
(oracle/pruning_oracle.py): cluster ids, registration, the cluster count and every integer statistic exactly."""
import os
import subprocess
import sys

import numpy as np
import pytest

from glomap_b200 import _lib, colmap_io as CI, estimators as E, mapper as MP, reconstruction_pruning as RP, synthetic as S
from oracle import pruning_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(tb, of, F, loop=None, min_obs=0, reg=None, **kw):
    dev = RP.prune_weakly_connected_images(tb, of, F, loop, min_obs, is_registered=reg, **kw)
    ref = O.prune(tb, of, F, loop, min_obs, reg)
    assert dev["num_clusters"] == ref["num_clusters"]
    assert dev["cluster_id"].tolist() == ref["cluster_id"].tolist()
    assert dev["is_registered"].tolist() == ref["is_registered"].tolist()
    for k, v in ref["stats"].items():
        assert dev["stats"][k] == v, (k, dev["stats"][k], v)
    return dev


@pytest.mark.parametrize("bridges", [[], [(0, 5, 35)], [(0, 5, 35), (1, 6, 35)], [(0, 5, 35), (1, 6, 29)], [(2, 9, 41)],
                                     [(0, 5, 50), (5, 12, 33), (6, 13, 31)]])
def test_cluster_scenes_match_the_oracle(bridges):
    d = S.make_cluster_tracks([5, 7, 6, 4], 40, bridges=bridges, seed=len(bridges))
    _check(d["track_begin"], d["obs_frame"], d["num_frames"])


def test_ten_pass_cap_on_the_device():
    n = 14
    pairs = [(0, 1, 60)] + [(k, k + 1, 26) for k in range(1, n - 1)] + [(k, k + 2, 26) for k in range(n - 2)]
    tracks = []
    for a, b, c in pairs:
        if c % 2:
            tracks.append([a, a, a, b])
            c -= 3
        tracks += [[a, a, b]] * (c // 2)
    tb = np.concatenate([[0], np.cumsum([len(t) for t in tracks])]).astype(np.int64)
    dev = _check(tb, np.concatenate(tracks).astype(np.int32), n)
    assert dev["stats"]["clustering_iterations"] == 11


@pytest.mark.parametrize("seed", range(8))
def test_random_tracks_match_the_oracle(seed):
    rng = np.random.default_rng([seed, 5])
    F = int(rng.integers(2, 300))
    T = int(rng.integers(1, 3000))
    lens = rng.integers(0, 12, size=T)
    tb = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    hot = rng.choice(F, size=max(2, F // 4), replace=False)
    of = np.where(rng.random(tb[-1]) < 0.7, rng.choice(hot, size=tb[-1]), rng.integers(0, F, size=tb[-1])).astype(np.int32)
    loop = (rng.random(F) < 0.2).astype(np.uint8) if seed % 2 else None
    reg = rng.random(F) < 0.5
    _check(tb, of, F, loop, [0, 10, 40, 0][seed % 4], reg)


def test_config2_sized_scene_matches_and_is_reproducible():
    sc = S.make_scene(1000, 200_000, 10.0, seed=1, chunk=25_000)
    dev = _check(sc.pt_obs_begin, sc.obs_cam, sc.C)
    again = RP.prune_weakly_connected_images(sc.pt_obs_begin, sc.obs_cam, sc.C)
    assert again["cluster_id"].tobytes() == dev["cluster_id"].tobytes()
    assert again["is_registered"].tobytes() == dev["is_registered"].tobytes() and again["stats"] == dev["stats"]


def test_small_passes_split_long_tracks():
    """100-view tracks (4950 slots each) with 1000 keys per pass: passes split tracks, the merge restores the counts."""
    rng = np.random.default_rng(11)
    F, T = 400, 300
    lens = np.where(rng.random(T) < 0.3, 100, rng.integers(3, 10, size=T))
    tb = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    of = (np.repeat(rng.integers(0, F, size=T), lens) + rng.integers(0, 40, size=tb[-1])).astype(np.int32) % F
    ref = _check(tb, of, F)
    for per_pass in (1000, 4949, 1):
        dev = RP.prune_weakly_connected_images(tb, of, F, max_pair_keys_per_pass=per_pass)
        assert dev["cluster_id"].tolist() == ref["cluster_id"].tolist() and dev["stats"] == ref["stats"]
        assert dev["is_registered"].tolist() == ref["is_registered"].tolist()


def test_edge_cases():
    reg = np.array([1, 0, 1, 1], bool)
    for tb, of, F in [(np.array([0]), np.zeros(0), 4),                               # T = 0
                      (np.array([0, 2, 4]), np.array([0, 1, 2, 3]), 4),              # all tracks <= 2
                      (np.array([0, 3, 6]), np.array([0, 1, 2, 0, 1, 3]), 4),        # no pair reaches 5
                      (np.array([0, 3, 6]), np.array([0, 0, 0, 0, 0, 0]), 1)]:       # F = 1
        r = reg[:F]
        dev = _check(tb, of, F, reg=r)
        assert dev["num_clusters"] == 0 and (dev["cluster_id"] == -1).all() and dev["is_registered"].tolist() == r.tolist()
    with pytest.raises(_lib.B200Error) as e:
        RP.prune_weakly_connected_images(np.array([0, 3]), np.array([0, 1, 4]), 4)
    assert e.value.code == 1 and "obs_frame" in str(e.value)
    with pytest.raises(_lib.B200Error) as e:
        RP.prune_weakly_connected_images(np.array([0, 3]), np.array([0, -1, 2]), 4)
    assert e.value.code == 1
    # the context still works after a rejected call
    d = S.make_cluster_tracks([5, 6], 40, bridges=[(0, 5, 35)])
    _check(d["track_begin"], d["obs_frame"], d["num_frames"])


def test_every_edge_dropped_leaves_no_pending_launch_error():
    """A chain 0 - 1 - 2 of weight 10: thr = 20, no edge is strong or >= 0.75 thr, so 5d drops every edge (0 clusters
    with 2 visibility edges).  The call checks for launch errors before it returns, so a launch over zero edges would
    fail it; repeated calls, other entries on the same context and torch's own kernels keep working."""
    import torch
    tracks = [[0, 0, 1]] * 5 + [[1, 1, 2]] * 5
    tb = np.concatenate([[0], np.cumsum([len(t) for t in tracks])]).astype(np.int64)
    of = np.concatenate(tracks).astype(np.int32)
    for _ in range(2):
        dev = _check(tb, of, 3)
        assert dev["stats"]["visibility_edges"] == 2 and dev["num_clusters"] == 0 and dev["is_registered"].all()
    d = S.make_cluster_tracks([5, 6], 40, bridges=[(0, 5, 35)])
    _check(d["track_begin"], d["obs_frame"], d["num_frames"])
    x = torch.arange(1000, device="cuda", dtype=torch.float64)
    assert float((x * 2).sum().item()) == 999000.0
    torch.cuda.synchronize()


def test_multi_rank_context_is_unsupported():
    """Two ranks on two GPUs (one thread each): the call is refused on either rank before any device work."""
    import ctypes as ct
    import threading
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs for a two-rank context")
    lib = _lib.load()
    uid = ct.create_string_buffer(_lib.NCCL_ID_BYTES)
    assert lib.b200sfm_nccl_unique_id(uid) == 0
    handles, rcs = [ct.c_void_p(), ct.c_void_p()], [None, None]

    def make(r):
        rcs[r] = lib.b200sfm_create_dist(r, r, 2, uid, ct.byref(handles[r]))
    threads = [threading.Thread(target=make, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    try:
        assert rcs == [0, 0]
        tb, cid, reg = np.array([0], np.int64), np.zeros(2, np.int32), np.ones(2, np.uint8)
        nc = ct.c_int32()
        p = lambda a: a.ctypes.data_as(ct.c_void_p)   # noqa: E731
        assert lib.b200sfm_prune_weakly_connected(handles[0], 2, 0, p(tb), None, None, 0, 0, p(cid), p(reg), ct.byref(nc),
                                                  None) == 5
    finally:
        threads = [threading.Thread(target=lib.b200sfm_destroy, args=(h,)) for h in handles if h.value]
        for t in threads:
            t.start()
        for t in threads:
            t.join()


def test_global_mapper_prunes_its_final_tracks():
    sc = S.make_scene(30, 2000, mean_track_len=6, seed=21, pixel_sigma=0.5)
    vg = S.view_graph_from_scene(sc, min_shared=15, noise_deg=0.5)
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]; start.trans[:] = 0; start.points[:] = 0
    m = MP.GlobalMapper(MP.GlobalMapperOptions(skip_pruning=False))
    ok, out = m.Solve(vg, start)
    assert ok, m.log
    ref = O.prune(out.pt_obs_begin, out.obs_cam, out.C)
    assert m.frame_cluster_id.tolist() == ref["cluster_id"].tolist()
    assert m.frame_registered.tolist() == ref["is_registered"].tolist()
    assert ref["num_clusters"] >= 1
    default = MP.GlobalMapper()
    assert default.options_.skip_pruning and default.frame_cluster_id is None


def test_colmap_io_prune_writes_one_model_per_cluster(tmp_path):
    d = S.make_cluster_tracks([5, 6], 40, bridges=[(0, 5, 35)], seed=9)
    F, tb, of = d["num_frames"], d["track_begin"], d["obs_frame"]
    N = len(of)
    sc = S.Scene(np.tile([0, 0, 0, 1.0], (F, 1)), np.tile([0, 0, 5.0], (F, 1)), np.zeros((len(tb) - 1, 3)), tb, of,
                 np.random.default_rng(0).uniform(0, 100, size=(N, 2)), np.zeros(F, np.int32), np.zeros(1, np.int32),
                 np.array([[500.0, 50, 50] + [0] * 9]))
    model = tmp_path / "model"
    CI.write_model(str(model), *CI.model_from_scene(sc))
    out = tmp_path / "out"
    r = subprocess.run([sys.executable, "-m", "glomap_b200.colmap_io", "prune", str(model), str(out)], cwd=ROOT,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert sorted(os.listdir(out)) == ["0", "1"]
    want = {c: sorted(int(i) + 1 for i in np.flatnonzero(d["group"] == g)) for c, g in [(0, 1), (1, 0)]}   # 6 frames first
    for c in (0, 1):
        _, ims, pts = CI.read_model(str(out / str(c)))
        assert sorted(ims) == want[c]
        for p in pts.values():
            assert set(p.image_ids.tolist()) <= set(want[c]) and len(p.image_ids) >= 2
