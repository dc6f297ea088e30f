"""Reconstruction pruning without a GPU: the oracle (oracle/pruning_oracle.py) against a literal loop-and-dict
transcription of PruneWeaklyConnectedImages / EstablishStrongClusters / KeepLargestConnectedComponents /
MarkConnectedComponents on random scenes with rigs, hand cases for every rule, the C ABI's argument checks and struct
layout, the C++ shim over a recording test double, and ``colmap_io.write_clustered_model``."""
import ctypes as ct
import os
import subprocess
from collections import deque

import numpy as np
import pytest

from glomap_b200 import _lib, colmap_io as CI, synthetic as S
from oracle import pruning_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- literal transcription of the reference (image and frame ids, dicts, a union-find, BFS) ----------------------------
def _pair_id(a, b):                          # colmap::ImagePairToPairId
    a, b = min(a, b), max(a, b)
    return a * 2147483647 + b


def _pair_from_id(pid):
    return pid // 2147483647, pid % 2147483647


class _UnionFind:                            # colmap::UnionFind
    def __init__(self):
        self.parent = {}

    def find(self, x):
        self.parent.setdefault(x, x)
        while self.parent[x] != x:
            self.parent[x] = self.parent[self.parent[x]]
            x = self.parent[x]
        return x

    def union(self, x, y):
        rx, ry = self.find(x), self.find(y)
        if rx != ry:
            self.parent[rx] = ry


def _components(pairs, images):
    """FindConnectedComponents(CreateFrameAdjacencyList): components in the order of their smallest frame."""
    adj = {}
    for p in pairs.values():
        if p["is_valid"]:
            f1, f2 = images[p["image_id1"]], images[p["image_id2"]]
            adj.setdefault(f1, set()).add(f2)
            adj.setdefault(f2, set()).add(f1)
    seen, comps = set(), []
    for f in sorted(adj):
        if f in seen:
            continue
        comp, q = {f}, deque([f])
        seen.add(f)
        while q:
            for nb in adj[q.popleft()]:
                if nb not in seen:
                    seen.add(nb)
                    comp.add(nb)
                    q.append(nb)
        comps.append(comp)
    return comps


def reference_prune(frames, images, tracks, min_num_observations=0):
    """frames: {frame_id: {"images": [image ids], "is_registered": bool}}; images: {image_id: frame_id};
    tracks: {track_id: [image ids]}.  Returns (num_comp, cluster_id {frame: id}, is_registered {frame: bool}, stats)."""
    cluster = {f: -1 for f in frames}
    reg = {f: frames[f]["is_registered"] for f in frames}
    cov, obs = {}, {}
    for tid in tracks:
        t = tracks[tid]
        if len(t) <= 2:
            continue
        for i in range(len(t)):
            f1 = images[t[i]]
            obs[f1] = obs.get(f1, 0) + 1
            for j in range(i + 1, len(t)):
                f2 = images[t[j]]
                if f1 == f2:
                    continue
                pid = _pair_id(f1, f2)
                cov[pid] = cov.get(pid, 0) + 1
    counter, vis_frame, pair_count = 0, {}, []
    for pid, count in cov.items():
        if count >= 5:
            counter += 1
            f1, f2 = _pair_from_id(pid)
            if obs.get(f1, 0) < min_num_observations or obs.get(f2, 0) < min_num_observations:
                continue
            vis_frame[pid] = count
            pair_count.append(count)
    stats = dict(covisible_pairs=len(cov), pairs_min5=counter, visibility_edges=len(pair_count))
    if not pair_count:                                             # rule (iii)
        return 0, cluster, reg, stats
    begin = {}
    for f in frames:
        for i in frames[f]["images"]:
            if i in images:
                begin[f] = i
                break
    pairs = {}
    for pid, w in vis_frame.items():
        f1, f2 = _pair_from_id(pid)
        pairs[pid] = dict(image_id1=begin[f1], image_id2=begin[f2], weight=w, is_valid=True)
    max_weight = int(np.argmax(pair_count))
    for f in frames:
        for i in frames[f]["images"]:
            if i == begin.get(f) or i not in images:
                continue
            pairs[_pair_id(begin[f], i)] = dict(image_id1=begin[f], image_id2=i, weight=max_weight, is_valid=True)
    pair_count.sort()
    median = float(pair_count[len(pair_count) // 2])
    diff = sorted(int(abs(c - median)) for c in pair_count)
    mad = float(diff[len(diff) // 2])
    thr = max(median - mad, 20.0)
    stats["strong_threshold"] = thr
    # EstablishStrongClusters: KeepLargestConnectedComponents
    comps = _components(pairs, images)
    largest = max(comps, key=len)                                  # first of the largest: rule (i)
    stats["largest_component_frames"] = len(largest)
    for f in reg:
        reg[f] = False
    for f in largest:
        reg[f] = True
    for p in pairs.values():
        if not reg[images[p["image_id1"]]] or not reg[images[p["image_id2"]]]:
            p["is_valid"] = False
    uf = _UnionFind()
    for p in pairs.values():
        if p["is_valid"] and p["weight"] > thr:
            uf.union(images[p["image_id1"]], images[p["image_id2"]])
    status, iteration = True, 0
    while status:
        status = False
        iteration += 1
        if iteration > 10:
            break
        num_pairs = {}
        for p in pairs.values():
            if not p["is_valid"] or p["weight"] < 0.75 * thr:
                continue
            r1, r2 = uf.find(images[p["image_id1"]]), uf.find(images[p["image_id2"]])
            if r1 == r2:
                continue
            num_pairs.setdefault(r1, {})
            num_pairs.setdefault(r2, {})
            num_pairs[r1][r2] = num_pairs[r1].get(r2, 0) + 1
            num_pairs[r2][r1] = num_pairs[r2].get(r1, 0) + 1
        for r1 in num_pairs:
            for r2, count in num_pairs[r1].items():
                if r1 <= r2:
                    continue
                if count >= 2:
                    status = True
                    uf.union(r1, r2)
    stats["clustering_iterations"] = iteration
    for p in pairs.values():
        if p["is_valid"] and uf.find(images[p["image_id1"]]) != uf.find(images[p["image_id2"]]):
            p["is_valid"] = False
    comps = _components(pairs, images)
    order = sorted(range(len(comps)), key=lambda c: (-len(comps[c]), min(comps[c])))   # rule (ii)
    for rank, c in enumerate(order):
        for f in comps[c]:
            cluster[f] = rank
    return len(comps), cluster, reg, stats


def _random_scene(rng, F, T, rig_frac=0.3, max_len=9):
    """Frames 0..F-1 (frame id = 10 + index); a rig frame has 2-3 images.  Image ids start at 1000 so that an intra-frame
    pair id never equals a frame-pair id."""
    frames, images, img = {}, {}, 1000
    for k in range(F):
        n = int(rng.integers(2, 4)) if rng.random() < rig_frac else 1
        frames[10 + k] = dict(images=list(range(img, img + n)), is_registered=bool(rng.random() < 0.8))
        for i in range(img, img + n):
            images[i] = 10 + k
        img += n
    ids = sorted(images)
    tracks = {}
    hot = rng.choice(F, size=max(2, F // 2), replace=False)    # denser covisibility among some frames
    for t in range(T):
        L = int(rng.integers(1, max_len + 1))
        pool = [i for i in ids if images[i] - 10 in hot] if rng.random() < 0.7 else ids
        tracks[t] = [int(rng.choice(pool)) for _ in range(L)]      # duplicates of images / frames included
    return frames, images, tracks


def _flatten(frames, images, tracks):
    fids = sorted(frames)
    fidx = {f: k for k, f in enumerate(fids)}
    begin, of = [0], []
    for t in sorted(tracks):
        of += [fidx[images[i]] for i in tracks[t]]
        begin.append(len(of))
    loop = np.array([sum(i in images for i in frames[f]["images"]) >= 2 for f in fids], np.uint8)
    reg = np.array([frames[f]["is_registered"] for f in fids], bool)
    return fids, np.array(begin, np.int64), np.array(of, np.int32), loop, reg


def _seeded(seed):
    """Seeds 0-11: dense scenes; 12-15: a few tracks only (few or no visibility edges)."""
    rng = np.random.default_rng(seed)
    F = int(rng.integers(3, 25))
    frames, images, tracks = _random_scene(rng, F, int(rng.integers(40, 400)) if seed < 12 else int(rng.integers(3, 30)))
    return F, frames, images, tracks, [0, 0, 5, 30][seed % 4]


@pytest.mark.parametrize("seed", range(16))
def test_oracle_equals_the_literal_transcription(seed):
    F, frames, images, tracks, min_obs = _seeded(seed)
    n_ref, cl_ref, reg_ref, st_ref = reference_prune(frames, images, tracks, min_obs)
    fids, tb, of, loop, reg = _flatten(frames, images, tracks)
    out = O.prune(tb, of, F, loop, min_obs, reg)
    assert out["num_clusters"] == n_ref
    assert out["cluster_id"].tolist() == [cl_ref[f] for f in fids]
    assert out["is_registered"].tolist() == [reg_ref[f] for f in fids]
    for k, v in st_ref.items():
        assert out["stats"][k] == v, k


def test_random_scenes_reach_every_branch():
    """The random scenes above are not degenerate: some cluster, some split, some take the empty rule."""
    seen = set()
    for seed in range(16):
        F, frames, images, tracks, min_obs = _seeded(seed)
        n, *_ = reference_prune(frames, images, tracks, min_obs)
        seen.add(min(n, 2))
    assert seen == {0, 1, 2}, seen


# ---- hand cases ----------------------------------------------------------------------------------------------------
def _prune(d, **kw):
    return O.prune(d["track_begin"], d["obs_frame"], d["num_frames"], **kw)


def _same_partition(cluster_id, group):
    """Frames of one group share one cluster id, and different groups have different ids."""
    pairs = set(zip(group.tolist(), cluster_id.tolist()))
    return len(pairs) == len(set(group.tolist())) == len(set(cluster_id.tolist()))


def test_groups_are_clusters_and_the_threshold_is_the_median():
    d = S.make_cluster_tracks([5, 7, 6], 40, bridges=[(0, 5, 50), (5, 12, 50)], seed=3)
    out = _prune(d)
    assert out["stats"]["strong_threshold"] == d["threshold"] == 40.0
    assert out["num_clusters"] == 1 and (out["cluster_id"] == 0).all() and out["is_registered"].all()


@pytest.mark.parametrize("bridges,merged", [([(0, 5, 35)], False), ([(0, 5, 35), (1, 6, 35)], True),
                                            ([(0, 5, 35), (1, 6, 29)], False), ([(0, 5, 35), (1, 6, 30)], True),
                                            ([(0, 5, 41)], True), ([(0, 5, 40)], False)])
def test_bridges(bridges, merged):
    """thr = 40: one weak bridge (30 <= c <= 40) does not merge two groups, two do; 29 < 0.75 thr = 30 is not counted;
    a bridge above thr is a strong edge."""
    d = S.make_cluster_tracks([5, 6], 40, bridges=bridges, seed=4)
    out = _prune(d)
    assert out["stats"]["strong_threshold"] == 40.0
    assert out["is_registered"].all() and out["stats"]["largest_component_frames"] == 11
    if merged:
        assert out["num_clusters"] == 1 and (out["cluster_id"] == 0).all()
    else:
        assert out["num_clusters"] == 2 and _same_partition(out["cluster_id"], d["group"])
        assert out["cluster_id"][d["group"] == 1].tolist() == [0] * 6     # the larger group is cluster 0


def test_threshold_floor_of_20():
    d = S.make_cluster_tracks([5, 6], 15, bridges=[(0, 5, 16), (1, 6, 15)], seed=5)
    out = _prune(d)
    assert out["stats"]["strong_threshold"] == 20.0                    # median - MAD = 15
    assert out["num_clusters"] == 1                                    # 15 = 0.75 * 20: both bridges count


def test_ties_of_rules_i_and_ii():
    # (i) two equal components: the one with frame 0 is kept
    d = S.make_cluster_tracks([5, 5], 40, seed=6)
    out = _prune(d)
    keep = d["group"][0]
    assert out["is_registered"].tolist() == (d["group"] == keep).tolist()
    assert out["num_clusters"] == 1 and (out["cluster_id"][d["group"] == keep] == 0).all()
    # (ii) two equal clusters in one component: numbered by their smallest frame
    d = S.make_cluster_tracks([5, 5], 40, bridges=[(0, 5, 35)], seed=7)
    out = _prune(d)
    assert out["num_clusters"] == 2
    first = d["group"][0]
    assert (out["cluster_id"][d["group"] == first] == 0).all() and (out["cluster_id"][d["group"] != first] == 1).all()


def test_empty_rule_iii():
    reg = np.array([1, 0, 1, 1], bool)
    for tb, of in [(np.array([0, 2, 4]), np.array([0, 1, 2, 3])),                      # tracks of <= 2 observations
                   (np.array([0, 3, 6]), np.array([0, 1, 2, 0, 1, 3])),                # no pair reaches 5
                   (np.array([0]), np.array([], np.int64))]:                           # no track
        out = O.prune(tb, of, 4, is_registered=reg)
        assert out["num_clusters"] == 0 and (out["cluster_id"] == -1).all()
        assert out["is_registered"].tolist() == reg.tolist()
        assert out["stats"]["clustering_iterations"] == 0


def _tracks_from_pairs(pairs):
    tracks = []
    for a, b, c in pairs:
        if c % 2:
            tracks.append([a, a, a, b])
            c -= 3
        tracks += [[a, a, b]] * (c // 2)
    lens = [len(t) for t in tracks]
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), np.concatenate(tracks).astype(np.int32)


def test_ten_pass_cap():
    """A ladder: (0, 1) strong, (k, k+1) and (k, k+2) weak.  Frame k joins the set of 0 in pass k - 1, so frames 2..11
    join in passes 1..10; the 11th pass is cut off (iteration = 11) and frames 12, 13 stay outside every cluster."""
    n = 14
    pairs = [(0, 1, 60)] + [(k, k + 1, 26) for k in range(1, n - 1)] + [(k, k + 2, 26) for k in range(n - 2)]
    tb, of = _tracks_from_pairs(pairs)
    out = O.prune(tb, of, n)
    assert out["stats"]["strong_threshold"] == 26.0
    assert out["stats"]["clustering_iterations"] == 11
    assert out["cluster_id"].tolist() == [0] * 12 + [-1, -1]
    assert out["is_registered"].all() and out["num_clusters"] == 1
    frames = {k: dict(images=[k + 100], is_registered=True) for k in range(n)}
    images = {k + 100: k for k in range(n)}
    tracks = {t: [int(f) + 100 for f in of[tb[t]:tb[t + 1]]] for t in range(len(tb) - 1)}
    n_ref, cl_ref, _, st_ref = reference_prune(frames, images, tracks)
    assert st_ref["clustering_iterations"] == 11 and [cl_ref[k] for k in range(n)] == out["cluster_id"].tolist()


def test_self_loops_make_singleton_components():
    """A rig frame without any other edge is a component of its own, but never part of the largest one here."""
    d = S.make_cluster_tracks([5, 6], 40, bridges=[(0, 5, 35)], shuffle=False)
    F = d["num_frames"] + 2
    loop = np.zeros(F, np.uint8)
    loop[[3, F - 1]] = 1
    out = O.prune(d["track_begin"], d["obs_frame"], F, loop)
    assert out["cluster_id"][F - 1] == -1 and not out["is_registered"][F - 1]
    assert out["num_clusters"] == 2 and out["cluster_id"][F - 2] == -1


# ---- C ABI ---------------------------------------------------------------------------------------------------------
def test_abi_null_arguments_are_invalid_without_a_device():
    lib = _lib.load()
    tb = np.zeros(1, np.int64)
    cid, reg, nc, st = np.zeros(2, np.int32), np.ones(2, np.uint8), ct.c_int32(), _lib.PruneStats()
    p = lambda a: a.ctypes.data_as(ct.c_void_p)   # noqa: E731
    assert lib.b200sfm_prune_weakly_connected(None, 2, 0, p(tb), None, None, 0, 0, p(cid), p(reg), ct.byref(nc), ct.byref(st)) == 1
    assert lib.b200sfm_prune_weakly_connected(None, 2, 0, None, None, None, 0, 0, p(cid), p(reg), ct.byref(nc), None) == 1
    assert lib.b200sfm_prune_weakly_connected(None, -1, 0, p(tb), None, None, 0, 0, None, None, None, None) == 1


def test_prune_stats_layout_matches_ctypes(tmp_path):
    fields = [f for f, _ in _lib.PruneStats._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sfm.h"\nint main(void) {\n' +
                   "".join(f'  printf("%zu\\n", offsetof(b200sfm_prune_stats, {f}));\n' for f in fields) +
                   '  printf("%zu\\n", sizeof(b200sfm_prune_stats));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True, capture_output=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [getattr(_lib.PruneStats, f).offset for f in fields] + [ct.sizeof(_lib.PruneStats)]


# ---- C++ shim ------------------------------------------------------------------------------------------------------
def test_shim_flattens_in_sorted_id_order_and_writes_back(tmp_path):
    lib, exe, dump = tmp_path / "libb200sfm.so", tmp_path / "prune_driver", tmp_path / "dump.txt"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c"),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_prune.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "shim_mock", "prune_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe)], env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rec = {}
    for line in dump.read_text().splitlines()[1:]:
        name, n, *vals = line.split()
        rec[name] = [int(v) for v in vals]
        assert len(vals) == int(n)
    assert rec["scalars"] == [4, 0, 3]                       # min_num_observations, default pass size, F
    # tracks in sorted id order (3, 5, 7); frames 10, 20, 30 -> 0, 1, 2; images 201 / 202 are frame 20
    assert rec["track_begin"] == [0, 2, 6, 9]
    assert rec["obs_frame"] == [1, 1, 0, 2, 1, 0, 2, 0, 1]
    assert rec["frame_self_loop"] == [0, 1, 0]               # frame 20 has two images
    assert rec["is_registered"] == [1, 1, 0]
    assert r.stdout.splitlines()[:4] == ["clusters 2", "frame 10 registered 1 cluster 0", "frame 20 registered 1 cluster 1",
                                         "frame 30 registered 0 cluster -1"]


def test_shim_prune_typechecks_against_the_glomap_api():
    """Inside a glomap build the shim takes glomap's Frame (is_registered, cluster_id), Image (frame_id) and Track."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(ROOT, "tests", "shim_mock", "glomap_stub_prune"),
                        "-I" + os.path.join(ROOT, "glomap_b200", "host"),
                        os.path.join(ROOT, "tests", "shim_mock", "prune_typecheck.cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


# ---- clustered model output ----------------------------------------------------------------------------------------
def _hand_scene():
    """4 images; points: 0 seen by images 0, 1, 2; 1 by 2, 3; 2 by 0, 3; 3 by 1, 2, 3."""
    begin = np.array([0, 3, 5, 7, 10], np.int64)
    obs_cam = np.array([0, 1, 2, 2, 3, 0, 3, 1, 2, 3], np.int32)
    C = 4
    return S.Scene(np.tile([0, 0, 0, 1.0], (C, 1)), np.array([[0, 0, 5.0]] * C), np.arange(12, dtype=float).reshape(4, 3) * 0.1,
                   begin, obs_cam, np.arange(20, dtype=float).reshape(10, 2), np.zeros(C, np.int32), np.zeros(1, np.int32),
                   np.array([[500.0, 50, 50] + [0] * 9]))


def test_write_clustered_model(tmp_path):
    sc = _hand_scene()
    written = CI.write_clustered_model(str(tmp_path), sc, None, [0, 0, 1, 1], [True] * 4)
    assert written == [str(tmp_path / "0"), str(tmp_path / "1")]
    cams0, ims0, pts0 = CI.read_model(str(tmp_path / "0"))
    cams1, ims1, pts1 = CI.read_model(str(tmp_path / "1"))
    assert sorted(ims0) == [1, 2] and sorted(ims1) == [3, 4] and len(cams0) == len(cams1) == 1
    # cluster 0 (images 1, 2): point 1 keeps (1, 2); point 4 keeps (2) only -> dropped; points 2, 3 have < 2 elements
    assert sorted(pts0) == [1] and pts0[1].image_ids.tolist() == [1, 2]
    # cluster 1 (images 3, 4): point 2 (3, 4), point 4 (3, 4); point 1 keeps (3) -> dropped
    assert sorted(pts1) == [2, 4] and pts1[4].image_ids.tolist() == [3, 4]
    inv = CI.INVALID_POINT3D
    assert ims1[3].point3D_ids.tolist().count(inv) == len(ims1[3].point3D_ids) - 2
    # every id -1: the registered images in 0/ (the reference deregisters the other frames before writing)
    written = CI.write_clustered_model(str(tmp_path / "all"), sc, None, [-1] * 4, [True, True, True, False])
    assert written == [str(tmp_path / "all" / "0")]
    _, ims, pts = CI.read_model(written[0])
    assert sorted(ims) == [1, 2, 3] and sorted(pts) == [1, 4]          # point 2 keeps image 1 only
    assert pts[1].image_ids.tolist() == [1, 2, 3] and pts[4].image_ids.tolist() == [2, 3]
    # all registered: the same images and points as model_from_scene
    written = CI.write_clustered_model(str(tmp_path / "whole"), sc, None, [-1] * 4, [True] * 4)
    _, ims, pts = CI.read_model(written[0])
    _, ims_w, pts_w = CI.model_from_scene(sc)
    assert sorted(ims) == sorted(ims_w) and sorted(pts) == sorted(pts_w)
    for i in ims:
        assert ims[i].point3D_ids.tolist() == ims_w[i].point3D_ids.tolist()


def test_prune_wrapper_rejects_inputs_that_would_wrap_or_overrun():
    """Checked on the host before any device call: no GPU needed."""
    from glomap_b200 import reconstruction_pruning as RP
    tb = np.array([0, 3], np.int64)
    with pytest.raises(ValueError, match="range of int32"):
        RP.prune_weakly_connected_images(tb, np.array([0, 1, 2**31], np.int64), 4)
    with pytest.raises(ValueError, match="entries"):
        RP.prune_weakly_connected_images(tb, np.array([0, 1], np.int32), 4)               # shorter than track_begin[-1]
    with pytest.raises(ValueError, match="integer"):
        RP.prune_weakly_connected_images(tb, np.array([0.0, 1.0, 2.0]), 4)
    with pytest.raises(ValueError, match="is_registered"):
        RP.prune_weakly_connected_images(tb, np.array([0, 1, 2], np.int32), 4, is_registered=np.ones(3, bool))
    with pytest.raises(ValueError, match="frame_self_loop"):
        RP.prune_weakly_connected_images(tb, np.array([0, 1, 2], np.int32), 4, frame_self_loop=np.ones(5, np.uint8))


def test_prune_subcommand_names_the_camera_model_restriction(tmp_path):
    sc = _hand_scene()
    cams, ims, pts = CI.model_from_scene(sc)
    for c in cams.values():
        c.model_id, c.params = 4, np.array([500.0, 500, 50, 50, 0, 0, 0, 0])   # OPENCV
    CI.write_model(str(tmp_path / "m"), cams, ims, pts)
    with pytest.raises(SystemExit, match="camera models 0-3"):
        CI._main(["prune", str(tmp_path / "m"), str(tmp_path / "out")])
