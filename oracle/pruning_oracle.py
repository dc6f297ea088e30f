"""CPU restatement of PruneWeaklyConnectedImages (glomap/processors/reconstruction_pruning.cc:6-131) with
EstablishStrongClusters (processors/view_graph_manipulation.cc:70-176), KeepLargestConnectedComponents and
MarkConnectedComponents (scene/view_graph.cc:56-126), in frame space: frames 0..F-1, a track is the frame index of each
of its observations (CSR ``track_begin`` over ``obs_frame``), ``frame_self_loop[f]`` marks a frame with >= 2 images
present (its intra-frame edges are self-loops in frame space, :63-104).

Pair counts by numpy ``unique``, connected components by scipy, the merge passes of EstablishStrongClusters over the
component labels.  Where the reference depends on hash-map order or is undefined, the same rules as
``b200sfm_prune_weakly_connected`` (include/b200sfm.h):
  (i)   between equally large components in KeepLargestConnectedComponents, the one with the smallest frame is kept;
  (ii)  equally large clusters are numbered by their smallest frame, ascending;
  (iii) with no visibility edge: num_clusters = 0, every cluster id -1, is_registered as given."""
from __future__ import annotations

import numpy as np


def _components(F: int, a, b, in_adj):
    """Root (= smallest frame) of every frame's component over the edges (a, b); -1 outside ``in_adj``."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    g = sp.coo_matrix((np.ones(len(a)), (a, b)), shape=(F, F))
    _, lab = connected_components(g, directed=False)
    first = np.full(lab.max() + 1 if F else 0, F, np.int64)
    np.minimum.at(first, lab, np.arange(F))
    root = first[lab]
    return np.where(np.asarray(in_adj, bool), root, -1)


def covisibility(track_begin, obs_frame, F: int):
    """Per-frame observation counts and the (lo, hi, count) of every covisible frame pair (:14-36)."""
    tb = np.asarray(track_begin, np.int64)
    of = np.asarray(obs_frame, np.int64)
    lens = np.diff(tb)
    obs_count = np.zeros(F, np.int64)
    keys = []
    for L in np.unique(lens[lens > 2]):
        t = np.flatnonzero(lens == L)
        fr = of[tb[t][:, None] + np.arange(L)[None, :]]          # [tracks, L]
        np.add.at(obs_count, fr.ravel(), 1)
        i, j = np.triu_indices(int(L), 1)
        a, b = fr[:, i].ravel(), fr[:, j].ravel()
        m = a != b
        keys.append(np.minimum(a[m], b[m]) * F + np.maximum(a[m], b[m]))
    k = np.concatenate(keys) if keys else np.zeros(0, np.int64)
    uk, cnt = np.unique(k, return_counts=True)
    return obs_count, uk // max(F, 1), uk % max(F, 1), cnt


def prune(track_begin, obs_frame, F: int, frame_self_loop=None, min_num_observations: int = 0, is_registered=None):
    """Returns dict(cluster_id [F] int32, is_registered [F] bool, num_clusters, stats)."""
    reg_in = np.ones(F, bool) if is_registered is None else np.asarray(is_registered, bool).copy()
    of = np.asarray(obs_frame, np.int64)
    if len(of) and (of.min() < 0 or of.max() >= F):
        raise ValueError("obs_frame outside [0, F)")
    loop = np.zeros(F, bool) if frame_self_loop is None else np.asarray(frame_self_loop, bool)
    stats = dict(covisible_pairs=0, pairs_min5=0, visibility_edges=0, strong_threshold=0.0, clustering_iterations=0,
                 largest_component_frames=0)
    out = dict(cluster_id=np.full(F, -1, np.int32), is_registered=reg_in, num_clusters=0, stats=stats)
    if F < 2:
        return out
    obs_count, lo, hi, cnt = covisibility(track_begin, obs_frame, F)
    stats["covisible_pairs"] = len(cnt)
    m5 = cnt >= 5
    stats["pairs_min5"] = int(m5.sum())
    e = m5 & (obs_count[lo] >= min_num_observations) & (obs_count[hi] >= min_num_observations)
    a, b, w = lo[e], hi[e], cnt[e].astype(np.int64)
    E = len(w)
    stats["visibility_edges"] = E
    if E == 0:                                                     # rule (iii)
        return out
    ws = np.sort(w)
    median = ws[E // 2]
    mad = np.sort(np.abs(ws - median))[E // 2]
    thr = max(float(median) - float(mad), 20.0)
    stats["strong_threshold"] = thr
    # 5a. KeepLargestConnectedComponents
    in_adj = loop.copy()
    in_adj[a] = True
    in_adj[b] = True
    root = _components(F, a, b, in_adj)
    size = np.bincount(root[in_adj], minlength=F)
    best = int(np.argmax(size))                                    # first maximum: the smallest root, rule (i)
    reg = in_adj & (root == best)
    stats["largest_component_frames"] = int(size[best])
    valid = reg[a] & reg[b]
    # 5b. strong edges
    s = valid & (w > thr)
    lab = _components(F, a[s], b[s], np.ones(F, bool))
    # 5c. merge passes
    iteration, status = 0, True
    while status:
        status = False
        iteration += 1
        if iteration > 10:
            break
        c = valid & ~(w < 0.75 * thr) & (lab[a] != lab[b])
        r1, r2 = lab[a[c]], lab[b[c]]
        pk, pc = np.unique(np.minimum(r1, r2) * F + np.maximum(r1, r2), return_counts=True)
        sel = pk[pc >= 2]
        if len(sel):
            status = True
            f = np.arange(F)
            lab = _components(F, np.concatenate([f, sel // F]), np.concatenate([lab, sel % F]), np.ones(F, bool))
    stats["clustering_iterations"] = iteration
    # 5d-e. drop the edges between sets, MarkConnectedComponents
    keep = valid & (lab[a] == lab[b])
    adj2 = loop & reg
    adj2[a[keep]] = True
    adj2[b[keep]] = True
    root2 = _components(F, a[keep], b[keep], adj2)
    roots = np.flatnonzero(adj2 & (root2 == np.arange(F)))
    sizes = np.bincount(root2[adj2], minlength=F)[roots]
    order = np.lexsort((roots, -sizes))                            # size descending, smallest frame ascending: rule (ii)
    rank = np.full(F, -1, np.int64)
    rank[roots[order]] = np.arange(len(roots))
    cid = np.where(adj2, rank[np.maximum(root2, 0)], -1).astype(np.int32)
    out.update(cluster_id=cid, is_registered=reg, num_clusters=len(roots))
    return out
