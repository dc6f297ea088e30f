"""numpy restatement of the device InitializeFromMaximumSpanningTree (glomap_b200/csrc/mst_kernels.cuh), step for step:
ranks from a stable sort of max_w - w, Boruvka by rank with the mutual-pair rule and pointer jumping, Euler-tour rooting
with Wyllie list ranking, and the composition R_v = A_v A_parent ... R_root by synchronous pointer jumping.  It checks
the data-parallel form against the host function (scipy MST + BFS) without a device."""
from __future__ import annotations

import numpy as np

NONE = np.iinfo(np.int64).max


def ranks(weight) -> np.ndarray:
    """Edge indices in rank order: key max_w - w (-0 folded into +0), ties by edge index."""
    w = np.asarray(weight, np.float64)
    key = w.max() - w if len(w) else w
    key = np.where(key == 0.0, 0.0, key)
    return np.argsort(key, kind="stable")


def flatten(p: np.ndarray) -> np.ndarray:
    while True:
        q = p[p]
        if np.array_equal(q, p):
            return p
        p = q


def boruvka(n: int, eu: np.ndarray, ev: np.ndarray):
    """eu, ev: endpoints in rank order.  Returns (in_tree [E] by rank, comp [n] = root of each node's component, rounds)."""
    E = len(eu)
    comp = np.arange(n)
    act = np.arange(E)
    in_tree = np.zeros(E, bool)
    rounds = 0
    while True:
        act = act[comp[eu[act]] != comp[ev[act]]]
        if len(act) == 0:
            return in_tree, comp, rounds
        rounds += 1
        best = np.full(n, NONE)
        np.minimum.at(best, comp[eu[act]], act)
        np.minimum.at(best, comp[ev[act]], act)
        v = np.nonzero((comp == np.arange(n)) & (best != NONE))[0]
        r = best[v]
        a, b = comp[eu[r]], comp[ev[r]]
        other = np.where(a == v, b, a)
        in_tree[r] = True
        hook = comp.copy()
        hook[v] = np.where((best[other] == r) & (v < other), v, other)
        comp = flatten(hook)


def euler_parents(n: int, tu: np.ndarray, tv: np.ndarray, comp: np.ndarray, root: int):
    """Tree edges k = (tu[k], tv[k]).  Returns (k, child, parent) for the tree edges of the root's component."""
    m = len(tu)
    A = 2 * m
    src = np.empty(A, np.int64)
    src[0::2], src[1::2] = tu, tv
    sarc = np.argsort(src, kind="stable")
    ssrc = src[sarc]
    pos = np.empty(A, np.int64)
    pos[sarc] = np.arange(A)
    lo, hi = np.searchsorted(ssrc, np.arange(n), "left"), np.searchsorted(ssrc, np.arange(n), "right")
    t = np.arange(A) ^ 1
    v = src[t]
    p = pos[t] + 1
    p = np.where(p == hi[v], lo[v], p)
    succ = sarc[p]
    inc = comp[src] == comp[root]
    if lo[root] < hi[root]:
        succ = np.where(succ == sarc[lo[root]], -1, succ)
    succ[~inc] = -2
    dist = (succ >= 0).astype(np.int64)
    nx, span = succ, 1
    while span < A:                                       # Wyllie, synchronous
        ok = nx >= 0
        d2, n2 = dist.copy(), nx.copy()
        d2[ok] += dist[nx[ok]]
        n2[ok] = nx[nx[ok]]
        dist, nx, span = d2, n2, 2 * span
    k = np.nonzero(comp[tu] == comp[root])[0]
    down = dist[2 * k] > dist[2 * k + 1]                   # tu -> tv comes first in the tour
    return k, np.where(down, tv[k], tu[k]), np.where(down, tu[k], tv[k])


def mst_init(n: int, ei, ej, R_rel, weight, root: int = 0, R_init=None):
    """Returns (R [n,3,3], parent [n], stats dict) like b200sfm_ra_mst_init."""
    ei, ej = np.asarray(ei, np.int64), np.asarray(ej, np.int64)
    R_rel = np.asarray(R_rel, np.float64).reshape(-1, 3, 3)
    R = np.tile(np.eye(3), (n, 1, 1)) if R_init is None else np.array(R_init, np.float64, copy=True)
    order = ranks(weight)
    eu, ev = ei[order], ej[order]
    in_tree, comp, rounds = boruvka(n, eu, ev)
    te = np.nonzero(in_tree)[0]
    k, child, par = euler_parents(n, eu[te], ev[te], comp, root)
    parent = np.full(n, -1, np.int64)
    parent[root] = root
    parent[child] = par
    anc = parent.copy()
    depth = np.zeros(n, np.int64)
    depth[child] = 1
    M = np.zeros((n, 3, 3))
    Rt = R_rel[order[te[k]]]
    M[child] = np.where((child == ev[te[k]])[:, None, None], Rt, np.swapaxes(Rt, 1, 2))
    while True:                                           # synchronous pointer jumping over the ancestors
        go = np.nonzero((anc >= 0) & (anc != root))[0]
        if len(go) == 0:
            break
        a = anc[go]
        M2, anc2, depth2 = M.copy(), anc.copy(), depth.copy()
        M2[go] = M[go] @ M[a]
        anc2[go] = anc[a]
        depth2[go] = depth[go] + depth[a]
        M, anc, depth = M2, anc2, depth2
    R[child] = M[child] @ R[root]
    stats = dict(num_reached=int((parent >= 0).sum()), num_tree_edges=len(te), boruvka_rounds=rounds,
                 max_depth=int(depth.max()))
    return R, parent, stats
