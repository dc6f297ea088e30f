"""Maximum-spanning-tree initialisation without a device: b200sfm_ra_mst_init's argument checks and stats struct, and
the numpy restatement of its data-parallel form (oracle/mst_oracle.py) against the host function
initialize_from_maximum_spanning_tree (scipy MST + BFS) and, for repeated pairs, a plain Kruskal transcription."""
import ctypes as ct
import os
import subprocess

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E, geometry as G
from glomap_b200.synthetic import ViewGraph
from oracle import mst_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = 1


def random_graph(rng, n, E_, repeated=False, self_loops=True, wmax=5):
    ei, ej = rng.integers(0, n, E_), rng.integers(0, n, E_)
    if not self_loops:
        keep = ei != ej
        ei, ej = ei[keep], ej[keep]
    if not repeated:     # one edge per unordered pair, as glomap's pair ids give
        _, first = np.unique(np.minimum(ei, ej) * n + np.maximum(ei, ej), return_index=True)
        first = np.sort(first)
        ei, ej = ei[first], ej[first]
    R_rel = G.so3_exp(rng.normal(size=(len(ei), 3)))
    w = rng.integers(0, wmax + 1, len(ei)).astype(np.float64)
    return ViewGraph(n, ei.astype(np.int32), ej.astype(np.int32), R_rel, w, np.tile(np.eye(3), (n, 1, 1)))


def scipy_parents(vg, root=0):
    """The host function's tree (same keys and index tie-break) and BFS from root; -1 = unreached."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import breadth_first_order, minimum_spanning_tree
    n, m = vg.n_images, vg.E
    wmax = float(vg.weight.max()) if m else 0.0
    cost = (wmax - vg.weight) + 1e-9 * (1 + np.arange(m) / max(m, 1))
    Gm = sp.coo_matrix((cost, (vg.ei, vg.ej)), shape=(n, n)).tocsr()
    T = minimum_spanning_tree(Gm.maximum(Gm.T))
    _, pred = breadth_first_order(T.maximum(T.T).tocsr(), root, directed=False)
    par = np.where(pred < 0, -1, pred)
    par[root] = root
    return par


def kruskal_parents(vg, root=0):
    """Plain Kruskal over (max_w - w, index) with union-find, then BFS from root."""
    n = vg.n_images
    w = np.asarray(vg.weight, np.float64)
    key = (w.max() - w) if vg.E else w
    uf = list(range(n))

    def find(x):
        while uf[x] != x:
            uf[x] = uf[uf[x]]
            x = uf[x]
        return x
    adj = [[] for _ in range(n)]
    for e in sorted(range(vg.E), key=lambda e: (key[e] + 0.0, e)):
        a, b = find(int(vg.ei[e])), find(int(vg.ej[e]))
        if a != b:
            uf[a] = b
            adj[vg.ei[e]].append((int(vg.ej[e]), e))
            adj[vg.ej[e]].append((int(vg.ei[e]), e))
    par, edge = np.full(n, -1), np.full(n, -1)
    par[root], queue = root, [root]
    for u in queue:
        for v, e in adj[u]:
            if par[v] < 0:
                par[v], edge[v] = u, e
                queue.append(v)
    return par, edge


def host_rooted(vg, R_init, root):
    """initialize_from_maximum_spanning_tree rooted at `root`: swap the labels root <-> 0 (the tree depends on the edge
    order only), run the host function, swap back."""
    perm = np.arange(vg.n_images)
    perm[[0, root]] = perm[[root, 0]]
    vg2 = ViewGraph(vg.n_images, perm[vg.ei].astype(np.int32), perm[vg.ej].astype(np.int32), vg.R_rel, vg.weight, vg.R_gt)
    R0 = None if R_init is None else R_init[perm]
    return E.initialize_from_maximum_spanning_tree(vg2, R0)[perm]


def test_invalid_arguments_are_refused_without_a_device():
    lib = _lib.load()
    st = _lib.MSTStats()
    ei, ej = (ct.c_int32 * 2)(0, 1), (ct.c_int32 * 2)(1, 2)
    Rr, w = (ct.c_double * 18)(), (ct.c_double * 2)(1.0, 2.0)
    R, par = (ct.c_double * 27)(), (ct.c_int32 * 3)()
    call = lambda *a: lib.b200sfm_ra_mst_init(*a, ct.byref(st))   # noqa: E731
    assert call(None, 3, 2, ei, ej, Rr, w, 0, R, par) == INVALID                 # null context
    for bad in ((None, 3, 2, ei, ej, Rr, w, 0, None, par),                      # null R
                (None, 3, 2, None, ej, Rr, w, 0, R, par),                       # null edge arrays
                (None, 3, 2, ei, ej, None, w, 0, R, par),
                (None, 3, 2, ei, ej, Rr, None, 0, R, par),
                (None, 0, 2, ei, ej, Rr, w, 0, R, par),                         # n_nodes < 1
                (None, 3, -1, ei, ej, Rr, w, 0, R, par),                        # n_edges < 0
                (None, 3, 2**31, ei, ej, Rr, w, 0, R, par),                     # n_edges > INT32_MAX
                (None, 3, 2, ei, ej, Rr, w, 3, R, par),                         # root out of range
                (None, 3, 2, ei, ej, Rr, w, -1, R, par),
                (None, 2, 2, ei, ej, Rr, w, 0, R, par),                         # endpoint out of range
                (None, 3, 2, ei, ej, Rr, (ct.c_double * 2)(1.0, float("nan")), 0, R, par)):   # NaN weight
        assert call(*bad) == INVALID


def test_stats_struct_matches_the_c_header(tmp_path):
    cls = _lib.MSTStats
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "b200sfm.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(b200sfm_mst_stats));']
    lines += [f'  printf("{f} %zu\\n", offsetof(b200sfm_mst_stats, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "mst.c", tmp_path / "mst"
    src.write_text("\n".join(lines))
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out["size"]) == ct.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f


def test_prototype_is_bound():
    fn = _lib.load().b200sfm_ra_mst_init
    assert fn.argtypes[-1] == ct.POINTER(_lib.MSTStats) and len(fn.argtypes) == 11


def test_oracle_matches_the_host_function_on_random_graphs():
    rng = np.random.default_rng(7)
    for it in range(300):
        n = int(rng.integers(1, 40))
        vg = random_graph(rng, n, int(rng.integers(0, 3 * n + 1)), wmax=int(rng.choice([0, 1, 5, 50])))
        root = 0 if it % 3 else int(rng.integers(0, n))
        R_init = None if it % 2 else G.so3_exp(rng.normal(size=(n, 3)))
        R, par, st = MO.mst_init(n, vg.ei, vg.ej, vg.R_rel, vg.weight, root, R_init)
        ref = scipy_parents(vg, root)
        assert np.array_equal(par, ref), it
        assert np.abs(R - host_rooted(vg, R_init, root)).max() <= 1e-12, it
        assert st["num_reached"] == int((ref >= 0).sum())
        assert st["boruvka_rounds"] <= int(np.ceil(np.log2(n)))


def test_oracle_matches_kruskal_with_repeated_pairs():
    rng = np.random.default_rng(11)
    for it in range(200):
        n = int(rng.integers(2, 25))
        vg = random_graph(rng, n, int(rng.integers(1, 4 * n)), repeated=True, wmax=3)
        root = int(rng.integers(0, n))
        R, par, _ = MO.mst_init(n, vg.ei, vg.ej, vg.R_rel, vg.weight, root)
        kpar, kedge = kruskal_parents(vg, root)
        assert np.array_equal(par, kpar), it
        for v in np.nonzero((kpar >= 0) & (np.arange(n) != root))[0]:     # R_v = A_v R_parent along Kruskal's edges
            e = kedge[v]
            A = vg.R_rel[e] if vg.ej[e] == v else vg.R_rel[e].T
            assert np.abs(R[v] - A @ R[kpar[v]]).max() <= 1e-12


def test_oracle_depth_is_logarithmic_on_a_path():
    n = 4096
    ei = np.arange(n - 1, dtype=np.int32)
    vg = ViewGraph(n, ei, ei + 1, G.so3_exp(np.full((n - 1, 3), 0.01)), np.ones(n - 1), None)
    R, par, st = MO.mst_init(n, vg.ei, vg.ej, vg.R_rel, vg.weight)
    assert np.array_equal(par, np.concatenate([[0], np.arange(n - 1)])) and st["max_depth"] == n - 1
    assert np.abs(R - E.initialize_from_maximum_spanning_tree(vg)).max() <= 1e-12


@pytest.mark.parametrize("n", [1, 5])
def test_oracle_without_edges(n):
    R, par, st = MO.mst_init(n, np.zeros(0), np.zeros(0), np.zeros((0, 9)), np.zeros(0), n - 1)
    assert par.tolist() == [-1] * (n - 1) + [n - 1] and np.array_equal(R, np.tile(np.eye(3), (n, 1, 1)))
    assert st == dict(num_reached=1, num_tree_edges=0, boruvka_rounds=0, max_depth=0)
