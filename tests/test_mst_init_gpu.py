"""b200sfm_ra_mst_init on the device: parents equal to the host tree (scipy MST + BFS, or plain Kruskal for repeated
pairs) exactly, rotations within 1e-10 of initialize_from_maximum_spanning_tree, bit-identical repeated calls, a launch
count that does not grow with the depth, and EstimateRotations starting from it above MST_DEVICE_MIN_EDGES."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_mst_init_cpu import host_rooted, kruskal_parents, random_graph, scipy_parents  # noqa: E402

from glomap_b200 import _lib, estimators as E, geometry as G, synthetic as S  # noqa: E402
from glomap_b200.synthetic import ViewGraph  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    return E.default_context()


def forest_edges(vg):
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    n = vg.n_images
    return n - connected_components(sp.coo_matrix((np.ones(vg.E), (vg.ei, vg.ej)), shape=(n, n)), directed=False)[0]


def dev(ctx, vg, R_init=None, root=0):
    st = _lib.MSTStats()
    R, par = E.initialize_from_maximum_spanning_tree_device(vg, R_init, ctx, root, stats=st)
    return R, par, st


def check(ctx, vg, R_init=None, root=0, tol=1e-10):
    R, par, st = dev(ctx, vg, R_init, root)
    ref = scipy_parents(vg, root)
    assert np.array_equal(par, ref)
    assert np.abs(R - host_rooted(vg, R_init, root)).max() <= tol
    reached = par >= 0
    assert np.abs(np.swapaxes(R[reached], 1, 2) @ R[reached] - np.eye(3)).max() <= tol
    R0 = np.tile(np.eye(3), (vg.n_images, 1, 1)) if R_init is None else R_init
    assert R[~reached].tobytes() == np.asarray(R0)[~reached].tobytes()            # unreached rows bitwise untouched
    assert st.num_reached == int(reached.sum())
    return R, par, st


def test_random_graphs_with_heavy_ties(ctx):
    rng = np.random.default_rng(3)
    for it in range(60):
        n = int(rng.integers(2, 3000))
        vg = random_graph(rng, n, int(rng.integers(0, 6 * n)), wmax=int(rng.choice([1, 3, 20, 200])))
        root = 0 if it % 2 else int(rng.integers(0, n))
        check(ctx, vg, G.so3_exp(rng.normal(size=(n, 3))) if it % 3 else None, root)


def test_all_equal_weights_break_ties_by_edge_index(ctx):
    rng = np.random.default_rng(4)
    vg = random_graph(rng, 2000, 20000, wmax=0)
    _, _, st = check(ctx, vg)
    assert st.num_tree_edges == forest_edges(vg)


def test_self_loops_never_enter_the_tree(ctx):
    rng = np.random.default_rng(5)
    n = 50
    vg = random_graph(rng, n, 400, wmax=10)
    loops = np.arange(0, n, 2, dtype=np.int32)
    vg = ViewGraph(n, np.concatenate([loops, vg.ei]), np.concatenate([loops, vg.ej]),
                   np.concatenate([G.so3_exp(rng.normal(size=(len(loops), 3))), vg.R_rel]),
                   np.concatenate([np.full(len(loops), 100.0), vg.weight]), None)   # the heaviest edges are the loops
    check(ctx, vg)
    only = ViewGraph(4, np.array([0, 1, 1], np.int32), np.array([0, 1, 1], np.int32), np.tile(np.eye(3), (3, 1, 1)) * 2,
                     np.ones(3), None)
    R, par, st = dev(ctx, only)
    assert par.tolist() == [0, -1, -1, -1] and st.num_tree_edges == 0 and np.array_equal(R, np.tile(np.eye(3), (4, 1, 1)))


def test_forest_leaves_unreached_rows_untouched(ctx):
    rng = np.random.default_rng(6)
    a = random_graph(rng, 300, 1500, wmax=5)
    b = random_graph(rng, 200, 1000, wmax=5)
    n = 600                                                        # nodes 500..599 isolated
    vg = ViewGraph(n, np.concatenate([b.ei + 300, a.ei]).astype(np.int32), np.concatenate([b.ej + 300, a.ej]).astype(np.int32),
                   np.concatenate([b.R_rel, a.R_rel]), np.concatenate([b.weight, a.weight]), None)
    R_init = G.so3_exp(rng.normal(size=(n, 3)))
    for root in (0, 350, 550):
        R, par, st = check(ctx, vg, R_init, root)
        assert np.array_equal(R[root], R_init[root])
        assert st.num_tree_edges == forest_edges(vg)
    assert st.num_reached == 1


@pytest.mark.parametrize("n", [1, 7])
def test_no_edges(ctx, n):
    vg = ViewGraph(n, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 3, 3)), np.zeros(0), None)
    R_init = G.so3_exp(np.random.default_rng(n).normal(size=(n, 3)))
    R, par, st = dev(ctx, vg, R_init, n - 1)
    assert par.tolist() == [-1] * (n - 1) + [n - 1] and R.tobytes() == R_init.tobytes()
    assert (st.num_reached, st.num_tree_edges, st.max_depth) == (1, 0, 0)


def test_repeated_pairs_against_kruskal(ctx):
    rng = np.random.default_rng(8)
    for it in range(30):
        n = int(rng.integers(2, 500))
        vg = random_graph(rng, n, int(rng.integers(1, 8 * n)), repeated=True, wmax=3)
        root = int(rng.integers(0, n))
        R_init = G.so3_exp(rng.normal(size=(n, 3)))
        R, par, _ = dev(ctx, vg, R_init, root)
        kpar, kedge = kruskal_parents(vg, root)
        assert np.array_equal(par, kpar), it
        v = np.nonzero((kpar >= 0) & (np.arange(n) != root))[0]
        A = np.where((vg.ej[kedge[v]] == v)[:, None, None], vg.R_rel[kedge[v]], np.swapaxes(vg.R_rel[kedge[v]], 1, 2))
        # R_v = A_v R_parent: compose the Kruskal tree in BFS order (parents come first)
        Rk = R_init.copy()
        order = [root]
        children = {}
        for c, p in zip(v, kpar[v]):
            children.setdefault(int(p), []).append(int(c))
        Av = dict(zip(v.tolist(), A))
        for u in order:
            for c in children.get(u, []):
                Rk[c] = Av[c] @ Rk[u]
                order.append(c)
        assert np.abs(R - Rk).max() <= 1e-10


def path_graph(n, weight=1.0, seed=0):
    ei = np.arange(n - 1, dtype=np.int32)
    R_rel = G.so3_exp(np.random.default_rng(seed).normal(size=(n - 1, 3)) * 0.3)
    return ViewGraph(n, ei, ei + 1, R_rel, np.full(n - 1, weight), None)


def test_path_depth_does_not_drive_the_launch_count(ctx):
    _, _, small = check(ctx, path_graph(1024))
    R_init = G.so3_exp(np.random.default_rng(1).normal(size=(131072, 3)))
    R, par, big = check(ctx, path_graph(131072), R_init, root=70000)
    assert big.max_depth == 70000 and small.max_depth == 1023
    assert big.kernel_launches <= 2 * small.kernel_launches, (big.kernel_launches, small.kernel_launches)


def test_star(ctx):
    n = 131072
    rng = np.random.default_rng(2)
    vg = ViewGraph(n, np.zeros(n - 1, np.int32), np.arange(1, n, dtype=np.int32), G.so3_exp(rng.normal(size=(n - 1, 3))),
                   rng.integers(0, 100, n - 1).astype(np.float64), None)
    _, _, st = check(ctx, vg, root=5)
    assert st.max_depth == 2 and st.boruvka_rounds == 1


def test_config5_lattice_and_repeated_calls_are_bit_identical(ctx):
    vg = S.make_lattice_view_graph(100_000)
    R, par, st = check(ctx, vg)
    assert st.num_reached == 100_000 and st.num_tree_edges == 99_999
    assert st.boruvka_rounds <= 17
    R2, par2, _ = dev(ctx, vg)
    assert R.tobytes() == R2.tobytes() and par.tobytes() == par2.tobytes()


def test_invalid_arguments_with_a_context(ctx):
    vg = path_graph(4)
    for bad, msg in ((dict(root=4), "root out of range"),
                     (dict(ei=np.array([0, 1, 4], np.int32)), "edge index out of range"),
                     (dict(weight=np.array([1.0, np.nan, 1.0])), "non-finite edge weight"),
                     (dict(weight=np.array([1.0, np.inf, 1.0])), "non-finite edge weight")):
        g = ViewGraph(4, bad.get("ei", vg.ei), vg.ej, vg.R_rel, bad.get("weight", vg.weight), None)
        with pytest.raises(_lib.B200Error, match=msg) as e:
            E.initialize_from_maximum_spanning_tree_device(g, None, ctx, bad.get("root", 0))
        assert e.value.code == 1


def test_estimate_rotations_starts_from_the_device_tree_above_the_gate(ctx):
    vg = S.make_lattice_view_graph(2000, seed=4)
    assert vg.E >= E.MST_DEVICE_MIN_EDGES
    o = dict(pcg_rel_tolerance=1e-12)
    ok, R = E.RotationEstimator(E.RotationEstimatorOptions(**o), ctx).EstimateRotations(vg)
    R0 = E.initialize_from_maximum_spanning_tree(vg)
    ok2, R2 = E.RotationEstimator(E.RotationEstimatorOptions(skip_initialization=True, **o), ctx).EstimateRotations(vg, R0)
    assert ok and ok2
    assert np.abs(R - R2).max() <= 1e-9
