"""CPU checks of oracle/ra_system.py, the FP64 reference tests/test_ra_system_gpu.py compares the device rotation
averager with: its operators against a dense construction written row by row from the reference's rules, its PCG
against a direct solve, its two-level preconditioner, and its pieces composed into ra_oracle's first L1 step."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import ra_oracle as RO
from oracle import ra_system as RS


def rand_rot(rng, n, deg):
    return RO.aa_to_R(rng.normal(size=(n, 3)) * np.radians(deg))


def tiny(rng, gravity=True, rig=True):
    """8 frames (3 with gravity), 2 unknown cameras.  Every row kind: 3-DoF, y-only, mixed, a duplicate and a reversed
    pair, a same-frame pair (ei == ej) and same-camera pairs (eci == ecj), the gauge on a frame that is not frame 0."""
    nf, nc = 8, (2 if rig else 0)
    ei = np.array([0, 1, 2, 3, 4, 5, 6, 0, 1, 2, 2, 6, 3])
    ej = np.array([1, 2, 3, 4, 5, 6, 7, 7, 0, 3, 5, 6, 7])
    E = len(ei)
    g = np.zeros(nf, bool)
    if gravity:
        g[[2, 3, 5]] = True                                 # (2, 3) y-only twice, (3, 4) mixed, (2, 5) y-only
    theta = rng.normal(size=(nf + nc, 3)) * 0.3
    theta[:nf][g] = np.stack([np.zeros(g.sum()), theta[:nf][g, 1], np.zeros(g.sum())], 1)
    kw = {}
    if rig:
        eci = np.full(E, -1); ecj = np.full(E, -1)
        eci[[0, 4, 11]] = nf; ecj[[0, 4, 11]] = nf          # same camera in both images (11 is also a same-frame pair)
        ecj[[5, 6]] = nf + 1; eci[7] = nf + 1; ecj[8] = nf
        kw = dict(n_cams=nc, eci=eci, ecj=ecj, cam_frames=[[0, 1, 4, 5, 6], [0, 6, 7]])
    R_rel = rand_rot(rng, E, 40)
    w = rng.uniform(0.5, 2.0, E)
    w[3] = -1.0                                             # negative: weight 1 (.cc:390-393)
    return RS.RASystem(nf, ei, ej, R_rel, theta, fixed=6, edge_w=w, use_weight=True, has_grav=g, **kw)


def dense_rows(s):
    """Rows a[(e, k)] of A, written out edge by edge from the reference's rules (duplicate columns summed)."""
    n = s.n
    rows = {}
    for e in range(s.E):
        i, j, ci, cj = s.ei[e], s.ej[e], s.eci[e], s.ecj[e]
        gi = i >= 0 and s.grav[i]
        gj = s.grav[j]
        one_row = (gi and gj) if i >= 0 else gj
        for k in ((1,) if one_row else (0, 1, 2)):
            a = np.zeros(3 * n)
            if not gj or k == 1:
                a[3 * j + k] += 1
            if i >= 0:
                if not gi or k == 1:
                    a[3 * i + k] -= 1
                if cj >= 0:
                    a[3 * cj + k] += 1
                if ci >= 0:
                    a[3 * ci + k] -= 1
            rows[(e, k)] = a
    return rows


@pytest.mark.parametrize("gravity,rig", [(True, True), (False, True), (True, False), (False, False)])
@pytest.mark.parametrize("square", [0, 1])
def test_laplacian_rhs_and_diagonal_match_a_dense_row_by_row_construction(gravity, rig, square):
    rng = np.random.default_rng(3)
    s = tiny(rng, gravity, rig)
    res = s.residuals()
    w = s.weights(res, 1, np.radians(5.0) ** 2)
    wp = w ** (2 if square else 1)
    L = np.zeros((3 * s.n, 3 * s.n))
    b = np.zeros(3 * s.n)
    rows = dense_rows(s)
    for (e, k), a in rows.items():
        L += wp[e] * np.outer(a, a)
        b += wp[e] * res[e, k] * a
    assert len(rows) == s.rows_total
    Ls = s.laplacian(w, square).toarray()
    assert np.abs(Ls - L).max() <= 1e-13 * np.abs(L).max()
    assert np.abs(s.rhs(w, square, res) - b).max() <= 1e-13 * np.abs(b).max()
    d, dinv = s.jacobi(sp.csr_matrix(L))
    assert np.array_equal(d, np.diag(L))
    assert np.all(dinv[d == 0] == 1.0) and np.allclose(dinv[d > 0], 1 / d[d > 0])
    if rig:   # the same camera in both images of a pair contributes nothing to the camera's diagonal
        cam0 = 3 * s.n_frames
        same = [e for e in range(s.E) if s.eci[e] == s.ecj[e] == s.n_frames]
        others = [e for e in range(s.E) if (s.eci[e] == s.n_frames) != (s.ecj[e] == s.n_frames)]
        assert same and L[cam0, cam0] == pytest.approx(sum(wp[e] for e in others))
    if gravity:   # a gravity frame's x / z columns are empty
        assert np.all(np.diag(L)[[3 * 2, 3 * 2 + 2, 3 * 5, 3 * 5 + 2]] == 0)


def test_residuals_follow_ra_oracle():
    rng = np.random.default_rng(5)
    n = 12
    ei = np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 0, 3])
    ej = np.array([1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 11, 8])
    R_rel = rand_rot(rng, len(ei), 150)          # includes residuals beyond 120 degrees
    theta = rng.normal(size=(n, 3)) * 0.5
    theta[4] = 0.0
    s = RS.RASystem(n, ei, ej, R_rel, theta, fixed=3)
    ref = RO.compute_residuals(theta, ei, ej, R_rel, 3, theta[3])
    assert np.abs(s.residuals().ravel() - ref).max() < 1e-12


def test_pcg_after_3n_iterations_equals_a_direct_solve():
    rng = np.random.default_rng(7)
    for gravity, rig in ((True, False), (False, True), (False, False)):
        s = tiny(rng, gravity, rig)
        res = s.residuals()
        w = s.weights(res, 2)
        L = s.laplacian(w, 0)
        b = s.rhs(w, 0, res)
        d, dinv = s.jacobi(L)
        act = np.nonzero(d > 0)[0]
        x_ref = np.zeros_like(b)
        x_ref[act] = spla.spsolve(L[act][:, act].tocsc(), b[act])
        its, k = s.pcg(L, b, s.precond(dinv), 3 * s.n)
        assert k == 3 * s.n
        assert np.abs(its[-1] - x_ref).max() <= 1e-9 * np.abs(x_ref).max()
        # warm-started from the solution, the stopping rule fires at the head of iteration 1
        its, k = s.pcg(L, b, s.precond(dinv), 10, x0=x_ref, rel_tol=1e-8)
        assert k == 0 and its == []


def lattice(n_side, rng):
    n = n_side * n_side
    idx = np.arange(n).reshape(n_side, n_side)
    ei = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
    ej = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    return n, ei, ej, rand_rot(rng, len(ei), 3)


def test_two_level_preconditioner_is_spd_and_exact_on_the_coarse_space():
    rng = np.random.default_rng(9)
    n, ei, ej, R_rel = lattice(12, rng)
    s = RS.RASystem(n, ei, ej, R_rel, np.zeros((n, 3)), fixed=17)
    w = rng.uniform(0.1, 3.0, s.E)
    L = s.laplacian(w, 1)
    agg_of = (np.arange(n) // 12) // 3                      # 4 aggregates of 3 lattice rows
    P, Ac = s.coarse(L, agg_of, 4)
    Ls = L[0::3, 0::3].toarray()
    assert np.allclose(Ac, P.T.toarray() @ Ls @ P.toarray())
    _, dinv = s.jacobi(L)
    M = s.precond(dinv, P, np.linalg.inv(Ac))
    Md = np.stack([M(np.eye(3 * n)[c]) for c in range(3 * n)], 1)
    assert np.abs(Md - Md.T).max() < 1e-12 * np.abs(Md).max()
    assert np.linalg.eigvalsh(Md).min() > 0
    # the coarse correction inverts L on the coarse space: P^T L (M^-1 - D^-1) r = P^T r
    r = rng.normal(size=3 * n)
    zc = M(r) - dinv * r
    for k in range(3):
        assert np.allclose(P.T @ (Ls @ zc[k::3]), P.T @ r[k::3])


def test_admm_step_gives_the_next_x_update_of_l1_admm():
    rng = np.random.default_rng(11)
    s = tiny(rng, gravity=False, rig=True)
    res = s.residuals()
    w = s.weights(res, 0)
    L = s.laplacian(w, 1).tocsc()
    b = np.repeat(w, 3) * res.ravel()
    Aw = (sp.diags(np.repeat(w, 3)) @ s.A).tocsc()
    for k in (1, 2, 3):
        x_ref, its = RO.l1_admm(Aw, b, max_iter=k, abs_tol=0.0, rel_tol=0.0)
        assert its == k
        z = np.zeros(3 * s.E); u = np.zeros(3 * s.E)
        rhs = s.rhs(w, 1, res)
        for _ in range(k):
            x = spla.spsolve(L, rhs)
            z, u, rhs, _, _, _ = s.admm_step(w, x, b, z, u, 1.0)
        assert np.abs(x - x_ref).max() < 1e-10 * np.abs(x_ref).max()


def first_l1_step(s, o=RO.RAOptions()):
    """solve()'s first L1 outer iteration composed from the reference pieces (ra_solver.cuh)."""
    res = s.residuals()
    w = s.weights(res, 0)
    L = s.laplacian(w, 1)
    rhs = s.rhs(w, 1, res)
    b = np.repeat(w, 3) * res.ravel()
    act = np.nonzero(L.diagonal() > 0)[0]
    z = np.zeros(3 * s.E); u = np.zeros(3 * s.E)
    eps_pri_thr = np.sqrt(s.rows_total) * 1e-4
    eps_dual_thr = np.sqrt(3.0 * s.n) * 1e-4
    for _ in range(10):
        x = np.zeros(3 * s.n)
        x[act] = spla.spsolve(L[act][:, act].tocsc(), rhs[act])
        z, u, rsu_r, svec, uvec, nm = s.admm_step(w, x, b, z, u, 1.0)
        rhs = rsu_r
        eps_pri = eps_pri_thr + 1e-2 * np.sqrt(max(b @ b, nm[1], nm[2]))
        eps_dual = eps_dual_thr + 1e-2 * np.sqrt(nm[4])
        if np.sqrt(nm[0]) < eps_pri and np.sqrt(nm[3]) < eps_dual:
            break
    return s.update(x)[0]


def test_composed_pieces_reproduce_the_first_l1_step():
    rng = np.random.default_rng(13)
    n, ei, ej, R_rel = lattice(5, rng)
    theta0 = rng.normal(size=(n, 3)) * 0.05
    o = RO.RAOptions(max_num_l1_iterations=1, max_num_irls_iterations=0)
    ref, info = RO.estimate_rotations(n, ei, ej, R_rel, theta0, opts=o, fixed=7)
    assert info["l1_iterations"] == 1
    s = RS.RASystem(n, ei, ej, R_rel, theta0, fixed=7)
    assert np.abs(first_l1_step(s) - ref).max() < 1e-10
    # with unknown cameras (ra_oracle's sum_duplicates construction)
    s = tiny(rng, gravity=False, rig=True)
    th0 = s.theta.copy()
    E = s.E - 1
    ref, info = RO.estimate_rotations_rig_unknown(s.n_frames, s.n_cams, s.ei[:E], s.ej[:E], s.eci[:E], s.ecj[:E],
                                                  s.Rrel[:E], th0, s.cam_frames, opts=o, fixed=s.fixed,
                                                  edge_weight=s.w_edge[:E])
    s_unw = RS.RASystem(s.n_frames, s.ei[:E], s.ej[:E], s.Rrel[:E], th0, fixed=s.fixed, n_cams=s.n_cams,
                        eci=s.eci[:E], ecj=s.ecj[:E], cam_frames=s.cam_frames)
    assert np.abs(first_l1_step(s_unw) - ref).max() < 1e-9
