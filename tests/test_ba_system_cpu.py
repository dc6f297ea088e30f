"""CPU checks of the FP64 linear-system reference oracle/ba_system.py, the yardstick of the operator-level GPU tests
(tests/test_ba_system_gpu.py): its sparse operator, its step bookkeeping, its column layout and its gradient."""
import numpy as np
import pytest

from glomap_b200 import synthetic as S
from oracle import ba_oracle as B
from oracle import ba_system as BS


def _problem(opts, model=S.SIMPLE_RADIAL, K=3, mask=None):
    sc = S.make_scene(8, 60, mean_track_len=5, seed=3, model=model, num_intrinsics=K)
    st = S.perturb_scene(sc, rot_deg=1.0, center_frac=0.02, point_frac=0.02)
    rng = np.random.default_rng(0)
    xy = sc.obs_xy + rng.normal(size=sc.obs_xy.shape) * 2.0     # a share of the residuals beyond the Huber threshold
    if mask is None:
        mask = np.zeros(sc.C, np.uint8)
        mask[0], mask[1], mask[2] = 3, 1, 2
    prob = B.BAProblem(st.quat, st.trans, st.points, sc.pt_obs_begin, sc.obs_cam, xy, sc.cam_intr, sc.intr_model,
                       st.intr_params, opts, mask)
    nbk = sc.C + (K if opts.optimize_intrinsics else 0)
    return prob, nbk


@pytest.fixture(params=["frames", "intrinsics"])
def system(request):
    opts = B.BAOptions(optimize_intrinsics=request.param == "intrinsics")
    prob, nbk = _problem(opts)
    return BS.BASystem(prob, prob.x0, radius=50.0, nbk=nbk, precond="schur")


def test_every_oracle_column_maps_to_exactly_one_device_slot(system):
    cam, pt = system.cam_idx, system.pt_idx
    assert np.all((cam >= 0) ^ (pt >= 0))
    assert len(np.unique(cam[cam >= 0])) == (cam >= 0).sum()
    assert len(np.unique(pt[pt >= 0])) == (pt >= 0).sum()
    # masked dofs (camera 1: rotation, camera 2: translation, camera 0: both) have no column
    blk = cam[cam >= 0] // 6
    slot = cam[cam >= 0] % 6
    assert 0 not in blk
    assert not np.any((blk == 1) & (slot < 3)) and not np.any((blk == 2) & (slot >= 3))


def test_sparse_schur_operator_equals_the_dense_schur_complement(system):
    """(S + D) x of the sparse reference against the Schur complement of the dense, damped normal equations."""
    p = system.prob
    H = (system.J.T @ system.J).toarray() + np.diag(system.damping_full())
    cols_c = np.nonzero(system.cam_idx >= 0)[0]
    cols_p = np.nonzero(system.pt_idx >= 0)[0]
    Hcc, Hcp, Hpp = H[np.ix_(cols_c, cols_c)], H[np.ix_(cols_c, cols_p)], H[np.ix_(cols_p, cols_p)]
    Sdense = Hcc - Hcp @ np.linalg.solve(Hpp, Hcp.T)
    rng = np.random.default_rng(1)
    for _ in range(3):
        x = np.where(system.var_c, rng.normal(size=system.var_c.size), 0.0)
        y = system.apply(x)
        want = Sdense @ x[system.cam_idx[cols_c]]
        assert np.abs(y[system.cam_idx[cols_c]] - want).max() <= 1e-11 * np.abs(want).max()
        assert np.all(y[~system.var_c] == 0.0)
    assert p.ncols == len(cols_c) + len(cols_p)


def test_direct_model_decrease_equals_the_reduced_formula_for_an_inexact_step(system):
    """The device's 1/2 (-g^T d + d_c^T rho + d^T D d) is the undamped model decrease for ANY camera step when the point
    step is the exact back-substitution.  For PCG iterates from x_0 = 0, d_c^T rho vanishes up to rounding (the residual
    is orthogonal to the Krylov space that holds the iterate), so the identity is checked on a perturbed iterate too."""
    it = system.pcg(2)[-1]                         # two PCG iterations: far from the exact solution
    rng = np.random.default_rng(4)
    for dc in (it, it + np.where(system.var_c, rng.normal(size=it.size), 0.0) * 0.3 * np.abs(it).max()):
        rho = system.b - system.apply(dc)
        assert np.linalg.norm(rho) > 1e-3 * np.linalg.norm(system.b)
        direct = system.model_cost_change(system.full_step(dc))
        reduced = system.model_cost_change_reduced(dc)
        assert abs(direct - reduced) <= 1e-10 * abs(direct)
    assert abs(it @ (system.b - system.apply(it))) <= 1e-10 * abs(system.model_cost_change(system.full_step(it)))
    # off the Krylov space the rho term is not negligible: without it the two differ
    delta = system.full_step(dc)
    no_rho = 0.5 * (-(system.J.T @ system.r) @ delta + delta @ (system.damping_full() * delta))
    assert abs(no_rho - direct) > 1e-3 * abs(direct)


def test_gradient_and_rhs_agree_with_finite_differences(system):
    """g = J^T r is the derivative of the robust cost along the tangent step; b = -(reduced model gradient)."""
    p = system.prob
    rng = np.random.default_rng(2)
    g_full = np.zeros(p.ncols)
    mc, mp = system.cam_idx >= 0, system.pt_idx >= 0
    g_full[mc] = system.g_c[system.cam_idx[mc]]
    g_full[mp] = system.g_p[system.pt_idx[mp]]
    for _ in range(3):
        d = rng.normal(size=p.ncols)
        h = 1e-6
        fd = (p.evaluate(p.plus(p.x0, h * d), False)[0] - p.evaluate(p.plus(p.x0, -h * d), False)[0]) / (2 * h)
        assert abs(fd - g_full @ d) <= 1e-6 * (abs(fd) + np.abs(g_full).max())
    # reduced model m(dc) = min over the point step of the damped quadratic model: grad at 0 = -b
    def m(dc):
        delta = system.full_step(dc)
        Jd = system.J @ delta
        return Jd @ (system.r + 0.5 * Jd) + 0.5 * delta @ (system.damping_full() * delta)
    for _ in range(2):
        u = np.where(system.var_c, rng.normal(size=system.var_c.size), 0.0)
        h = 1e-4
        fd = (m(h * u) - m(-h * u)) / (2 * h)
        assert abs(fd + system.b @ u) <= 1e-7 * (abs(fd) + np.abs(system.b).max())


def test_pcg_converges_to_the_reduced_solution_and_preconditioners_differ():
    prob, nbk = _problem(B.BAOptions())
    sj = BS.BASystem(prob, prob.x0, radius=50.0, nbk=nbk, precond="schur")
    bj = BS.BASystem(prob, prob.x0, radius=50.0, nbk=nbk, precond="jacobi")
    it = sj.pcg(60)
    res = np.linalg.norm(sj.b - sj.apply(it[-1]))
    assert res <= 1e-9 * np.linalg.norm(sj.b)
    # the Schur-Jacobi block really subtracts the point coupling: its inverse differs from block-Jacobi
    c = 3
    assert np.abs(sj.Minv_blocks[c] - bj.Minv_blocks[c]).max() > 1e-2 * np.abs(bj.Minv_blocks[c]).max()
    # ... and is the exact diagonal block of the damped reduced system
    e = np.zeros(6 * nbk)
    blk = np.zeros((6, 6))
    for j in range(6):
        e[:] = 0.0
        e[6 * c + j] = 1.0
        blk[:, j] = sj.apply(e)[6 * c:6 * c + 6]
    assert np.abs(np.linalg.inv(blk) - sj.Minv_blocks[c]).max() <= 1e-9 * np.abs(sj.Minv_blocks[c]).max()
