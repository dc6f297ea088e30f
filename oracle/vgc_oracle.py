"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of ViewGraphCalibrator::Solve
(glomap/estimators/view_graph_calibration.cc:11-185) with FetzerFocalLengthCost / FetzerFocalLengthSameCameraCost
(glomap/estimators/cost_function.h:138-310).

UPSTREAM-UNVERIFIED: the reference's Ceres solve (LM, CauchyLoss, the corrector, bounds with the projected line search)
is restated through oracle/ceres_lm.py, and Eigen's JacobiSVD through numpy.linalg.svd (LAPACK); neither Ceres nor
Eigen can be built here.  The singular vectors' signs differ between the two SVDs; the Fetzer constants d_01, d_12 change
sign as a whole under a joint (u_k, v_k) flip, which leaves the residuals unchanged (tests/test_view_graph_calibration_cpu.py).

Restated:
  * unknowns: one focal per camera used by a qualifying pair, initialised to Camera::Focal(); lower bound 1e-3; cameras
    with has_prior_focal_length constant (.cc:105-120); no variable camera: return true, nothing written (.cc:30-35);
  * G = K1^T F K0 (K = I with the principal point in its last column), SVD, d_01 = fetzer_d(.., 1, 0),
    d_12 = fetzer_d(.., 2, 1);
  * r0 = (fi^2 - K0_01) / fi^2, K0_01 = -(fj^2 d01[2] + d01[3]) / di, di = fj^2 d01[0] + d01[1];
    r1 = (fj^2 - K1_12) / fj^2, K1_12 = -(fi^2 d12[1] + d12[3]) / dj, dj = fi^2 d12[0] + d12[2];
    an exact zero di / dj becomes 1e-6 (a constant: no derivative); same camera: fi = fj = f;
  * CauchyLoss(a): rho = b log(1 + s / b), rho' = max(DBL_MIN, 1 / (1 + s / b)), b = a^2; rho'' < 0, so the corrector
    scales residual and Jacobian by sqrt(rho');
  * CopyBackResults (.cc:122-148) and FilterImagePairs (.cc:150-185).

Only tests/ and profiles/ may import this module."""
from __future__ import annotations

import dataclasses

import numpy as np
import scipy.sparse as sp

from .ceres_lm import LMOptions, solve_lm

LOWER_BOUND = 1e-3


@dataclasses.dataclass
class VGCOptions:
    """ViewGraphCalibratorOptions (view_graph_calibration.h:10-29) + the OptimizationBaseOptions solver settings."""
    thres_lower_ratio: float = 0.1
    thres_higher_ratio: float = 10.0
    thres_two_view_error: float = 2.0
    thres_loss_function: float = 1e-2
    max_num_iterations: int = 100
    function_tolerance: float = 1e-5


def fetzer_d(ai, bi, aj, bj, u, v):
    """cost_function.h:144-157 over [E, 3] arrays -> [E, 4]."""
    return np.stack([ai[:, u] * aj[:, v] - ai[:, v] * aj[:, u], ai[:, u] * bj[:, v] - ai[:, v] * bj[:, u],
                     bi[:, u] * aj[:, v] - bi[:, v] * aj[:, u], bi[:, u] * bj[:, v] - bi[:, v] * bj[:, u]], 1)


def fetzer_from_svd(s, U, V):
    """d_01, d_12 ([E, 4] each) from the singular values s [E, 3] and the singular vectors (columns of U, V [E, 3, 3])
    (cost_function.h:159-202)."""
    v0, v1, u0, u1 = V[:, :, 0], V[:, :, 1], U[:, :, 0], U[:, :, 1]
    s0, s1 = s[:, 0], s[:, 1]
    ai = np.stack([s0 * s0 * (v0[:, 0] * v0[:, 0] + v0[:, 1] * v0[:, 1]), s0 * s1 * (v0[:, 0] * v1[:, 0] + v0[:, 1] * v1[:, 1]),
                   s1 * s1 * (v1[:, 0] * v1[:, 0] + v1[:, 1] * v1[:, 1])], 1)
    aj = np.stack([u1[:, 0] * u1[:, 0] + u1[:, 1] * u1[:, 1], -(u0[:, 0] * u1[:, 0] + u0[:, 1] * u1[:, 1]),
                   u0[:, 0] * u0[:, 0] + u0[:, 1] * u0[:, 1]], 1)
    bi = np.stack([s0 * s0 * v0[:, 2] * v0[:, 2], s0 * s1 * v0[:, 2] * v1[:, 2], s1 * s1 * v1[:, 2] * v1[:, 2]], 1)
    bj = np.stack([u1[:, 2] * u1[:, 2], -(u0[:, 2] * u1[:, 2]), u0[:, 2] * u0[:, 2]], 1)
    return fetzer_d(ai, bi, aj, bj, 1, 0), fetzer_d(ai, bi, aj, bj, 2, 1)


def g_matrix(F, pp0, pp1):
    """G = K1^T F K0 for [E, 3, 3] F and [E, 2] principal points."""
    E = len(F)
    K0 = np.tile(np.eye(3), (E, 1, 1))
    K0[:, 0, 2], K0[:, 1, 2] = pp0[:, 0], pp0[:, 1]
    K1 = np.tile(np.eye(3), (E, 1, 1))
    K1[:, 0, 2], K1[:, 1, 2] = pp1[:, 0], pp1[:, 1]
    return np.swapaxes(K1, 1, 2) @ F @ K0


def fetzer_constants(F, pp0, pp1):
    """d_01, d_12 of every pair; a non-finite G gives NaN constants."""
    G = g_matrix(np.asarray(F, np.float64).reshape(-1, 3, 3), np.asarray(pp0, np.float64), np.asarray(pp1, np.float64))
    E = len(G)
    ok = np.isfinite(G.reshape(E, 9)).all(1)
    U = np.full((E, 3, 3), np.nan)
    V = np.full((E, 3, 3), np.nan)
    s = np.full((E, 3), np.nan)
    if ok.any():
        u, sv, vt = np.linalg.svd(G[ok])
        U[ok], s[ok], V[ok] = u, sv, np.swapaxes(vt, 1, 2)
    return fetzer_from_svd(s, U, V)


def residuals(d01, d12, fi, fj, jacobian=False):
    """r [E, 2] (and dr/dfi, dr/dfj [E, 2] each) at focal arrays fi, fj (cost_function.h:211-229)."""
    di = fj * fj * d01[:, 0] + d01[:, 1]
    dj = fi * fi * d12[:, 0] + d12[:, 2]
    nzi, nzj = di != 0, dj != 0
    di = np.where(nzi, di, 1e-6)
    dj = np.where(nzj, dj, 1e-6)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        K0 = -(fj * fj * d01[:, 2] + d01[:, 3]) / di
        K1 = -(fi * fi * d12[:, 1] + d12[:, 3]) / dj
        r = np.stack([(fi * fi - K0) / (fi * fi), (fj * fj - K1) / (fj * fj)], 1)
        if not jacobian:
            return r
        # d r0 / d fi = 2 K0 / fi^3; d r0 / d fj = 2 fj (d01[2] + K0 d01[0]) / (di fi^2) (no d01[0] term after the 1e-6
        # replacement); symmetrically for r1
        dri = np.stack([2.0 * K0 / (fi * fi * fi), 2.0 * fi * (d12[:, 1] + K1 * d12[:, 0] * nzj) / (dj * fj * fj)], 1)
        drj = np.stack([2.0 * fj * (d01[:, 2] + K0 * d01[:, 0] * nzi) / (di * fi * fi), 2.0 * K1 / (fj * fj * fj)], 1)
    return r, dri, drj


def cauchy(s, a):
    """CauchyLoss(a) (ceres loss_function.cc): rho, rho'."""
    b = a * a
    c = 1.0 / b
    with np.errstate(invalid="ignore", over="ignore"):
        sm = 1.0 + s * c
        return b * np.log(sm), np.maximum(np.finfo(float).tiny, 1.0 / sm)


class VGCProblem:
    def __init__(self, principal_point, focal, focal_constant, cam1, cam2, F, opts: VGCOptions):
        self.K = len(focal)
        self.c1 = np.asarray(cam1, np.int64)
        self.c2 = np.asarray(cam2, np.int64)
        pp = np.asarray(principal_point, np.float64).reshape(-1, 2)
        self.d01, self.d12 = fetzer_constants(F, pp[self.c1], pp[self.c2])
        self.has_block = np.zeros(self.K, bool)
        self.has_block[self.c1] = True
        self.has_block[self.c2] = True
        const = np.zeros(self.K, bool) if focal_constant is None else np.asarray(focal_constant, bool)
        self.var = self.has_block & ~const
        self.col = np.full(self.K, -1, np.int64)
        self.col[self.var] = np.arange(int(self.var.sum()))
        self.same = self.c1 == self.c2
        self.a = opts.thres_loss_function

    def evaluate(self, x, want_jacobian):
        fi, fj = x[self.c1], x[self.c2]
        if not want_jacobian:
            r = residuals(self.d01, self.d12, fi, fj)
            rho, _ = cauchy((r * r).sum(1), self.a)
            return 0.5 * float(rho.sum()), None, None
        r, dri, drj = residuals(self.d01, self.d12, fi, fj, True)
        rho, rho1 = cauchy((r * r).sum(1), self.a)
        sq = np.sqrt(rho1)[:, None]
        rc = (r * sq).ravel()
        Ji = np.where(self.same[:, None], dri + drj, dri) * sq
        Jj = drj * sq
        E = len(r)
        rows = np.arange(2 * E)
        ci, cj = self.col[self.c1], self.col[self.c2]
        mi = np.repeat(ci >= 0, 2)
        mj = np.repeat((cj >= 0) & ~self.same, 2)
        J = sp.csr_matrix((np.concatenate([Ji.ravel()[mi], Jj.ravel()[mj]]),
                           (np.concatenate([rows[mi], rows[mj]]), np.concatenate([np.repeat(ci, 2)[mi], np.repeat(cj, 2)[mj]]))),
                          shape=(2 * E, int(self.var.sum())))
        return 0.5 * float(rho.sum()), rc, J

    def plus(self, x, delta):
        out = x.copy()
        out[self.var] = np.maximum(x[self.var] + delta[self.col[self.var]], LOWER_BOUND)
        return out

    def project(self, x, step):
        return np.maximum(x[self.var] + step[self.col[self.var]], LOWER_BOUND) - x[self.var]

    def x_norm(self, x, y=None):
        a = x[self.var] if y is None else x[self.var] - y[self.var]
        return float(np.sqrt((a * a).sum()))


def solve_vgc(principal_point, focal, focal_constant, cam1, cam2, F, opts: VGCOptions | None = None, lm: LMOptions | None = None):
    """The ABI's contract (b200sfm_view_graph_calibrate) on the CPU.  Returns a dict: focal [K] (estimates of the cameras
    with a block, others unchanged), cam_accepted [K], pair_valid [E], residual [E, 2], summary (None on the early return,
    where nothing is written: cam_accepted all 0, pair_valid all 1, residual None)."""
    o = opts or VGCOptions()
    f0 = np.asarray(focal, np.float64).copy()
    E = len(cam1)
    out = dict(focal=f0.copy(), cam_accepted=np.zeros(len(f0), bool), pair_valid=np.ones(E, bool), residual=None,
               summary=None, problem=None)
    if E == 0:
        return out
    prob = VGCProblem(principal_point, f0, focal_constant, cam1, cam2, F, o)
    out["problem"] = prob
    if not prob.var.any():
        return out
    lm = lm or LMOptions(max_num_iterations=o.max_num_iterations, function_tolerance=o.function_tolerance)
    cost0, _, _ = prob.evaluate(f0, False)
    if np.isfinite(cost0):
        x, summ = solve_lm(f0, prob.evaluate, prob.plus, lm, project=prob.project, x_norm_fn=prob.x_norm)
    else:   # the initial evaluation fails: Ceres returns FAILURE, the parameters untouched
        from .ceres_lm import LMSummary
        x, summ = f0.copy(), LMSummary(initial_cost=cost0, final_cost=cost0, termination="initial evaluation failed",
                                       usable=False)
    ratio = x / f0
    accepted = prob.has_block & ~((ratio > o.thres_higher_ratio) | (ratio < o.thres_lower_ratio))
    r = residuals(prob.d01, prob.d12, x[prob.c1], x[prob.c2])
    out.update(focal=np.where(prob.has_block, x, f0), cam_accepted=accepted,
               pair_valid=~((r * r).sum(1) > o.thres_two_view_error ** 2), residual=r, summary=summ)
    return out
