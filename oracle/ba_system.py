"""ORACLE (test infrastructure, NOT product code) -- FP64 sparse restatement of
one Levenberg-Marquardt step of the device bundle adjuster, in the device's
coordinates, for the operator-level tests (tests/test_ba_system_gpu.py against
the probe of include/b200sfm_testing.h).

Built from ``BAProblem.evaluate`` (the Huber-corrected sparse Jacobian of
oracle/ba_oracle.py) and nothing else; no quantity is taken from the device.

Device layout (include/b200sfm_testing.h): the camera side is ``nbk`` blocks
of 6 dofs, block order frame f | C + intrinsics k | C + K + sensor s.  A frame
block holds rotation (slots 0-2) and translation (3-5); an intrinsics block
holds its variable parameters in ascending parameter index; a sensor block
holds the cam_from_rig rotation (0-2) and translation (3-5).  Dofs that are
not variables -- masked, unobserved, or without curvature -- are identity rows
with zero gradient and Jacobi scale -1 (ba_finalize_cams).  Symmetric blocks
are packed upper triangle, row by row.

What is formed (compute_step in glomap_b200/csrc/ba_solver.cuh):
  * U, g_c, V, g_p of the linearisation; Jacobi scales js = 1/(1+sqrt(diag));
  * damping D = clamp(diag js^2, 1e-6, 1e32) / (radius js^2);
  * the reduced camera system S = U + D - W (V + D_p)^-1 W^T (no Schur term with
    constant points), b = -(g_c - W (V + D_p)^-1 g_p), applied with sparse products;
  * preconditioner blocks: exact Schur-Jacobi (U_c + D_c - sum_p W_cp (V_p + D_p)^-1 W_cp^T)^-1,
    or block-Jacobi (U_c + D_c)^-1, per block as the path documents it;
  * textbook PCG from x_0 = 0 with that preconditioner (all iterates);
  * back-substitution of the point step, the candidate state (BAProblem.plus)
    and its cost, and the model decrease -g^T d - 1/2 d^T J^T J d formed directly
    over the full, unreduced system (the device forms it from the reduced system's
    identity 1/2 (-g^T d + d_c^T rho + d^T D d), rho the PCG residual).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from .ba_oracle import BAProblem

SYM6 = [(i, j) for i in range(6) for j in range(i, 6)]
SYM3 = [(i, j) for i in range(3) for j in range(i, 3)]


def pack_sym(M):
    """[..., n, n] -> [..., n(n+1)/2] upper triangle, row by row."""
    n = M.shape[-1]
    return np.stack([M[..., i, j] for i in range(n) for j in range(i, n)], -1)


def unpack_sym(a, n):
    """[..., n(n+1)/2] -> [..., n, n]."""
    M = np.zeros(a.shape[:-1] + (n, n))
    for k, (i, j) in enumerate([(i, j) for i in range(n) for j in range(i, n)]):
        M[..., i, j] = a[..., k]
        M[..., j, i] = a[..., k]
    return M


def device_index(prob: BAProblem, nbk: int):
    """Oracle column -> device camera dof (block * 6 + slot) or point dof (point * 3 + slot); -1 where not that side."""
    C, K = prob.C, prob.K
    cam_idx = np.full(prob.ncols, -1, np.int64)
    pt_idx = np.full(prob.ncols, -1, np.int64)
    for c in range(C):
        if prob.rot_col[c] >= 0:
            cam_idx[prob.rot_col[c] + np.arange(3)] = 6 * c + np.arange(3)
        if prob.trn_col[c] >= 0:
            cam_idx[prob.trn_col[c] + np.arange(3)] = 6 * c + 3 + np.arange(3)
    for k, ent in enumerate(prob.intr_cols):
        for slot, (_, col) in enumerate(ent):      # ent is sorted by parameter index
            cam_idx[col] = 6 * (C + k) + slot
    for s in range(prob.S):
        if prob.sq_col[s] >= 0:
            cam_idx[prob.sq_col[s] + np.arange(3)] = 6 * (C + K + s) + np.arange(3)
            cam_idx[prob.st_col[s] + np.arange(3)] = 6 * (C + K + s) + 3 + np.arange(3)
    for p in np.nonzero(prob.pt_col >= 0)[0]:
        pt_idx[prob.pt_col[p] + np.arange(3)] = 3 * p + np.arange(3)
    assert cam_idx.max(initial=-1) < 6 * nbk, "a variable block lies beyond nbk"
    return cam_idx, pt_idx


def _selector(idx, n):
    cols = np.nonzero(idx >= 0)[0]
    return sp.csr_matrix((np.ones(len(cols)), (cols, idx[cols])), shape=(len(idx), n))


def _diag_blocks(M, nb, b):
    """Diagonal b x b blocks of the sparse [nb*b, nb*b] matrix M -> dense [nb, b, b]."""
    M = M.tocoo()
    keep = (M.row // b) == (M.col // b)
    out = np.zeros((nb, b, b))
    np.add.at(out, (M.row[keep] // b, M.row[keep] % b, M.col[keep] % b), M.data[keep])
    return out


def _damping(diag, js, radius):
    js2 = js * js
    return np.clip(diag * js2, 1e-6, 1e32) / (radius * js2)


class BASystem:
    """The linear system of the first LM iteration of a solve at state ``x`` (``first = true``: Jacobi scales set).

    precond: "schur" (Schur-Jacobi on every block), "schur_frames" (Schur-Jacobi on the frame blocks, block-Jacobi
    on the rest: the stored-row intrinsics path), "jacobi" (block-Jacobi on U + D) or "schur_per_obs" (the frame blocks
    minus sum_o W_o (V_p + D_p)^-1 W_o^T over single observations: what ba2_schur_diag forms with known rigs, where a
    frame that sees a point through two sensors has two observations of it and the exact block has their cross terms
    as well)."""

    def __init__(self, prob: BAProblem, x: dict, radius: float, nbk: int, precond: str = "schur"):
        assert precond in ("schur", "schur_frames", "jacobi", "schur_per_obs")
        self.prob, self.x, self.radius, self.nbk = prob, x, radius, nbk
        self.points_var = bool(prob.opts.optimize_points)
        C, P = prob.C, prob.P
        nc, npt = 6 * nbk, 3 * P
        self.cam_idx, self.pt_idx = device_index(prob, nbk)
        self.cost, r, J = prob.evaluate(x, True)
        J = J.tocsr()
        self.J, self.r = J, r
        Jc = (J @ _selector(self.cam_idx, nc)).tocsr()
        Jp = (J @ _selector(self.pt_idx, npt)).tocsr()
        # ---- camera side: U blocks, gradient, variable dofs --------------------------------------------------------
        self.Hcc = (Jc.T @ Jc).tocsr()
        Ub = _diag_blocks(self.Hcc, nbk, 6)
        d = np.einsum("bii->bi", Ub).ravel()
        mapped = np.zeros(nc, bool)
        mapped[self.cam_idx[self.cam_idx >= 0]] = True
        self.var_c = mapped & (d > 0)                    # ba_finalize_cams: dofs without curvature are decoupled too
        off = ~self.var_c.reshape(nbk, 6)
        Ub[off[:, :, None] | off[:, None, :]] = 0.0
        Ub[off[:, :, None] & np.eye(6, dtype=bool)[None]] = 1.0
        self.U_blocks = Ub
        self.g_c = np.where(self.var_c, Jc.T @ r, 0.0)
        self.jscale_c = np.where(self.var_c, 1.0 / (1.0 + np.sqrt(np.maximum(d, 0.0))), -1.0)
        self.Dc = np.where(self.var_c, _damping(d, np.abs(self.jscale_c), radius), 0.0)
        # ---- point side ---------------------------------------------------------------------------------------------
        if self.points_var:
            Vb = _diag_blocks(Jp.T @ Jp, P, 3)
            self.V_blocks = Vb
            self.g_p = Jp.T @ r
            dv = np.einsum("pii->pi", Vb)
            self.jscale_p = 1.0 / (1.0 + np.sqrt(dv))
            self.Dp = _damping(dv, self.jscale_p, radius)
            self.Vinv_blocks = np.linalg.inv(Vb + self.Dp[:, :, None] * np.eye(3)[None])
            self.Vinv = sp.bsr_matrix((self.Vinv_blocks, np.arange(P), np.arange(P + 1)), shape=(npt, npt)).tocsr()
            self.W = (Jc.T @ Jp).tocsr()
        # ---- preconditioner blocks ------------------------------------------------------------------------------------
        M = Ub + self.Dc.reshape(nbk, 6)[:, :, None] * np.eye(6)[None]
        self.jacobi_inv = np.linalg.inv(M)
        if self.points_var:
            self.Sd_blocks = _diag_blocks(self.W @ self.Vinv @ self.W.T, nbk, 6)
            self.schur_jacobi_inv = np.linalg.inv(M - self.Sd_blocks)
        if precond == "schur_per_obs":
            self.schur_jacobi_inv = np.linalg.inv(M - self._per_observation_schur_diag(Jc, Jp, nbk))
            precond = "schur"
        if precond == "jacobi" or not self.points_var:
            self.Minv_blocks = self.jacobi_inv
        elif precond == "schur":
            self.Minv_blocks = self.schur_jacobi_inv
        else:
            self.Minv_blocks = self.jacobi_inv.copy()
            self.Minv_blocks[:C] = self.schur_jacobi_inv[:C]
        # ---- right-hand side ------------------------------------------------------------------------------------------
        self.b = -self.g_c
        if self.points_var:
            self.b = -(self.g_c - self.W @ (self.Vinv @ self.g_p))

    def _per_observation_schur_diag(self, Jc, Jp, nbk):
        p = self.prob
        rows = 2 * np.arange(p.N)
        f, pt = p.obs_cam, p.obs_pt
        Jcd = np.zeros((p.N, 2, 6))
        Jpd = np.zeros((p.N, 2, 3))
        for a in range(2):
            for k in range(6):
                Jcd[:, a, k] = np.asarray(Jc[rows + a, 6 * f + k]).ravel()
            for k in range(3):
                Jpd[:, a, k] = np.asarray(Jp[rows + a, 3 * pt + k]).ravel()
        Wo = np.einsum("nai,naj->nij", Jcd, Jpd)
        T = np.einsum("nij,njk,nlk->nil", Wo, self.Vinv_blocks[pt], Wo)
        out = np.zeros((nbk, 6, 6))
        np.add.at(out, f, T)
        return out

    # -- the reduced camera system ------------------------------------------------------------------------------------
    def apply(self, xc):
        """(S + D) x with S never formed: U + cross terms (J_c^T J_c), identity on non-variable dofs, damping, minus the
        Schur term W (V + D_p)^-1 W^T x."""
        xv = np.where(self.var_c, xc, 0.0)
        y = self.Hcc @ xv + self.Dc * xv + np.where(self.var_c, 0.0, xc)
        if self.points_var:
            y -= self.W @ (self.Vinv @ (self.W.T @ xv))
        return y

    def precondition(self, rc):
        return np.einsum("bij,bj->bi", self.Minv_blocks, rc.reshape(-1, 6)).ravel()

    def pcg(self, iters: int):
        """Textbook PCG from x_0 = 0 with the block preconditioner: the iterates x_1 .. x_iters."""
        x = np.zeros_like(self.b)
        r = self.b.copy()
        z = self.precondition(r)
        p = z.copy()
        rz = r @ z
        out = []
        for _ in range(iters):
            q = self.apply(p)
            alpha = rz / (p @ q)
            x = x + alpha * p
            r = r - alpha * q
            z = self.precondition(r)
            rz_new = r @ z
            p = z + (rz_new / rz) * p
            rz = rz_new
            out.append(x.copy())
        return out

    # -- the step ---------------------------------------------------------------------------------------------------------
    def full_step(self, dc):
        """Camera step (device layout) -> full oracle tangent step, the point step by back-substitution."""
        delta = np.zeros(self.prob.ncols)
        m = self.cam_idx >= 0
        delta[m] = dc[self.cam_idx[m]]
        if self.points_var:
            dp = -(self.Vinv @ (self.g_p + self.W.T @ np.where(self.var_c, dc, 0.0)))
            mp = self.pt_idx >= 0
            delta[mp] = dp[self.pt_idx[mp]]
        return delta

    def damping_full(self):
        D = np.zeros(self.prob.ncols)
        m = self.cam_idx >= 0
        D[m] = self.Dc[self.cam_idx[m]]
        if self.points_var:
            mp = self.pt_idx >= 0
            D[mp] = self.Dp.ravel()[self.pt_idx[mp]]
        return D

    def model_cost_change(self, delta):
        """Decrease of the undamped linear model, -(J d)^T (r + J d / 2) = -g^T d - 1/2 d^T J^T J d, formed directly over
        the full system (Ceres: the step quality divides by it; oracle/ceres_lm.py)."""
        Jd = self.J @ delta
        return float(-(Jd @ (self.r + 0.5 * Jd)))

    def candidate(self, dc):
        """(candidate state, its cost, step norm, x norm, model cost change) of camera step ``dc``."""
        delta = self.full_step(dc)
        cand = self.prob.plus(self.x, delta)
        cost = self.prob.evaluate(cand, False)[0]
        return cand, cost, self.prob.x_norm(cand, self.x), self.prob.x_norm(self.x), self.model_cost_change(delta)

    def model_cost_change_reduced(self, dc):
        """The device's bookkeeping: 1/2 (-g^T d + d_c^T rho + d^T D d), rho = b - (S + D) d_c the PCG residual."""
        delta = self.full_step(dc)
        g = self.J.T @ self.r
        rho = self.b - self.apply(dc)
        D = self.damping_full()
        return float(0.5 * (-(g @ delta) + np.where(self.var_c, dc, 0.0) @ rho + delta @ (D * delta)))
