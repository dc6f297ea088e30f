"""ORACLE (test infrastructure, NOT product code) -- FP64 sparse restatement of
one Levenberg-Marquardt step of the device global positioner, in the device's
coordinates, for the operator-level tests (tests/test_gp_system_gpu.py against
the probe of include/b200sfm_testing.h).

Built from ``GPProblem.evaluate`` (the Huber-corrected sparse Jacobian of
oracle/gp_oracle.py) and nothing else; no quantity is taken from the device.

Device layout: CB = C + S_u blocks of 3 dofs, the frame centres then the
unknown cam_from_rig centres; points [P][3]; one scale per observation in the
problem's observation order, short tracks included.  Blocks that are not
variables -- constant, masked or unobserved -- are identity rows with zero
gradient, zero right-hand side and Jacobi scale -1 (gp_finalize_cams).
Symmetric 3x3 blocks are packed upper triangle, row by row.

What is formed (compute_step in glomap_b200/csrc/gp_solver.cuh):
  * Jacobi scales js = 1/(1+sqrt(colnorm)) of the linearisation, damping
    D = clamp(colnorm js^2, 1e-6, 1e32) / (radius js^2), H = J^T J + D, g = J^T r;
  * the scales eliminated from H (H_ss is diagonal): per observation the
    3x3 block M_o, the rhs term b_o and the pivot h, formed generically from
    the Jacobian rows of a problem with every centre variable; then over the
    reduced program, the points eliminated: V, g_X, U, g_c, S, b;
  * the preconditioner: the Schur-Jacobi block summed per observation,
    (U + D - sum_o M_o Vinv M_o)^-1, or block-Jacobi (U + D)^-1;
  * plain PCG from x = 0, the exact solve, the back-substitution of dX and ds
    from a given block step, g.delta, the model decrease
    -(J delta)^T (r + J delta / 2), the candidate Project(x + alpha delta), the
    reduced-program norms and the projected raw-gradient max-norm.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from .gp_oracle import GPProblem

SYM3 = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]


def pack_sym3(M):
    """[..., 3, 3] -> [..., 6] upper triangle, row by row."""
    return np.stack([M[..., i, j] for i, j in SYM3], -1)


def unpack_sym3(a):
    M = np.zeros(a.shape[:-1] + (3, 3))
    for k, (i, j) in enumerate(SYM3):
        M[..., i, j] = a[..., k]
        M[..., j, i] = a[..., k]
    return M


def _block_diag(blocks):
    """[n, 3, 3] -> sparse block-diagonal (3n x 3n)."""
    n = len(blocks)
    rows = np.repeat(3 * np.arange(n), 9) + np.tile(np.repeat(np.arange(3), 3), n)
    cols = np.repeat(3 * np.arange(n), 9) + np.tile(np.tile(np.arange(3), 3), n)
    return sp.csr_matrix((blocks.reshape(-1), (rows, cols)), shape=(3 * n, 3 * n))


def _selector(idx, n_dev):
    """Oracle column -> device dof selector (ncols x n_dev); idx[col] = -1 where the column is not on that side."""
    m = idx >= 0
    return sp.csr_matrix((np.ones(int(m.sum())), (np.nonzero(m)[0], idx[m])), shape=(len(idx), n_dev))


class GPSystem:
    """One LM step at ``prob.x0`` with damping ``radius``; the Jacobi scales are those of this same state (a solve's
    first linearisation).  ``full`` is the same problem with every centre and point variable (same scales option): its
    Jacobian rows give the per-observation blocks, which the device forms whether a centre is variable or not."""

    def __init__(self, prob: GPProblem, full: GPProblem, radius: float, schur_jacobi: bool):
        self.prob, self.radius = prob, radius
        x = prob.x0
        C, P = prob.C, prob.P
        S_u = len(prob.u_col)
        self.C, self.P, self.S_u, self.CB = C, P, S_u, C + S_u
        self.kept = np.nonzero(prob.keep)[0]          # device observation of each oracle observation
        self.N_dev = len(prob.keep)
        nc3 = 3 * self.CB
        cost, r, J = prob.evaluate(x, True)
        self.cost, self.r, self.J = cost, r, J
        n = J.shape[1]
        colnorm = np.asarray(J.multiply(J).sum(axis=0)).ravel()
        js = 1.0 / (1.0 + np.sqrt(colnorm))
        D = np.clip(colnorm * js * js, 1e-6, 1e32) / (radius * js * js)
        self.D = D
        H = (J.T @ J + sp.diags(D)).tocsr()
        g = J.T @ r
        self.g = g
        # index maps: oracle columns -> device dofs
        cam_dev = np.full(n, -1, np.int64)
        for c in np.nonzero(prob.cam_col >= 0)[0]:
            cam_dev[prob.cam_col[c] + np.arange(3)] = 3 * c + np.arange(3)
        for u in np.nonzero(prob.u_col >= 0)[0]:
            cam_dev[prob.u_col[u] + np.arange(3)] = 3 * (C + u) + np.arange(3)
        pt_dev = np.full(n, -1, np.int64)
        for p in np.nonzero(prob.pt_col >= 0)[0]:
            pt_dev[prob.pt_col[p] + np.arange(3)] = 3 * p + np.arange(3)
        s_dev = np.full(n, -1, np.int64)
        sv = prob.s_col >= 0
        s_dev[prob.s_col[sv]] = np.nonzero(sv)[0]
        Sc, Sp, Ss = _selector(cam_dev, nc3), _selector(pt_dev, 3 * P), _selector(s_dev, prob.N)
        self.Sc, self.Sp, self.Ss = Sc, Sp, Ss
        self.var_c = np.zeros(self.CB, bool)
        self.var_c[cam_dev[cam_dev >= 0] // 3] = True
        self.var_p = prob.pt_col >= 0
        self.var_s = sv
        # eliminate the scales (H_ss diagonal)
        Sa = sp.hstack([Sc, Sp]).tocsr()
        Haa = (Sa.T @ H @ Sa).tocsr()
        Has = (Sa.T @ H @ Ss).tocsr()
        hs = np.asarray((Ss.T @ H @ Ss).diagonal()).ravel()
        self.inv_h = np.where(hs > 0, 1.0 / np.where(hs > 0, hs, 1.0), 0.0)
        self.g_s = Ss.T @ g
        H1 = (Haa - Has @ sp.diags(self.inv_h) @ Has.T).tocsr()
        g1 = Sa.T @ g - Has @ (self.inv_h * self.g_s)
        self.Has = Has
        H1cc, H1cp, H1pp = H1[:nc3, :nc3], H1[:nc3, nc3:], H1[nc3:, nc3:].tocsr()
        self.H1cp = H1cp.tocsr()
        # points
        Vb = np.zeros((P, 3, 3))
        for i in range(3):
            for j in range(3):
                Vb[:, i, j] = np.asarray(H1pp[np.arange(P) * 3 + i, np.arange(P) * 3 + j]).ravel()
        self.Vinv_blocks = np.zeros((P, 3, 3))
        self.Vinv_blocks[self.var_p] = np.linalg.inv(Vb[self.var_p])
        self.Vinv = _block_diag(self.Vinv_blocks)
        self.gX = g1[nc3:].reshape(P, 3)
        self.Dp = np.zeros(P)
        self.jscale_p = np.zeros(P)
        self.Dp[self.var_p] = D[prob.pt_col[self.var_p]]
        self.jscale_p[self.var_p] = js[prob.pt_col[self.var_p]]
        # reduced block system, identity rows on the constant blocks
        fixed3 = np.repeat(~self.var_c, 3).astype(float)
        self.S = (H1cc - H1cp @ self.Vinv @ H1cp.T + sp.diags(fixed3)).tocsr()
        gc = g1[:nc3]
        self.b = np.where(fixed3 > 0, 0.0, -(gc - H1cp @ (self.Vinv @ g1[nc3:])))
        colD = np.zeros(nc3)
        colD[cam_dev[cam_dev >= 0]] = D[cam_dev >= 0]
        colJs = np.full(nc3, -1.0)
        colJs[cam_dev[cam_dev >= 0]] = js[cam_dev >= 0]
        self.Dc = colD.reshape(-1, 3)
        self.jscale_c = colJs.reshape(-1, 3)[:, 0]
        self.gc = gc.reshape(-1, 3)
        Ub = np.zeros((self.CB, 3, 3))
        for i in range(3):
            for j in range(3):
                Ub[:, i, j] = np.asarray(H1cc[np.arange(self.CB) * 3 + i, np.arange(self.CB) * 3 + j]).ravel()
        Ub -= self.Dc[:, :, None] * np.eye(3)
        Ub[~self.var_c] = np.eye(3)
        self.U_blocks = Ub
        # per-observation blocks from the problem with every centre variable
        self._per_obs(full)
        # preconditioner
        Mb = Ub + self.Dc[:, :, None] * np.eye(3)
        if schur_jacobi:
            cam = prob.obs_cam
            pt = prob.obs_pt
            Mo = unpack_sym3(self.M[self.kept])
            T = np.einsum("nij,njk,nkl->nil", Mo, self.Vinv_blocks[pt], Mo)
            Sd = np.zeros((self.CB, 3, 3))
            np.add.at(Sd, cam, T)
            Mb = Mb - np.where(self.var_c[:, None, None], Sd, 0.0)
        self.Minv_blocks = np.linalg.inv(Mb)

    def _per_obs(self, full: GPProblem):
        """M_o, b_o, h, w s^2 per observation (device order; zero rows for short tracks), by eliminating the scale from
        the observation's rows of the Jacobian of ``full``."""
        _, r, J = full.evaluate(full.x0, True)
        J = J.tocsr()
        colnorm = np.asarray(J.multiply(J).sum(axis=0)).ravel()
        js = 1.0 / (1.0 + np.sqrt(colnorm))
        D = np.clip(colnorm * js * js, 1e-6, 1e32) / (self.radius * js * js)
        Nk = full.N
        rows = 3 * np.arange(Nk)[:, None] + np.arange(3)                      # [Nk, 3]
        c0 = full.cam_col[full.obs_cam]
        Jc = np.zeros((Nk, 3, 3))
        for m in range(3):
            Jc[:, :, m] = np.asarray(J[rows.ravel(), np.repeat(c0 + m, 3)]).reshape(Nk, 3)
        sv = full.s_col >= 0
        Js = np.zeros((Nk, 3))
        if sv.any():
            Js[sv] = np.asarray(J[rows[sv].ravel(), np.repeat(full.s_col[sv], 3)]).reshape(-1, 3)
        Ds = np.zeros(Nk)
        Ds[sv] = D[full.s_col[sv]]
        h = (Js * Js).sum(1) + Ds
        rr = r.reshape(Nk, 3)
        JcJs = np.einsum("nki,nk->ni", Jc, Js)
        inv_h = np.where(h > 0, 1.0 / np.where(h > 0, h, 1.0), 0.0)
        M = np.einsum("nki,nkj->nij", Jc, Jc) - inv_h[:, None, None] * JcJs[:, :, None] * JcJs[:, None, :]
        b = np.einsum("nki,nk->ni", Jc, rr) - (inv_h * (Js * rr).sum(1))[:, None] * JcJs
        self.M = np.zeros((self.N_dev, 6))
        self.bw = np.zeros((self.N_dev, 4))
        self.h = np.zeros(self.N_dev)
        self.jscale_s = np.zeros(self.N_dev)
        self.M[self.kept] = pack_sym3(M)
        self.bw[self.kept, :3] = b
        self.bw[self.kept, 3] = np.einsum("nii->n", np.einsum("nki,nkj->nij", Jc, Jc)) / 3.0
        self.h[self.kept[sv]] = h[sv]
        self.jscale_s[self.kept[sv]] = js[full.s_col[sv]]

    # ---- the reduced system --------------------------------------------------------------------------------------
    @property
    def U(self):
        return pack_sym3(self.U_blocks)

    @property
    def Minv(self):
        return pack_sym3(self.Minv_blocks)

    def apply(self, x):
        return self.S @ x

    def pcg(self, k):
        """Textbook PCG from x = 0 with the block preconditioner: the iterates after 1..k iterations."""
        Minv = _block_diag(self.Minv_blocks)
        x = np.zeros_like(self.b)
        r = self.b.copy()
        z = Minv @ r
        p = z.copy()
        rz = r @ z
        out = []
        for _ in range(k):
            q = self.S @ p
            pq = p @ q
            alpha = rz / pq if pq > 0 else 0.0        # as pcg_update: no step on an empty system
            x = x + alpha * p
            r = r - alpha * q
            z = Minv @ r
            rz_new = r @ z
            p = z + (rz_new / rz if rz > 0 else 0.0) * p
            rz = rz_new
            out.append(x.copy())
        return out

    def solve(self):
        return spla.spsolve(self.S.tocsc(), self.b)

    # ---- the step ------------------------------------------------------------------------------------------------
    def back_sub(self, dc):
        """dX [P, 3] and ds [N_dev] (device order) from a block step dc [CB*3]."""
        dc = np.where(np.repeat(self.var_c, 3), dc, 0.0)
        dX = -(self.Vinv @ (self.gX.ravel() + self.H1cp.T @ dc))
        a = np.concatenate([dc, dX])
        ds_k = -self.inv_h * (self.g_s + self.Has.T @ a)
        ds = np.zeros(self.N_dev)
        ds[self.kept] = ds_k
        return dX.reshape(-1, 3), ds

    def delta(self, dc):
        """The full step over the oracle's columns: dc, then the back-substitution."""
        dX, ds = self.back_sub(dc)
        dc = np.where(np.repeat(self.var_c, 3), dc, 0.0)
        return self.Sc @ dc + self.Sp @ dX.ravel() + self.Ss @ ds[self.kept]

    def step_scalars(self, dc):
        """(g.delta, model_cost_change = -(J delta)^T (r + J delta / 2)) of the step dc + its back-substitution."""
        d = self.delta(dc)
        Jd = self.J @ d
        return float(self.g @ d), -float(Jd @ (self.r + 0.5 * Jd))

    def candidate(self, dc, alpha):
        """Project(x + alpha delta) as a state dict, its cost, step_norm and x_norm over the reduced program."""
        x = self.prob.x0
        cand = self.prob.plus(x, alpha * self.delta(dc))
        cost, _, _ = self.prob.evaluate(cand, False)
        return cand, cost, self.prob.x_norm(cand, x), self.prob.x_norm(x)

    def gmax(self):
        """Ceres' gradient max-norm: the projected raw gradient |Project(x - g) - x|_inf over the reduced program."""
        return float(np.abs(self.prob.project(self.prob.x0, -self.g)).max())
