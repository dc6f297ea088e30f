"""ORACLE (test infrastructure, NOT product code) -- FP64 sparse restatement of the linear algebra one rotation-averaging
iteration forms on the device, operator by operator, so that tests/test_ra_system_gpu.py can compare every kernel of
the solver (include/b200sfm_testing.h) with it.

Layout: the device's.  Unknowns are n = n_frames + n_cams nodes of 3 slots (a gravity frame's unknown is its y slot;
its x and z columns are empty).  Rows are 3 per edge, row 3e + k, and edge E - 1 is the gauge pseudo-edge
(identity -> fixed frame).  A row that does not exist (x / z of a 1-DoF row) is empty.  A is built from the reference's
triplet rules (global_rotation_averaging.cc:386-460) with duplicates summed, as the reference's sparse matrix does:
  * 3-DoF rows: -I at image 1's frame, +I at image 2's frame; a gravity frame only in slot y (.cc:396-415);
  * pairs of two gravity frames: one row in slot y (.cc:387-394);
  * unknown sensors: -I at image 1's camera node, +I at image 2's (.cc:425-440).  The same sensor in both images of
    a pair cancels, and so does the same frame;
  * gauge rows: +I at the fixed frame, or one y row when it has gravity (.cc:449-460).
Residuals, weights, the update and the quaternion average reuse oracle/ra_oracle.py.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from oracle import ra_oracle as RO


class RASystem:
    """One problem as b200sfm_test_ra_problem_create receives it.  theta [n, 3]: the state (a gravity frame holds
    (0, phi, 0)); R_rel [E_real, 3, 3] (gravity-aligned where a frame has gravity)."""

    def __init__(self, n_frames, ei, ej, R_rel, theta, fixed, edge_w=None, use_weight=False, has_grav=None,
                 n_cams=0, eci=None, ecj=None, cam_frames=None):
        self.n_frames, self.n_cams = int(n_frames), int(n_cams)
        self.n = n = self.n_frames + self.n_cams
        E_real = len(ei)
        self.E = E = E_real + 1
        self.fixed = int(fixed)
        self.ei = np.append(np.asarray(ei, np.int64), -1)
        self.ej = np.append(np.asarray(ej, np.int64), self.fixed)
        none = np.full(E_real, -1, np.int64)
        self.eci = np.append(np.asarray(eci, np.int64) if eci is not None else none, -1)
        self.ecj = np.append(np.asarray(ecj, np.int64) if ecj is not None else none, -1)
        self.cam_frames = cam_frames or []
        self.theta = np.array(theta, np.float64).reshape(n, 3)
        self.grav = np.zeros(n, bool) if has_grav is None else np.append(np.asarray(has_grav, bool), np.zeros(self.n_cams, bool))
        self.Rrel = np.concatenate([np.asarray(R_rel, np.float64).reshape(E_real, 3, 3),
                                    RO.aa_to_R(self.theta[self.fixed][None])])
        self.w_edge = np.ones(E)
        if use_weight and edge_w is not None:
            self.w_edge[:E_real] = np.where(np.asarray(edge_w) >= 0, edge_w, 1.0)
        gi = np.where(self.ei >= 0, self.grav[np.maximum(self.ei, 0)], False)
        gj = self.grav[self.ej]
        self.y_only = np.where(self.ei >= 0, gi & gj, gj)
        aa = RO.R_to_aa(self.Rrel)
        self.angle_rel = np.where(self.y_only, aa[:, 1], 0.0)
        self.angle_rel[-1] = self.theta[self.fixed, 1]          # gravity gauge row: phi_fixed(initial)
        self.xz_err = np.where(self.y_only, aa[:, 0] ** 2 + aa[:, 2] ** 2, 0.0)
        self.row_exists = np.ones((E, 3), bool)
        self.row_exists[self.y_only, 0] = self.row_exists[self.y_only, 2] = False
        self.A = self._build_A(gi, gj)

    def _build_A(self, gi, gj):
        rows, cols, vals = [], [], []
        for e in range(self.E):
            i, j, ci, cj = self.ei[e], self.ej[e], self.eci[e], self.ecj[e]
            for k in range(3):
                if not self.row_exists[e, k]:
                    continue
                r = 3 * e + k
                if not gj[e] or k == 1:
                    rows.append(r); cols.append(3 * j + k); vals.append(1.0)
                if i >= 0 and (not gi[e] or k == 1):
                    rows.append(r); cols.append(3 * i + k); vals.append(-1.0)
                if i >= 0 and cj >= 0:
                    rows.append(r); cols.append(3 * cj + k); vals.append(1.0)
                if i >= 0 and ci >= 0:
                    rows.append(r); cols.append(3 * ci + k); vals.append(-1.0)
        A = sp.csr_matrix((vals, (rows, cols)), shape=(3 * self.E, 3 * self.n))
        A.sum_duplicates()
        A.eliminate_zeros()
        return A

    @property
    def rows_total(self):
        return int(self.row_exists.sum())

    # ---- residuals and weights (ra_oracle's conventions) ------------------------------------------------------
    def residuals(self, theta=None):
        th = self.theta if theta is None else theta
        i, j = self.ei, self.ej
        Ri = RO.aa_to_R(th[np.maximum(i, 0)])
        Ri[i < 0] = np.eye(3)
        m = (self.eci >= 0) & (i >= 0)
        if m.any():
            Ri[m] = RO.aa_to_R(th[self.eci[m]]) @ Ri[m]
        Rj = RO.aa_to_R(th[j])
        m = (self.ecj >= 0) & (i >= 0)
        if m.any():
            Rj[m] = RO.aa_to_R(th[self.ecj[m]]) @ Rj[m]
        res = -RO.R_to_aa(np.swapaxes(Rj, -1, -2) @ self.Rrel @ Ri)
        yo = np.nonzero(self.y_only)[0]
        res[yo] = 0.0
        for e in yo:
            if i[e] >= 0:
                res[e, 1] = RO.rel_angle_error(self.angle_rel[e], th[i[e], 1], th[j[e], 1])
            else:
                res[e, 1] = th[j[e], 1] - self.angle_rel[e]
        return res

    def weights(self, res, mode, sigma2=0.0):
        """ra_residuals' w: the L1 rows' weights (mode 0), Geman-McClure (1) or half-norm (2); the gauge keeps w_edge."""
        w = self.w_edge.copy()
        if mode == 0:
            return w
        e2 = np.where(self.y_only, res[:, 1] ** 2 + self.xz_err, (res ** 2).sum(1))
        with np.errstate(divide="ignore"):
            wi = sigma2 / (e2 + sigma2) ** 2 if mode == 1 else e2 ** ((0.5 - 2.0) / 2.0)
        real = self.ei >= 0
        w[real] *= wi[real]
        return w

    # ---- the linear system --------------------------------------------------------------------------------------
    def row_weights(self, w, square):
        return np.repeat(w ** (2 if square else 1), 3)

    def laplacian(self, w, square):
        """L = A^T W^p A."""
        return (self.A.T @ sp.diags(self.row_weights(w, square)) @ self.A).tocsr()

    def rhs(self, w, square, res):
        return self.A.T @ (self.row_weights(w, square) * res.ravel())

    @staticmethod
    def jacobi(L):
        """diag(L) and its inverse as ra_build_precond forms it (1 where the diagonal is 0)."""
        d = L.diagonal()
        return d, np.where(d > 0, 1.0 / np.where(d > 0, d, 1.0), 1.0)

    def coarse(self, L, agg_of, nc):
        """P (nodes -> aggregates, one slot) and Ac = P^T L_slot P of one slot: on the two-level paths every node has 3
        DoF and L = L_slot (x) I3."""
        P = sp.csr_matrix((np.ones(self.n), (np.arange(self.n), np.asarray(agg_of))), shape=(self.n, nc))
        Ls = L[0::3, 0::3]
        return P, (P.T @ Ls @ P).toarray()

    @staticmethod
    def precond(Dinv, P=None, Ac_inv=None):
        """r -> M^-1 r = D^-1 r + P Ac^-1 P^T r (per slot)."""
        def apply(r):
            z = Dinv * r
            if P is not None:
                r3 = r.reshape(-1, 3)
                z = z + (P @ (Ac_inv @ (P.T @ r3))).ravel()
            return z
        return apply

    @staticmethod
    def pcg(L, b, Minv, k, x0=None, rel_tol=0.0):
        """Plain PCG, the device's recurrence and stopping rule (pcg.cuh): at the head of iteration it, stop when
        |r|^2 <= rel_tol^2 ref, ref = |r_0|^2 cold or |b|^2 warm.  Returns (iterates after every iteration, count)."""
        x = np.zeros_like(b) if x0 is None else np.array(x0, np.float64)
        r = b - L @ x if x0 is not None else b.copy()
        z = Minv(r)
        ref = float(b @ b) if x0 is not None else float(r @ r)
        rz = float(r @ z)
        p = None
        out = []
        for it in range(1, k + 1):
            rr = float(r @ r)
            if not ref > 0 or rr <= rel_tol ** 2 * ref:
                return out, it - 1
            p = z.copy() if p is None else z + (rz / rz_prev if rz_prev > 0 else 0.0) * p
            q = L @ p
            pq = float(p @ q)
            alpha = rz / pq if pq > 0 else 0.0
            x = x + alpha * p
            r = r - alpha * q
            z = Minv(r)
            rz_prev, rz = rz, float(r @ z)
            out.append(x.copy())
        return out, k

    # ---- ADMM step and update ---------------------------------------------------------------------------------
    def admm_step(self, w, x, b, z, u, rho):
        """ra_admm_step: one iteration after the x-update on |A_w x - b|_1, A_w = diag(w) A (rows that do not exist
        keep z and u).  Returns (z, u, rhs, svec, uvec, norms[5])."""
        ex = self.row_exists.ravel()
        Aw = sp.diags(np.repeat(w, 3)) @ self.A
        a = Aw @ x
        v = a - b + u
        zn = np.maximum(0, v - 1 / rho) - np.maximum(0, -v - 1 / rho)
        un = u + a - zn - b
        zn, un = np.where(ex, zn, z), np.where(ex, un, u)
        pr = np.where(ex, a - zn - b, 0.0)
        rhs = Aw.T @ np.where(ex, b + zn - un, 0.0)
        svec = Aw.T @ np.where(ex, zn - z, 0.0)
        uvec = Aw.T @ np.where(ex, un, 0.0)
        norms = np.array([pr @ pr, a @ a, zn[ex] @ zn[ex], svec @ svec, uvec @ uvec])
        return zn, un, rhs, svec, uvec, norms

    def update(self, step, theta=None):
        """UpdateGlobalRotations: the frames (1-DoF: phi -= step), then the unknown cameras' quaternion average over
        the updated frames.  Returns (theta, [average frame step, |step|, NaN flag])."""
        th = self.theta if theta is None else theta
        st = np.asarray(step, np.float64).reshape(self.n, 3)
        nf = self.n_frames
        out = th.copy()
        g = self.grav[:nf]
        out[:nf] = RO.update_rotations(th[:nf], st[:nf])
        out[:nf][g] = np.stack([np.zeros(g.sum()), th[:nf][g, 1] - st[:nf][g, 1], np.zeros(g.sum())], 1)
        Rf = RO.aa_to_R(out[:nf])
        for c in range(self.n_cams):
            if len(self.cam_frames[c]) == 0:
                continue
            R_ori = RO.aa_to_R(th[nf + c][None])[0]
            R_upd = RO.aa_to_R(-st[nf + c][None])[0]
            out[nf + c] = RO.R_to_aa(RO.average_quaternions([R_ori @ Rf[f] @ R_upd @ Rf[f].T for f in self.cam_frames[c]])[None])[0]
        sums = np.array([np.linalg.norm(st[:nf], axis=1).sum() / nf, np.linalg.norm(st), float(np.isnan(st).any())])
        return out, sums
