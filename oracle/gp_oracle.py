"""ORACLE (test infrastructure, NOT product code) -- CPU/numpy restatement of
the reference's BATA global positioning, glomap/estimators/global_positioning.cc
with the cost functor of glomap/estimators/cost_function.h:15-41.

PARITY UNPINNED (see oracle/ceres_lm.py): Ceres cannot be built here and the
reference holds no golden vectors for GlobalPositioner.  The reference's random
initialisation (std::mt19937 consumed in unordered_map order,
global_positioning.cc:123-165,262) cannot be reproduced bit for bit either, so
parity is on the converged solution after Sim3 alignment.

What is restated, with the reference lines it follows:
  * one residual block per (track, observation), tracks with fewer than
    min_num_view_per_track observations skipped (.cc:257-258):
        r = t_obs - s * (X - c),   t_obs = R_cw^T * bearing     (.cc:294-296, cost_function.h:26-29)
    parameters: camera centre c (3), point X (3), scale s (1) initialised to 1 (.cc:298).
  * loss: Huber(thres_loss_function = 0.1) for cameras with a prior focal
    length, ScaledLoss(Huber, 0.5) otherwise (.cc:242-255,313-316).
  * every scale has the lower bound 1e-5 (.cc:373); the FIRST scale is held
    constant (.cc:484-489); optimize_{positions,points,scales} flags (.cc:456-482).
  * ONLY_POINTS constraints (the mapper enforces it, controllers/global_mapper.cc:145-149).
  * Ceres LM with bounds (projection in Plus + projected Armijo line search)
    -> oracle/ceres_lm.py; the reference eliminates the scales with
    SPARSE_SCHUR and factors the rest (.cc:553-555) -- an exact solve, as here.
  * ConvertResults: t = -R c (.cc:562-572) is left to the caller.
"""
from __future__ import annotations

import dataclasses

import numpy as np
import scipy.sparse as sp

from .ceres_lm import LMOptions, LMSummary, huber_rho, solve_lm

SCALE_LOWER_BOUND = 1e-5


@dataclasses.dataclass
class GPOptions:
    """Mirror of GlobalPositionerOptions (global_positioning.h:9-54)."""
    optimize_positions: bool = True
    optimize_points: bool = True
    optimize_scales: bool = True
    thres_loss_function: float = 0.1
    min_num_view_per_track: int = 3
    max_num_iterations: int = 100
    function_tolerance: float = 1e-5


class GPProblem:
    def __init__(self, centers, points, pt_obs_begin, obs_cam, obs_dir, cam_calibrated, opts: GPOptions, scales=None,
                 obs_offset=None, rig_unknown=None, cam_const=None, obs_calibrated=None):
        """``obs_offset`` [N,3]: known-rig term of RigBATAPairwiseDirectionError (cost_function.h:49-82) with the rig
        scale held at 1 (global_positioning.cc:493-497): r = t_obs - s (X - c_frame + t_rig), t_rig = R_cw^T t_cam_from_rig
        (.cc:339-345).
        ``rig_unknown`` = dict(obs_sensor [N] (-1: none), R_rw [N,3,3] rig_from_world rotation of the observation's frame,
        centers [S,3]): RigUnknownBATAPairwiseDirectionError (cost_function.h:90-134, global_positioning.cc:347-364) --
        the camera centre in the rig frame u_s of a sensor whose cam_from_rig is not known yet is an unknown block shared
        by all its images:  r = t_obs - s (X - c_frame - R_rw^T u_s).
        ``cam_const`` [C]: centres held constant (SetParameterBlockConstant) on top of optimize_positions.
        ``obs_calibrated`` [N]: the prior-focal flag of the observing camera of a rig, overriding cam_calibrated."""
        self.opts = opts
        self.C, self.P = len(centers), len(points)
        lens = np.diff(pt_obs_begin)
        keep_pt = lens >= opts.min_num_view_per_track
        pt_of_obs = np.repeat(np.arange(self.P), lens)
        self.keep = keep_pt[pt_of_obs]
        self.obs_pt = pt_of_obs[self.keep]
        self.obs_cam = np.asarray(obs_cam)[self.keep].astype(np.int64)
        self.obs_dir = np.asarray(obs_dir, dtype=np.float64)[self.keep]
        self.obs_off = None if obs_offset is None else np.asarray(obs_offset, dtype=np.float64)[self.keep]
        self.N = len(self.obs_pt)
        cal = np.ones(self.C, bool) if cam_calibrated is None else np.asarray(cam_calibrated).astype(bool)
        ocal = cal[self.obs_cam] if obs_calibrated is None else np.asarray(obs_calibrated).astype(bool)[self.keep]
        self.loss_scale = np.where(ocal, 1.0, 0.5)
        s0 = np.ones(self.N) if scales is None else np.asarray(scales, dtype=np.float64)[self.keep]
        self.x0 = dict(centers=np.array(centers, dtype=np.float64), points=np.array(points, dtype=np.float64), scales=s0)
        self.ru = None
        if rig_unknown is not None:
            os_ = np.asarray(rig_unknown["obs_sensor"]).astype(np.int64)[self.keep]
            self.ru = dict(obs_sensor=os_, R_rw=np.asarray(rig_unknown["R_rw"], dtype=np.float64)[self.keep])
            self.x0["rig_centers"] = np.array(rig_unknown["centers"], dtype=np.float64)
        cam_used = np.zeros(self.C, bool); cam_used[self.obs_cam] = True
        pt_used = np.zeros(self.P, bool); pt_used[self.obs_pt] = True
        col = 0
        self.cam_col = np.full(self.C, -1)
        if cam_const is not None:
            cam_used &= ~np.asarray(cam_const).astype(bool)
        if opts.optimize_positions:
            idx = np.nonzero(cam_used)[0]
            self.cam_col[idx] = 3 * np.arange(len(idx)); col = 3 * len(idx)
        self.pt_col = np.full(self.P, -1)
        if opts.optimize_points:
            idx = np.nonzero(pt_used)[0]
            self.pt_col[idx] = col + 3 * np.arange(len(idx)); col += 3 * len(idx)
        self.s_col = np.full(self.N, -1)
        if opts.optimize_scales and self.N > 1:
            self.s_col[1:] = col + np.arange(self.N - 1)      # first scale constant (.cc:484-489)
            col += self.N - 1
        self.u_col = np.zeros(0, dtype=np.int64)
        if self.ru is not None:
            S_ = len(self.x0["rig_centers"])
            self.u_col = np.full(S_, -1)
            used = np.zeros(S_, bool); used[self.ru["obs_sensor"][self.ru["obs_sensor"] >= 0]] = True
            # always variable: .cc:440-453 only RANDOMISES them with optimize_positions, nothing sets them constant
            idx = np.nonzero(used)[0]
            self.u_col[idx] = col + 3 * np.arange(len(idx)); col += 3 * len(idx)
        self.ncols = col

    def plus(self, x, delta):
        out = {k: v.copy() for k, v in x.items()}
        uv = self.u_col >= 0
        if uv.any():
            out["rig_centers"][uv] += delta[self.u_col[uv][:, None] + np.arange(3)]
        cv = self.cam_col >= 0
        out["centers"][cv] += delta[self.cam_col[cv][:, None] + np.arange(3)]
        pv = self.pt_col >= 0
        out["points"][pv] += delta[self.pt_col[pv][:, None] + np.arange(3)]
        sv = self.s_col >= 0
        out["scales"][sv] = np.maximum(x["scales"][sv] + delta[self.s_col[sv]], SCALE_LOWER_BOUND)   # Plus() projects
        return out

    def project(self, x, step):
        """Project(x + step) - x over the tangent vector (for the projected gradient norm)."""
        out = step.copy()
        sv = self.s_col >= 0
        cols = self.s_col[sv]
        out[cols] = np.maximum(x["scales"][sv] + step[cols], SCALE_LOWER_BOUND) - x["scales"][sv]
        return out

    def x_norm(self, x, y=None):
        tot = 0.0
        for key, m in (("centers", self.cam_col >= 0), ("points", self.pt_col >= 0), ("scales", self.s_col >= 0)):
            a = x[key][m] if y is None else x[key][m] - y[key][m]
            tot += float((a * a).sum())
        if (self.u_col >= 0).any():
            m = self.u_col >= 0
            a = x["rig_centers"][m] if y is None else x["rig_centers"][m] - y["rig_centers"][m]
            tot += float((a * a).sum())
        return np.sqrt(tot)

    def evaluate(self, x, want_jac):
        d = x["points"][self.obs_pt] - x["centers"][self.obs_cam]
        if self.obs_off is not None:
            d = d + self.obs_off
        if self.ru is not None:       # - R_rw^T u_sensor
            os_ = self.ru["obs_sensor"]
            mu = os_ >= 0
            d = d.copy()
            d[mu] -= np.einsum("nji,nj->ni", self.ru["R_rw"][mu], x["rig_centers"][os_[mu]])
        s = x["scales"]
        res = self.obs_dir - s[:, None] * d
        sq = (res * res).sum(1)
        rho0, rho1 = huber_rho(sq, self.opts.thres_loss_function)
        rho0, rho1 = rho0 * self.loss_scale, rho1 * self.loss_scale
        cost = 0.5 * float(rho0.sum())
        w = np.sqrt(rho1)
        r = (res * w[:, None]).ravel()
        if not want_jac:
            return cost, r, None
        rows, cols, vals = [], [], []
        row0 = 3 * np.arange(self.N)
        cc = self.cam_col[self.obs_cam]
        m = cc >= 0
        for k in range(3):     # dr/dc = +s I
            rows.append(row0[m] + k); cols.append(cc[m] + k); vals.append((w * s)[m])
        pc = self.pt_col[self.obs_pt]
        m = pc >= 0
        for k in range(3):     # dr/dX = -s I
            rows.append(row0[m] + k); cols.append(pc[m] + k); vals.append(-(w * s)[m])
        m = self.s_col >= 0
        for k in range(3):     # dr/ds = -(X - c)
            rows.append(row0[m] + k); cols.append(self.s_col[m]); vals.append(-(w * d[:, k])[m])
        if self.ru is not None and (self.u_col >= 0).any():     # dr/du = + s R_rw^T
            os_ = self.ru["obs_sensor"]
            uc = np.where(os_ >= 0, self.u_col[np.maximum(os_, 0)], -1)
            m = uc >= 0
            for k in range(3):
                for j in range(3):
                    rows.append(row0[m] + k); cols.append(uc[m] + j); vals.append((w * s)[m] * self.ru["R_rw"][m][:, j, k])
        J = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(3 * self.N, self.ncols))
        return cost, r, J


def solve_gp(centers, points, pt_obs_begin, obs_cam, obs_dir, cam_calibrated=None, opts: GPOptions | None = None,
             scales=None, verbose=False, obs_offset=None, rig_unknown=None):
    """Oracle counterpart of the ceres::Solve inside GlobalPositioner::Solve
    (global_positioning.cc:83) on already-initialised centres/points.
    Returns (state dict with centers, points, scales (valid observations only), LMSummary)."""
    opts = opts or GPOptions()
    prob = GPProblem(centers, points, pt_obs_begin, obs_cam, obs_dir, cam_calibrated, opts, scales, obs_offset, rig_unknown)
    if prob.N == 0 or prob.ncols == 0:
        return prob.x0, LMSummary(termination="empty problem")
    lm = LMOptions(max_num_iterations=opts.max_num_iterations, function_tolerance=opts.function_tolerance, verbose=verbose)
    has_bounds = opts.optimize_scales
    x, summ = solve_lm(prob.x0, prob.evaluate, prob.plus, lm, project=prob.project if has_bounds else None,
                       x_norm_fn=prob.x_norm)
    x["keep"] = prob.keep
    return x, summ


def world_bearings(quat, bearings_cam, obs_cam):
    """t_obs = R_cw^T * bearing (global_positioning.cc:294-296)."""
    from .ba_oracle import quat_rotmat
    R = quat_rotmat(np.asarray(quat, dtype=np.float64))[np.asarray(obs_cam)]
    return np.einsum("nji,nj->ni", R, bearings_cam)
