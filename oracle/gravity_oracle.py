"""ORACLE (test infrastructure, NOT product code) -- numpy restatement of GravityRefiner::RefineGravity
(glomap/estimators/gravity_refinement.cc:9-181) in frame space, under the rules of include/b200sfm.h:
  (i)   every error-prone frame is refined against the gravities as they were on entry (Jacobi)
  (ii)  a sign tie of AverageGravity goes toward the frame's prior
  (iii) R_align is the caller's (the error test depends on its completion)

Ceres pieces restated from the public Ceres 2.x sources and flagged UPSTREAM-UNVERIFIED:
  * SphereManifold<3> (sphere_manifold.h, internal/sphere_manifold_functions.h): Householder vector v, beta of x
    with (I - beta v v^T) x = |x| e_3 (sigma <= DBL_EPSILON: beta = 2 if x_3 < 0 else 0);
    Plus(x, d) = |x| H (0.5 sin(|d|/2) / (|d|/2) d, cos(|d|/2)), PlusJacobian = 0.5 |x| H[:, :2]
  * ArctanLoss(a) (loss_function.cc): rho(s) = a atan2(s, a), rho'(s) = max(DBL_MIN, 1 / (1 + s^2 / a^2)),
    rho'' <= 0 so the corrector scales residual and Jacobian by sqrt(rho')
The LM is ceres_lm.solve_lm (no line search; the gradient norm is the manifold one, max |x [+] -g - x|)."""
from __future__ import annotations

import dataclasses

import numpy as np
import scipy.sparse as sp
from scipy.spatial.transform import Rotation

from oracle import ceres_lm

EPS = 1e-12   # glomap/types.h


@dataclasses.dataclass
class GravityOptions:
    max_outlier_ratio: float = 0.5
    max_gravity_error: float = 1.0
    min_num_neighbors: int = 7
    max_num_iterations: int = 100
    function_tolerance: float = 1e-5
    gradient_tolerance: float = 1e-10
    parameter_tolerance: float = 1e-8


def householder(x):
    sigma = float(x[0] * x[0] + x[1] * x[1])
    v = np.array([x[0], x[1], 1.0])
    if sigma <= np.finfo(np.float64).eps:
        return v, (2.0 if x[2] < 0 else 0.0)
    mu = np.sqrt(x[2] * x[2] + sigma)
    vp = x[2] - mu if x[2] <= 0 else -sigma / (x[2] + mu)
    beta = 2 * vp * vp / (sigma + vp * vp)
    v[:2] /= vp
    return v, beta


def sphere_plus(x, d):
    nd = float(np.linalg.norm(d))
    if nd == 0.0:
        return np.array(x, dtype=np.float64)
    v, beta = householder(x)
    h = 0.5 * nd
    y = np.array([0.5 * np.sin(h) / h * d[0], 0.5 * np.sin(h) / h * d[1], np.cos(h)])
    return np.linalg.norm(x) * (y - v * (beta * (v @ y)))


def sphere_plus_jacobian(x):
    v, beta = householder(x)
    return 0.5 * np.linalg.norm(x) * (np.eye(3) - beta * np.outer(v, v))[:, :2]


def arctan_rho(s, a):
    return a * np.arctan2(s, a), np.maximum(np.finfo(np.float64).tiny, 1.0 / (1.0 + s * s / (a * a)))


def rot_up_angle(R):
    """RotUpToAngle (math/gravity.cc:26-28): the y component of the rotation vector."""
    return Rotation.from_matrix(R).as_rotvec()[..., 1]


def angle_to_rot_up(t):
    """AngleToRotUp (math/gravity.cc:30-33) through AngleAxisToRotation's first-order branch below EPS."""
    t = np.asarray(t, dtype=np.float64)
    c, s = np.cos(t), np.sin(t)
    small = np.abs(t) <= EPS
    c = np.where(small, 1.0, c)
    R = np.zeros(t.shape + (3, 3))
    R[..., 0, 0] = c; R[..., 0, 2] = s; R[..., 1, 1] = 1; R[..., 2, 0] = -s; R[..., 2, 2] = c
    return R


def pair_angles(R_align, f1, f2, M):
    """CalcAngle(R, AngleToRotUp(RotUpToAngle(R))) in degrees for R = Ra2^T M Ra1 (.cc:150-158)."""
    R = np.swapaxes(R_align[f2], -1, -2) @ M @ R_align[f1]
    Rup = angle_to_rot_up(rot_up_angle(R))
    c = np.clip((np.einsum("nij,nij->n", R, Rup) - 1) / 2, -1, 1)
    return np.degrees(np.arccos(c))


def average_gravity(gs, prior):
    """AverageGravity (math/gravity.cc:37-91) with the sign tie toward ``prior``."""
    A = (gs[:, :, None] * gs[:, None, :]).sum(0) / len(gs)
    w, V = np.linalg.eigh(A)
    x = V[:, int(np.argmax(w))].copy()
    neg = int((gs @ x < 0).sum())
    if neg > len(gs) // 2 or (2 * neg == len(gs) and x @ prior < 0):
        x = -x
    return x


def solve_sphere_lm(gs, x0, opts: GravityOptions):
    """The Ceres problem of .cc:54-109: one GravError block per observation under ArctanLoss on SphereManifold<3>."""
    a = 1.0 - np.cos(np.radians(opts.max_gravity_error))
    n = len(gs)

    def evaluate(x, want_j):
        r = x[None, :] - gs
        s = (r * r).sum(1)
        rho, rho1 = arctan_rho(s, a)
        cost = 0.5 * float(rho.sum())
        sq = np.sqrt(rho1)
        rc = (r * sq[:, None]).ravel()
        J = None
        if want_j:
            P = sphere_plus_jacobian(x)
            J = sp.csr_matrix((sq[:, None, None] * P[None]).reshape(3 * n, 2))
        return cost, rc, J

    lm = ceres_lm.LMOptions(max_num_iterations=opts.max_num_iterations, function_tolerance=opts.function_tolerance,
                            gradient_tolerance=opts.gradient_tolerance, parameter_tolerance=opts.parameter_tolerance,
                            max_num_line_search_step_size_iterations=0)
    x_norm = lambda x, prev=None: float(np.linalg.norm(x if prev is None else x - prev))   # noqa: E731
    return ceres_lm.solve_lm(x0, evaluate, sphere_plus, lm, project=lambda x, d: sphere_plus(x, d) - x, x_norm_fn=x_norm)


def refine_gravity(R_align, has_gravity, frame1, frame2, M, opts: GravityOptions | None = None) -> dict:
    """Frame-space inputs as b200sfm_gravity_refine takes them.  Returns dict(status [F] uint8, gravity [F,3] (NaN where
    status != 2), iterations {frame: LM iterations}, error_prone [sorted frames], mistakes [F], total [F], margin = the
    smallest distance in degrees of a pair angle from max_gravity_error or of a refined frame's term from its bound)."""
    opts = opts or GravityOptions()
    R_align = np.asarray(R_align, dtype=np.float64).reshape(-1, 3, 3)
    F = len(R_align)
    has = np.asarray(has_gravity, bool)
    f1, f2 = np.asarray(frame1, np.int64), np.asarray(frame2, np.int64)
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3, 3)
    keep = has[f1] & has[f2]
    f1, f2, M = f1[keep], f2[keep], M[keep]
    ang = pair_angles(R_align, f1, f2, M) if len(f1) else np.zeros(0)
    mis = ang > opts.max_gravity_error
    total = np.bincount(f1, minlength=F) + np.bincount(f2, minlength=F)
    mistakes = np.bincount(f1, weights=mis, minlength=F).astype(np.int64) + np.bincount(f2, weights=mis, minlength=F).astype(np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        ep = (total >= opts.min_num_neighbors) & (mistakes / total >= opts.max_outlier_ratio)
    g = R_align[:, :, 1]
    status = np.zeros(F, np.uint8)
    out = np.full((F, 3), np.nan)
    iters = {}
    margin = float(np.abs(ang - opts.max_gravity_error).min()) if len(ang) else np.inf
    for f in np.nonzero(ep)[0]:
        terms = []
        for e in range(len(f1)):                    # incidence order 2 e + side
            if f1[e] == f:
                terms.append(M[e].T @ g[f2[e]])
            elif f2[e] == f:
                terms.append(M[e] @ g[f1[e]])
        if len(terms) < opts.min_num_neighbors:
            status[f] = 1
            continue
        gs = np.array(terms)
        x0 = average_gravity(gs, g[f])
        x, summ = solve_sphere_lm(gs, x0, opts)
        iters[int(f)] = summ.iterations
        err = np.degrees(np.arccos(np.clip(gs @ x, -1, 1)))
        outl = int((err > 2 * opts.max_gravity_error).sum())
        margin = min(margin, float(np.abs(err - 2 * opts.max_gravity_error).min()))
        if outl / len(gs) < opts.max_outlier_ratio:
            status[f] = 2
            out[f] = x
        else:
            status[f] = 3
    return dict(status=status, gravity=out, iterations=iters, error_prone=np.nonzero(ep)[0], mistakes=mistakes, total=total,
                margin=margin)
