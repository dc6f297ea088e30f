"""ORACLE (test infrastructure, NOT product code) -- high-precision (mpmath, 50 digits) restatements of the small
numerical routines under the gravity refiner (glomap_b200/csrc/gravity_kernels.cuh) and the rig rotation averages
(rig_init_kernels.cuh, ra_kernels.cuh quat_avg_eig):

  * SphereManifold<3>: the Householder vector, Plus and PlusJacobian (oracle/gravity_oracle.py states the formulas)
  * symmetric 3x3 / 4x4 eigenvectors (mpmath.eigsy), AverageGravity's start with its sign rule
  * CalcAngle(R, AngleToRotUp(RotUpToAngle(R))) of the error test
  * the per-frame LM of oracle/gravity_oracle.solve_sphere_lm, restated step by step as the device runs it (the closed
    form 2x2 system) with every quantity in mpmath, and the trust-region bookkeeping (radius, decrease factor) in IEEE
    double from the rounded step quality, as the device keeps it; it returns the per-iteration trace of the device probe
  * the rig samples q_i conj(q_ref) and their average (colmap::AverageQuaternions, unit weights, canonical w >= 0)

Inputs are doubles; every helper returns mpmath numbers or lists of them unless stated."""
from __future__ import annotations

import math

import mpmath as mp
import numpy as np

DPS = 50
DBL_EPSILON = float(np.finfo(np.float64).eps)
DBL_MIN = float(np.finfo(np.float64).tiny)


def _v(x):
    return [mp.mpf(float(t)) if not isinstance(t, mp.mpf) else t for t in x]


# ---- SphereManifold<3> -----------------------------------------------------------------------------------------------
def householder(x):
    """(v [3], beta, branch): (I - beta v v^T) x = |x| e_3.  branch 0: sigma <= DBL_EPSILON (decided on the exact sigma
    of the double x), 1: x_3 <= 0, 2: x_3 > 0."""
    with mp.workdps(DPS):
        x = _v(x)
        sigma = x[0] ** 2 + x[1] ** 2
        v = [x[0], x[1], mp.mpf(1)]
        if sigma <= DBL_EPSILON:
            return v, (mp.mpf(2) if x[2] < 0 else mp.mpf(0)), 0
        mu = mp.sqrt(x[2] ** 2 + sigma)
        vp = x[2] - mu if x[2] <= 0 else -sigma / (x[2] + mu)
        beta = 2 * vp * vp / (sigma + vp * vp)
        return [v[0] / vp, v[1] / vp, v[2]], beta, (1 if x[2] <= 0 else 2)


def sphere_plus(x, d):
    """x [+] d.  |d| == 0 returns x; as in Ceres (Eigen's norm(), an unscaled sqrt of the squared norm) that test is
    made on the double |d|^2, so a step whose square underflows (|d| below ~1e-162) also returns x."""
    with mp.workdps(DPS):
        if all(isinstance(t, float) for t in d) and d[0] * d[0] + d[1] * d[1] == 0.0:
            return _v(x)
        x, d = _v(x), _v(d)
        nd = mp.sqrt(d[0] ** 2 + d[1] ** 2)
        if nd == 0:
            return list(x)
        v, beta, _ = householder(x)
        nx = mp.sqrt(sum(t * t for t in x))
        h = nd / 2
        sbd = mp.sin(h) / h
        y = [sbd * d[0] / 2, sbd * d[1] / 2, mp.cos(h)]
        vy = beta * sum(a * b for a, b in zip(v, y))
        return [nx * (y[k] - v[k] * vy) for k in range(3)]


def sphere_plus_jacobian(x):
    """[3][2] row-major as a flat list of 6."""
    with mp.workdps(DPS):
        v, beta, _ = householder(x)
        nx = mp.sqrt(sum(t * t for t in _v(x)))
        return [nx / 2 * ((1 if r == c else 0) - beta * v[r] * v[c]) for r in range(3) for c in range(2)]


def sphere_plus_jacobian_fd(x, h=mp.mpf("1e-25")):
    """Central differences of sphere_plus at d = 0 (in mpmath: truncation O(h^2), rounding 10^-DPS / h)."""
    with mp.workdps(DPS):
        cols = []
        for c in range(2):
            d = [mp.mpf(0), mp.mpf(0)]
            d[c] = h
            p = sphere_plus(x, d)
            d[c] = -h
            m = sphere_plus(x, d)
            cols.append([(a - b) / (2 * h) for a, b in zip(p, m)])
        return [cols[c][r] for r in range(3) for c in range(2)]


# ---- symmetric eigenvectors --------------------------------------------------------------------------------------------
def eig_sym(A):
    """(eigenvalues ascending [n], eigenvectors as columns [n][n]) of the symmetric double matrix A (n x n, any nesting)."""
    A = np.asarray(A, dtype=np.float64)
    with mp.workdps(DPS):
        E, Q = mp.eigsy(mp.matrix(A.tolist()))
        n = A.shape[0]
        order = sorted(range(n), key=lambda i: E[i])
        return [E[i] for i in order], [[Q[r, i] for i in order] for r in range(n)]


def dominant(A):
    """(unit eigenvector of the largest eigenvalue, relative gap (l1 - l2) / |l1|) of the symmetric double A."""
    E, Q = eig_sym(A)
    n = len(E)
    with mp.workdps(DPS):
        v = [Q[r][n - 1] for r in range(n)]
        gap = (E[n - 1] - E[n - 2]) / abs(E[n - 1]) if E[n - 1] != 0 else mp.mpf(0)
        return v, gap


def angle_to(a, b):
    """Angle in radians between the lines of a and b (sign-invariant), accurate near 0, as a float."""
    with mp.workdps(DPS):
        a, b = _v(a), _v(b)
        na = mp.sqrt(sum(t * t for t in a))
        nb = mp.sqrt(sum(t * t for t in b))
        d = abs(sum(x * y for x, y in zip(a, b))) / (na * nb)
        s = mp.sqrt(max(mp.mpf(0), sum((x / na - y / nb) ** 2 for x, y in zip(a, b)) * sum((x / na + y / nb) ** 2 for x, y in zip(a, b)))) / 2
        return float(mp.atan2(s, d))


def average_gravity(gs, prior):
    """AverageGravity (math/gravity.cc:37-91) of the double terms gs [n][3] with the sign tie toward ``prior``:
    (x [3], relative eigengap, sign margin = min |g . x| over the terms, as a float)."""
    gs = np.asarray(gs, np.float64)
    with mp.workdps(DPS):
        n = len(gs)
        A = [[mp.fsum(mp.mpf(float(g[i])) * mp.mpf(float(g[j])) for g in gs) / n for j in range(3)] for i in range(3)]
        E, Q = mp.eigsy(mp.matrix(A))
        order = sorted(range(3), key=lambda i: E[i])
        x = [Q[r, order[2]] for r in range(3)]
        gap = (E[order[2]] - E[order[1]]) / abs(E[order[2]])
        dots = [mp.fsum(mp.mpf(float(g[k])) * x[k] for k in range(3)) for g in gs]
        neg = sum(1 for d in dots if d < 0)
        pr = mp.fsum(mp.mpf(float(prior[k])) * x[k] for k in range(3))
        if neg > n // 2 or (2 * neg == n and pr < 0):
            x = [-t for t in x]
        margin = float(min(abs(d) for d in dots))
        if 2 * neg == n:
            margin = min(margin, float(abs(pr)))
        return x, gap, margin


# ---- the error test ----------------------------------------------------------------------------------------------------
def _R_to_quat(R):
    """Unit quaternion (x, y, z, w), w >= 0, of the rotation matrix R (mpmath, Shepperd's branches)."""
    t = R[0][0] + R[1][1] + R[2][2]
    if t > 0:
        s = mp.sqrt(t + 1) * 2
        q = [(R[2][1] - R[1][2]) / s, (R[0][2] - R[2][0]) / s, (R[1][0] - R[0][1]) / s, s / 4]
    else:
        i = max(range(3), key=lambda k: R[k][k])
        j, k = (i + 1) % 3, (i + 2) % 3
        s = mp.sqrt(R[i][i] - R[j][j] - R[k][k] + 1) * 2
        q = [0, 0, 0, (R[k][j] - R[j][k]) / s]
        q[i] = s / 4
        q[j] = (R[j][i] + R[i][j]) / s
        q[k] = (R[k][i] + R[i][k]) / s
    n = mp.sqrt(sum(c * c for c in q))
    q = [c / n for c in q]
    return [-c for c in q] if q[3] < 0 else q


def pair_angle(R):
    """(RotUpToAngle(R), CalcAngle(R, AngleToRotUp(RotUpToAngle(R))) in degrees) of the double R [3][3], through R's
    quaternion in mpmath (R is a rotation to rounding; the angle is exact to about eps / sin(angle))."""
    R = np.asarray(R, np.float64).reshape(3, 3)
    with mp.workdps(DPS):
        q = _R_to_quat([[mp.mpf(float(R[i, j])) for j in range(3)] for i in range(3)])
        nv = mp.sqrt(q[0] ** 2 + q[1] ** 2 + q[2] ** 2)
        theta = 2 * mp.atan2(nv, q[3])
        up = theta * q[1] / nv if nv > 0 else mp.mpf(0)
        # angle between the rotation q and the rotation about y by up: 2 atan2(|v|, |w|) of q_up^-1 q
        c, s = mp.cos(up / 2), mp.sin(up / 2)
        # conj(q_up) q with q_up = (0, s, 0, c)
        x = c * q[0] - s * q[2]
        y = c * q[1] - s * q[3]
        z = c * q[2] + s * q[0]
        w = c * q[3] + s * q[1]
        ang = 2 * mp.atan2(mp.sqrt(x * x + y * y + z * z), abs(w))
        return up, ang * 180 / mp.pi


# ---- the per-frame LM --------------------------------------------------------------------------------------------------
TERM = {-1: "too few terms", 0: "gradient tolerance at x0", 1: "max iterations", 2: "min radius", 3: "too many invalid steps",
        4: "parameter tolerance", 5: "function tolerance", 6: "gradient tolerance"}


def _eval_mp(gs, x, a):
    cost, w, rs = [], [], [[], [], []]
    for g in gs:
        d = [x[k] - mp.mpf(float(g[k])) for k in range(3)]
        s = d[0] ** 2 + d[1] ** 2 + d[2] ** 2
        cost.append(a * mp.atan2(s, a))
        rho1 = 1 / (1 + s * s / (a * a))
        w.append(rho1)
        for k in range(3):
            rs[k].append(rho1 * d[k])
    return mp.fsum(cost) / 2, mp.fsum(w), [mp.fsum(r) for r in rs]


def _eval_fp64(gs, x, a):
    """The same sums in IEEE double with exactly rounded accumulation (math.fsum): for frames too large for mpmath."""
    xf = np.array([float(t) for t in x])
    a = float(a)
    d = xf[None, :] - gs
    s = (d * d).sum(1)
    c = a * np.arctan2(s, a)
    rho1 = np.maximum(DBL_MIN, 1.0 / (1.0 + s * s / (a * a)))
    return (mp.mpf(math.fsum(c)) / 2, mp.mpf(math.fsum(rho1)), [mp.mpf(math.fsum(rho1 * d[:, k])) for k in range(3)])


def lm_trace(gs, x0, opts, fp64=False, near_rel=1e4 * DBL_EPSILON):
    """The LM of grv_refine from the double start x0 over the terms gs [n][3] (skipped terms removed).  opts has the
    fields of GravityOptions.  Returns dict(x [3] floats, term, iterations, trace [it][5] floats as the device records
    them, near = list of (iteration, decision) whose margin to its bound is within rounding: the trace after the first
    one is not a comparison)."""
    gs = np.asarray(gs, np.float64)
    ev = _eval_fp64 if fp64 else _eval_mp
    with mp.workdps(DPS):
        # ArctanLoss's parameter is the double 1 - cos(max_gravity_error) the solver forms (the cancellation there costs
        # ~1e-12 relative, more than the comparison allows): the loss is evaluated exactly at that parameter
        a = mp.mpf(1.0 - math.cos(opts.max_gravity_error * math.pi / 180.0))
        x = _v(x0)
        cost, wsum, rs = ev(gs, x, a)

        def jac(x):
            P = sphere_plus_jacobian(x)
            return P, [P[0] ** 2 + P[2] ** 2 + P[4] ** 2, P[0] * P[1] + P[2] * P[3] + P[4] * P[5], P[1] ** 2 + P[3] ** 2 + P[5] ** 2]

        def grad(P, rs):
            return [P[0] * rs[0] + P[2] * rs[1] + P[4] * rs[2], P[1] * rs[0] + P[3] * rs[1] + P[5] * rs[2]]

        def gmax(x, g):
            p = sphere_plus(x, [-g[0], -g[1]])
            return max(abs(p[k] - x[k]) for k in range(3))

        def norm(x):
            return mp.sqrt(sum(t * t for t in x))

        P, PtP = jac(x)
        sc0, sc1 = 1 / (1 + mp.sqrt(wsum * PtP[0])), 1 / (1 + mp.sqrt(wsum * PtP[2]))
        g = grad(P, rs)
        radius, decrease = 1e4, 2.0
        invalid, it, trace, near = 0, 0, [], []
        x_norm = norm(x)
        gtol, ptol, ftol = opts.gradient_tolerance, opts.parameter_tolerance, opts.function_tolerance

        def check_near(it, what, val, bound, scale):
            if abs(val - bound) <= near_rel * scale:
                near.append((it, what))

        gm = gmax(x, g)
        check_near(0, "gradient", gm, gtol, x_norm)
        term = 0
        if gm > gtol:
            while True:
                if it >= opts.max_num_iterations:
                    term = 1
                    break
                if not radius >= 1e-32:
                    term = 2
                    break
                it += 1
                H00, H01, H11 = wsum * PtP[0] * sc0 * sc0, wsum * PtP[1] * sc0 * sc1, wsum * PtP[2] * sc1 * sc1
                D0 = min(max(H00, mp.mpf(1e-6)), mp.mpf(1e32)) / radius
                D1 = min(max(H11, mp.mpf(1e-6)), mp.mpf(1e32)) / radius
                a00, a11 = H00 + D0, H11 + D1
                q0, q1 = -sc0 * g[0], -sc1 * g[1]
                det = a00 * a11 - H01 * H01
                y0, y1 = (a11 * q0 - H01 * q1) / det, (a00 * q1 - H01 * q0) / det
                mcc = (y0 * q0 + y1 * q1) - (y0 * (H00 * y0 + H01 * y1) + y1 * (H01 * y0 + H11 * y1)) / 2
                if mcc <= 0:
                    trace.append([float(cost), radius, float(mcc), math.nan, -1])
                    invalid += 1
                    if invalid >= 5:
                        term = 3
                        break
                    radius /= decrease
                    decrease *= 2.0
                    continue
                invalid = 0
                xc = sphere_plus(x, [y0 * sc0, y1 * sc1])
                ccost, cw, crs = ev(gs, xc, a)
                sn = norm([xc[k] - x[k] for k in range(3)])
                bound = ptol * (x_norm + ptol)
                check_near(it, "parameter", sn, bound, x_norm)
                if sn <= bound:
                    trace.append([float(cost), radius, float(mcc), float(ccost), 2])
                    term = 4
                    break
                change = cost - ccost
                check_near(it, "function", abs(change), ftol * cost, cost)
                if abs(change) <= ftol * cost:
                    trace.append([float(cost), radius, float(mcc), float(ccost), 3])
                    term = 5
                    break
                check_near(it, "step quality", change, mp.mpf(1e-3) * mcc, cost)
                rel = change / mcc
                ok = rel > mp.mpf(1e-3)
                trace.append([float(cost), radius, float(mcc), float(ccost), 1 if ok else 0])
                if ok:
                    x, cost, wsum, rs = xc, ccost, cw, crs
                    P, PtP = jac(x)
                    g = grad(P, rs)
                    x_norm = norm(x)
                    t = 2.0 * float(rel) - 1.0
                    radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - t * t * t))
                    decrease = 2.0
                    gm = gmax(x, g)
                    check_near(it, "gradient", gm, gtol, x_norm)
                    if gm <= gtol:
                        term = 6
                        break
                else:
                    radius /= decrease
                    decrease *= 2.0
        return dict(x=[float(t) for t in x], term=term, iterations=it, trace=trace, near=near)


# ---- rig rotation averages ---------------------------------------------------------------------------------------------
def qunit(q):
    with mp.workdps(DPS):
        q = _v(q)
        n = mp.sqrt(sum(t * t for t in q))
        return [t / n for t in q]


def qmul(a, b):
    """Eigen's quaternion product, xyzw."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return [aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
            aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz]


def cam_sample(q_i, q_ref):
    """q_i conj(q_ref) over the normalised inputs, normalised (rig_cam_samples)."""
    with mp.workdps(DPS):
        qi, qr = qunit(q_i), qunit(q_ref)
        return qunit(qmul(qi, [-qr[0], -qr[1], -qr[2], qr[3]]))


def average_quaternions(qs):
    """(average [4], relative gap (l1 - l2) / l1 of sum q q^T) with unit weights over the normalised samples; a single
    sample as it is; canonical sign w >= 0 (w < 0 flips)."""
    with mp.workdps(DPS):
        qs = [qunit(q) for q in qs]
        if len(qs) == 1:
            v, gap = qs[0], mp.mpf(1)
        else:
            M = mp.matrix(4, 4)
            for i in range(4):
                for j in range(4):
                    M[i, j] = mp.fsum(q[i] * q[j] for q in qs)
            E, Q = mp.eigsy(M)
            order = sorted(range(4), key=lambda i: E[i])
            v = [Q[r, order[3]] for r in range(4)]
            gap = (E[order[3]] - E[order[2]]) / E[order[3]]
        if v[3] < 0:
            v = [-t for t in v]
        return v, gap
