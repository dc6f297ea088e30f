"""The gravity refiner stage by stage (b200sfm_test_gravity, b200sfm_test_device_helpers) against the high-precision
restatements of oracle/gravity_mp.py: the per-pair error test at its bound, the incidence CSR and the counts, the observed
gravities, AverageGravity's start and sign rule, the sphere-manifold helpers and the LM trace, iteration by iteration."""
import ctypes as ct
import math
import os

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E_, geometry as geo
from glomap_b200.gravity_refinement import GravityRefinerOptions, get_align_rot_householder
from oracle import gravity_mp as GM
from test_gravity_refinement_cpu import frame_inputs, make_scene

pytestmark = pytest.mark.gpu
EPS = float(np.finfo(np.float64).eps)
HERE = os.path.dirname(os.path.abspath(__file__))
OUT_W = [4, 3, 6, 3, 4, 2]


def ptr(a):
    return a.ctypes.data_as(ct.c_void_p)


def helpers(op, rows):
    """b200sfm_test_device_helpers over the rows (one input per row)."""
    rows = np.ascontiguousarray(np.atleast_2d(rows), np.float64)
    out = np.full((len(rows), OUT_W[op]), np.nan)
    ctx = E_.default_context()
    _lib.check(ctx.handle, ctx.lib.b200sfm_test_device_helpers(ctx.handle, op, len(rows), ptr(rows), ptr(out)))
    return out


def probe(R_align, has, f1, f2, M, opts=None, cap=128):
    """Every stage's output of b200sfm_test_gravity; rows of the per-k arrays are trimmed to the error-prone frames."""
    R_align = np.ascontiguousarray(np.asarray(R_align, np.float64).reshape(-1, 9))
    F, E = len(R_align), len(f1)
    a = dict(mistake=np.zeros(E, np.uint8), angle=np.full(E, np.nan), offs=np.zeros(F + 1, np.int32),
             inc=np.zeros(2 * E, np.int32), total=np.zeros(F, np.int32), mistakes=np.zeros(F, np.int32),
             error_prone=np.zeros(F, np.uint8), ep=np.zeros(F, np.int32), gobs=np.zeros((2 * E, 3)), x=np.zeros((F, 3)),
             status=np.zeros(F, np.uint8), iterations=np.zeros(F, np.int32), trace=np.zeros((F, 5 + 5 * cap)))
    out = _lib.GravityProbeOut(**{k: ptr(v) for k, v in a.items()}, trace_cap=cap)
    ctx = E_.default_context()
    o = (opts or GravityRefinerOptions()).to_c()
    _lib.check(ctx.handle, ctx.lib.b200sfm_test_gravity(
        ctx.handle, ct.byref(o), F, ptr(R_align), ptr(np.ascontiguousarray(has, np.uint8)), E,
        ptr(np.ascontiguousarray(f1, np.int32)), ptr(np.ascontiguousarray(f2, np.int32)),
        ptr(np.ascontiguousarray(np.asarray(M, np.float64).reshape(-1, 9))), ct.byref(out)))
    k = out.n_error_prone
    for f in ("ep", "x", "status", "iterations", "trace"):
        a[f] = a[f][:k]
    a["n_error_prone"] = k
    return a


def production(R_align, has, f1, f2, M, opts=None):
    """b200sfm_gravity_refine with every output (the frames' gravity is written only for error-prone frames)."""
    F = len(has)
    ctx = E_.default_context()
    g = np.full((F, 3), 7.0)
    st = np.full(F, 9, np.uint8)
    s = _lib.GravityStats()
    _lib.check(ctx.handle, ctx.lib.b200sfm_gravity_refine(
        ctx.handle, ct.byref((opts or GravityRefinerOptions()).to_c()), F,
        ptr(np.ascontiguousarray(np.asarray(R_align, np.float64).reshape(-1, 9))), ptr(np.ascontiguousarray(has, np.uint8)),
        len(f1), ptr(np.ascontiguousarray(f1, np.int32)), ptr(np.ascontiguousarray(f2, np.int32)),
        ptr(np.ascontiguousarray(np.asarray(M, np.float64).reshape(-1, 9))), ptr(g), ptr(st), ct.byref(s)))
    return g, st, s


def terms_of(p, k):
    """The error-prone frame k's terms in incidence order (skipped rows removed) and its incidence ids."""
    f = p["ep"][k]
    rows = np.arange(p["offs"][f], p["offs"][f + 1])
    g = p["gobs"][rows]
    keep = ~np.isnan(g[:, 0])
    return g[keep], p["inc"][rows]


def near_bound(values, bound, tol):
    """Indices of the decisions `value > bound` that lie within `tol` of the bound: rounding could flip them, so they are
    reported instead of compared."""
    return np.nonzero(np.abs(np.asarray(values, np.float64) - bound) <= tol)[0]


def rot(axis, deg):
    w = np.zeros(3)
    w[axis] = math.radians(deg)
    return geo.so3_exp(w[None])[0]


def exact_angles(R_align, f1, f2, M):
    R_align = np.asarray(R_align, np.float64).reshape(-1, 3, 3)
    R = np.swapaxes(R_align[f2], -1, -2) @ np.asarray(M).reshape(-1, 3, 3) @ R_align[f1]
    return np.array([float(GM.pair_angle(r)[1]) for r in R])


def angle_tol_deg(a_deg):
    """CalcAngle's rounding through acos: about eps / sin(angle) radians."""
    s = np.maximum(np.sin(np.radians(a_deg)), np.sqrt(EPS))
    return np.degrees(16 * EPS / s) + 1e-13


# ---- 1. the error test ------------------------------------------------------------------------------------------------
def star(angles, F=None, seed=0, self_pairs=0, frames=None):
    """Frame 0 paired with frames 1..n: pair e has R = Ra2^T M Ra1 = Rx(angle_e) (or Rz), random R_align."""
    rng = np.random.default_rng(seed)
    n = len(angles)
    F = F or n + 1
    Ra = get_align_rot_householder(rng.normal(size=(F, 3)))
    f1 = np.zeros(n, np.int32) if frames is None else np.asarray(frames[0], np.int32)
    f2 = np.arange(1, n + 1, dtype=np.int32) if frames is None else np.asarray(frames[1], np.int32)
    Q = np.array([rot(0 if e % 2 else 2, a) for e, a in enumerate(angles)])
    M = Ra[f2] @ Q @ np.swapaxes(Ra[f1], -1, -2)
    return Ra, np.ones(F, np.uint8), f1, f2, M


def test_mistake_flags_at_the_bound():
    bound = 1.0
    angles = np.array([bound + d for d in (1e-6, -1e-6, 1e-5, -1e-5)] + [0.0, 0.3, 2.0, 179.0, 90.0])
    Ra, has, f1, f2, M = star(angles)
    p = probe(Ra, has, f1, f2, M)
    ex = exact_angles(Ra, f1, f2, M)
    assert len(near_bound(ex, bound, 1e-9)) == 0
    np.testing.assert_array_equal(p["mistake"], (ex > bound).astype(np.uint8))
    assert (np.abs(p["angle"] - ex) <= angle_tol_deg(ex)).all(), np.abs(p["angle"] - ex).max()


def test_pair_angle_helper_against_mpmath():
    rng = np.random.default_rng(3)
    Rs = list(geo.so3_exp(rng.normal(size=(40, 3)) * rng.uniform(0, 3, size=(40, 1))))
    Rs += [rot(0, 1.0 + 1e-6), rot(2, 1.0 - 1e-6), rot(1, 30.0) @ rot(0, 1.0), rot(0, 179.9), rot(1, 179.999)]
    out = helpers(5, np.array(Rs).reshape(-1, 9))
    ex = np.array([[float(v) for v in GM.pair_angle(R)] for R in Rs])
    assert (np.abs(out[:, 1] - ex[:, 1]) <= angle_tol_deg(ex[:, 1])).all()
    up_ok = np.abs(np.abs(out[:, 0]) - np.abs(ex[:, 0])) <= 1e-12 * np.maximum(1.0, np.abs(ex[:, 0]))
    assert up_ok.all()


def check_counts(p, has, f1, f2, opts):
    F = len(has)
    valid = has[f1].astype(bool) & has[f2].astype(bool)
    mis = p["mistake"].astype(np.int64) * valid
    total = np.bincount(f1[valid], minlength=F) + np.bincount(f2[valid], minlength=F)
    mistakes = np.bincount(f1, weights=mis, minlength=F).astype(np.int64) + np.bincount(f2, weights=mis, minlength=F).astype(np.int64)
    np.testing.assert_array_equal(p["total"], total)
    np.testing.assert_array_equal(p["mistakes"], mistakes)
    with np.errstate(invalid="ignore", divide="ignore"):
        ep = (total >= opts.min_num_neighbors) & (mistakes / total >= opts.max_outlier_ratio)
    np.testing.assert_array_equal(p["error_prone"], ep.astype(np.uint8))
    np.testing.assert_array_equal(p["ep"], np.nonzero(ep)[0])
    # the CSR: each frame's incidences 2 e + side, ascending
    for f in range(F):
        ids = p["inc"][p["offs"][f]:p["offs"][f + 1]]
        want = sorted([2 * e for e in np.nonzero(valid & (f1 == f))[0]] + [2 * e + 1 for e in np.nonzero(valid & (f2 == f))[0]])
        np.testing.assert_array_equal(ids, want)
    return total, mistakes


@pytest.mark.parametrize("min_nb", [0, 7])
def test_counts_on_rigs_without_gravity_and_isolated_frames(min_nb):
    sc = make_scene(F=30, sensors=2, seed=21, pair_prob=0.25, noise_deg=0.3, outlier_ratio=0.3, no_gravity=0.2)
    R_align, has, f1, f2, M = frame_inputs(sc)
    # two frames with gravity and no pair at all
    R_align = np.concatenate([R_align, get_align_rot_householder(np.array([[0.1, 1.0, 0.2], [0.0, -1.0, 0.3]]))])
    has = np.concatenate([has, [True, True]]).astype(np.uint8)
    opts = GravityRefinerOptions(min_num_neighbors=min_nb)
    p = probe(R_align, has, f1, f2, M, opts)
    ex = exact_angles(R_align, f1[has[f1] & has[f2] > 0], f2[has[f1] & has[f2] > 0],
                      M[(has[f1] & has[f2]) > 0])
    assert len(near_bound(ex, opts.max_gravity_error, 1e-9)) == 0
    total, _ = check_counts(p, has, f1, f2, opts)
    assert (f1 == f2).any() and (~has.astype(bool)).any() and (total[-2:] == 0).all()
    assert not p["error_prone"][-2:].any()       # 0 / 0 does not flag a frame, also with min_num_neighbors 0
    # pairs inside a frame count twice (above) and give one term: the second incidence is skipped
    for k, f in enumerate(p["ep"]):
        rows = np.arange(p["offs"][f], p["offs"][f + 1])
        for r in rows:
            e, side = divmod(int(p["inc"][r]), 2)
            g = p["gobs"][r]
            if side == 1 and f1[e] == f2[e]:
                assert np.isnan(g).all()
                continue
            o = R_align.reshape(-1, 3, 3)[f2[e] if side == 0 else f1[e]][:, 1]
            Me = M[e].reshape(3, 3)
            want = Me.T @ o if side == 0 else Me @ o
            assert np.abs(g - want).max() <= 4 * EPS


def test_ratio_exactly_at_the_bound():
    """Frame 0: 5 pairs, 2 mistakes (2 / 5 == 0.4 in double); frame 1..: one pair each."""
    angles = [5.0, 5.0, 0.1, 0.2, 0.3]
    Ra, has, f1, f2, M = star(angles)
    for ratio, flagged in ((0.4, 1), (np.nextafter(0.4, 1.0), 0)):
        opts = GravityRefinerOptions(max_outlier_ratio=ratio, min_num_neighbors=5)
        p = probe(Ra, has, f1, f2, M, opts)
        total, mistakes = check_counts(p, has, f1, f2, opts)
        assert total[0] == 5 and mistakes[0] == 2 and p["error_prone"][0] == flagged


# ---- 2. AverageGravity ------------------------------------------------------------------------------------------------
def sym_with_gap(rng, gap, repeated=False):
    Q = geo.so3_exp(rng.normal(size=(1, 3)))[0]
    l1 = 1.0
    l2 = l1 if repeated else l1 * (1 - gap)
    A = Q @ np.diag([l1, l2, 0.25 * l2]) @ Q.T
    return (A + A.T) / 2


@pytest.mark.parametrize("gap", [1.0, 1e-1, 1e-2, 1e-4, 1e-6, 1e-8])
def test_principal_eigenvector_against_mpmath(gap):
    rng = np.random.default_rng(int(-math.log10(gap)) + 40)
    As = [sym_with_gap(rng, gap) for _ in range(16)]
    out = helpers(3, np.array(As).reshape(-1, 9))
    worst = 0.0
    for A, v in zip(As, out):
        e, g = GM.dominant(A)
        err = GM.angle_to(v, e)
        worst = max(worst, err * float(g) / EPS)
        assert err <= 32 * EPS / float(g), (gap, err, float(g))
    print(f"gap {gap:g}: worst angle {worst:.2f} eps / gap")


def test_principal_eigenvector_of_a_repeated_eigenvalue_is_in_the_subspace():
    rng = np.random.default_rng(7)
    As = [sym_with_gap(rng, 0.0, repeated=True) for _ in range(16)]
    out = helpers(3, np.array(As).reshape(-1, 9))
    for A, v in zip(As, out):
        E, Q = GM.eig_sym(A)
        w = np.array([[float(Q[r][c]) for c in (1, 2)] for r in range(3)])
        resid = v - w @ (w.T @ v)
        assert np.linalg.norm(resid) <= 32 * EPS and abs(np.linalg.norm(v) - 1) <= 8 * EPS


@pytest.mark.parametrize("n,neg,toward", [(8, 4, 1.0), (8, 4, -1.0), (9, 4, 1.0), (9, 5, 1.0), (7, 3, -1.0), (7, 4, 1.0)])
def test_sign_rule_majority_and_tie(n, neg, toward):
    """Frame 0 with n neighbours, `neg` of them with the reversed gravity; the prior leans toward +g or -g."""
    rng = np.random.default_rng(100 + n + neg)
    R = geo.so3_exp(rng.normal(size=(n + 1, 3)))
    g = R[:, :, 1].copy()
    g[1:neg + 1] = -g[1:neg + 1]
    perp = np.cross(g[0], [0.3, 0.5, 0.8])
    g[0] = toward * 0.3 * g[0] + perp / np.linalg.norm(perp)
    Ra = get_align_rot_householder(g)
    f1, f2 = np.zeros(n, np.int32), np.arange(1, n + 1, dtype=np.int32)
    M = R[f2] @ np.swapaxes(R[f1], -1, -2)
    opts = GravityRefinerOptions(min_num_neighbors=5, max_outlier_ratio=0.3)
    p = probe(Ra, np.ones(n + 1, np.uint8), f1, f2, M, opts)
    assert p["ep"][0] == 0
    terms, _ = terms_of(p, 0)
    x0 = p["trace"][0, :3]
    xm, gap, margin = GM.average_gravity(terms, Ra[0][:, 1])
    assert margin > 1e-3
    assert GM.angle_to(x0, xm) <= 32 * EPS / float(gap)
    assert float(np.dot(x0, [float(t) for t in xm])) > 0   # the same sign
    flip = neg > n // 2 or (2 * neg == n and toward < 0)
    assert np.dot(x0, R[0][:, 1]) * (-1 if flip else 1) > 0


# ---- 3. the sphere-manifold helpers -----------------------------------------------------------------------------------
def manifold_points():
    s = 2.0 ** -26                                        # s^2 == DBL_EPSILON exactly
    pts = [[0, 0, 1], [0, 0, -1], [0, 0, 3.0], [s, 0, 1], [0, s, -1], [s * (1 - 2 ** -20), 0, 1],
           [s * (1 + 2 ** -20), 0, 1], [0, s * (1 + 2 ** -20), -1], [s * (1 + 2 ** -20), 0, -1], [s * (1 - 2 ** -20), 0, -1],
           [1e-9, -2e-9, 1], [1e-9, 2e-9, -1], [0.6, -0.48, 0.64], [-0.6, 0.48, -0.64], [1, 0, 0], [0.3, 0.4, 0.0]]
    return np.array(pts, np.float64)


def test_householder_and_plus_jacobian_against_mpmath():
    X = manifold_points()
    H = helpers(0, X)
    P = helpers(2, X)
    for x, h, pj in zip(X, H, P):
        v, beta, branch = GM.householder(x)
        sig = x[0] * x[0] + x[1] * x[1]
        assert (sig <= EPS) == (branch == 0)   # the device decides on the double sigma: no input is within rounding
        nx = np.linalg.norm(x)
        # the reflector's action, not (v, beta) alone: beta v v^T is what Plus and PlusJacobian use
        for r in range(3):
            for c in range(3):
                want = float(beta * v[r] * v[c])
                got = h[3] * h[r] * h[c]
                assert abs(got - want) <= 16 * EPS * max(1.0, abs(want)), (x, r, c, got, want)
        want = [float(t) for t in GM.sphere_plus_jacobian(x)]
        assert np.abs(pj - want).max() <= 16 * EPS * nx, (x, pj, want)


def test_plus_against_mpmath():
    X = manifold_points()
    rng = np.random.default_rng(5)
    rows = []
    for x in X:
        for nd in (1e-300, 1e-200, 1e-20, 1e-8, 1e-3, 0.5, 2.0, np.pi):
            u = rng.normal(size=2)
            rows.append(np.concatenate([x, nd * u / np.linalg.norm(u)]))
        rows.append(np.concatenate([x, [0.0, 0.0]]))
    rows = np.array(rows)
    out = helpers(1, rows)
    for r, o in zip(rows, out):
        want = np.array([float(t) for t in GM.sphere_plus(r[:3], r[3:])])
        assert np.abs(o - want).max() <= 16 * EPS * np.linalg.norm(r[:3]), (r, o, want)


# ---- 4. the LM trace ---------------------------------------------------------------------------------------------------
def compare_frame(p, k, opts, prior, fp64=False):
    terms, _ = terms_of(p, k)
    tr = p["trace"][k]
    x0, term, ln = tr[:3], int(tr[3]), int(tr[4])
    ref = GM.lm_trace(terms, x0, opts, fp64=fp64)
    assert not ref["near"], ref["near"]                  # no decision within rounding of its bound in these scenes
    got = tr[5:5 + 5 * ln].reshape(-1, 5)
    want = np.array(ref["trace"]).reshape(-1, 5)
    assert term == ref["term"] and int(p["iterations"][k]) == ref["iterations"] == len(want) == ln, (term, ref["term"], ln, len(want))
    np.testing.assert_array_equal(got[:, 4], want[:, 4])                         # accept / reject / stop decisions
    for col in (0, 3):                                                           # cost, candidate cost
        ok = np.isnan(want[:, col]) | (np.abs(got[:, col] - want[:, col]) <= 1e-13 * np.abs(want[:, col]))
        assert ok.all(), (col, got[:, col], want[:, col])
    rr = np.abs(got[:, 1] - want[:, 1]) / want[:, 1]
    assert rr.max() <= 1e-12, rr
    mr = np.abs(got[:, 2] - want[:, 2]) / np.maximum(np.abs(want[:, 2]), 1e-300)
    assert mr.max() <= 1e-9, mr
    ang = GM.angle_to(p["x"][k], ref["x"])
    assert ang <= 1e-12, ang
    return dict(cost=float(np.nanmax(np.abs(got[:, [0, 3]] - want[:, [0, 3]]) / np.abs(want[:, [0, 3]]))),
                radius=float(rr.max()), radius_exact=int((got[:, 1] == want[:, 1]).sum()), n=len(want),
                mcc=float(mr.max()), x=ang)


def hub(n, seed, wrong=0.0, noise_deg=0.5, self_pairs=0):
    """Frame 0 (a wrong prior) paired with n other frames whose priors carry noise; `self_pairs` pairs of frame 0 with
    itself (a rig's two cameras), which give one term each."""
    rng = np.random.default_rng(seed)
    R = geo.so3_exp(rng.normal(size=(n + 1, 3)))
    g = R[:, :, 1] + rng.normal(size=(n + 1, 3)) * math.radians(noise_deg)
    g[0] = [1.0, 0.2, 0.1]
    f1 = np.concatenate([np.zeros(n, np.int32), np.zeros(self_pairs, np.int32)])
    f2 = np.concatenate([np.arange(1, n + 1, dtype=np.int32), np.zeros(self_pairs, np.int32)])
    M = R[f2] @ np.swapaxes(R[f1], -1, -2)
    if self_pairs:                                                  # rig_from_rig of a pair inside the frame: ~identity
        M[n:] = geo.so3_exp(rng.normal(size=(self_pairs, 3)) * 0.01)
    Ra = get_align_rot_householder(g)
    return Ra, np.ones(n + 1, np.uint8), f1, f2, M


LM_CASES = [("warp", 20, 0), ("33", 33, 0), ("rig_self_pairs", 24, 6), ("1e4", 10_000, 0)]


@pytest.mark.parametrize("name,n,self_pairs", LM_CASES)
def test_lm_trace_against_the_restatement(name, n, self_pairs):
    Ra, has, f1, f2, M = hub(n, seed=50 + n, self_pairs=self_pairs)
    opts = GravityRefinerOptions()
    p = probe(Ra, has, f1, f2, M, opts)
    assert 0 in p["ep"]
    k = int(np.nonzero(p["ep"] == 0)[0][0])
    terms, inc = terms_of(p, k)
    assert len(terms) == n + self_pairs and p["total"][0] == n + 2 * self_pairs
    res = compare_frame(p, k, opts, Ra[0][:, 1], fp64=n > 200)
    assert res["n"] >= 2
    print(f"{name}: {res}")


def test_lm_trace_on_a_scene():
    """Every error-prone frame of a seeded two-camera rig scene (pairs inside frames included)."""
    sc = make_scene(F=40, sensors=2, seed=8, pair_prob=0.3, noise_deg=0.8, rel_noise_deg=0.2, outlier_ratio=0.3)
    R_align, has, f1, f2, M = frame_inputs(sc)
    opts = GravityRefinerOptions()
    p = probe(R_align, has, f1, f2, M, opts)
    assert p["n_error_prone"] >= 5 and (p["status"] == 2).any()
    worst = {}
    for k in range(p["n_error_prone"]):
        if p["status"][k] == 1:
            assert int(p["trace"][k, 3]) == -1
            continue
        r = compare_frame(p, k, opts, R_align[p["ep"][k]][:, 1])
        for key in ("cost", "radius", "mcc", "x"):
            worst[key] = max(worst.get(key, 0.0), r[key])
    print(f"scene worst: {worst}")


# ---- 5. the probe is the production path ------------------------------------------------------------------------------
def test_probe_equals_production_bit_for_bit_and_repeats():
    sc = make_scene(F=60, sensors=2, seed=12, pair_prob=0.3, noise_deg=0.5, rel_noise_deg=0.3, outlier_ratio=0.3)
    R_align, has, f1, f2, M = frame_inputs(sc)
    g, st, s = production(R_align, has, f1, f2, M)
    p = probe(R_align, has, f1, f2, M, cap=4)                 # a cap below the iteration count: the trace is cut, not the LM
    assert s.error_prone_frames == p["n_error_prone"] > 0 and int(p["trace"][:, 4].max()) == 4
    for k, f in enumerate(p["ep"]):
        assert st[f] == p["status"][k]
        if st[f] == 2:
            assert g[f].tobytes() == p["x"][k].tobytes()
    assert s.lm_iterations == p["iterations"].sum()
    q = probe(R_align, has, f1, f2, M, cap=4)
    for key in ("mistake", "angle", "inc", "gobs", "x", "status", "iterations", "trace"):
        assert np.asarray(p[key]).tobytes() == np.asarray(q[key]).tobytes(), key


GOLDEN = os.path.join(HERE, "golden", "gravity_refine_outputs.npz")


def golden_scenes():
    for seed, sensors in ((12, 2), (31, 1)):
        sc = make_scene(F=60, sensors=sensors, seed=seed, pair_prob=0.3, noise_deg=0.5, rel_noise_deg=0.3, outlier_ratio=0.3)
        yield f"s{seed}", frame_inputs(sc)


def test_production_outputs_equal_the_recorded_ones():
    """The refined gravities, statuses and iteration totals of two seeded scenes, bit for bit, as recorded before the
    LM trace existed (tests/golden/gravity_refine_outputs.npz)."""
    ref = np.load(GOLDEN)
    for name, (R_align, has, f1, f2, M) in golden_scenes():
        g, st, s = production(R_align, has, f1, f2, M)
        assert g.tobytes() == ref[name + "_g"].tobytes() and st.tobytes() == ref[name + "_status"].tobytes()
        assert s.lm_iterations == int(ref[name + "_its"][0]) and s.rectified_frames == int(ref[name + "_its"][1])
