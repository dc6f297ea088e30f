"""CPU tests of oracle/gp_system.py, the FP64 reference of one device global-positioning LM step: the per-observation
scale elimination against its closed form, the Schur solve against a dense solve of the full system, the model-decrease
identity the device uses, the exact step against the first step of oracle/ceres_lm.py, and the option masks against
GPProblem's columns."""
import numpy as np
import pytest

from oracle import gp_oracle as GP
from oracle import gp_system as GS
from oracle.ceres_lm import LMOptions, huber_rho, solve_lm

RADIUS = 300.0


def make_scene(seed=0, C=9, P=70, unknown=0, offsets=False, near=False):
    """Tracks of length 0, 1, 2 first (the first valid observation is not observation 0), then 3..6, a short track
    between valid ones; half the cameras uncalibrated; optional known-rig offsets and unknown sensors."""
    rng = np.random.default_rng(seed)
    cen = rng.normal(size=(C, 3)) * 3
    pts = rng.normal(size=(P, 3)) * 3
    lens = rng.integers(3, 7, size=P)
    lens[:3] = [0, 1, 2]
    lens[10] = 2
    tracks = [rng.choice(C, n, replace=False) for n in lens]
    ptb = np.zeros(P + 1, np.int64)
    np.cumsum(lens, out=ptb[1:])
    obs_cam = np.concatenate(tracks).astype(np.int32)
    obs_pt = np.repeat(np.arange(P), lens)
    N = len(obs_cam)
    off = rng.normal(size=(N, 3)) * 0.2 if offsets else None
    ru = None
    d = pts[obs_pt] - cen[obs_cam] + (off if off is not None else 0.0)
    if unknown:
        frame_rot = np.stack([np.linalg.qr(rng.normal(size=(3, 3)))[0] for _ in range(C)])
        frame_rot *= np.sign(np.linalg.det(frame_rot))[:, None, None]
        obs_us = np.where(rng.uniform(size=N) < 0.4, rng.integers(0, unknown, size=N), -1)
        u_true = rng.normal(size=(unknown, 3)) * 0.3
        m = obs_us >= 0
        d[m] -= np.einsum("nji,nj->ni", frame_rot[obs_cam[m]], u_true[obs_us[m]])
        ru = dict(obs_sensor=obs_us, R_rw=frame_rot[obs_cam], centers=u_true + rng.normal(size=u_true.shape) * 0.1)
    t = d / np.linalg.norm(d, axis=1, keepdims=True) + rng.normal(size=(N, 3)) * 0.02
    cal = (np.arange(C) % 2).astype(np.uint8)
    if near:
        c0 = cen + rng.normal(size=cen.shape) * 0.01
        X0 = pts + rng.normal(size=pts.shape) * 0.01
        s0 = 1.0 / np.linalg.norm(d, axis=1)
    else:
        c0, X0, s0 = 100 * rng.uniform(-1, 1, size=(C, 3)), 100 * rng.uniform(-1, 1, size=(P, 3)), np.ones(N)
    return dict(centers=c0, points=X0, pt_obs_begin=ptb, obs_cam=obs_cam, obs_dir=t, cam_calibrated=cal, scales=s0,
                obs_offset=off, rig_unknown=ru)


def problems(sc, min_views=3, cam_const=None, **flags):
    opts = GP.GPOptions(min_num_view_per_track=min_views, **flags)
    full = GP.GPOptions(min_num_view_per_track=min_views, optimize_scales=opts.optimize_scales)
    return GP.GPProblem(opts=opts, cam_const=cam_const, **sc), GP.GPProblem(opts=full, **sc)


def system(sc, schur_jacobi=True, **kw):
    prob, full = problems(sc, **kw)
    return prob, GS.GPSystem(prob, full, RADIUS, schur_jacobi and prob.opts.optimize_points and prob.ru is None)


@pytest.mark.parametrize("kind", ["plain", "offsets", "unknown", "near", "scales_const"])
def test_per_observation_blocks_match_their_closed_form(kind):
    sc = make_scene(1, offsets=kind == "offsets", unknown=2 if kind == "unknown" else 0, near=kind == "near")
    prob, sysm = system(sc, optimize_scales=kind != "scales_const")
    x = prob.x0
    d = x["points"][prob.obs_pt] - x["centers"][prob.obs_cam]
    if prob.obs_off is not None:
        d = d + prob.obs_off
    if prob.ru is not None:
        m = prob.ru["obs_sensor"] >= 0
        d[m] -= np.einsum("nji,nj->ni", prob.ru["R_rw"][m], x["rig_centers"][prob.ru["obs_sensor"][m]])
    s = x["scales"]
    r = prob.obs_dir - s[:, None] * d
    _, rho1 = huber_rho((r * r).sum(1), 0.1)
    w = prob.loss_scale * rho1
    dd = (d * d).sum(1)
    js = 1.0 / (1.0 + np.sqrt(w * dd))
    Ds = np.clip(w * dd * js * js, 1e-6, 1e32) / (RADIUS * js * js)
    k = np.where(prob.s_col >= 0, w / (w * dd + Ds), 0.0)
    dr = (d * r).sum(1)
    M = (w * s * s)[:, None, None] * (np.eye(3) - k[:, None, None] * d[:, :, None] * d[:, None, :])
    b = (w * s)[:, None] * (r - (k * dr)[:, None] * d)
    kept = sysm.kept
    assert np.abs(sysm.M[kept] - GS.pack_sym3(M)).max() <= 1e-12 * np.abs(M).max()
    assert np.abs(sysm.bw[kept, :3] - b).max() <= 1e-12 * np.abs(b).max()
    assert np.allclose(sysm.bw[kept, 3], w * s * s, rtol=1e-14)
    short = np.setdiff1d(np.arange(sysm.N_dev), kept)
    assert len(short) and not sysm.M[short].any() and not sysm.bw[short].any()
    # the point blocks: V + Dp = sum M_o + Dp, g_X = -sum b_o
    for p in np.nonzero(prob.pt_col >= 0)[0][:10]:
        m = prob.obs_pt == p
        V = M[m].sum(0) + sysm.Dp[p] * np.eye(3)
        assert np.allclose(np.linalg.inv(V), sysm.Vinv_blocks[p], rtol=1e-10, atol=1e-12 * np.abs(sysm.Vinv_blocks[p]).max())
        assert np.allclose(sysm.gX[p], -b[m].sum(0), rtol=1e-10, atol=1e-12 * np.abs(b).max())


@pytest.mark.parametrize("kind", ["plain", "offsets", "unknown", "positions_const", "points_const", "cam_mask"])
def test_schur_solve_and_back_substitution_match_a_dense_solve(kind):
    sc = make_scene(2, offsets=kind == "offsets", unknown=2 if kind == "unknown" else 0)
    kw = dict(optimize_positions=kind != "positions_const", optimize_points=kind != "points_const")
    if kind == "cam_mask":
        kw["cam_const"] = np.arange(sc["centers"].shape[0]) % 3 == 0
    prob, sysm = system(sc, **kw)
    Hd = (sysm.J.T @ sysm.J).toarray() + np.diag(sysm.D)
    full = np.linalg.solve(Hd, -sysm.g)
    dc = sysm.solve()
    delta = sysm.delta(dc)
    assert np.abs(delta - full).max() <= 1e-8 * np.abs(full).max()
    assert not dc[np.repeat(~sysm.var_c, 3)].any()


@pytest.mark.parametrize("kind", ["plain", "unknown", "cam_mask"])
def test_model_cost_change_identity_holds_for_an_inexact_step(kind):
    """The device forms model_cost_change = 1/2 (-g.delta + dc.res + delta^T D delta), res = b - S dc the PCG residual;
    it equals -(J delta)^T (r + J delta / 2) for any dc when dX and ds are back-substituted."""
    sc = make_scene(3, unknown=2 if kind == "unknown" else 0)
    prob, sysm = system(sc, cam_const=(np.arange(9) % 4 == 1) if kind == "cam_mask" else None)
    for k in (1, 3):
        dc = sysm.pcg(k)[-1]
        res = sysm.b - sysm.apply(dc)
        gd, mcc = sysm.step_scalars(dc)
        delta = sysm.delta(dc)
        ident = 0.5 * (-gd + dc @ res + delta @ (sysm.D * delta))
        assert abs(ident - mcc) <= 1e-9 * abs(mcc), (k, ident, mcc)


@pytest.mark.parametrize("scales", [True, False])
def test_exact_step_is_the_first_step_of_ceres_lm(scales):
    sc = make_scene(4, near=False)
    prob, sysm = problems(sc, optimize_scales=scales)
    steps = []

    def plus(x, d):
        steps.append(d.copy())
        return prob.plus(x, d)
    solve_lm(prob.x0, prob.evaluate, plus, LMOptions(max_num_iterations=1), project=prob.project if scales else None,
             x_norm_fn=prob.x_norm)
    ref = GS.GPSystem(prob, sysm, 1e4, True)                 # Ceres' initial trust-region radius
    delta = ref.delta(ref.solve())
    assert np.abs(steps[0] - delta).max() <= 1e-8 * np.abs(delta).max()


@pytest.mark.parametrize("flags", [dict(), dict(optimize_positions=False), dict(optimize_points=False),
                                   dict(optimize_scales=False), dict(cam_const=True), dict(min_views=2),
                                   dict(min_views=4)])
def test_option_masks_follow_the_problem_columns(flags):
    sc = make_scene(5, unknown=1)
    flags = dict(flags)
    if flags.pop("cam_const", False):
        flags["cam_const"] = np.arange(9) % 2 == 0
    prob, sysm = system(sc, **flags)
    assert np.array_equal(sysm.var_c[:prob.C], prob.cam_col >= 0)
    assert np.array_equal(sysm.var_c[prob.C:], prob.u_col >= 0)
    assert np.array_equal(sysm.var_p, prob.pt_col >= 0)
    assert np.array_equal(sysm.jscale_c < 0, ~sysm.var_c)
    kept = np.nonzero(prob.keep)[0]
    assert kept[0] == sc["pt_obs_begin"][np.nonzero(np.diff(sc["pt_obs_begin"]) >= prob.opts.min_num_view_per_track)[0][0]]
    assert not sysm.var_s[0] and sysm.var_s[1:].all() == prob.opts.optimize_scales
    if not prob.opts.optimize_points:
        assert not sysm.Vinv_blocks.any() and not sysm.gX.any()
    assert np.array_equal(sysm.U_blocks[~sysm.var_c], np.broadcast_to(np.eye(3), (int((~sysm.var_c).sum()), 3, 3)))
    assert not sysm.b.reshape(-1, 3)[~sysm.var_c].any()
