"""Operator-level tests of the device global positioner: every quantity one Levenberg-Marquardt step forms on the GPU,
read through the test probe (include/b200sfm_testing.h), against the FP64 sparse reference oracle/gp_system.py.

The trajectory tests (test_gp_gpu.py, test_rig_gpu.py) run PCG to 1e-8..1e-13 and compare the converged answer; a wrong
preconditioner, rhs term, back-substitution, step scalar or norm costs iterations there but leaves the answer alone.
Here each path takes the first LM step of a scene built to reach the kernels' edge shapes, and the test compares,
relative to the magnitude of each compared row:
  * per observation M_o, (b_o, w s^2) and the scale Jacobi scales; per point Vinv, g_X, D_p and the Jacobi scales;
    per block U, g_c, D_c, the Jacobi scales, the preconditioner and the right-hand side;
  * (S + D) x through the kernels of one PCG iteration (b200sfm_test_gp_apply) for random x on the variable blocks;
  * the PCG iterate after k = 1, 2, 5 iterations (tolerance 0) against reference PCG, and at convergence against the
    exact solve; the PCG residual;
  * dX and ds against the back-substitution of the device's own block step; g.delta, the model decrease, the cost,
    Ceres' gradient max-norm, the candidate state and cost, and the step and x norms.

The errors of every comparison are printed per path with `-s`; the bounds and the worst measured values are listed
beside BOUNDS.
"""
import ctypes as ct

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E
from oracle import gp_oracle as GP
from oracle import gp_system as GS

pytestmark = pytest.mark.gpu

C_MAIN, P_ORD = 280, 2600
FRONT_LENS = [0, 1, 2, 3, 127, 128, 129, 257]     # kTile = 128: the last three take the multi-chunk paths
N_TWO_VIEW = 64                                   # kTilePts = 64 two-view points: one full tile at min_views = 2
SPECIAL_CAMS = {0: 383, 1: 384, 2: 385, 3: 700}   # valid observations per camera at min_views = 3 (seg_split at 384)
EMPTY_CAM = 4                                     # observed only in tracks shorter than min_views = 3
ONLY_UNKNOWN_FRAME = 5                            # seen only through unknown sensor 0 on the rig paths
MASKED = (6, 7, 8, 9)                             # cam_const_mask
RADIUS = 300.0
FIRST_RADIUS = 1e4
PCG_KS = (1, 2, 5)

# bound per comparison, relative to the magnitude of the compared row (the PCG residual: relative to max|b|); the worst
# value measured over all paths on an H100 is in the comment (DESIGN.md §5)
BOUNDS = dict(M=5e-14,          # 1.4e-15
              bw=5e-12,         # 1.3e-13
              jscale_s=1e-14,   # 5.1e-16
              Vinv=1e-12,       # 2.6e-14
              gX=1e-11,         # 3.8e-13
              Dp=1e-14,         # 8.6e-16
              jscale_p=1e-14,   # 4.7e-16
              U=2e-13,          # 8.6e-15
              gc=2e-11,         # 7.8e-13
              Dc=2e-13,         # 6.7e-15
              jscale_c=2e-14,   # 9.6e-16
              Minv=5e-13,       # 1.1e-14
              b=1e-11,          # 3.2e-13
              apply=5e-13,      # 1.2e-14
              fixed=0.0,        # 0
              pcg=1e-11,        # 3.5e-13
              exact=2e-11,      # 8.6e-13
              resid=1e-11,      # see DESIGN.md
              dX=2e-11,         # 7.5e-13
              ds=5e-9,          # 3.0e-10: a scale step is a difference of two nearly equal terms near convergence
              scalars=2e-14,    # 9.0e-16
              gmax=5e-14,       # 1.8e-15
              cand=2e-12,       # 6.8e-14
              norms=2e-14)      # 6.8e-16


def make_scene(min_views=3, rig=None, start="random", seed=11):
    """C_MAIN cameras around a ball of points, tracks of FRONT_LENS first, N_TWO_VIEW two-view points, then ordinary
    tracks of 3..8 with every 7th one short; the SPECIAL_CAMS observation counts; 5% outlier bearings.
    rig: None, "known" (per-observation offsets and prior-focal flags, a frame that sees a point through two sensors),
    "unknown1" / "unknown2" (one / two unknown sensors on top of known offsets, a third that only sees short tracks)."""
    rng = np.random.default_rng(seed)
    C = C_MAIN
    cen = rng.normal(size=(C, 3)) * 4.0
    normal = np.arange(10, C)
    tracks = [list(rng.choice(normal, n, replace=False)) for n in FRONT_LENS]
    tracks += [list(rng.choice(normal, 2, replace=False)) for _ in range(N_TWO_VIEW)]
    n_fixed = len(tracks)
    ordinary = []
    for i in range(P_ORD):
        if i % 7 == 3:
            tracks.append([EMPTY_CAM] + list(rng.choice(normal, int(rng.integers(0, 2)), replace=False)))
        else:
            ordinary.append(len(tracks))
            tracks.append(list(rng.choice(np.concatenate([normal, MASKED, [ONLY_UNKNOWN_FRAME]]),
                                          int(rng.integers(3, 9)), replace=False)))
    for c, n in SPECIAL_CAMS.items():
        for p in rng.choice(ordinary, n, replace=False):
            tracks[p].append(c)
    if rig == "known":
        for p in rng.choice(ordinary, 40, replace=False):       # the same frame through a second sensor
            tracks[p].append(tracks[p][0])
    P = len(tracks)
    pts = rng.normal(size=(P, 3)) * 3.0
    lens = np.array([len(t) for t in tracks])
    ptb = np.zeros(P + 1, np.int64)
    np.cumsum(lens, out=ptb[1:])
    obs_cam = np.concatenate([np.asarray(t, np.int32) for t in tracks])
    obs_pt = np.repeat(np.arange(P), lens)
    N = len(obs_cam)
    d = pts[obs_pt] - cen[obs_cam]
    sc = dict(pt_obs_begin=ptb, obs_cam=obs_cam, n_fixed=n_fixed, C=C, P=P, N=N, min_views=min_views)
    if rig is None:
        sc["cam_calibrated"] = (np.arange(C) % 3 != 0).astype(np.uint8)
    else:
        off = rng.normal(size=(N, 3)) * 0.3
        d += off
        sc["obs_offset"] = off
        sc["obs_calibrated"] = (rng.uniform(size=N) < 0.6).astype(np.uint8)
    if rig in ("unknown1", "unknown2"):
        S_u = 1 if rig == "unknown1" else 3
        frot = np.stack([np.linalg.qr(rng.normal(size=(3, 3)))[0] for _ in range(C)])
        frot *= np.sign(np.linalg.det(frot))[:, None, None]
        obs_us = np.where(rng.uniform(size=N) < 0.3, 0, -1)
        if S_u == 3:
            obs_us[(obs_us < 0) & (rng.uniform(size=N) < 0.3)] = 1
            short = np.repeat(lens < min_views, lens)
            obs_us[short & (obs_us < 0)] = 2                     # sensor 2 sees only short tracks
        obs_us[obs_cam == ONLY_UNKNOWN_FRAME] = 0
        u_gt = rng.normal(size=(S_u, 3)) * 0.5
        m = obs_us >= 0
        d[m] -= np.einsum("nji,nj->ni", frot[obs_cam[m]], u_gt[obs_us[m]])
        sc.update(obs_us=obs_us.astype(np.int32), frame_rot=frot, u_gt=u_gt)
    t = d / np.linalg.norm(d, axis=1, keepdims=True) + rng.normal(size=(N, 3)) * 0.01
    out = rng.uniform(size=N) < 0.05
    v = rng.normal(size=(int(out.sum()), 3))
    t[out] = v / np.linalg.norm(v, axis=1, keepdims=True)
    sc["obs_dir"] = t
    if start == "random":          # the reference's start: 100 U(-1, 1), scales 1 (Huber active everywhere)
        sc["centers"], sc["points"], sc["scales"] = (100 * rng.uniform(-1, 1, size=(C, 3)),
                                                     100 * rng.uniform(-1, 1, size=(P, 3)), np.ones(N))
        ucen = rng.uniform(-1, 1, size=(len(sc.get("u_gt", [])), 3))
    else:                          # near converged: Huber inactive but on the outliers
        sc["centers"] = cen + rng.normal(size=cen.shape) * 0.01
        sc["points"] = pts + rng.normal(size=pts.shape) * 0.01
        sc["scales"] = 1.0 / np.linalg.norm(d, axis=1) * (1 + 0.01 * rng.normal(size=N))
        ucen = sc.get("u_gt", np.zeros((0, 3))) + rng.normal(size=(len(sc.get("u_gt", [])), 3)) * 0.01
    if "obs_us" in sc:
        sc["ucen"] = ucen
    return sc


# name: (scene spec, option overrides, probe settings)
PATHS = {
    "default_random": (dict(), {}, {}),
    "default_near": (dict(start="near"), {}, {}),
    "scale_bound": (dict(start="near"), {}, dict(alpha=40.0)),
    "block_jacobi": (dict(), dict(preconditioner=0), {}),
    "scales_const": (dict(), dict(optimize_scales=0), {}),
    "points_const": (dict(), dict(optimize_points=0), {}),
    "positions_const": (dict(), dict(optimize_positions=0), {}),
    "cam_const_mask": (dict(), {}, dict(mask=True)),
    "second_radius": (dict(), {}, dict(first_radius=FIRST_RADIUS)),
    "min_views_2": (dict(min_views=2), {}, {}),
    "min_views_4": (dict(min_views=4), {}, {}),
    "rig_known": (dict(rig="known"), {}, {}),
    "rig_unknown1": (dict(rig="unknown1"), {}, {}),
    "rig_unknown2": (dict(rig="unknown2"), {}, {}),
    "rig_unknown2_positions_const": (dict(rig="unknown2"), dict(optimize_positions=0), {}),
    "pcg_depth_3": (dict(), {}, dict(depth=3)),
}


def _ptr(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(ct.c_void_p)


class Probe:
    """One resident problem and its oracle counterpart."""

    def __init__(self, ctx, sc, opts: dict, mask):
        self.ctx, self.sc, self.lib = ctx, sc, _lib.load()
        self.o = _lib.GPOpts()
        self.lib.b200sfm_gp_default_opts(ct.byref(self.o))
        self.o.min_num_view_per_track = sc["min_views"]
        for k, v in opts.items():
            setattr(self.o, k, v)
        self.mask = mask
        self.keep = []            # arrays handed to the library
        h = ct.c_void_p()
        a = lambda x, t: self.keep.append(np.ascontiguousarray(x, t)) or self.keep[-1]
        _lib.check(ctx.handle, self.lib.b200sfm_gp_problem_create(
            ctx.handle, sc["C"], sc["P"], sc["N"], _ptr(a(sc["pt_obs_begin"], np.int64)), _ptr(a(sc["obs_cam"], np.int32)),
            _ptr(a(sc["obs_dir"], np.float64)),
            _ptr(a(sc["cam_calibrated"], np.uint8)) if "cam_calibrated" in sc else None,
            _ptr(a(mask, np.uint8)) if mask is not None else None, sc["min_views"], ct.byref(h)))
        self.h = h
        if "obs_offset" in sc:
            _lib.check(ctx.handle, self.lib.b200sfm_gp_problem_set_rig_terms(
                h, _ptr(a(sc["obs_offset"], np.float64)), _ptr(a(sc["obs_calibrated"], np.uint8))))
        self.S_u = len(sc["ucen"]) if "ucen" in sc else 0
        if self.S_u:
            _lib.check(ctx.handle, self.lib.b200sfm_gp_problem_set_rig_unknown(
                h, self.S_u, _ptr(a(sc["obs_us"], np.int32)), _ptr(a(sc["frame_rot"].reshape(-1, 9), np.float64)),
                _ptr(a(sc["ucen"], np.float64))))
        _lib.check(ctx.handle, self.lib.b200sfm_gp_problem_set_state(
            h, _ptr(a(sc["centers"], np.float64)), _ptr(a(sc["points"], np.float64)), _ptr(a(sc["scales"], np.float64))))

    def close(self):
        self.lib.b200sfm_gp_problem_free(self.h)

    def step(self, k, first_radius=0.0, alpha=1.0, rel_tol=0.0):
        """b200sfm_test_gp_step after exactly k PCG iterations (rel_tol = 0), or at convergence (rel_tol > 0)."""
        o = self.o
        o.pcg_min_iterations, o.pcg_max_iterations, o.pcg_rel_tolerance = (k, k, 0.0) if rel_tol == 0 else (0, k, rel_tol)
        sc, CB = self.sc, self.sc["C"] + self.S_u
        N, P = sc["N"], sc["P"]
        bufs = dict(M=np.zeros((N, 6)), bw=np.zeros((N, 4)), jscale_s=np.zeros(N), ds=np.zeros(N),
                    Vinv=np.zeros((P, 6)), gX=np.zeros((P, 3)), Dp=np.zeros(P), jscale_p=np.zeros(P), dX=np.zeros((P, 3)),
                    U=np.zeros((CB, 6)), gc=np.zeros((CB, 3)), Dc=np.zeros((CB, 3)), Minv=np.zeros((CB, 6)),
                    jscale_c=np.zeros(CB), b=np.zeros(CB * 3), px=np.zeros(CB * 3), resid=np.zeros(CB * 3),
                    cand_centers=np.zeros((sc["C"], 3)), cand_points=np.zeros((P, 3)), cand_scales=np.zeros(N))
        if self.S_u:
            bufs["cand_ucen"] = np.zeros((self.S_u, 3))
        out = _lib.GPStepProbeOut()
        for f, arr in bufs.items():
            setattr(out, f, _ptr(arr))
        _lib.check(self.ctx.handle, self.lib.b200sfm_test_gp_step(self.h, ct.byref(o), first_radius, RADIUS, alpha,
                                                                      ct.byref(out)))
        return out, bufs

    def apply(self, x):
        y = np.zeros_like(x)
        _lib.check(self.ctx.handle, self.lib.b200sfm_test_gp_apply(self.h, _ptr(x), _ptr(y)))
        return y

    def oracle(self, schur_jacobi):
        sc, o = self.sc, self.o
        ru = None
        if self.S_u:
            ru = dict(obs_sensor=sc["obs_us"], R_rw=sc["frame_rot"][sc["obs_cam"]], centers=sc["ucen"])
        kw = dict(centers=sc["centers"], points=sc["points"], pt_obs_begin=sc["pt_obs_begin"], obs_cam=sc["obs_cam"],
                  obs_dir=sc["obs_dir"], cam_calibrated=sc.get("cam_calibrated"), scales=sc["scales"],
                  obs_offset=sc.get("obs_offset"), rig_unknown=ru, obs_calibrated=sc.get("obs_calibrated"))
        opts = GP.GPOptions(optimize_positions=bool(o.optimize_positions), optimize_points=bool(o.optimize_points),
                            optimize_scales=bool(o.optimize_scales), min_num_view_per_track=sc["min_views"])
        full = GP.GPOptions(optimize_scales=opts.optimize_scales, min_num_view_per_track=sc["min_views"])
        prob = GP.GPProblem(opts=opts, cam_const=self.mask, **kw)
        return GS.GPSystem(prob, GP.GPProblem(opts=full, **kw), RADIUS, schur_jacobi)


def rowerr(dev, ref, width):
    """max over rows of max|dev - ref| / max|ref| of that row (rows that are zero in the reference: relative to the
    largest row)."""
    dev, ref = np.asarray(dev, float).reshape(-1, width), np.asarray(ref, float).reshape(-1, width)
    if ref.size == 0:
        return 0.0
    scale = np.abs(ref).max(1)
    scale = np.maximum(scale, 1e-14 * max(scale.max(), 1e-300))
    return float((np.abs(dev - ref).max(1) / scale).max())


@pytest.fixture(scope="module")
def scenes():
    cache = {}

    def get(spec):
        key = tuple(sorted(spec.items()))
        if key not in cache:
            cache[key] = make_scene(**spec)
        return cache[key]
    return get


def test_scene_reaches_the_shapes_it_is_built_for(scenes):
    sc = scenes({})
    lens = np.diff(sc["pt_obs_begin"])
    assert list(lens[:len(FRONT_LENS)]) == FRONT_LENS
    two = lens[len(FRONT_LENS):sc["n_fixed"]]
    assert len(two) == N_TWO_VIEW and (two == 2).all() and 2 * N_TWO_VIEW == 128
    valid = np.repeat(lens >= 3, lens)
    used = np.bincount(sc["obs_cam"][valid], minlength=sc["C"])
    assert all(used[c] == n for c, n in SPECIAL_CAMS.items())
    assert used[EMPTY_CAM] == 0 and (sc["obs_cam"] == EMPTY_CAM).any()
    # first valid observation is not observation 0; short tracks lie between valid ones
    assert sc["pt_obs_begin"][3] == 3 and lens[3] == 3
    assert ((lens[sc["n_fixed"]:] < 3) & (lens[sc["n_fixed"]:] > 0)).any()
    rs = scenes(dict(rig="unknown2"))
    short = np.repeat(np.diff(rs["pt_obs_begin"]) < 3, np.diff(rs["pt_obs_begin"]))
    assert (rs["obs_us"] == 2).any() and short[rs["obs_us"] == 2].all()
    assert (rs["obs_us"][rs["obs_cam"] == ONLY_UNKNOWN_FRAME] == 0).all()
    kr = scenes(dict(rig="known"))
    ptb = kr["pt_obs_begin"]
    assert any(len(set(kr["obs_cam"][ptb[p]:ptb[p + 1]])) < ptb[p + 1] - ptb[p] for p in range(len(ptb) - 1))


@pytest.mark.parametrize("name", list(PATHS))
def test_device_step_matches_the_fp64_reference(name, scenes, monkeypatch):
    spec, opts, pset = PATHS[name]
    sc = scenes(spec)
    ctx = None
    if pset.get("depth"):
        monkeypatch.setenv("B200SFM_PCG_DEPTH", str(pset["depth"]))
        ctx = E.Context(0)          # the depth is read when a context runs its first PCG
    mask = None
    if pset.get("mask"):
        mask = np.zeros(sc["C"], np.uint8)
        mask[list(MASKED)] = 1
    probe = Probe(ctx or E.default_context(), sc, opts, mask)
    try:
        fr, alpha = pset.get("first_radius", 0.0), pset.get("alpha", 1.0)
        runs = {k: probe.step(k, fr, alpha) for k in PCG_KS}
        conv_out, conv = probe.step(500, fr, alpha, rel_tol=1e-13)
        out, dev = runs[PCG_KS[-1]]
        rng = np.random.default_rng(3)
        ref = probe.oracle(bool(out.schur_jacobi))
        xs = [np.where(np.repeat(ref.var_c, 3), rng.normal(size=3 * ref.CB), 0.0) for _ in range(3)]
        applied = [probe.apply(x) for x in xs]
    finally:
        probe.close()
        if ctx is not None:
            ctx.close()
    if ref.var_c.any():
        assert all(runs[k][0].pcg_iterations == k for k in PCG_KS)
    assert out.CB == ref.CB and out.n_us == probe.S_u
    assert out.schur_jacobi == int(bool(probe.o.optimize_points) and probe.o.preconditioner == 1 and probe.S_u == 0)
    if pset.get("depth"):
        assert out.pcg_depth == pset["depth"]
    err = {}
    err["M"] = rowerr(dev["M"], ref.M, 6)
    err["bw"] = rowerr(dev["bw"], ref.bw, 4)
    vs = np.zeros(sc["N"], bool)
    vs[ref.kept[ref.var_s]] = True
    err["jscale_s"] = rowerr(dev["jscale_s"][vs], ref.jscale_s[vs], 1)
    err["Vinv"] = rowerr(dev["Vinv"], GS.pack_sym3(ref.Vinv_blocks), 6)
    err["gX"] = rowerr(dev["gX"], ref.gX, 3)
    err["Dp"] = rowerr(dev["Dp"], ref.Dp, 1)
    err["jscale_p"] = rowerr(dev["jscale_p"][ref.var_p], ref.jscale_p[ref.var_p], 1)
    err["U"] = rowerr(dev["U"], ref.U, 6)
    err["gc"] = rowerr(dev["gc"], ref.gc, 3)
    err["Dc"] = rowerr(dev["Dc"], ref.Dc, 3)
    assert np.array_equal(dev["jscale_c"] < 0, ~ref.var_c)
    err["jscale_c"] = rowerr(dev["jscale_c"], ref.jscale_c, 1)
    err["Minv"] = rowerr(dev["Minv"], ref.Minv, 6)
    err["b"] = rowerr(dev["b"], ref.b, 3)
    fixed3 = np.repeat(~ref.var_c, 3)
    err["apply"] = max(rowerr(y, ref.apply(x), 3) for x, y in zip(xs, applied))
    # identity rows, fed zeros; constant blocks take no step (exactly 0)
    err["fixed"] = max([np.abs(y[fixed3]).max(initial=0.0) for y in applied] +
                       [np.abs(runs[k][1]["px"][fixed3]).max(initial=0.0) for k in PCG_KS])
    iters = ref.pcg(max(PCG_KS))
    err["pcg"] = max(rowerr(runs[k][1]["px"], iters[k - 1], 3) for k in PCG_KS)
    err["exact"] = rowerr(conv["px"], ref.solve(), 3)
    px = dev["px"]
    err["resid"] = np.abs(dev["resid"] - (ref.b - ref.apply(px))).max() / max(np.abs(ref.b).max(), 1e-300)
    dX, ds = ref.back_sub(px)
    err["dX"] = rowerr(dev["dX"], dX, 3)
    err["ds"] = rowerr(dev["ds"], ds, 1)
    gd, mcc = ref.step_scalars(px)
    err["scalars"] = max(abs(out.cost - ref.cost) / ref.cost, abs(out.g_dot_delta - gd) / abs(gd),
                         abs(out.model_cost_change - mcc) / abs(mcc))
    err["gmax"] = abs(out.gmax - ref.gmax()) / ref.gmax()
    cand, cost, step_norm, x_norm = ref.candidate(px, alpha)
    x0 = ref.prob.x0
    kept = ref.kept

    def rel(d, r, x):   # error of the candidate relative to the size of the step it takes
        return np.abs(d - r).max() / max(np.abs(r - x).max(), 1e-6 * (np.abs(x).max() + 1.0))
    cerr = [rel(dev["cand_centers"], cand["centers"], x0["centers"]), rel(dev["cand_points"], cand["points"], x0["points"]),
            rel(dev["cand_scales"][kept], cand["scales"], x0["scales"]), abs(out.cand_cost - cost) / cost]
    if probe.S_u:
        cerr.append(rel(dev["cand_ucen"], cand["rig_centers"], x0["rig_centers"]))
    err["cand"] = max(cerr)
    err["norms"] = max(abs(out.step_norm - step_norm) / step_norm, abs(out.x_norm - x_norm) / x_norm)
    if name == "scale_bound":
        assert (dev["cand_scales"][kept] == GP.SCALE_LOWER_BOUND).sum() > 10
    print(name, f"pcg_conv={conv_out.pcg_iterations}", " ".join(f"{k}={v:.1e}" for k, v in err.items()))
    bad = {k: v for k, v in err.items() if not v <= BOUNDS[k]}
    assert not bad, (name, bad)
