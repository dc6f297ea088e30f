"""Operator-level tests of the device bundle adjuster: every quantity one Levenberg-Marquardt step forms on the GPU,
read through the test probe (include/b200sfm_testing.h), against the FP64 sparse reference oracle/ba_system.py.

The trajectory tests (test_ba_gpu.py, test_rig_gpu.py, test_config2_gpu.py) run PCG to 1e-10..1e-13 and compare the
converged answer; they cannot see a wrong preconditioner, a wrong inexact-step bookkeeping or a mat-vec branch that
only a shape reaches.  Here each path solves the same first LM step of a scene built to reach those shapes, and the
test compares, relative to the magnitude of each compared block row:
  * the linearisation U, g_c, V, g_p, the Jacobi scales, the damping Dc and the right-hand side b;
  * the preconditioner blocks Minv against the exact Schur-Jacobi / block-Jacobi inverses;
  * (S + D) x through the production mat-vec chain (b200sfm_test_ba_apply) for random x on the variable dofs;
  * the PCG iterate after k = 1, 2, 3, 5, 8 iterations (tolerance 0, min = max = k), which also goes through
    ba2_pcg_direction_pack;
  * at k = 3, after a first step at a larger radius that is not accepted (the solve's path after a rejection): all of
    the above, the model cost change (against the direct formula), the candidate state and cost, the step and x norms.

The errors of every comparison are printed per path with `-s`; the bounds and the worst measured values are listed
beside BOUNDS.
"""
import ctypes as ct

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E, geometry as G, synthetic as S
from oracle import ba_oracle as B
from oracle import ba_system as BS

pytestmark = pytest.mark.gpu

C_MAIN, P_MAIN, MIN_VIEWS = 300, 2600, 3
SPECIAL_CAMS = {1: 256, 2: 257, 3: 512}     # cameras with exactly this many used observations (kSeg = 256 segments)
EMPTY_CAM = 4                               # all its observations belong to tracks shorter than min_num_view_per_track
BEHIND_CAM, BEHIND_PT = 5, 300              # one observation behind its camera (z <= kZEps)
LONG_TRACKS = {100: 31, 101: 32, 102: 33, 103: 280}   # inside the first ELL window; 280 > 256
EXCLUDED_PTS = range(200, 210)              # tracks of length MIN_VIEWS - 1
EXACT_MIN_PTS = range(210, 220)             # tracks of length MIN_VIEWS
MASKED = {6: 1, 7: 2, 8: 3}                 # per-camera constant masks (bit0 rotation, bit1 translation)
RADIUS = 200.0
PCG_KS = (1, 2, 3, 5, 8)
LOOSE_K = 3

# bound per comparison, relative to the magnitude of the compared block row (worst measured values: DESIGN.md §5)
BOUNDS = dict(U=1e-11, g_c=1e-11, V=1e-11, g_p=1e-11, jscale_c=1e-12, jscale_p=1e-12, Dc=1e-11, b=5e-11,
              Minv=1e-10, apply=2e-10, pcg=5e-9, model=1e-9, cand=1e-9, cand_cost=1e-12, norms=1e-9)
# the step at LOOSE_K comes after a step at FIRST_RADIUS that is not accepted (same linearisation), as in the solve
FIRST_RADIUS = 1e4


def make_scene(K=1, model=S.SIMPLE_PINHOLE, seed=7):
    """C = 300 cameras looking at a unit ball of P = 2600 points (three ELL windows of 1024, the last partial), with
    every shape of the module docstring built in on purpose."""
    rng = np.random.default_rng(seed)
    R, t = S.make_cameras(C_MAIN, seed, jitter_deg=2.0)
    cam_intr, intr_model, intr_params = S.make_intrinsics(C_MAIN, model, 1000.0, 1000, K)
    d = rng.normal(size=(P_MAIN, 3))
    pts = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0, 1, size=(P_MAIN, 1)) ** (1 / 3)
    centres = G.centers_from_pose(R, t)
    pts[BEHIND_PT] = 1.5 * centres[BEHIND_CAM]          # behind BEHIND_CAM, in front of the cameras facing it
    normal = np.arange(9, C_MAIN)
    tracks = []
    for p in range(P_MAIN):
        if p in LONG_TRACKS:
            tr = list(rng.choice(normal, LONG_TRACKS[p], replace=False))
        elif p in EXCLUDED_PTS:
            tr = [EMPTY_CAM, int(rng.choice(normal))]
        elif p in EXACT_MIN_PTS:
            tr = list(rng.choice(normal, MIN_VIEWS, replace=False))
        elif p == BEHIND_PT:
            z = np.einsum("cj,cj->c", R[:, 2], pts[p][None] - centres)
            tr = [BEHIND_CAM] + list(rng.choice(np.nonzero(z > 1.0)[0][10:], 4, replace=False))
        else:
            tr = list(rng.choice(np.concatenate([normal, list(MASKED)]), min(3 + rng.poisson(3), 10), replace=False))
        tracks.append(tr)
    ordinary = [p for p in range(P_MAIN)
                if p not in LONG_TRACKS and p not in EXCLUDED_PTS and p not in EXACT_MIN_PTS and p != BEHIND_PT]
    for c, n in SPECIAL_CAMS.items():
        for p in rng.choice(ordinary, n, replace=False):
            tracks[p].append(c)
    obs_cam = np.concatenate([np.asarray(tr, np.int32) for tr in tracks])
    obs_pt = np.repeat(np.arange(P_MAIN), [len(tr) for tr in tracks])
    Xc = np.einsum("nij,nj->ni", R[obs_cam], pts[obs_pt]) + t[obs_cam]
    xy = np.empty((len(obs_cam), 2))
    for k in range(K):
        m = cam_intr[obs_cam] == k
        xy[m] = S.project(int(intr_model[k]), intr_params[k], np.where(Xc[m, 2:3] > 0, Xc[m], 1.0))
    xy += rng.normal(size=xy.shape) * 0.8                # a share of the residuals beyond the Huber threshold
    ptb = np.zeros(P_MAIN + 1, np.int64)
    np.cumsum([len(tr) for tr in tracks], out=ptb[1:])
    sc = S.Scene(G.rotmat_to_quat_xyzw_fast(R), t, pts, ptb, obs_cam, xy, cam_intr, intr_model, intr_params)
    st = S.perturb_scene(sc, rot_deg=0.05, center_frac=0.001, point_frac=0.001, seed=seed)
    st.intr_params = sc.intr_params.copy()
    st.intr_params[:, 0] *= 1.002
    return st


def make_rig(model=S.SIMPLE_RADIAL, seed=21):
    rs = S.make_rig_scene(30, 3, 1500, seed=seed, pixel_sigma=0.8, model=model)
    st = S.perturb_rig_scene(rs, rot_deg=0.05, center_frac=0.001, point_frac=0.001)
    rng = np.random.default_rng(seed)
    st.sensor_quat = st.sensor_quat.copy()
    st.sensor_quat[1:] = G.rotmat_to_quat_xyzw_fast(G.so3_exp(rng.normal(size=(2, 3)) * 0.002) @
                                                    G.quat_xyzw_to_rotmat(st.sensor_quat[1:]))
    return st


# name: (scene, options, environment, expected path)
SC1 = dict(K=1)
PATHS = {
    "v1": (SC1, dict(design=1), {}, dict(use_v2=0, ext=0)),
    "v2_tile": (SC1, {}, {"B200SFM_ELL": "0"}, dict(use_v2=1, use_ell=0, ext=0)),
    "ell": (SC1, {}, {}, dict(use_v2=1, use_ell=1, ext=0)),
    "kfast_nk1_K200": (dict(K=200), dict(optimize_intrinsics=True), {}, dict(use_ell=1, kfast=1, nk=1)),
    "kfast_nk1_K300": (dict(K=300), dict(optimize_intrinsics=True), {}, dict(use_ell=1, kfast=1, nk=1)),
    "kfast_nk2_simple_radial_K300": (dict(K=300, model=S.SIMPLE_RADIAL), dict(optimize_intrinsics=True), {},
                                     dict(kfast=1, nk=2)),
    "kfast_nk2_pinhole_K200": (dict(K=200, model=S.PINHOLE), dict(optimize_intrinsics=True), {}, dict(kfast=1, nk=2)),
    "ext_radial_nk3": (dict(K=200, model=S.RADIAL), dict(optimize_intrinsics=True), {}, dict(ext=1, ext_k=1, kfast=0)),
    "ext_kfast_off": (dict(K=300, model=S.SIMPLE_RADIAL), dict(optimize_intrinsics=True), {"B200SFM_KFAST": "0"},
                      dict(ext=1, kfast=0)),
    "rig_known": ("rig", {}, {}, dict(use_ell=1, ext=0)),
    "rig_poses": ("rig", dict(optimize_rig_poses=True), {}, dict(ext=1, ext_s=1, ext_k=0, kfast=0)),
    "rig_poses_intrinsics": ("rig", dict(optimize_rig_poses=True, optimize_intrinsics=True), {},
                             dict(ext=1, ext_s=1, ext_k=1, kfast=0)),
    "constant_points": (SC1, dict(optimize_points=False), {}, dict(schur_jacobi=0)),
    "constant_points_kfast_K300": (dict(K=300), dict(optimize_points=False, optimize_intrinsics=True), {},
                                   dict(kfast=1, schur_jacobi=0)),
    "block_jacobi": (SC1, dict(preconditioner=0), {}, dict(schur_jacobi=0)),
    "constant_rotations": (SC1, dict(optimize_rotations=False), {}, dict(ext=0)),
}


def _ptr(a):
    return a.ctypes.data_as(ct.c_void_p)


class Probe:
    """One resident problem and its oracle counterpart."""

    def __init__(self, scene, opts: dict, mask):
        self.scene, self.mask = scene, mask
        self.rig = hasattr(scene, "obs_sensor")
        self.o = E.BundleAdjusterOptions(optimize_intrinsics=False)
        for k, v in opts.items():
            if k in ("preconditioner",):
                setattr(self.o.solver_options, k, v)
            else:
                setattr(self.o, k, v)
        self.lib = _lib.load()
        self.ctx = E.default_context()
        self.prob = E.BAProblem(self.ctx, scene, MIN_VIEWS, mask)
        self.prob.set_state(scene.intr_params, scene.quat, scene.trans, scene.points)
        if self.rig and self.o.optimize_rig_poses:
            self.prob.set_sensor_variable((np.arange(scene.S) != 0).astype(np.uint8))
        self.C, self.P, self.K = scene.C, scene.P, len(scene.intr_model)
        self.S = scene.S if self.rig else 0
        self.nmax = self.C + self.K + self.S

    def step(self, k, first_radius=0.0):
        """b200sfm_test_ba_step after exactly k PCG iterations (after a rejected step at first_radius if > 0)."""
        so = self.o.solver_options
        so.pcg_min_iterations = so.pcg_max_iterations = k
        so.pcg_rel_tolerance = 0.0
        oc = self.o.to_c()
        n = self.nmax
        bufs = dict(U=np.zeros(n * 21), g_c=np.zeros(n * 6), jscale_c=np.zeros(n * 6), V=np.zeros(self.P * 6),
                    g_p=np.zeros(self.P * 3), jscale_p=np.zeros(self.P * 3), Dc=np.zeros(n * 6), Minv=np.zeros(n * 21),
                    b=np.zeros(n * 6), px=np.zeros(n * 6), cand_points=np.zeros((self.P, 3)),
                    cand_quat=np.zeros((self.C, 4)), cand_trans=np.zeros((self.C, 3)),
                    cand_intr=np.zeros((self.K, _lib.INTR_STRIDE)))
        if self.S:
            bufs.update(cand_sensor_quat=np.zeros((self.S, 4)), cand_sensor_trans=np.zeros((self.S, 3)))
        out = _lib.BAStepProbeOut()
        for f, a in bufs.items():
            setattr(out, f, _ptr(a))
        _lib.check(self.ctx.handle, self.lib.b200sfm_test_ba_step(self.prob.handle, ct.byref(oc), first_radius, RADIUS,
                                                                      ct.byref(out)))
        nb = out.nbk
        for f in ("U", "Minv"):
            bufs[f] = bufs[f][:nb * 21].reshape(nb, 21)
        for f in ("g_c", "jscale_c", "Dc", "b", "px"):
            bufs[f] = bufs[f][:nb * 6]
        bufs["V"] = bufs["V"].reshape(self.P, 6)
        return out, bufs

    def apply(self, x):
        y = np.zeros_like(x)
        _lib.check(self.ctx.handle, self.lib.b200sfm_test_ba_apply(self.prob.handle, _ptr(np.ascontiguousarray(x)), _ptr(y)))
        return y

    def oracle(self, nbk, precond):
        sc = self.scene
        bo = B.BAOptions(optimize_rotations=self.o.optimize_rotations, optimize_translation=self.o.optimize_translation,
                         optimize_intrinsics=self.o.optimize_intrinsics,
                         optimize_principal_point=self.o.optimize_principal_point, optimize_points=self.o.optimize_points,
                         optimize_rig_poses=self.o.optimize_rig_poses, thres_loss_function=self.o.thres_loss_function,
                         min_num_view_per_track=MIN_VIEWS)
        if self.rig:
            p = B.BAProblem(sc.quat, sc.trans, sc.points, sc.pt_obs_begin, sc.obs_frame, sc.obs_xy, np.zeros(sc.F, np.int32),
                            sc.intr_model, sc.intr_params, bo, self.mask, rig=sc.rig_dict())
        else:
            p = B.BAProblem(sc.quat, sc.trans, sc.points, sc.pt_obs_begin, sc.obs_cam, sc.obs_xy, sc.cam_intr,
                            sc.intr_model, sc.intr_params, bo, self.mask)
        return BS.BASystem(p, p.x0, RADIUS, nbk, precond)


def blockerr(dev, ref, width):
    """max over block rows of max|dev - ref| / max|ref| of that row (rows that are zero in the reference: relative to
    the largest row)."""
    dev, ref = np.asarray(dev).reshape(-1, width), np.asarray(ref).reshape(-1, width)
    scale = np.abs(ref).max(1)
    scale = np.maximum(scale, 1e-14 * scale.max())
    return float((np.abs(dev - ref).max(1) / scale).max())


def intr_param_masks(prob: B.BAProblem):
    """[K, INTR_STRIDE] masks of the reference problem: (parameters that are unknowns, parameters of the block's model)."""
    ivar = np.zeros((prob.K, _lib.INTR_STRIDE), bool)
    own = np.zeros_like(ivar)
    for k, ent in enumerate(prob.intr_cols):
        own[k, :S.MODEL_NUM_PARAMS[int(prob.intr_model[k])]] = True
        ivar[k, [i for i, _ in ent]] = True
    return ivar, own


def expected_precond(probe: Probe, flags):
    if not probe.o.optimize_points or probe.o.solver_options.preconditioner == 0 or (flags.ext and not flags.kfast):
        return "jacobi"
    if probe.rig:
        # ba2_schur_diag sums per observation; the exact block (Ceres SCHUR_JACOBI) also has the cross terms of a frame
        # that sees a point through two sensors -- pinned to what the kernel forms until the kernel forms the exact one
        return "schur_per_obs"
    return "schur_frames" if flags.kfast else "schur"


@pytest.fixture(scope="module")
def scenes():
    cache = {}

    def get(spec):
        key = "rig" if spec == "rig" else tuple(sorted(spec.items()))
        if key not in cache:
            cache[key] = make_rig() if spec == "rig" else make_scene(**spec)
        return cache[key]
    return get


def test_scene_reaches_the_shapes_it_is_built_for(scenes):
    sc = scenes(SC1)
    assert sc.P % 32 != 0 and sc.P > 2 * 1024 and sc.P % 1024 != 0
    lens = np.diff(sc.pt_obs_begin)
    assert all(lens[p] == n for p, n in LONG_TRACKS.items()) and max(LONG_TRACKS) < 1024 and lens.max() > 256
    assert all(lens[p] == MIN_VIEWS - 1 for p in EXCLUDED_PTS) and all(lens[p] == MIN_VIEWS for p in EXACT_MIN_PTS)
    valid = np.repeat(lens >= MIN_VIEWS, lens)
    used = np.bincount(sc.obs_cam[valid], minlength=sc.C)
    assert all(used[c] == n for c, n in SPECIAL_CAMS.items())
    assert used[EMPTY_CAM] == 0 and np.count_nonzero(sc.obs_cam == EMPTY_CAM) == len(EXCLUDED_PTS)
    p = B.BAProblem(sc.quat, sc.trans, sc.points, sc.pt_obs_begin, sc.obs_cam, sc.obs_xy, sc.cam_intr, sc.intr_model,
                    sc.intr_params, B.BAOptions(), None)
    res, jac = p.residuals(p.x0, True)
    assert (~jac[4]).sum() == 1                                    # exactly one observation behind its camera
    outlier = (res * res).sum(1) > 1.0
    assert 0.1 <= outlier.mean() <= 0.9, outlier.mean()            # Huber outliers next to inliers


@pytest.mark.parametrize("name", list(PATHS))
def test_device_step_matches_the_fp64_reference(name, scenes, monkeypatch):
    spec, opts, env, want = PATHS[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sc = scenes(spec)
    mask = E.first_frame_mask(sc.C)
    if spec != "rig":
        for c, m in MASKED.items():
            mask[c] = m
    probe = Probe(sc, opts, mask)
    runs = {k: probe.step(k, FIRST_RADIUS if k == LOOSE_K else 0.0) for k in PCG_KS}
    out, dev = runs[LOOSE_K]
    for f, v in want.items():
        assert getattr(out, f) == v, (f, getattr(out, f), v)
    assert all(runs[k][0].pcg_iterations == k for k in PCG_KS)
    ref = probe.oracle(out.nbk, expected_precond(probe, out))
    err = {}
    err["U"] = blockerr(dev["U"], BS.pack_sym(ref.U_blocks), 21)
    for f, w in (("g_c", 6), ("jscale_c", 6), ("Dc", 6), ("b", 6)):
        err[f] = blockerr(dev[f], getattr(ref, f), w)
    assert np.array_equal(dev["jscale_c"] < 0, ~ref.var_c)
    if ref.points_var:
        err["V"] = blockerr(dev["V"], BS.pack_sym(ref.V_blocks), 6)
        err["g_p"] = blockerr(dev["g_p"], ref.g_p, 3)
        err["jscale_p"] = blockerr(dev["jscale_p"], ref.jscale_p.ravel(), 3)
    err["Minv"] = blockerr(dev["Minv"], BS.pack_sym(ref.Minv_blocks), 21)
    rng = np.random.default_rng(3)
    err["apply"] = max(blockerr(probe.apply(x), ref.apply(x), 6)
                       for x in (np.where(ref.var_c, rng.normal(size=ref.var_c.size), 0.0) for _ in range(3)))
    iters = ref.pcg(max(PCG_KS))
    err["pcg"] = max(blockerr(runs[k][1]["px"], iters[k - 1], 6) for k in PCG_KS)
    # the step at the loose k: candidate of the device's own camera step
    cand, cost, step_norm, x_norm, mcc = ref.candidate(dev["px"])
    err["model"] = abs(out.model_cost_change - mcc) / abs(mcc)
    err["cand_cost"] = abs(out.cand_cost - cost) / cost
    err["norms"] = max(abs(out.step_norm - step_norm) / step_norm, abs(out.x_norm - x_norm) / x_norm)
    def rel(d, r, x0):   # error of the candidate relative to the size of the step it takes
        return np.abs(d - r).max() / max(np.abs(r - x0).max(), 1e-6 * (np.abs(x0).max() + 1.0))
    def unit(q):   # the device normalises the state's quaternions on upload
        return q / np.linalg.norm(q, axis=1, keepdims=True)
    qd, qr = unit(dev["cand_quat"]), unit(cand["quat"])
    qd = qd * np.sign((qd * qr).sum(1, keepdims=True))
    cerr = [rel(dev["cand_points"], cand["points"], sc.points), rel(dev["cand_trans"], cand["trans"], sc.trans),
            rel(qd, qr, unit(sc.quat))]
    # intrinsics, each block over its own parameters: the variable ones (the reference's columns) against the reference
    # candidate, the others (the principal point when held, every parameter of a constant or unused block) unchanged
    ivar, own = intr_param_masks(ref.prob)
    assert np.array_equal(dev["cand_intr"][own & ~ivar], sc.intr_params[own & ~ivar]), "a constant intrinsic moved"
    if ivar.any():
        cerr.append(rel(dev["cand_intr"][ivar], cand["intr"][ivar], sc.intr_params[ivar]))
    if probe.S and probe.o.optimize_rig_poses:
        sq = dev["cand_sensor_quat"] * np.sign((dev["cand_sensor_quat"] * cand["sq"]).sum(1, keepdims=True))
        cerr += [rel(sq, cand["sq"], sc.sensor_quat), rel(dev["cand_sensor_trans"], cand["st"], sc.sensor_trans)]
    err["cand"] = max(cerr)
    print(name, " ".join(f"{k}={v:.1e}" for k, v in err.items()))
    bad = {k: v for k, v in err.items() if not v <= BOUNDS[k]}
    assert not bad, (name, bad)
