"""Gravity priors in stage 3 of the mapper (glomap_b200/mapper.py, ``GlobalMapper.Solve(..., gravity=...)``) and in the
rig driver (``rotation_averager.solve_rotation_averaging_rig(..., gravity=...)``) on the CPU, the rotation averages
replaced by the ORACLE (oracle/ra_oracle.py, as in tests/test_mapper_oracle_cpu.py): the Image::HasGravity rule, the
R_align alignment of the folded pairs, the 0 / 95 % switch of the 1-DoF pass, the gauge, and the refusal of use_gravity
with an unknown cam_from_rig, on small hand-built graphs.  The GPU counterpart is tests/test_mapper_gravity_gpu.py."""
import numpy as np
import pytest

from glomap_b200 import estimators as E, geometry as G, mapper as M, rotation_averager as RA, synthetic as S
from oracle import ra_oracle as RO, rig_init_oracle as RIO


def _ra_opts(o):
    return RO.RAOptions(max_num_l1_iterations=o.max_num_l1_iterations, l1_step_convergence_threshold=o.l1_step_convergence_threshold,
                        max_num_irls_iterations=o.max_num_irls_iterations,
                        irls_step_convergence_threshold=o.irls_step_convergence_threshold,
                        irls_loss_parameter_sigma=o.irls_loss_parameter_sigma, use_weight=o.use_weight)


def oracle_estimate(o, vg, R_init, gravity):
    """RotationEstimator::EstimateRotations on the oracle: the 1-DoF frames with use_gravity and a prior."""
    n = vg.n_images
    R0 = np.tile(np.eye(3), (n, 1, 1)) if R_init is None else np.asarray(R_init, np.float64)
    if o.use_gravity and gravity is not None:
        hg = ~np.isnan(gravity).any(axis=1)
        R_align = np.tile(np.eye(3), (n, 1, 1))
        for i in np.flatnonzero(hg):
            R_align[i] = E.get_align_rot(gravity[i])
        R, info = RO.estimate_rotations_gravity(n, vg.ei, vg.ej, vg.R_rel, R0, hg, R_align, _ra_opts(o))
        return not info.get("failed", False), R
    if not o.skip_initialization and not o.use_gravity:
        R0 = E.initialize_from_maximum_spanning_tree(vg, R_init)
    th, info = RO.estimate_rotations(vg.n_images, vg.ei, vg.ej, vg.R_rel, RO.R_to_aa(R0), vg.weight, _ra_opts(o))
    return not info.get("failed", False), RO.aa_to_R(th)


class FakeRA:
    def __init__(self, options, ctx=None):
        self.o = options

    def EstimateRotations(self, vg, R_init=None, fixed=0, gravity=None):
        return oracle_estimate(self.o, vg, R_init, gravity)


class Ops(RIO.OracleOps):
    """The rig driver's numeric steps on the oracle, with the gravity-aligned solve; records every call."""
    calls = []

    def __init__(self, options):
        super().__init__(options)
        self.o = options

    def estimate_gravity(self, vg, R0, gravity):
        Ops.calls.append(("gravity", vg, np.array(gravity, copy=True)))
        return oracle_estimate(self.o, vg, R0, gravity)

    def estimate(self, vg, R0):
        Ops.calls.append(("estimate", vg, None))
        return super().estimate(vg, R0)


@pytest.fixture
def oracle_solvers(monkeypatch):
    monkeypatch.setattr(RA, "RotationEstimator", FakeRA)
    monkeypatch.setattr(M.E, "RotationEstimator", FakeRA)
    monkeypatch.setattr(RA, "_DeviceOps", lambda options, ctx: Ops(options))
    monkeypatch.setattr(M, "VIEW_GRAPH_DEVICE_MIN_PAIRS", 1 << 40)
    monkeypatch.setattr(M.E, "default_context", lambda: None)
    Ops.calls = []


def _rot(rng, n, deg=180.0):
    w = rng.normal(size=(n, 3))
    return G.so3_exp(w / np.linalg.norm(w, axis=1, keepdims=True) * np.radians(rng.uniform(5, deg, size=(n, 1))))


def _rig_graph(seed=0, F=6, gravity_frames=(0, 2, 3, 5)):
    """One rig of two sensors (0 the reference, 1 known), F frames, image 2f + s = (frame f, sensor s); the pairs (2f, 2f+1)
    inside every frame and every pair of images of consecutive frames, noise free.  Exact priors R_f e_y on
    ``gravity_frames``."""
    rng = np.random.default_rng(seed)
    R_f, R_s = _rot(rng, F), _rot(rng, 2, 30.0)
    R_s[0] = np.eye(3)
    fr, cam = np.repeat(np.arange(F), 2).astype(np.int32), np.tile([0, 1], F).astype(np.int32)
    R_img = np.einsum("nij,njk->nik", R_s[cam], R_f[fr])
    pairs = [(2 * f, 2 * f + 1) for f in range(F)]
    pairs += [(2 * f + a, 2 * f + 2 + b) for f in range(F - 1) for a in (0, 1) for b in (0, 1)]
    ei, ej = np.array(pairs, np.int32).T
    vg = S.ViewGraph(2 * F, ei, ej, R_img[ej] @ np.swapaxes(R_img[ei], -1, -2), np.ones(len(ei)), R_img)
    g = np.full((F, 3), np.nan)
    g[list(gravity_frames)] = R_f[list(gravity_frames)][:, :, 1]
    return vg, fr, cam, R_f, R_s, g


def _solve_rig(vg, fr, cam, R_s, g, known=(True, True), **opts):
    info = {}
    out = RA.solve_rotation_averaging_rig(vg, fr, cam, np.array(known), G.rotmat_to_quat_xyzw_fast(R_s),
                                          np.zeros(fr.max() + 1, np.int64), RA.RotationAveragerOptions(use_gravity=True, **opts),
                                          info=info, gravity=g)
    return out, info


def test_has_gravity_follows_image_h():
    """Image::HasGravity: the frame has a prior and the image's camera is the frame's reference camera or has a known
    cam_from_rig.  Rig 0: cameras 0 (reference), 1 (known), 2 (unknown); frame 0 has a prior, frame 1 none."""
    image_frame = np.array([0, 0, 0, 1, 1, 1])
    image_camera = np.array([0, 1, 2, 0, 1, 2])
    g = np.array([[0.0, 1.0, 0.0], [np.nan, np.nan, np.nan]])
    has = RA.image_has_gravity(image_frame, image_camera, np.array([0, 0]), np.array([False, True, False]), g)
    assert has.tolist() == [True, True, False, False, False, False]
    # the reference camera counts even when its flag says unknown (a rig's reference sensor has the identity)
    has = RA.image_has_gravity(image_frame, image_camera, np.array([2, 2]), np.array([False, False, False]), g)
    assert has.tolist() == [False, False, True, False, False, False]


def test_folded_pairs_are_aligned_with_the_frames_r_align():
    vg, fr, cam, R_f, R_s, g = _rig_graph(1)
    keep, fi, fj, R_rel = RA.fold_pairs(vg, fr.astype(np.int64), R_s, cam)
    assert (fi != fj).all() and keep.sum() == vg.E - 6                   # the 6 pairs inside a frame are dropped
    fg = S.ViewGraph(len(R_f), fi.astype(np.int32), fj.astype(np.int32), R_rel, np.ones(len(fi)), R_f)
    R0 = np.tile(np.eye(3), (len(R_f), 1, 1))
    hg, R_align, theta, Rr, fixed = E.gravity_aligned_inputs(fg, R0, g)
    assert hg.tolist() == [True, False, True, True, False, True]
    for e in range(fg.E):
        i, j = fi[e], fj[e]
        want = R_f[j] @ R_f[i].T                                        # rig2_from_rig1 from the folded image pair
        assert np.abs(R_rel[e] - want).max() < 1e-12
        want = (R_align[j].T if hg[j] else np.eye(3)) @ want @ (R_align[i] if hg[i] else np.eye(3))
        assert np.abs(Rr[e] - want).max() < 1e-12
        if hg[i] and hg[j]:                                             # a rotation about the aligned up-axis
            aa = G.so3_log(Rr[e][None])[0]
            phi = [G.so3_log((R_align[k].T @ R_f[k])[None])[0, 1] for k in (i, j)]
            assert abs(aa[0]) < 1e-9 and abs(aa[2]) < 1e-9
            assert abs((aa[1] - (phi[1] - phi[0]) + np.pi) % (2 * np.pi) - np.pi) < 1e-9
    # theta: (0, RotUpToAngle(R_align^T R0), 0) for the frames with a prior, the angle-axis of R0 elsewhere
    assert np.array_equal(theta[~hg], G.so3_log(R0)[~hg]) and not theta[hg][:, [0, 2]].any()


def test_gauge_is_the_first_frame_with_gravity():
    vg, fr, cam, R_f, R_s, g = _rig_graph(2, gravity_frames=(3, 4))
    _, fi, fj, R_rel = RA.fold_pairs(vg, fr.astype(np.int64), R_s, cam)
    fg = S.ViewGraph(len(R_f), fi.astype(np.int32), fj.astype(np.int32), R_rel, np.ones(len(fi)), R_f)
    assert E.gravity_aligned_inputs(fg, R_f, g)[4] == 3
    assert E.gravity_aligned_inputs(fg, R_f, np.full_like(g, np.nan))[4] is None
    # the 1-DoF solve keeps the gauge frame's angle and puts every prior on its frame's up-axis
    ok, R = oracle_estimate(RA.RotationAveragerOptions(use_gravity=True), fg, R_f, g)
    assert ok
    assert np.abs(R[3] - R_f[3]).max() < 1e-9
    assert np.abs(R[[3, 4]][:, :, 1] - g[[3, 4]]).max() < 1e-9
    assert G.rotation_angle_deg(R, R_f).max() < 1e-4                   # noise free: the ground truth, gauge included


@pytest.mark.parametrize("frames,stratified", [((), False), ((0, 1, 2, 3, 4, 5), False), ((0, 2, 3, 5), True)])
def test_the_1dof_pass_runs_between_0_and_95_percent(oracle_solvers, frames, stratified):
    vg, fr, cam, R_f, R_s, g = _rig_graph(3, gravity_frames=frames)
    (ok, R, _, reg), info = _solve_rig(vg, fr, cam, R_s, g)
    assert ok and reg.all()
    assert info["stratified"] == stratified
    # image pairs, the ones inside a frame included (rotation_averager.cc:22-40)
    img_g = ~np.isnan(g).any(axis=1)[fr]
    assert info["total_pairs"] == vg.E and info["gravity_pairs"] == int((img_g[vg.ei] & img_g[vg.ej]).sum())
    kinds = [c[0] for c in Ops.calls]
    assert kinds == ["gravity"] * (2 if stratified else 1)
    if stratified:                                                      # the gravity frames' largest component
        sub = Ops.calls[0][1]
        assert sub.n_images == 2 and sub.E == 4                         # frames 2 and 3 (0 and 5 are alone)
        assert not np.isnan(Ops.calls[0][2]).any()
    A = R[0].T @ R_f[0]
    assert G.rotation_angle_deg(R @ A, R_f).max() < 1e-6


def test_unknown_cam_from_rig_refuses_before_any_solve(oracle_solvers):
    vg, fr, cam, R_f, R_s, g = _rig_graph(5)
    (ok, R, _, _), info = _solve_rig(vg, fr, cam, R_s, g, known=(True, False))
    assert not ok and Ops.calls == []                                   # neither the pre-pass nor a solve ran
    assert np.array_equal(R, np.tile(np.eye(3), (len(R_f), 1, 1)))
    assert any("use_gravity" in line and "[1]" in line for line in info["log"])
    # without use_gravity the same call runs the pre-pass and the solve
    info = {}
    ok, *_ = RA.solve_rotation_averaging_rig(vg, fr, cam, np.array([True, False]), G.rotmat_to_quat_xyzw_fast(R_s),
                                             np.zeros(len(R_f), np.int64), RA.RotationAveragerOptions(), info=info, gravity=g)
    assert ok and Ops.calls and "log" not in info


def test_mapper_refuses_use_gravity_with_an_unknown_cam_from_rig(oracle_solvers):
    d = S.make_rig_dataset(2, 2, 4, 60, seed=6)
    start = d.scene.copy()
    start.quat[:] = [0, 0, 0, 1]; start.trans[:] = 0; start.points[:] = 0
    start.sensor_known[3] = False
    g = S.make_frame_gravity(G.quat_xyzw_to_rotmat(d.scene.quat), share=0.7, seed=6)
    opts = M.GlobalMapperOptions()
    opts.opt_ra.use_gravity = True
    mapper = M.GlobalMapper(opts)
    before = start.copy()
    ok, out = mapper.Solve(d.view_graph, start, gravity=g)
    assert not ok and Ops.calls == []
    assert sum("use_gravity needs every cam_from_rig" in line for line in mapper.log) == 2     # both runs refuse
    for name in ("quat", "trans", "sensor_quat", "sensor_trans", "sensor_known"):
        assert np.array_equal(getattr(out, name), getattr(before, name)) and np.array_equal(getattr(start, name), getattr(before, name))


def test_known_rigs_reduce_to_the_frame_graph(oracle_solvers):
    d = S.make_rig_dataset(2, 2, 6, 120, seed=9, rotation_noise_deg=3.0)
    sc = d.scene
    R_gt = G.quat_xyzw_to_rotmat(sc.quat)
    g = S.make_frame_gravity(R_gt, share=0.7, noise_deg=0.5, seed=9)
    o = RA.RotationAveragerOptions(use_gravity=True)
    info = {}
    ok, R, _, reg = RA.solve_rotation_averaging_rig(d.view_graph, sc.image_frame, sc.image_sensor, sc.sensor_known, sc.sensor_quat,
                                                    sc.rig_ref_sensor[sc.frame_rig], o, info=info, gravity=g)
    fg = E.rig_view_graph(d.view_graph, sc.image_frame, sc.image_sensor, sc.sensor_quat)
    info_f = {}
    ok_f, R_f, reg_f = RA.solve_rotation_averaging(fg, g, o, info=info_f)
    assert ok and ok_f and info["stratified"] and info_f["stratified"]
    assert np.array_equal(reg, reg_f) and np.array_equal(R, R_f)


def _trivial(seed=8, noise=3.0):
    sc = S.make_scene(16, 600, mean_track_len=6, seed=seed)
    vg = S.view_graph_from_scene(sc, min_shared=15, noise_deg=noise, seed=seed)
    g = S.make_frame_gravity(G.quat_xyzw_to_rotmat(sc.quat), share=0.7, noise_deg=0.5, seed=seed)
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]
    return sc, vg, g, start


def _stage_3_only(use_gravity=False):
    o = M.GlobalMapperOptions(skip_global_positioning=True, skip_bundle_adjustment=True)
    o.opt_ra.use_gravity = use_gravity
    return o


def test_gravity_without_use_gravity_changes_nothing(oracle_solvers):
    sc, vg, g, start = _trivial()
    a, b = M.GlobalMapper(_stage_3_only()), M.GlobalMapper(_stage_3_only())
    (ok_a, out_a), (ok_b, out_b) = a.Solve(vg, start), b.Solve(vg, start, gravity=g)
    assert ok_a and ok_b and np.array_equal(out_a.quat, out_b.quat) and a.log == b.log
    d = S.make_rig_dataset(2, 2, 4, 60, seed=6, rotation_noise_deg=2.0)
    rs = d.scene.copy()
    rs.quat[:] = [0, 0, 0, 1]
    g = S.make_frame_gravity(G.quat_xyzw_to_rotmat(d.scene.quat), share=0.7, seed=6)
    a, b = M.GlobalMapper(_stage_3_only()), M.GlobalMapper(_stage_3_only())
    (ok_a, out_a), (ok_b, out_b) = a.Solve(d.view_graph, rs), b.Solve(d.view_graph, rs, gravity=g)
    assert ok_a and ok_b and np.array_equal(out_a.quat, out_b.quat) and a.log == b.log
    with pytest.raises(ValueError):
        o = _stage_3_only(True)
        M.GlobalMapper(o).Solve(vg, start, gravity=g[:-1])


def stage_3_by_hand(mapper, vg, g):
    """Two runs of rotation_averager.solve_rotation_averaging on the registered pairs, each followed by the mapper's
    FilterRotations and largest component; the first from R_align / the identity, the second from the first."""
    from glomap_b200.gravity_refinement import get_align_rot_householder
    has = ~np.isnan(g).any(axis=1)
    R = np.tile(np.eye(3), (vg.n_images, 1, 1))
    R[has] = get_align_rot_householder(g[has])
    q_rel = G.rotmat_to_quat_xyzw_fast(vg.R_rel)
    valid, reg = np.ones(vg.E, bool), np.ones(vg.n_images, bool)
    stratified = []
    for _ in range(2):
        valid, reg, _ = mapper._largest_component(vg, valid, reg)
        sub, idx = M.registered_view_graph(vg, valid, reg)
        info = {}
        ok, R_sub, _ = RA.solve_rotation_averaging(sub, g[idx], M._ra_options(mapper.options_.opt_ra), R_init=R[idx], info=info)
        assert ok
        stratified.append(info["stratified"])
        R[idx] = R_sub
        valid, _ = mapper._filter_rotations(vg, q_rel, R, valid, reg, mapper.options_.inlier_thresholds.max_rotation_error)
        valid, reg, _ = mapper._largest_component(vg, valid, reg)
    return R, reg, stratified


def test_trivial_stage_3_is_the_stratified_driver(oracle_solvers):
    sc, vg, g, start = _trivial(9)
    mapper = M.GlobalMapper(_stage_3_only(True))
    ok, out = mapper.Solve(vg, start, gravity=g)
    assert ok, mapper.log
    R, reg, stratified = stage_3_by_hand(M.GlobalMapper(_stage_3_only(True)), vg, g)
    assert stratified == [True, True]
    assert np.array_equal(mapper.image_registered, reg)
    assert np.array_equal(out.quat, np.where(reg[:, None], G.rotmat_to_quat_xyzw_fast(R), start.quat))
    assert sum("pairs with gravity, 1-DoF pass run" in line for line in mapper.log) == 2
