"""Gravity priors in stage 3 of the mapper on the GPU (``GlobalMapper.Solve(..., gravity=...)`` with
``opt_ra.use_gravity``): nothing changes without use_gravity, the trivial-frame stage 3 is the stratified driver
``rotation_averager.solve_rotation_averaging``, known rigs reduce to the frame graph, the priors lower the rotation error,
and an unknown cam_from_rig fails the solve as in the reference.  The CPU counterpart with the oracle is
tests/test_mapper_gravity_cpu.py.

The device rotation averager sums with FP64 atomics, so two identical calls may differ in the last bits: results are
compared bit for bit wherever two identical calls agree bit for bit, and to 1e-9 otherwise."""
import numpy as np
import pytest

from glomap_b200 import estimators as E, geometry as G, mapper as M, rotation_averager as RA, synthetic as S
from glomap_b200.gravity_refinement import get_align_rot_householder

pytestmark = pytest.mark.gpu


def _same(x, repeat, y, name, tol=1e-9):
    """y is x bit for bit when a repeat of x is, else within ``tol``."""
    assert x.shape == y.shape, name
    if np.array_equal(x, repeat):
        assert np.array_equal(x, y), (name, np.abs(x - y).max())
    else:
        assert np.abs(x - y).max() <= tol, (name, np.abs(x - y).max(), np.abs(x - repeat).max())


def _stage_3_only(use_gravity):
    o = M.GlobalMapperOptions(skip_global_positioning=True, skip_bundle_adjustment=True)
    o.opt_ra.use_gravity = use_gravity
    return o


def _rig_start(sc):
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]; start.trans[:] = 0; start.points[:] = 0
    return start


def test_gravity_without_use_gravity_changes_nothing_trivial():
    sc = S.make_scene(30, 2000, mean_track_len=6, seed=21, pixel_sigma=0.5)          # tests/test_mapper_gpu.py
    vg = S.view_graph_from_scene(sc, min_shared=15, noise_deg=0.5)
    start = _rig_start(sc)
    g = S.make_frame_gravity(G.quat_xyzw_to_rotmat(sc.quat), share=0.7, noise_deg=0.5, seed=21)
    runs = [M.GlobalMapper() for _ in range(3)]
    outs = [runs[0].Solve(vg, start), runs[1].Solve(vg, start), runs[2].Solve(vg, start, gravity=g)]
    assert all(ok for ok, _ in outs), runs[2].log
    (_, a), (_, r), (_, b) = outs
    assert np.array_equal(runs[0].image_registered, runs[2].image_registered)
    for name in ("pt_obs_begin", "obs_cam", "obs_xy"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    for name in ("quat", "trans", "points", "intr_params"):
        _same(getattr(a, name), getattr(r, name), getattr(b, name), name, tol=1e-6)


def test_gravity_without_use_gravity_changes_nothing_rigs():
    d = S.make_rig_dataset(2, 2, 7, 100, seed=11)                                   # tests/test_mapper_rig_gpu.py
    sc = d.scene
    g = S.make_frame_gravity(G.quat_xyzw_to_rotmat(sc.quat), share=0.7, noise_deg=0.5, seed=11)
    runs = [M.GlobalMapper() for _ in range(3)]
    kw = dict(image_pairs=d.image_pairs, features=d.features)
    outs = [runs[0].Solve(d.view_graph, _rig_start(sc), **kw), runs[1].Solve(d.view_graph, _rig_start(sc), **kw),
            runs[2].Solve(d.view_graph, _rig_start(sc), gravity=g, **kw)]
    assert all(ok for ok, _ in outs), runs[2].log
    (_, a), (_, r), (_, b) = outs
    assert np.array_equal(runs[0].image_registered, runs[2].image_registered)
    for name in ("pt_obs_begin", "obs_frame", "obs_sensor", "obs_xy"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    for name in ("quat", "trans", "points", "sensor_quat", "sensor_trans"):
        _same(getattr(a, name), getattr(r, name), getattr(b, name), name, tol=1e-6)


def _stage_3_by_hand(vg, g):
    """Two runs of solve_rotation_averaging on the registered pairs, each followed by the mapper's FilterRotations and
    largest component; the first from R_align / the identity, the second from the first."""
    mapper = M.GlobalMapper(_stage_3_only(True))
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


def test_trivial_stage_3_is_the_stratified_driver():
    sc = S.make_scene(60, 3000, mean_track_len=6, seed=22)
    vg = S.view_graph_from_scene(sc, min_shared=15, noise_deg=3.0, seed=22)
    assert vg.E >= M.VIEW_GRAPH_DEVICE_MIN_PAIRS                                    # the view-graph passes on the device
    g = S.make_frame_gravity(G.quat_xyzw_to_rotmat(sc.quat), share=0.7, noise_deg=0.5, seed=22)
    start = _rig_start(sc)
    mapper = M.GlobalMapper(_stage_3_only(True))
    ok, out = mapper.Solve(vg, start, gravity=g)
    assert ok, mapper.log
    R, reg, stratified = _stage_3_by_hand(vg, g)
    R2, reg2, _ = _stage_3_by_hand(vg, g)
    assert stratified == [True, True]
    assert np.array_equal(mapper.image_registered, reg) and np.array_equal(reg, reg2)
    q = [np.where(reg[:, None], G.rotmat_to_quat_xyzw_fast(x), start.quat) for x in (R, R2)]
    _same(q[0], q[1], out.quat, "rotations")
    assert sum("pairs with gravity, 1-DoF pass run" in line for line in mapper.log) == 2


def test_known_rigs_reduce_to_the_frame_graph():
    d = S.make_rig_dataset(3, 2, 10, 300, seed=23, rotation_noise_deg=4.0)
    sc = d.scene
    g = S.make_frame_gravity(G.quat_xyzw_to_rotmat(sc.quat), share=0.7, noise_deg=0.5, seed=23)
    has = ~np.isnan(g).any(axis=1)
    R0 = np.tile(np.eye(3), (sc.F, 1, 1))
    R0[has] = get_align_rot_householder(g[has])
    o = RA.RotationAveragerOptions(use_gravity=True)
    info = {}
    ok, R, _, reg = RA.solve_rotation_averaging_rig(d.view_graph, sc.image_frame, sc.image_sensor, sc.sensor_known,
                                                    sc.sensor_quat, sc.rig_ref_sensor[sc.frame_rig], o, R_init=R0, info=info,
                                                    gravity=g)
    fg = E.rig_view_graph(d.view_graph, sc.image_frame, sc.image_sensor, sc.sensor_quat)
    runs, infos = [], [{}, {}]
    for i in infos:
        runs.append(RA.solve_rotation_averaging(fg, g, o, R_init=R0, info=i))
    assert ok and all(r[0] for r in runs)
    assert info["stratified"] and all(i["stratified"] for i in infos)
    assert np.array_equal(reg, runs[0][2])
    _same(runs[0][1], runs[1][1], R, "frame rotations")


def _median_error(R, R_gt):
    """Median rotation error in degrees after the best global rotation."""
    U, _, Vt = np.linalg.svd(np.einsum("nji,njk->ik", R, R_gt))
    return float(np.median(G.rotation_angle_deg(R @ (U @ Vt), R_gt)))


def _up_error(R, g):
    """Largest angle in degrees between R e_y (the world's up-axis seen from the frame) and the frame's prior."""
    gn = g / np.linalg.norm(g, axis=1, keepdims=True)
    return float(np.degrees(np.arccos(np.clip((R[:, :, 1] * gn).sum(1), -1.0, 1.0))).max())


@pytest.mark.parametrize("kind,seed", [("trivial", 31), ("trivial", 32), ("rig", 33), ("rig", 34)])
def test_gravity_lowers_the_rotation_error(kind, seed):
    """Relative rotations at 3-5 degrees of noise, priors on 70-80 % of the frames at 0.5 degrees: stage 3 with the
    priors ends closer to the ground truth than without, and every prior is its frame's up-axis."""
    if kind == "trivial":
        sc = S.make_scene(60, 3000, mean_track_len=6, seed=seed)
        vg = S.view_graph_from_scene(sc, min_shared=15, noise_deg=4.0, seed=seed)
        share = 0.7
    else:
        d = S.make_rig_dataset(3, 2, 10, 300, seed=seed, rotation_noise_deg=5.0)
        sc, vg, share = d.scene, d.view_graph, 0.8
    R_gt = G.quat_xyzw_to_rotmat(sc.quat)
    g = S.make_frame_gravity(R_gt, share=share, noise_deg=0.5, seed=seed)
    err = {}
    for use in (False, True):
        mapper = M.GlobalMapper(_stage_3_only(use))
        ok, out = mapper.Solve(vg, _rig_start(sc), gravity=g)
        assert ok, mapper.log
        reg = mapper.frame_in_component if kind == "rig" else mapper.image_registered
        assert reg.sum() >= 0.9 * len(reg), mapper.log
        R = G.quat_xyzw_to_rotmat(out.quat)
        err[use] = _median_error(R[reg], R_gt[reg])
    has = ~np.isnan(g).any(axis=1) & reg
    up = _up_error(R[has], g[has])
    print(f"{kind} seed {seed}: {int(has.sum())} / {len(has)} priors, median rotation error {err[False]:.4f} deg without "
          f"gravity, {err[True]:.4f} deg with; largest up-axis to prior angle {up:.2e} deg")
    assert err[True] < err[False], err
    assert up < 0.5


def test_use_gravity_with_an_unknown_cam_from_rig_fails():
    d = S.make_rig_dataset(2, 3, 7, 100, seed=12)
    sc = d.scene
    start = _rig_start(sc)
    ref = sc.sensor_is_ref
    start.sensor_known[~ref] = False
    start.sensor_quat[~ref] = [0, 0, 0, 1]
    start.sensor_trans[~ref] = 0
    before = start.copy()
    g = S.make_frame_gravity(G.quat_xyzw_to_rotmat(sc.quat), share=0.7, noise_deg=0.5, seed=12)
    opts = M.GlobalMapperOptions()
    opts.opt_ra.use_gravity = True
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(d.view_graph, start, image_pairs=d.image_pairs, features=d.features, gravity=g)
    assert not ok
    assert any("use_gravity needs every cam_from_rig" in line for line in mapper.log), mapper.log
    for name in ("quat", "trans", "points", "sensor_quat", "sensor_trans", "sensor_known"):
        assert np.array_equal(getattr(out, name), getattr(before, name)), name
        assert np.array_equal(getattr(start, name), getattr(before, name)), name
