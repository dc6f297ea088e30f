"""End-to-end runs of the mapper driver on camera rigs (``GlobalMapper.Solve`` on a ``synthetic.RigScene``) on the GPU,
in the shape of the reference's rig tests (glomap/controllers/global_mapper_test.cc:89-175): 2 rigs, 7 frames per rig,
known or unknown cam_from_rig, with its thresholds after a Sim3 alignment on the projection centres (:15-39,84-86,
211-215).  Stages 3-6 and 4 all run on the device; the CPU counterpart with the oracle is tests/test_mapper_rig_cpu.py."""
import numpy as np
import pytest

from glomap_b200 import estimators as E, geometry as G, mapper as M, synthetic as S

pytestmark = pytest.mark.gpu


def _start(sc, reset_sensors=False):
    """Nothing but the tracks, the relative rotations and the known cam_from_rig."""
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]; start.trans[:] = 0; start.points[:] = 0
    if reset_sensors:                                 # Rig::ResetSensorFromRig of every non-reference sensor (:154-161)
        ref = sc.sensor_is_ref
        start.sensor_known[~ref] = False
        start.sensor_quat[~ref] = [0, 0, 0, 1]
        start.sensor_trans[~ref] = 0
    return start


def _errors(out, sc):
    Ri, ti = out.image_poses()
    Rg, tg = sc.image_poses()
    return G.compare_reconstructions(Ri, ti, Rg, tg)[:2]


def _solve(d, start, opts=None):
    mapper = M.GlobalMapper(opts or M.GlobalMapperOptions())
    ok, out = mapper.Solve(d.view_graph, start, image_pairs=d.image_pairs, features=d.features)
    assert ok, mapper.log
    return mapper, out


def test_known_rigs_without_noise():
    d = S.make_rig_dataset(2, 2, 7, 100, seed=11)
    sc = d.scene
    assert d.view_graph.E >= M.VIEW_GRAPH_DEVICE_MIN_PAIRS       # the view-graph passes run on the device
    mapper, out = _solve(d, _start(sc))
    assert mapper.image_registered.all() and mapper.frame_in_component.all()
    rot, cen = _errors(out, sc)
    assert rot < 1e-2 and cen < 1e-4, (rot, cen, mapper.log)
    assert out.N >= sc.N
    assert np.array_equal(out.sensor_quat, sc.sensor_quat)      # the known cam_from_rig rotations are kept


@pytest.mark.parametrize("optimize_rig_poses", [False, True])
def test_unknown_rigs_without_noise(optimize_rig_poses):
    """Rotation averaging estimates the unknown rotations (the trivial-rig pre-pass, then the rig solve), global
    positioning the translations (RigUnknownBATA), bundle adjustment refines them with optimize_rig_poses."""
    d = S.make_rig_dataset(2, 3, 7, 100, seed=12)
    sc = d.scene
    opts = M.GlobalMapperOptions()
    opts.opt_ba.optimize_rig_poses = optimize_rig_poses
    mapper, out = _solve(d, _start(sc, reset_sensors=True), opts)
    assert mapper.image_registered.all()
    assert out.sensor_known.all() and np.isfinite(out.sensor_trans).all()
    rot, cen = _errors(out, sc)
    assert rot < 1e-2 and cen < 1e-4, (rot, cen, mapper.log)
    assert out.N >= sc.N


def test_known_rigs_with_pixel_noise():
    d = S.make_rig_dataset(2, 2, 7, 200, seed=13, pixel_sigma=0.5, rotation_noise_deg=0.5)
    sc = d.scene
    mapper, out = _solve(d, _start(sc))
    assert mapper.image_registered.all()
    rot, cen = _errors(out, sc)
    assert rot < 1e-1 and cen < 1e-1, (rot, cen, mapper.log)    # global_mapper_test.cc:211-215
    assert out.N >= 0.98 * sc.N


@pytest.mark.parametrize("skip_rotation_averaging", [False, True])
def test_single_sensor_rigs_reproduce_the_trivial_mapper(skip_rotation_averaging):
    """One camera per rig: the rig path computes what the trivial-frame path computes, with or without rotation
    averaging.  The tracks are identical; the poses and points agree to 1e-5, not bit for bit: the rig problem runs the
    rig paths of global positioning and bundle adjustment (the cam_from_rig composed in) where the trivial path runs
    the one-shot solves, so the sums differ in rounding, and LM stops at a function tolerance of 1e-5 with PCG solved to
    a relative residual of 1e-2.  The two runs therefore stop about 1e-7 apart (measured 5e-7 on the quaternions)."""
    d = S.make_rig_dataset(2, 1, 7, 100, seed=14, pixel_sigma=0.5, rotation_noise_deg=0.5)
    sc = d.scene
    assert np.array_equal(sc.image_frame, np.arange(sc.F))       # image f = frame f
    opts = M.GlobalMapperOptions(skip_rotation_averaging=skip_rotation_averaging)
    start = _start(sc)
    if skip_rotation_averaging:
        start.quat = sc.quat.copy()
    _, rig = _solve(d, start, opts)
    flat = sc.images_scene()
    flat.quat[:] = start.quat; flat.trans[:] = 0; flat.points[:] = 0
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(d.view_graph, flat, image_pairs=d.image_pairs, features=d.features)
    assert ok, mapper.log
    assert np.array_equal(rig.pt_obs_begin, out.pt_obs_begin) and np.array_equal(rig.obs_frame, out.obs_cam)
    tol = 1e-5
    sign = np.where((rig.quat * out.quat).sum(1, keepdims=True) < 0, -1.0, 1.0)
    np.testing.assert_allclose(rig.quat * sign, out.quat, rtol=0, atol=tol)
    np.testing.assert_allclose(rig.trans, out.trans, rtol=0, atol=tol * np.abs(out.trans).max())
    np.testing.assert_allclose(rig.points, out.points, rtol=0, atol=tol * np.abs(out.points).max())


class _Recording:
    """Wraps a solver class and records (number of frames, observations) of every problem it is given."""
    seen = []

    @classmethod
    def wrap(cls, base):
        class W(base):
            def Solve(self, prob, *args, **kw):
                cls.seen.append((len(prob.quat), np.asarray(prob.obs_xy if hasattr(prob, "obs_xy") else prob.bearings).copy()))
                return super().Solve(prob, *args, **kw)
        return W


def test_a_cut_off_frame_is_unregistered_and_keeps_its_pose(monkeypatch):
    d = S.make_rig_dataset(2, 2, 7, 100, seed=15)
    sc, vg = d.scene, d.view_graph
    cut = 9
    # every pair of the frame's own images is off by 40-90 degrees, its pairs to other frames are gone
    rng = np.random.default_rng(3)
    fi, fj = sc.image_frame[vg.ei], sc.image_frame[vg.ej]
    inside, hit = (fi == cut) & (fj == cut), (fi == cut) | (fj == cut)
    assert inside.any()
    w = rng.normal(size=(int(inside.sum()), 3))
    w *= np.radians(rng.uniform(40, 90, size=(len(w), 1))) / np.linalg.norm(w, axis=1, keepdims=True)
    R_rel = vg.R_rel.copy()
    R_rel[inside] = G.so3_exp(w) @ R_rel[inside]
    k = ~hit | inside
    d.view_graph = S.ViewGraph(vg.n_images, vg.ei[k], vg.ej[k], R_rel[k], vg.weight[k], vg.R_gt)
    start = _start(sc)
    start.quat[cut] = [0.1, 0.2, 0.3, 0.9]; start.trans[cut] = [1.0, 2.0, 3.0]
    _Recording.seen = []
    monkeypatch.setattr(M.E, "GlobalPositioner", _Recording.wrap(E.GlobalPositioner))
    monkeypatch.setattr(M.E, "BundleAdjuster", _Recording.wrap(E.BundleAdjuster))
    mapper, out = _solve(d, start)
    assert np.flatnonzero(~mapper.frame_in_component).tolist() == [cut]
    assert np.array_equal(mapper.image_registered, sc.image_frame != cut)
    assert np.array_equal(out.quat[cut], start.quat[cut]) and np.array_equal(out.trans[cut], start.trans[cut])
    assert not (out.obs_frame == cut).any()
    assert len(_Recording.seen) >= 3 and all(F == sc.F - 1 for F, _ in _Recording.seen)
    cut_xy = {tuple(r) for r in sc.obs_xy[sc.obs_frame == cut]}
    for _, arr in _Recording.seen[1:]:                           # bundle adjustment: pixel observations
        assert not any(tuple(r) in cut_xy for r in arr.reshape(-1, 2))
    assert len(_Recording.seen[0][1]) <= int((sc.obs_frame != cut).sum())
    reg = mapper.image_registered
    Ri, ti = out.image_poses()
    Rg, tg = sc.image_poses()
    rot, cen = G.compare_reconstructions(Ri[reg], ti[reg], Rg[reg], tg[reg])[:2]
    assert rot < 1e-2 and cen < 1e-4, (rot, cen, mapper.log)
