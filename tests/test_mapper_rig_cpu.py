"""The rig path of the mapper driver (glomap_b200/mapper.py, ``GlobalMapper.Solve`` on a ``synthetic.RigScene``) on the
CPU: the compaction / scatter helpers, the track-to-rig-observation conversion, stage 3's image and frame registration,
and one end-to-end run with the rotation averager, the positioner, the bundle adjuster and the track filters replaced by
the ORACLE (test-only fakes, as in tests/test_mapper_oracle_cpu.py) on two rigs with one unknown sensor.  The GPU
counterpart is tests/test_mapper_rig_gpu.py."""
import dataclasses

import numpy as np
import pytest

from glomap_b200 import estimators as E, geometry as G, mapper as M, rotation_averager as RA, synthetic as S
from glomap_b200 import track_establishment as TE
from oracle import ba_oracle as B, filter_oracle as FO, gp_oracle as GPO, rig_init_oracle as RIO


def _two_rigs():
    """Rig 0: sensors 0 (reference), 1; rig 1: sensors 2 (reference), 3, 4.  Frames 0, 1 of rig 0, frames 2, 3 of rig 1;
    frame 3 lacks sensor 4's image.  Two tracks."""
    rng = np.random.default_rng(0)
    image_frame = np.array([0, 0, 1, 1, 2, 2, 2, 3, 3], np.int32)
    image_sensor = np.array([0, 1, 0, 1, 2, 3, 4, 2, 3], np.int32)
    q = lambda n: G.rotmat_to_quat_xyzw_fast(G.so3_exp(rng.normal(size=(n, 3))))   # noqa: E731
    return S.RigScene(q(4), rng.normal(size=(4, 3)), rng.normal(size=(2, 3)), np.array([0, 4, 9], np.int64),
                      np.array([0, 1, 2, 3, 1, 2, 2, 3, 3], np.int32), np.array([0, 1, 2, 2, 0, 3, 4, 2, 3], np.uint16),
                      rng.normal(size=(9, 2)), q(5), rng.normal(size=(5, 3)), np.array([0, 1, 2, 3, 4], np.int32),
                      np.zeros(5, np.int32), rng.normal(size=(5, S.INTR_STRIDE)), image_frame, image_sensor,
                      np.array([0, 0, 1, 1], np.int32), np.array([0, 0, 1, 1, 1], np.int32), np.array([0, 2], np.int32),
                      np.array([True, True, True, False, True]))


def test_dense_layout_is_the_default():
    rs = S.make_rig_scene(4, 3, 20, seed=1)
    assert rs.I == 12 and rs.image_frame.tolist() == np.repeat(np.arange(4), 3).tolist()
    assert rs.image_sensor.tolist() == np.tile(np.arange(3), 4).tolist()
    assert rs.sensor_is_ref.tolist() == [True, False, False] and rs.sensor_known.all()
    assert np.array_equal(rs.obs_image(), rs.obs_frame.astype(np.int64) * 3 + rs.obs_sensor)
    assert np.array_equal(rs.copy().image_sensor, rs.image_sensor)


def test_compact_and_scatter_frames():
    sc = _two_rigs()
    part, sensors = M.compact_frames(sc, np.array([1, 3]))
    assert sensors.tolist() == [0, 1, 2, 3]                     # sensor 4 has no image in frames 1 and 3
    assert part.F == 2 and part.S == 4 and part.I == 4
    assert part.image_frame.tolist() == [0, 0, 1, 1] and part.image_sensor.tolist() == [0, 1, 2, 3]
    assert part.rig_ref_sensor.tolist() == [0, 2] and part.sensor_is_ref.tolist() == [True, False, True, False]
    assert part.sensor_known.tolist() == [True, True, True, False]
    assert part.pt_obs_begin.tolist() == [0, 2, 5]              # every point kept, the observations of frames 0, 2 dropped
    assert part.obs_frame.tolist() == [0, 1, 0, 1, 1] and part.obs_sensor.tolist() == [1, 2, 0, 2, 3]
    assert np.array_equal(part.obs_xy, sc.obs_xy[[1, 3, 4, 7, 8]])
    assert np.array_equal(part.quat, sc.quat[[1, 3]]) and np.array_equal(part.sensor_trans, sc.sensor_trans[:4])
    # the composed image poses of the part are those of the full scene's images
    R, t = sc.image_poses()
    Rp, tp = part.image_poses()
    assert np.allclose(Rp, R[[2, 3, 7, 8]]) and np.allclose(tp, t[[2, 3, 7, 8]])
    # scatter: the solved part goes back, the other frames and sensor 4 keep theirs
    solved = part.copy()
    solved.quat[:] = [0, 0, 0, 1]; solved.trans[:] = 7.0; solved.sensor_trans[3] = [1.0, 2.0, 3.0]
    solved.sensor_known[3] = True
    solved = M.compact_observations(solved, np.array([True, False, True, True, True]))
    out = M.scatter_frames(sc, solved, np.array([1, 3]), sensors)
    assert np.array_equal(out.quat[[0, 2]], sc.quat[[0, 2]]) and (out.trans[[1, 3]] == 7.0).all()
    assert np.array_equal(out.sensor_quat[4], sc.sensor_quat[4]) and np.array_equal(out.sensor_trans[4], sc.sensor_trans[4])
    assert out.sensor_trans[3].tolist() == [1.0, 2.0, 3.0] and out.sensor_known.all()
    assert out.pt_obs_begin.tolist() == [0, 1, 4] and out.obs_frame.tolist() == [1, 1, 3, 3]
    assert out.obs_sensor.tolist() == [1, 0, 2, 3] and np.array_equal(out.obs_xy, sc.obs_xy[[1, 4, 7, 8]])
    assert np.array_equal(out.image_frame, sc.image_frame)      # the layout is the full scene's


def test_tracks_to_rig_scene_matches_tracks_to_scene():
    d = S.make_rig_dataset(2, 2, 3, 40, seed=4)
    sc = d.scene
    ids = sorted(d.features)
    tracks, _ = TE.establish_full_tracks(d.image_pairs, d.features)
    keep = [i for i in ids if sc.image_frame[i] != 2]             # frame 2 unregistered
    sel = TE.find_tracks_for_problem(tracks, keep)
    part, _ = M.compact_frames(sc, np.array([0, 1, 3, 4, 5]))
    rig = TE.tracks_to_rig_scene(sel, d.features, keep, part)
    flat = TE.tracks_to_scene(sel, d.features, keep, part.sensor_intr[part.image_sensor], sc.intr_model, sc.intr_params)
    assert np.array_equal(rig.pt_obs_begin, flat.pt_obs_begin) and np.array_equal(rig.obs_xy, flat.obs_xy)
    assert np.array_equal(rig.obs_image(), flat.obs_cam)          # image k of the part = the k-th registered id
    assert rig.P == len(sel) and not rig.points.any() and np.array_equal(rig.quat, part.quat)
    # the observations are the scene's own pixels of those images
    img = np.asarray(keep)[rig.obs_image()]
    assert np.array_equal(sc.image_frame[img], np.array([0, 1, 3, 4, 5])[rig.obs_frame])
    assert np.array_equal(sc.image_sensor[img], rig.obs_sensor)   # no sensor is dropped: sensor ids unchanged
    with pytest.raises(ValueError):
        TE.tracks_to_rig_scene(sel, d.features, keep[1:], part)


# ---- fakes --------------------------------------------------------------------------------------------------------
class FakeGP:
    def __init__(self, options, ctx=None):
        self.rng = np.random.default_rng(options.seed)

    def Solve(self, prob):
        cen = 100.0 * self.rng.uniform(-1, 1, size=(prob.C, 3))
        pts = 100.0 * self.rng.uniform(-1, 1, size=(prob.P, 3))
        S_ = len(prob.sensor_quat)
        unk = np.zeros(S_, bool) if prob.sensor_unknown is None else np.asarray(prob.sensor_unknown, bool)
        st = np.array(prob.sensor_trans, dtype=np.float64, copy=True)
        st[unk] = 0.0
        t_obs, t_rig = E.rig_world_terms(prob.quat, prob.sensor_quat, st, prob.bearings, prob.obs_cam, prob.obs_sensor)
        ru = None
        if unk.any():
            uidx = np.full(S_, -1, np.int64)
            uidx[unk] = np.arange(int(unk.sum()))
            Rf = G.quat_xyzw_to_rotmat(prob.quat)
            ru = dict(obs_sensor=uidx[prob.obs_sensor], R_rw=Rf[prob.obs_cam],
                      centers=self.rng.uniform(-1, 1, size=(int(unk.sum()), 3)))
        x, _ = GPO.solve_gp(cen, pts, prob.pt_obs_begin, prob.obs_cam, t_obs, None, GPO.GPOptions(), None, obs_offset=t_rig,
                            rig_unknown=ru)
        prob.centers, prob.points = x["centers"], x["points"]
        prob.trans = -np.einsum("nij,nj->ni", G.quat_xyzw_to_rotmat(prob.quat), prob.centers)
        if ru is not None:
            st[unk] = -np.einsum("sij,sj->si", G.quat_xyzw_to_rotmat(prob.sensor_quat)[unk], x["rig_centers"])
            prob.sensor_trans = st
        return True


@dataclasses.dataclass
class _Summary:
    final_cost: float = 0.0
    usable: int = 1


class FakeBA:
    def __init__(self, options, ctx=None):
        self.options_ = dataclasses.replace(options)
        self.summary = _Summary()

    def GetOptions(self):
        return self.options_

    def Solve(self, sc, cam_const_mask=None):
        o = self.options_
        opts = B.BAOptions(optimize_rotations=o.optimize_rotations, optimize_translation=o.optimize_translation,
                           optimize_intrinsics=o.optimize_intrinsics, optimize_points=o.optimize_points,
                           optimize_rig_poses=o.optimize_rig_poses)
        x, summ = B.solve_ba(sc.quat, sc.trans, sc.points, sc.pt_obs_begin, sc.obs_frame, sc.obs_xy, np.zeros(sc.F, np.int32),
                             sc.intr_model, sc.intr_params, opts, E.first_frame_mask(sc.F), rig=sc.rig_dict())
        sc.quat, sc.trans, sc.points, sc.intr_params = x["quat"], x["trans"], x["points"], x["intr"]
        if o.optimize_rig_poses:
            sc.sensor_quat, sc.sensor_trans = x["sq"], x["st"]
        self.summary = _Summary(summ.final_cost)
        return True


class FakeBAProblem:
    """The rig problem's filters are those of the same observations posed over its images (tests/test_rig_gpu.py checks
    the device's equality)."""

    def __init__(self, ctx, scene, min_views=3, mask=None):
        self.sc = scene.images_scene()

    def set_state(self, intr, quat, trans, points):
        pass

    def _bearings(self, bearings):
        from glomap_b200 import processors as PR
        return PR.undistort_images(self.sc) if isinstance(bearings, str) else bearings

    def filter_angle(self, bearings, thr, cal=None):
        return FO.filter_angle(self.sc, self._bearings(bearings), thr)

    def filter_reprojection(self, thr, bearings=None):
        return FO.filter_reprojection_normalized(self.sc, self._bearings(bearings), thr)

    def filter_triangulation_angle(self, thr):
        return FO.filter_triangulation_angle(self.sc, thr)

    def free(self):
        pass


def _host_passes(monkeypatch):
    """Rotation averaging on the oracle's numeric steps, the view-graph passes and stage 4 as the host restatements."""
    monkeypatch.setattr(RA, "_DeviceOps", lambda options, ctx: RIO.OracleOps(options))
    monkeypatch.setattr(M, "VIEW_GRAPH_DEVICE_MIN_PAIRS", 1 << 40)
    monkeypatch.setattr(M.TE, "establish_full_tracks_device", lambda pairs, feats, o, ctx: TE.establish_full_tracks(pairs, feats, o))
    monkeypatch.setattr(M.TE, "find_tracks_for_problem_device", lambda t, reg, o, ctx: TE.find_tracks_for_problem(t, reg, o))


def _cut_frame(vg, image_frame, f, seed=7):
    """Every pair of frame f's images rotated by 40-90 degrees, its pairs to other frames removed."""
    rng = np.random.default_rng(seed)
    fi, fj = image_frame[vg.ei], image_frame[vg.ej]
    inside, hit = (fi == f) & (fj == f), (fi == f) | (fj == f)
    w = rng.normal(size=(int(inside.sum()), 3))
    w *= np.radians(rng.uniform(40, 90, size=(len(w), 1))) / np.linalg.norm(w, axis=1, keepdims=True)
    R_rel = vg.R_rel.copy()
    R_rel[inside] = G.so3_exp(w) @ R_rel[inside]
    k = ~hit | inside
    return S.ViewGraph(vg.n_images, vg.ei[k], vg.ej[k], R_rel[k], vg.weight[k], vg.R_gt)


def test_stage_3_registers_the_frames_of_the_largest_component(monkeypatch):
    _host_passes(monkeypatch)
    d = S.make_rig_dataset(2, 2, 4, 40, seed=5)
    sc = d.scene
    vg = _cut_frame(d.view_graph, sc.image_frame, 5)
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]
    mapper = M.GlobalMapper()
    assert mapper._rotation_averaging_rig(vg, start), mapper.log
    assert np.flatnonzero(~mapper.frame_in_component).tolist() == [5]
    assert np.array_equal(mapper.image_registered, sc.image_frame != 5)
    assert mapper.frame_registered is None                     # stage 8's name is not used by stage 3
    assert np.array_equal(start.quat[5], [0, 0, 0, 1])          # the cut frame keeps its input rotation
    reg = mapper.frame_in_component
    Rf, Rt = G.quat_xyzw_to_rotmat(start.quat[reg]), G.quat_xyzw_to_rotmat(sc.quat[reg])
    A = Rf[0].T @ Rt[0]
    assert G.rotation_angle_deg(Rf @ A, Rt).max() < 1e-6


@pytest.mark.parametrize("unknown", [False, True])
def test_rig_mapper_end_to_end_with_oracle_solvers(monkeypatch, unknown):
    """Two rigs of two cameras, noise free.  With ``unknown``, rig 1's second camera starts without a cam_from_rig:
    rotation averaging estimates its rotation, global positioning its translation, and bundle adjustment refines it
    (optimize_rig_poses)."""
    _host_passes(monkeypatch)
    monkeypatch.setattr(M.E, "GlobalPositioner", FakeGP)
    monkeypatch.setattr(M.E, "BundleAdjuster", FakeBA)
    monkeypatch.setattr(M.E, "BAProblem", FakeBAProblem)
    monkeypatch.setattr(M.E, "default_context", lambda: None)
    d = S.make_rig_dataset(2, 2, 4, 60, seed=6)
    sc = d.scene
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]; start.trans[:] = 0; start.points[:] = 0
    opts = M.GlobalMapperOptions()
    opts.opt_ba.optimize_intrinsics = False
    if unknown:
        start.sensor_known[3] = False
        start.sensor_quat[3] = [0, 0, 0, 1]; start.sensor_trans[3] = 0
        opts.opt_ba.optimize_rig_poses = True
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(d.view_graph, start, image_pairs=d.image_pairs, features=d.features)
    assert ok, mapper.log
    assert mapper.image_registered.all() and out.sensor_known.all() and np.isfinite(out.sensor_trans).all()
    Ri, ti = out.image_poses()
    Rg, tg = sc.image_poses()
    rot, cen = G.compare_reconstructions(Ri, ti, Rg, tg)[:2]
    assert rot < 1e-2 and cen < 1e-4, (rot, cen, mapper.log)    # global_mapper_test.cc:84-86
    assert out.N >= sc.N
