"""The mapper's glue for cameras without a prior focal length (``GlobalMapper.Solve(..., camera_prior_focal=...)``) on
the CPU: stage 0 on the host restatement, stage 1 with the calibrator's back end replaced by the oracle
(oracle/vgc_oracle.py), and recording fakes for rotation averaging, global positioning and the filters (test-only,
monkeypatched into the driver).  Checked: an edge whose pair stage 1 invalidated does not reach stage 3, the refined
focals reach global positioning's bearings, and global positioning and the angle filter receive the prior flags."""
import numpy as np

from glomap_b200 import mapper as M, processors as PR, synthetic as S
from glomap_b200 import view_graph_calibration as VGC
from oracle import filter_oracle as FO, vgc_oracle as V

REC: dict = {}


def _oracle_backend(pp, focal, focal_constant, cam1, cam2, F, options=None, ctx=None, want_residual=False):
    o = options or VGC.ViewGraphCalibratorOptions()
    out = V.solve_vgc(pp, focal, focal_constant, cam1, cam2, F,
                      V.VGCOptions(thres_lower_ratio=o.thres_lower_ratio, thres_higher_ratio=o.thres_higher_ratio,
                                   thres_two_view_error=o.thres_two_view_error))
    usable = out["summary"].usable if out["summary"] is not None else True
    return dict(focal=out["focal"], cam_accepted=out["cam_accepted"], pair_valid=out["pair_valid"], residual=out["residual"],
                stats=dict(usable=int(usable)))


class FakeRA:
    """Records the view graph and returns its true rotations."""
    def __init__(self, options, ctx=None):
        pass

    def EstimateRotations(self, vg, R_init=None, fixed=0, gravity=None):
        REC.setdefault("ra_edges", []).append((np.asarray(vg.ei).copy(), np.asarray(vg.ej).copy()))
        return True, np.asarray(vg.R_gt).copy()


class FakeGP:
    """Records the problem and returns the true positions."""
    truth = None

    def __init__(self, options, ctx=None):
        pass

    def Solve(self, prob):
        REC["gp_bearings"] = np.asarray(prob.bearings).copy()
        REC["gp_cam_calibrated"] = None if prob.cam_calibrated is None else np.asarray(prob.cam_calibrated).copy()
        prob.trans, prob.points = FakeGP.truth.trans.copy(), FakeGP.truth.points.copy()
        return True


class FakeBAProblem:
    def __init__(self, ctx, scene, min_views=3, mask=None):
        self.sc = scene

    def set_state(self, intr, quat, trans, points):
        pass

    def filter_angle(self, bearings, thr, cal=None):
        REC["angle_cal"] = None if cal is None else np.asarray(cal).copy()
        return FO.filter_angle(self.sc, PR.undistort_images(self.sc), thr)

    def filter_reprojection(self, thr, bearings=None):
        return FO.filter_reprojection_normalized(self.sc, PR.undistort_images(self.sc), thr)

    def filter_triangulation_angle(self, thr):
        return FO.filter_triangulation_angle(self.sc, thr)

    def free(self):
        pass


def _setup(monkeypatch):
    REC.clear()
    monkeypatch.setattr(M.E, "RotationEstimator", FakeRA)
    monkeypatch.setattr(M.E, "GlobalPositioner", FakeGP)
    monkeypatch.setattr(M.E, "BAProblem", FakeBAProblem)
    monkeypatch.setattr(M.E, "default_context", lambda: None)
    monkeypatch.setattr(M, "VIEW_GRAPH_DEVICE_MIN_PAIRS", 1 << 40)
    monkeypatch.setattr(M, "UPDATE_PAIRS_CONFIG_DEVICE_MIN_PAIRS", 1 << 40)
    monkeypatch.setattr(VGC, "calibrate_arrays", _oracle_backend)
    sc = S.make_scene(12, 300, mean_track_len=5, seed=21, num_intrinsics=12)
    FakeGP.truth = sc
    vg = S.view_graph_from_scene(sc, min_shared=8)
    pairs, is_outlier = S.make_calibration_pairs(sc, np.stack([vg.ei, vg.ej], 1), seed=21, outlier_frac=0.1)
    assert is_outlier.sum() >= 2
    prior = np.arange(12) % 3 != 0                                  # blocks 0, 3, 6, 9 without a prior
    start = sc.copy()
    start.intr_params[~prior, 0] *= 1.15
    opts = M.GlobalMapperOptions(skip_bundle_adjustment=True)
    return sc, vg, pairs, is_outlier, prior, start, opts


def test_invalidated_pairs_refined_focals_and_prior_flags_reach_the_stages(monkeypatch):
    sc, vg, pairs, is_outlier, prior, start, opts = _setup(monkeypatch)
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(vg, start, image_pairs=pairs, camera_prior_focal=prior)
    assert ok, mapper.log
    # stage 1 invalidated the outlier pairs; their edges start stage 3 invalid and never reach rotation averaging
    cut = ~mapper.pair_valid_after_calibration
    assert cut[is_outlier].all()
    key = lambda a, b: np.minimum(a, b).astype(np.int64) * 12 + np.maximum(a, b)   # noqa: E731
    bad = key(vg.ei[cut], vg.ej[cut])
    assert len(REC["ra_edges"]) == 2
    for ei, ej in REC["ra_edges"]:
        assert not np.isin(key(ei, ej), bad).any()
        assert len(ei) == vg.E - cut.sum()
    # the refined focals (the truth up to the outliers' bounded pull) are written back and reach global positioning's
    # bearings
    assert mapper.focal_refined[~prior].all()
    np.testing.assert_allclose(out.intr_params[:, 0], sc.intr_params[:, 0], rtol=1e-4)
    assert np.array_equal(out.intr_params[prior], start.intr_params[prior])
    refined = sc.copy()
    refined.intr_params = out.intr_params
    assert np.array_equal(REC["gp_bearings"], PR.undistort_images(refined))
    # global positioning and the angle filter see the prior flags of every camera's block
    assert np.array_equal(REC["gp_cam_calibrated"], prior[sc.cam_intr])
    assert np.array_equal(REC["angle_cal"], prior[sc.cam_intr])
    assert all(p.is_valid for p in pairs)                           # the caller's pairs are not changed


def test_without_prior_flags_nothing_runs_and_every_camera_is_calibrated(monkeypatch):
    sc, vg, pairs, is_outlier, prior, start, opts = _setup(monkeypatch)
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(vg, start, image_pairs=pairs)
    assert ok
    assert mapper.focal_refined is None and mapper.pair_valid_after_calibration is None
    assert all(len(ei) == vg.E for ei, _ in REC["ra_edges"])
    assert REC["gp_cam_calibrated"] is None and REC["angle_cal"] is None
    assert np.array_equal(out.intr_params, start.intr_params)


def test_unusable_calibration_fails_the_solve(monkeypatch):
    sc, vg, pairs, is_outlier, prior, start, opts = _setup(monkeypatch)
    monkeypatch.setattr(VGC, "calibrate_arrays", lambda *a, **k: dict(
        focal=np.asarray(a[1], float), cam_accepted=np.zeros(len(a[1]), bool), pair_valid=np.ones(len(a[3]), bool),
        residual=None, stats=dict(usable=0)))
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(vg, start, image_pairs=pairs, camera_prior_focal=prior)
    assert not ok and "ra_edges" not in REC
    # with stage 1 skipped, stage 0 alone runs and the solve goes on
    opts.skip_view_graph_calibration = True
    ok, out = M.GlobalMapper(opts).Solve(vg, start, image_pairs=pairs, camera_prior_focal=prior)
    assert ok and np.array_equal(REC["gp_cam_calibrated"], prior[sc.cam_intr])
