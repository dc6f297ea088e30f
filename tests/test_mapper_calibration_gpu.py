"""End-to-end runs of the mapper with cameras whose focal length is only a guess (``GlobalMapper.Solve(...,
camera_prior_focal=...)``) on the GPU: stage 0 (UpdateImagePairsConfig) and stage 1 (ViewGraphCalibrator) before
rotation averaging, the uncalibrated loss of global positioning and the doubled threshold of the angle filter, on
trivial frames and on rigs.  Bundle adjustment keeps the intrinsics fixed here, so the focals of the result are those
stage 1 set."""
import dataclasses

import numpy as np
import pytest

from glomap_b200 import estimators as E, geometry as G, mapper as M, synthetic as S

pytestmark = pytest.mark.gpu


class _RecordingRA(E.RotationEstimator):
    edges: list = []

    def EstimateRotations(self, vg, *args, **kwargs):
        _RecordingRA.edges.append((np.asarray(vg.ei).copy(), np.asarray(vg.ej).copy()))
        return super().EstimateRotations(vg, *args, **kwargs)


def _perturb_focals(start, no_prior, rng):
    f_true = start.intr_params[:, 0].copy()
    sign = np.where(rng.random(len(f_true)) < 0.5, -1.0, 1.0)
    factor = 1.0 + sign * rng.uniform(0.1, 0.2, len(f_true))
    start.intr_params[no_prior, 0] *= factor[no_prior]
    return f_true


def _keys(a, b, n):
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    return np.minimum(a, b) * n + np.maximum(a, b)


def test_trivial_frames_calibrate_the_focals_without_a_prior(monkeypatch):
    monkeypatch.setattr(M.E, "RotationEstimator", _RecordingRA)
    _RecordingRA.edges = []
    rng = np.random.default_rng(41)
    sc = S.make_scene(40, 3000, mean_track_len=6, seed=41, pixel_sigma=0.5, num_intrinsics=40)
    vg = S.view_graph_from_scene(sc, min_shared=15, noise_deg=0.5)
    pairs, is_outlier = S.make_calibration_pairs(sc, np.stack([vg.ei, vg.ej], 1), seed=41, outlier_frac=0.04)
    assert 0 < is_outlier.sum() and vg.E >= M.UPDATE_PAIRS_CONFIG_DEVICE_MIN_PAIRS      # stage 0 runs on the device
    prior = np.arange(40) % 2 == 0
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]; start.trans[:] = 0; start.points[:] = 0
    f_true = _perturb_focals(start, ~prior, rng)
    opts = M.GlobalMapperOptions()
    opts.opt_ba.optimize_intrinsics = False
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(vg, start, image_pairs=pairs, camera_prior_focal=prior)
    assert ok, mapper.log
    assert mapper.focal_refined[~prior].all()
    rel = np.abs(out.intr_params[:, 0] - f_true) / f_true
    assert rel.max() < 1e-2, (rel, mapper.log)
    assert np.array_equal(out.intr_params[prior], start.intr_params[prior])            # the prior focals are constant
    # the outlier pairs are invalidated in stage 1 and none of their edges reaches rotation averaging
    assert not mapper.pair_valid_after_calibration[is_outlier].any()
    assert mapper.image_registered.all()
    bad = _keys(vg.ei[is_outlier], vg.ej[is_outlier], 40)
    assert len(_RecordingRA.edges) == 2
    for ei, ej in _RecordingRA.edges:
        assert not np.isin(_keys(ei, ej, 40), bad).any()
    rot, cen = G.compare_reconstructions(G.quat_xyzw_to_rotmat(out.quat), out.trans, G.quat_xyzw_to_rotmat(sc.quat), sc.trans)[:2]
    assert rot < 1e-1 and cen < 1e-1, (rot, cen, mapper.log)
    # the caller's pairs are not changed
    assert all(p.is_valid for p in pairs)


def test_rigs_calibrate_the_focals_without_a_prior(monkeypatch):
    monkeypatch.setattr(M.E, "RotationEstimator", _RecordingRA)
    d = S.make_rig_dataset(2, 2, 7, 100, seed=11)
    sc = d.scene
    rng = np.random.default_rng(12)
    prior = np.array([True, False, True, False])                 # one intrinsics block per sensor
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]; start.trans[:] = 0; start.points[:] = 0
    f_true = _perturb_focals(start, ~prior, rng)
    # the F of the true poses and true intrinsics; a few CALIBRATED outliers with the F of three times the focals
    images = sc.images_scene()
    pr = np.array([[p.image_id1, p.image_id2] for p in d.image_pairs])
    calib, is_outlier = S.make_calibration_pairs(images, pr, seed=12, outlier_frac=0.05)
    assert is_outlier.sum() > 0
    pairs = []
    for p, c in zip(d.image_pairs, calib):
        pairs.append(dataclasses.replace(p, F=c.F, config=c.config if p.config != 4 else 4))
    opts = M.GlobalMapperOptions()
    opts.opt_ba.optimize_intrinsics = False
    mapper = M.GlobalMapper(opts)
    ok, out = mapper.Solve(d.view_graph, start, image_pairs=pairs, features=d.features, camera_prior_focal=prior)
    assert ok, mapper.log
    assert mapper.focal_refined[~prior].all()
    rel = np.abs(out.intr_params[:, 0] - f_true) / f_true
    assert rel.max() < 1e-2, (rel, mapper.log)
    planar = np.array([p.config == 4 for p in pairs])
    assert not mapper.pair_valid_after_calibration[is_outlier & ~planar].any()
    assert mapper.image_registered.all()
    Ri, ti = out.image_poses()
    Rg, tg = sc.image_poses()
    rot, cen = G.compare_reconstructions(Ri, ti, Rg, tg)[:2]
    assert rot < 1e-2 and cen < 1e-4, (rot, cen, mapper.log)


def test_all_priors_with_both_stages_skipped_is_the_call_without_priors():
    """Every camera with a prior and stages 0 and 1 skipped is the call without prior flags: bit for bit wherever two
    identical calls are, within 1e-6 elsewhere: the solvers' FP64 atomics reorder sums from one call to the next, and two
    identical calls of this scene were measured 7e-9 apart in the points on an H100 (the flagged call 3.4e-8)."""
    sc = S.make_scene(30, 2000, mean_track_len=6, seed=21, pixel_sigma=0.5)
    vg = S.view_graph_from_scene(sc, min_shared=15, noise_deg=0.5)
    pairs, _ = S.make_calibration_pairs(sc, np.stack([vg.ei, vg.ej], 1), seed=21, outlier_frac=0.05)
    start = sc.copy()
    start.quat[:] = [0, 0, 0, 1]; start.trans[:] = 0; start.points[:] = 0
    ok_a, a = M.GlobalMapper().Solve(vg, start, image_pairs=pairs)
    ok_r, r = M.GlobalMapper().Solve(vg, start, image_pairs=pairs)
    opts = M.GlobalMapperOptions(skip_preprocessing=True, skip_view_graph_calibration=True)
    ok_b, b = M.GlobalMapper(opts).Solve(vg, start, image_pairs=pairs, camera_prior_focal=np.ones(len(sc.intr_model), bool))
    assert ok_a and ok_r and ok_b
    for name in ("pt_obs_begin", "obs_cam", "obs_xy"):
        assert np.array_equal(getattr(a, name), getattr(b, name)), name
    for name in ("quat", "trans", "points", "intr_params"):
        x, y, z = getattr(a, name), getattr(r, name), getattr(b, name)
        assert x.shape == z.shape, name
        if np.array_equal(x, y):
            assert np.array_equal(x, z), name
        else:
            assert np.abs(z - x).max() <= 1e-6, (name, np.abs(z - x).max(), np.abs(y - x).max())
