"""Device-resident NormalizeReconstruction / UndistortImages (SURVEY.md 8(f) item 2) against the host restatements of
glomap/processors/reconstruction_normalizer.cc:5-104 and image_undistorter.cc:7-53 (glomap_b200/processors.py, which
tests/test_processors_cpu.py pins to closed-form expectations)."""
import numpy as np
import pytest

from glomap_b200 import estimators as E, geometry as G, processors as PR, synthetic as S
from oracle import filter_oracle as FO
from test_filters_cpu import ALL_CAMERAS, _params, centres_scene, missing_sensor_rig_scene, rig_dataset_scene, sweep_pixels

pytestmark = pytest.mark.gpu


def _problem(sc):
    prob = E.BAProblem(E.default_context(), sc, 3, E.first_frame_mask(sc.C))
    prob.set_state(sc.intr_params, sc.quat, sc.trans, sc.points)
    return prob


@pytest.mark.parametrize("model", [S.SIMPLE_PINHOLE, S.PINHOLE, S.SIMPLE_RADIAL, S.RADIAL])
def test_undistort_matches_host_and_feeds_the_filters(model):
    sc = S.make_scene(25, 900, mean_track_len=6, seed=61, pixel_sigma=0.5, model=model, num_intrinsics=3)
    prob = _problem(sc)
    want = PR.undistort_images(sc)
    got = prob.undistort()
    assert np.abs(got - want).max() < 1e-14
    assert np.abs(np.linalg.norm(got, axis=1) - 1).max() < 1e-15
    # the bearing-based filters give the same masks from the resident bearings as from uploaded ones
    k1, n1 = prob.filter_angle(want, 1.0)
    k2, n2 = prob.filter_angle("resident", 1.0)
    assert np.array_equal(k1, k2) and n1 == n2
    k3, n3 = prob.filter_reprojection(1e-3, bearings=want)
    k4, n4 = prob.filter_reprojection(1e-3, bearings="resident")
    assert np.array_equal(k3, k4) and n3 == n4
    prob.free()


@pytest.mark.parametrize("fixed_scale", [False, True])
def test_normalize_matches_host(fixed_scale):
    sc = S.make_scene(200, 3000, mean_track_len=6, seed=62, pixel_sigma=0.5)
    prob = _problem(sc)
    ref = sc.copy()
    s_ref, t_ref = PR.normalize_reconstruction(ref, fixed_scale=fixed_scale)
    s_dev, t_dev = prob.normalize(fixed_scale=fixed_scale)
    assert abs(s_dev - s_ref) <= 1e-12 * s_ref and np.abs(t_dev - t_ref).max() <= 1e-10 * max(1.0, np.abs(t_ref).max())
    intr, q, t, X = prob.get_state()
    assert np.abs(G.quat_xyzw_to_rotmat(q) - G.quat_xyzw_to_rotmat(sc.quat)).max() < 1e-15    # rotations untouched (identity-rotation similarity)
    assert np.abs(t - ref.trans).max() < 1e-9 and np.abs(X - ref.points).max() < 1e-9
    # the robust box of the normalised scene has the requested extent and is centred
    c = G.centers_from_pose(G.quat_xyzw_to_rotmat(q), t)
    srt = np.sort(c.astype(np.float32), axis=0)
    i0, i1 = int(0.1 * (len(c) - 1)), int(0.9 * (len(c) - 1))
    if not fixed_scale:
        assert abs(np.linalg.norm(srt[i1].astype(float) - srt[i0].astype(float)) - 10.0) < 1e-4
    assert np.abs(srt[i0:i1 + 1].astype(float).mean(0)).max() < 1e-4
    # a second call is (numerically) the identity
    s2, t2 = prob.normalize(fixed_scale=fixed_scale)
    assert abs(s2 - 1) < 1e-5 and np.abs(t2).max() < 1e-4
    prob.free()


def test_normalize_rig_problem_scales_cam_from_rig():
    rsc = S.make_rig_scene(12, 3, 600, mean_track_len=6, seed=63, pixel_sigma=0.3)
    prob = E.BAProblem(E.default_context(), rsc, 3, E.first_frame_mask(rsc.F))
    prob.set_state(rsc.intr_params, rsc.quat, rsc.trans, rsc.points)
    ref = rsc.copy()
    s_ref, t_ref = PR.normalize_reconstruction(ref)
    s_dev, t_dev = prob.normalize()
    assert abs(s_dev - s_ref) <= 1e-12 * s_ref and np.abs(t_dev - t_ref).max() <= 1e-10 * max(1.0, np.abs(t_ref).max())
    intr, q, t, X = prob.get_state()
    assert np.abs(t - ref.trans).max() < 1e-9 and np.abs(X - ref.points).max() < 1e-9
    sq, st = prob.get_sensor_poses()
    assert np.abs(st - ref.sensor_trans).max() < 1e-12
    prob.free()


# ---- undistortion against the exact inverse ---------------------------------------------------------------------------
@pytest.mark.parametrize("model,k1,k2", ALL_CAMERAS)
def test_undistort_is_the_exact_inverse_up_to_the_fold(model, k1, k2):
    """Pixels from the centre out to where d/dr [r d(r^2)] falls to 0.05, plus the image box: bearings within 1e-12 of
    the long-double inverse, and within 1e-14 of the host restatement.  (Past the fold there is no inverse; what the
    kernel returns there is not pinned.)"""
    p = _params(model, 1000.0, 500.0, k1, k2)
    xy = sweep_pixels(model, p)
    n = len(xy)
    sc = S.Scene(np.array([[0.0, 0, 0, 1]]), np.array([[0.0, 0, 5]]), np.zeros((1, 3)), np.array([0, n]),
                 np.zeros(n, np.int32), xy, np.zeros(1, np.int32), np.array([model], np.int32), p[None])
    prob = _problem(sc)
    got = prob.undistort()
    prob.free()
    want = FO.bearings_exact(model, p, xy).astype(np.float64)
    assert np.abs(got - want).max() <= 1e-12, np.abs(got - want).max()
    assert np.abs(got - PR.undistort_images(sc)).max() <= 1e-14


# ---- normalisation over image counts, offsets, duplicates and rig tables ---------------------------------------------
def _compare_normalize(sc, fixed_scale=False, min_views=3):
    prob = E.BAProblem(E.default_context(), sc, min_views, E.first_frame_mask(sc.C))
    try:
        prob.set_state(sc.intr_params, sc.quat, sc.trans, sc.points)
        ref = sc.copy()
        s_ref, t_ref = PR.normalize_reconstruction(ref, fixed_scale=fixed_scale)
        s_dev, t_dev = prob.normalize(fixed_scale=fixed_scale)
        assert abs(s_dev - s_ref) <= 1e-12 * s_ref and np.abs(t_dev - t_ref).max() <= 1e-10 * max(1.0, np.abs(t_ref).max())
        _, _, t, X = prob.get_state()
        assert np.abs(t - ref.trans).max() < 1e-9 and np.abs(X - ref.points).max() < 1e-9
        if hasattr(sc, "obs_sensor"):
            assert np.abs(prob.get_sensor_poses()[1] - ref.sensor_trans).max() < 1e-12
    finally:
        prob.free()
    return s_ref


@pytest.mark.parametrize("fixed_scale", [False, True])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 330, 100_000])
def test_normalize_matches_host_for_every_image_count(n, fixed_scale):
    """1-3 images use the whole range; 330 images trim to 265 (more than one per thread of the 256-thread block sum)."""
    _compare_normalize(centres_scene(n, seed=n), fixed_scale, min_views=1)


@pytest.mark.parametrize("kw", [dict(offset=1e4), dict(duplicate=True)])
def test_normalize_offset_and_duplicate_centres(kw):
    """Centres near 1e4 (the float coordinates round at 1e-3); all centres at one point (zero extent: scale stays 1)."""
    s = _compare_normalize(centres_scene(50, seed=5, **kw), min_views=1)
    assert (s == 1.0) == bool(kw.get("duplicate"))


@pytest.mark.parametrize("fixed_scale", [False, True])
@pytest.mark.parametrize("which", ["rig_dataset", "missing_sensor"])
def test_normalize_rigs_over_the_image_table(which, fixed_scale):
    """Three rigs (36 images of 108 frame-sensor combinations) and a dense rig with missing images: the box and the mean
    run over the images of the table, which BAProblem passes with b200sfm_ba_problem_set_images."""
    sc = rig_dataset_scene()[0] if which == "rig_dataset" else missing_sensor_rig_scene()[0]
    _compare_normalize(sc, fixed_scale)
