"""Device ImagePairsInlierCount (b200sfm_image_pairs_inlier_count, pair_kernels.cuh) against the host restatement
(glomap_b200/image_pair_inliers.py, which tests/test_image_pair_inliers_cpu.py pins to a scalar transcription of the
reference).  Masks and per-pair counts are compared exactly; a match whose decision quantity lies so close to its bound that
an FMA contraction could flip it is reported, and the seeded inputs must have none."""
import ctypes as ct

import numpy as np
import pytest

from glomap_b200 import _lib, image_pair_inliers as IP, synthetic as S, track_establishment as T
from glomap_b200.mapper import InlierThresholdOptions
from glomap_b200.track_establishment import ImagePairMatches

pytestmark = pytest.mark.gpu

OPTS = InlierThresholdOptions(max_epipolar_error_H=40.0)     # the synthetic PLANAR pairs then have inliers and outliers


def _borderline(pairs, features, cameras, o, scored):
    """Matches whose host decision is within rounding of its bound: r2 within 1e-9 relative of thr2; the signum within
    1e-12 of 0 relative to the magnitude of its terms; cheirality depths, ray angle or epipole products within 1e-12
    (relative where the bound exceeds 1) of their bound -- the last three only where r2 < thr2 makes them count."""
    out, bear = [], {}
    near = lambda q, b: np.abs(q - b) <= 1e-12 * np.maximum(1.0, np.abs(b))   # noqa: E731
    for k in np.flatnonzero(scored):
        d = IP.score_image_pair(pairs[k], features, cameras, o, bear)
        flag = np.abs(d["r2"] - d["thr2"]) <= 1e-9 * d["thr2"]
        pre = d["r2"] < d["thr2"]
        if "signum" in d:
            flag |= pre & (np.abs(d["signum"]) <= 1e-12 * d["signum_scale"])
        if "lambda1" in d:
            for q in ("lambda1", "lambda2"):
                flag |= pre & (near(d[q], d["min_depth"]) | near(d[q], d["max_depth"]))
            flag |= pre & (near(d["diff_angle"], IP.ANGLE_THR) | near(d["diff_epipole1"], IP.COS_EPIPOLE_THR) |
                           near(d["diff_epipole2"], IP.COS_EPIPOLE_THR))
        out += [(int(k), int(r)) for r in np.flatnonzero(flag)]
    return out


def _copy(pairs):
    return [ImagePairMatches(p.image_id1, p.image_id2, p.matches, np.asarray(p.inliers).copy(), p.is_valid, p.config,
                             p.quat_xyzw, p.trans, p.F, p.H) for p in pairs]


def _compare(pairs, features, cameras, o=OPTS, clean_inliers=True):
    host_pairs, dev_pairs = _copy(pairs), _copy(pairs)
    want = IP.image_pairs_inlier_count(host_pairs, features, cameras, o, clean_inliers)
    got = IP.image_pairs_inlier_count_device(dev_pairs, features, cameras, o, clean_inliers)
    assert _borderline(host_pairs, features, cameras, o, want.scored) == []
    assert np.array_equal(got.scored, want.scored)
    for k in range(len(pairs)):
        assert np.array_equal(got.inliers[k], want.inliers[k]), k
        assert np.array_equal(dev_pairs[k].inliers, host_pairs[k].inliers)
    w, g = want.scores[want.scored], got.scores[want.scored]
    assert np.all(np.abs(g - w) <= 1e-12 * np.abs(w)), np.max(np.abs(g - w) / np.maximum(np.abs(w), 1e-300))
    return want, got, dev_pairs


@pytest.mark.parametrize("sigma", [0.0, 0.5])
@pytest.mark.parametrize("model", [S.SIMPLE_PINHOLE, S.PINHOLE, S.SIMPLE_RADIAL, S.RADIAL])
def test_device_matches_host_on_seeded_scenes(model, sigma):
    sc = S.make_scene(25, 2500, mean_track_len=6, seed=31 + model, pixel_sigma=sigma, model=model, num_intrinsics=3)
    d = S.make_pair_matches(sc, seed=5 + model, config_weights=(0.6, 0.25, 0.15))
    features, cameras, pairs = S.pairs_from_match_arrays(d)
    pairs[3].is_valid = False
    want, got, dev = _compare(pairs, features, cameras)
    cfg = np.array([p.config for p in pairs])
    n_inl = np.array([len(x) for x in want.inliers])
    n_m = np.diff(d["match_begin"])
    for c in (2, 3, 4):       # every config has pairs with both inliers and rejected matches
        assert (n_inl[cfg == c] > 0).any() and (n_inl[cfg == c] < n_m[cfg == c]).any(), c
    # bit-for-bit reproducible
    again = IP.image_pairs_inlier_count_device(_copy(pairs), features, cameras, OPTS)
    assert np.array_equal(again.scores.view(np.uint64), got.scores.view(np.uint64))
    assert all(np.array_equal(a, b) for a, b in zip(again.inliers, got.inliers))


def test_clean_inliers_false_zero_match_pair_and_shared_cameras():
    sc = S.make_scene(12, 900, mean_track_len=5, seed=41, pixel_sigma=0.5, model=S.PINHOLE)
    features, cameras, pairs = S.pairs_from_match_arrays(S.make_pair_matches(sc, seed=2))
    shared = cameras[0]
    cameras = {i: shared for i in cameras}                     # one camera block for every image
    pairs[0].inliers = np.array([0, 1, 4])
    pairs.append(ImagePairMatches(1, 2, np.zeros((0, 2), np.int64), np.zeros(0, np.int64), config=IP.TWO_VIEW_CALIBRATED))
    pairs.append(ImagePairMatches(2, 3, np.zeros((0, 2), np.int64), np.zeros(0, np.int64), config=IP.TWO_VIEW_UNCALIBRATED))
    want, got, dev = _compare(pairs, features, cameras, clean_inliers=False)
    assert dev[0].inliers.tolist() == [0, 1, 4] and not got.scored[0]
    assert got.scored[-1] and got.scored[-2] and got.scores[-1] == 0.0 and got.scores[-2] == 0.0
    assert len(dev[-1].inliers) == 0 and len(dev[-2].inliers) == 0


@pytest.mark.parametrize("config", [IP.TWO_VIEW_CALIBRATED, IP.TWO_VIEW_UNCALIBRATED])
def test_one_pair_with_more_than_200k_matches(config):
    sc = S.make_scene(2, 220_000, mean_track_len=2, seed=43, pixel_sigma=0.5, model=S.SIMPLE_RADIAL)
    d = S.make_pair_matches(sc, seed=3, config_weights=(1.0, 0.0, 0.0))
    features, cameras, pairs = S.pairs_from_match_arrays(d)
    assert len(pairs) == 1 and len(pairs[0].matches) > 200_000
    pairs[0].config = config
    want, got, dev = _compare(pairs, features, cameras)
    assert 0.5 * len(pairs[0].matches) < len(want.inliers[0]) < len(pairs[0].matches)


def test_no_pairs_out_of_range_index_and_unsupported_models():
    from glomap_b200 import estimators as E
    ctx = E.default_context()
    lib = ctx.lib
    fb = np.zeros(1, np.int64)
    assert lib.b200sfm_image_pairs_inlier_count(ctx.handle, 0, fb.ctypes.data_as(ct.c_void_p), None, None, 0, None, None, 0,
                                                *([None] * 9), 1.0, 4.0, 4.0, None, None, None) == 0
    sc = S.make_scene(10, 600, mean_track_len=5, seed=44, pixel_sigma=0.5)
    features, cameras, pairs = S.pairs_from_match_arrays(S.make_pair_matches(sc, seed=4))
    e = next(k for k, p in enumerate(pairs) if p.config == IP.TWO_VIEW_CALIBRATED)
    bad = _copy(pairs)
    m = np.array(bad[e].matches)
    m[len(m) // 2, 1] = len(features[bad[e].image_id2])        # one past the end of image 2's features
    bad[e].matches = m
    with pytest.raises(_lib.B200Error) as ei:
        IP.image_pairs_inlier_count_device(bad, features, cameras, OPTS)
    assert ei.value.code == 1
    bad[e].matches = np.array(pairs[e].matches)
    bad[e].matches[0, 0] = -1
    with pytest.raises(_lib.B200Error) as ei:
        IP.image_pairs_inlier_count_device(bad, features, cameras, OPTS)
    assert ei.value.code == 1
    # a camera model the device does not support, on an image used only by F / H pairs: accepted (no model is read) ...
    x = pairs[e].image_id1
    fh = [p for p in pairs if not (p.config == IP.TWO_VIEW_CALIBRATED and x in (p.image_id1, p.image_id2))]
    assert any(x in (p.image_id1, p.image_id2) for p in fh)
    cams = dict(cameras)
    cams[x] = IP.Camera(9, np.asarray(cameras[x].params))
    _compare(fh, features, cams)
    # ... but not on an image of a CALIBRATED pair
    with pytest.raises(_lib.B200Error) as ei:
        IP.image_pairs_inlier_count_device(_copy([pairs[e]]), features, cams, OPTS)
    assert ei.value.code == 5


def test_scoring_filters_and_track_establishment_end_to_end():
    sc = S.make_scene(40, 4000, mean_track_len=6, seed=45, pixel_sigma=0.5, model=S.SIMPLE_RADIAL)
    features, cameras, pairs = S.pairs_from_match_arrays(S.make_pair_matches(sc, seed=6))
    o = InlierThresholdOptions(min_inlier_num=12)
    chains = []
    for score in (IP.image_pairs_inlier_count, IP.image_pairs_inlier_count_device):
        ps = _copy(pairs)
        score(ps, features, cameras, o)
        IP.filter_inlier_num(ps, o.min_inlier_num)
        IP.filter_inlier_ratio(ps, o.min_inlier_ratio)
        chains.append(ps)
    assert [p.is_valid for p in chains[0]] == [p.is_valid for p in chains[1]]
    assert 0 < sum(not p.is_valid for p in chains[0]) < len(pairs)
    want, _ = T.establish_full_tracks(chains[0], features)
    got, _ = T.establish_full_tracks_device(chains[1], features)
    assert len(want) > 1000
    assert np.array_equal(got.track_ids, want.track_ids) and np.array_equal(got.begin, want.begin)
    assert np.array_equal(got.obs_image, want.obs_image) and np.array_equal(got.obs_feature, want.obs_feature)
