"""Track filters on the resident BA problem vs the numpy restatement of
glomap/processors/track_filter.cc (bit-exact masks: pure threshold tests).

The masks are compared exactly once the scene's smallest relative decision margin (``filter_oracle.smallest_margin``,
in long double) clears FP64_BOUND, so no decision can flip with the device's FP64 rounding or FMA contraction."""
import numpy as np
import pytest

from glomap_b200 import estimators as E, mapper as M, synthetic as S
from oracle import filter_oracle as FO
from test_filters_cpu import (FP64_BOUND, MAPPER_FILTERS, _params, bearings, image_scene, missing_sensor_rig_scene,
                              oracle_filter, rig_dataset_scene)

pytestmark = pytest.mark.gpu


def _problem(sc):
    prob = E.BAProblem(E.default_context(), sc, 3, E.first_frame_mask(sc.C))
    prob.set_state(sc.intr_params, sc.quat, sc.trans, sc.points)
    return prob


def _scene():
    sc = S.make_scene(30, 1500, mean_track_len=6, seed=51, pixel_sigma=1.0, model=S.SIMPLE_RADIAL, num_intrinsics=2)
    rng = np.random.default_rng(0)
    bad = rng.uniform(size=sc.N) < 0.05
    sc.obs_xy[bad] += rng.normal(scale=30.0, size=(int(bad.sum()), 2))      # outlier observations
    sc.quat = sc.quat / np.linalg.norm(sc.quat, axis=1, keepdims=True)
    return sc


def test_reprojection_filter_matches_reference_restatement():
    sc = _scene()
    prob = _problem(sc)
    for thr in (1.0, 3.0, 12.0):                                            # mapper uses max(3 - ite, 1) * thr
        keep, cnt = prob.filter_reprojection(thr)
        k0, c0 = FO.filter_reprojection(sc, thr, S.project)
        assert np.array_equal(keep, k0) and cnt == c0
    assert 0 < cnt < sc.P
    prob.free()


def test_angle_filter_matches_reference_restatement():
    sc = _scene()
    b = S.bearings_from_scene(sc)
    cal = (np.arange(sc.C) % 3 != 0).astype(np.uint8)
    prob = _problem(sc)
    for thr in (0.05, 1.0):
        keep, cnt = prob.filter_angle(b, thr, cal)
        k0, c0 = FO.filter_angle(sc, b, thr, cal)
        assert np.array_equal(keep, k0) and cnt == c0
    prob.free()


def test_triangulation_angle_filter_matches_reference_restatement():
    sc = _scene()
    prob = _problem(sc)
    for thr in (1.0, 8.0, 25.0):
        keep, cnt = prob.filter_triangulation_angle(thr)
        k0, c0 = FO.filter_triangulation_angle(sc, thr)
        assert np.array_equal(keep, k0) and cnt == c0
    prob.free()


def test_points_behind_cameras_are_dropped():
    sc = _scene()
    sc.points[:50] *= -40.0        # far behind most cameras -> z < EPS (track_filter.cc:20,71)
    prob = _problem(sc)
    keep, cnt = prob.filter_reprojection(1e9)
    k0, c0 = FO.filter_reprojection(sc, 1e9, S.project)
    assert np.array_equal(keep, k0) and cnt == c0 and not keep.all()
    prob.free()


def test_normalized_reprojection_filter_matches_oracle():
    sc = S.make_scene(12, 400, mean_track_len=5, seed=3, pixel_sigma=2.0)
    st = S.perturb_scene(sc, rot_deg=0.2)
    bear = S.bearings_from_scene(st)
    prob = E.BAProblem(E.default_context(), st, 3)
    prob.set_state(st.intr_params, st.quat, st.trans, st.points)
    for thr in (1e-3, 1e-2, 1e-1):
        keep, n = prob.filter_reprojection(thr, bear)
        k0, n0 = FO.filter_reprojection_normalized(st, bear, thr)
        assert np.array_equal(keep, k0) and n == n0
    prob.free()


# ---- the four filters at the mapper's thresholds, on image and rig scenes --------------------------------------------
SCENES = {"image": image_scene, "rig_dataset": rig_dataset_scene, "missing_sensor": missing_sensor_rig_scene}


def _device_filter(prob, kind, thr, bear, cal):
    if kind == "reprojection":
        return prob.filter_reprojection(thr)
    if kind == "normalized":
        return prob.filter_reprojection(thr, bearings=bear)
    if kind == "angle":
        return prob.filter_angle(bear, thr, cal)
    return prob.filter_triangulation_angle(thr)


def _compare_filters(sc, cal, filters):
    bear = bearings(sc)
    margin = FO.smallest_margin(sc, filters, bear, cal, S.project)
    assert margin > FP64_BOUND, margin
    prob = _problem(sc)
    try:
        for kind, thr in filters:
            want = oracle_filter(sc, kind, thr, bear, cal)
            for b in ((bear, "resident") if kind in ("normalized", "angle") else (None,)):
                keep, n = _device_filter(prob, kind, thr, b, cal)
                assert np.array_equal(keep, want[0]) and n == want[1], (kind, thr, None if b is None else str(type(b)))
    finally:
        prob.free()


@pytest.mark.parametrize("which", list(SCENES))
def test_filters_match_the_oracle_on_images_and_rigs(which):
    """Per-image models 0-3 and flags; three rigs of two sensors with per-sensor intrinsics and flags (36 of 108
    frame-sensor combinations); a dense rig with frames missing one sensor.  Uploaded and resident bearings."""
    sc, cal = SCENES[which]()
    _compare_filters(sc, cal, MAPPER_FILTERS)
    _compare_filters(sc, None, [("angle", 1.0)])


# ---- the triangulation-angle kernel's pair enumeration ----------------------------------------------------------------
def _pair(L, k):
    """(i, j) of the row-major pair index k of a track of length L, as the kernel enumerates them."""
    i = 0
    while k >= L - 1 - i:
        k -= L - 1 - i
        i += 1
    return i, i + 1 + k


def shapes_scene(seed=7):
    """One camera per observation (identity rotation) looking at its track's point along a chosen direction.  Track
    lengths 0, 1, 2, 31, 32, 33, 64, 65, 300 and 2000; for each, one track per placement of its only pair wider than 1
    deg (rays 0.3-0.7 deg off a common axis, the pair at 0 and 1.1 deg) at (0, 1), (L-2, L-1) and pair indices 31, 32,
    63, 64, one track without a wide pair and one whose rays spread over a hemisphere (Fibonacci directions).
    Then a track whose point sits on a camera centre (a zero ray, the other rays narrow) and two points seen at
    camera-frame z = 0.5e-12 and 2e-12.  Returns the scene and the expected keep of every track."""
    rng = np.random.default_rng(seed)
    arc = lambda a: np.stack([np.sin(np.radians(a)), 0 * a, np.cos(np.radians(a))], 1)   # noqa: E731
    tracks, expect = [], []                                   # (point, [camera centres])
    for L in (0, 1, 2, 31, 32, 33, 64, 65, 300, 2000):
        X = rng.normal(size=3)
        D = rng.uniform(2, 6, size=(L, 1))
        npairs = L * (L - 1) // 2
        places = sorted({(0, 1), (L - 2, L - 1)} | {_pair(L, k) for k in (31, 32, 63, 64) if k < npairs}) if L >= 2 else []
        for i, j in places:
            a = rng.uniform(0.3, 0.7, L)
            a[i], a[j] = 0.0, 1.1
            tracks.append((X, X - D * arc(a))); expect.append(True)
        tracks.append((X, X - D * arc(rng.uniform(0.3, 0.7, L)))); expect.append(False)
        if L >= 2:
            n = 3 * L + 6
            k = np.arange(n) + 0.5
            z = 1 - 2 * k / n
            ph = np.pi * (1 + 5 ** 0.5) * k
            d = np.stack([np.sqrt(1 - z * z) * np.cos(ph), np.sqrt(1 - z * z) * np.sin(ph), z], 1)
            d = d[d[:, 2] > 0.05][:L]
            tracks.append((X, X - D * d)); expect.append(True)
    tracks.append((np.zeros(3), np.stack([np.zeros(3), -2 * arc(np.array([0.3]))[0], -2 * arc(np.array([0.5]))[0]])))
    expect.append(True)
    for zz in (0.5e-12, 2e-12):
        X = np.array([0.0, 0.0, zz])
        tracks.append((X, np.stack([np.zeros(3), X - 3 * arc(np.array([10.0]))[0], X - 3 * arc(np.array([-10.0]))[0]])))
        expect.append(True)
    pts = np.array([t[0] for t in tracks])
    centres = np.concatenate([t[1] for t in tracks])
    lens = np.array([len(t[1]) for t in tracks])
    N = len(centres)
    p = _params(S.SIMPLE_PINHOLE, 1000.0, 500.0)
    Xc = np.repeat(pts, lens, axis=0) - centres
    with np.errstate(invalid="ignore"):                      # the zero ray projects to NaN: a pixel at the centre
        xy = np.nan_to_num(S.project(S.SIMPLE_PINHOLE, p, Xc), nan=500.0) + rng.normal(scale=0.5, size=(N, 2))
    sc = S.Scene(np.tile([0.0, 0, 0, 1], (N, 1)), -centres, pts, np.concatenate([[0], np.cumsum(lens)]).astype(np.int64),
                 np.arange(N, dtype=np.int32), xy, np.zeros(N, np.int32), np.zeros(1, np.int32), p[None])
    return sc, np.array(expect)


def test_triangulation_angle_pair_enumeration_and_edges():
    sc, expect = shapes_scene()
    keep, n = FO.filter_triangulation_angle(sc, 1.0)
    assert np.array_equal(keep, expect)                       # the builder places the wide pairs where it says
    _compare_filters(sc, None, [("triangulation", 1.0), ("reprojection", 3.0), ("normalized", 1e-2), ("angle", 1.0)])
    z = FO.decisions(sc, "z", 0.0)
    assert (~z[3]).sum() == 2                                 # the zero-ray observation and the one at z = 0.5e-12


def test_zero_ray_keeps_the_track():
    """Camera at t = 0, point at the origin, the other two rays 0.2 deg apart: the reference keeps the track (its zero
    ray has dot product 0 with every other); a NaN ray would drop it."""
    sc = S.Scene(np.tile([0.0, 0, 0, 1], (3, 1)), np.array([[0.0, 0, 0], [2 * np.sin(0.003), 0, 2 * np.cos(0.003)],
                                                             [2 * np.sin(0.0065), 0, 2 * np.cos(0.0065)]]),
                 np.zeros((1, 3)), np.array([0, 3]), np.arange(3, dtype=np.int32), np.full((3, 2), 500.0),
                 np.zeros(3, np.int32), np.zeros(1, np.int32), _params(S.SIMPLE_PINHOLE, 1000.0, 500.0)[None])
    prob = _problem(sc)
    keep, n = prob.filter_triangulation_angle(1.0)
    prob.free()
    assert keep.tolist() == [True] and n == 0
    assert FO.filter_triangulation_angle(sc, 1.0)[0].tolist() == [True]


# ---- stage 5's chain through the mapper -------------------------------------------------------------------------------
def test_mapper_filter_chain_on_rigs_with_per_sensor_flags():
    """GlobalMapper._filters on three rigs with per-sensor prior-focal flags: angle 1 deg, triangulation 1 deg,
    reprojection 0.1 (normalised image plane, resident bearings), each on the compacted output of the previous one,
    equals the oracle chain."""
    sc, cal = rig_dataset_scene()
    m = M.GlobalMapper()
    m._prior_focal = cal.astype(bool)          # per intrinsics block: sensor s has block s in this dataset
    chain = [("angle", 1.0), ("triangulation", 1.0), ("reprojection", 0.1)]
    got = m._filters(sc, chain)
    want = sc
    for kind, thr in chain:
        okind = "normalized" if kind == "reprojection" else kind
        bear = bearings(want)
        assert FO.smallest_margin(want, [(okind, thr)], bear, cal, S.project) > FP64_BOUND
        keep, _ = oracle_filter(want, okind, thr, bear, cal)
        want = M.drop_tracks(want, keep) if kind == "triangulation" else M.compact_observations(want, keep)
    assert want.N < sc.N
    for f in ("pt_obs_begin", "obs_frame", "obs_sensor", "obs_xy"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
