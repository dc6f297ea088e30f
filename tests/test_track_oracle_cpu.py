"""The transcription of TrackEngine::EstablishFullTracks (oracle/track_oracle.py) against the host restatement
(glomap_b200.track_establishment) on scenes with every kind of degenerate match, its distance margin against mpmath, and
the side of the bound every boundary construction of tests/test_track_establishment_gpu.py falls on."""
import math

import mpmath
import numpy as np
import pytest

from glomap_b200 import track_establishment as T
from oracle import track_oracle as O


def random_pairs(rng, n_images=6, n_feat=150, n_pairs=60, spread=40.0, max_matches=12):
    """(features, pairs) with reversed (image_id1 > image_id2), duplicate and self matches, pairs inside one image,
    inlier lists that repeat an index, invalid pairs and empty inlier lists.  Pixels are uniform in [0, spread)^2, so
    tracks that join features of one image are kept or discarded at thres 10 alike."""
    ids = rng.choice(np.arange(1, 4 * n_images), n_images, replace=False)
    features = {int(i): rng.uniform(0.0, spread, (n_feat, 2)) for i in ids}
    pairs = []
    for k in range(n_pairs):
        i1, i2 = (int(x) for x in rng.choice(ids, 2))
        if k % 9 == 0:
            i2 = i1                                          # a pair inside one image
        m = rng.integers(0, n_feat, (int(rng.integers(1, max_matches)), 2))
        if k % 5 == 0:
            m = np.concatenate([m, m[:1]])                   # a duplicate match
        if k % 7 == 0 and i1 == i2:
            m = np.concatenate([m, [[m[0, 0], m[0, 0]]]])    # a self match gid1 == gid2
        inl = np.arange(len(m))
        if k % 4 == 0:
            inl = rng.choice(len(m), len(m) + 2)             # repeated indices, not all rows
        if k % 11 == 3:
            inl = np.zeros(0, np.int64)
        pairs.append(T.ImagePairMatches(i1, i2, m, inl, is_valid=(k % 13 != 5)))
    return features, pairs


def same(a: T.Tracks, b: T.Tracks):
    assert a.track_ids.dtype == np.uint64 and b.track_ids.dtype == np.uint64
    assert np.array_equal(a.track_ids, b.track_ids)
    assert np.array_equal(a.begin, b.begin)
    assert np.array_equal(a.obs_image, b.obs_image) and np.array_equal(a.obs_feature, b.obs_feature)


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("thres", [10.0, 25.0, 0.0, math.inf])
def test_transcription_equals_host_restatement(seed, thres):
    rng = np.random.default_rng(seed)
    features, pairs = random_pairs(rng, n_images=3 + seed % 5, spread=20.0 + 10 * (seed % 4))
    want, dis_w = O.establish_canonical(pairs, features, thres)
    got, dis_g = T.establish_full_tracks(pairs, features, T.TrackEstablishmentOptions(thres_inconsistency=thres))
    assert O.smallest_margin(pairs, features, thres) > 1e-12
    same(got, want)
    assert dis_g == dis_w
    if thres == 10.0 and seed < 4:
        assert 0 < dis_w < len(want)                         # both outcomes occur


def test_transcription_roots_depend_on_order_but_canonical_tracks_do_not():
    """The reference's track id is the union-find root, which the pair order moves; the canonical form does not."""
    rng = np.random.default_rng(4)
    features, pairs = random_pairs(rng, n_feat=8)
    roots = set()
    canon = []
    for perm in (range(len(pairs)), reversed(range(len(pairs))), rng.permutation(len(pairs))):
        ps = [pairs[int(i)] for i in perm]
        tracks, track_map, dis = O.establish_full_tracks(ps, features)
        roots.add(frozenset(tracks))
        canon.append((O.canonical(tracks, track_map), dis))
    assert len(roots) > 1
    for c, d in canon[1:]:
        same(c, canon[0][0])
        assert d == canon[0][1]


def test_self_match_degenerate_pairs_and_empty_input():
    feats = {7: np.array([[1.0, 2.0], [1.5, 2.0], [40.0, 2.0]])}
    P = T.ImagePairMatches
    tr, dis = O.establish_canonical([P(7, 7, np.array([[0, 0]]), np.array([0]))], feats)
    assert dis == 0 and tr.track_ids.tolist() == [7 << 32] and tr.begin.tolist() == [0, 1]
    tr, dis = O.establish_canonical([P(7, 7, np.array([[0, 1]]), np.array([0, 0]))], feats)   # 0.5 px apart: kept
    assert dis == 0 and tr.obs_feature.tolist() == [0, 1]
    tr, dis = O.establish_canonical([P(7, 7, np.array([[2, 0]]), np.array([0]))], feats)      # 39 px: discarded
    assert dis == 1 and tr.track_ids.tolist() == [7 << 32] and tr.begin.tolist() == [0, 0]
    tr, dis = O.establish_canonical([P(7, 7, np.array([[2, 0]]), np.array([0]), is_valid=False),
                                     P(7, 7, np.array([[2, 0]]), np.zeros(0, np.int64))], feats)
    assert dis == 0 and len(tr) == 0 and tr.begin.tolist() == [0]
    host, _ = T.establish_full_tracks([], {})
    assert len(host) == 0 and host.begin.tolist() == [0]


@pytest.mark.filterwarnings("ignore:overflow encountered")
def test_host_decision_is_the_two_rounding_norm():
    """np.linalg.norm over the last axis of 2-vectors, the host's ``inconsistent`` and the oracle's ``norm_exceeds`` are
    the same FP64 operation: sqrt(fl(fl(dx*dx) + fl(dy*dy)))."""
    rng = np.random.default_rng(9)
    d = np.concatenate([rng.uniform(-12, 12, (20000, 2)), [[10.0, 1.2e-7], [6.0, 8.0], [1e200, 0.0], [0.0, 1e-170]],
                        np.array(O.circle_points(64))])
    two = np.array([math.sqrt(x * x + y * y) for x, y in d])
    assert np.array_equal(np.linalg.norm(d, axis=-1), two)
    for thres in (0.0, 0.1, 10.0, math.inf):
        want = np.array([O.norm_exceeds((x, y), (0.0, 0.0), thres) for x, y in d])
        assert np.array_equal(T.inconsistent(d[:, 0], d[:, 1], thres), want)
        assert np.array_equal(np.linalg.norm(d, axis=-1) > thres, want)


@pytest.mark.filterwarnings("ignore:overflow encountered")
@pytest.mark.parametrize("case", O.BOUNDARY_CASES, ids=[c[0] for c in O.BOUNDARY_CASES])
def test_boundary_construction_falls_on_its_claimed_side(case):
    name, thres, a, b, norm, squared = case
    assert O.norm_exceeds(a, b, thres) == norm and O.norm_exceeds(b, a, thres) == norm
    assert O.squared_exceeds(a, b, thres) == squared and O.squared_exceeds(b, a, thres) == squared
    assert T.inconsistent(np.array([b[0] - a[0]]), np.array([b[1] - a[1]]), thres)[0] == norm
    assert O.exact_margin(a, b, thres) < 1e-10 or math.isinf(thres) or thres == 0.0


def test_circle_points_split_the_fma_and_two_rounding_forms():
    """Each circle point is decided differently by a contracted squared form than by the two-rounding one; the norm
    keeps all of them (the distance rounds to 10), and the squared forms discard some."""
    pts = O.circle_points(64)
    assert len(set(pts)) == 64
    n_sq = 0
    for p in pts:
        sq = O.squared_exceeds(p, (0.0, 0.0), 10.0)
        assert any(f != sq for f in O.fma_exceeds(p, (0.0, 0.0), 10.0))
        assert not O.norm_exceeds(p, (0.0, 0.0), 10.0)
        assert O.exact_margin((0.0, 0.0), p, 10.0) < 1e-14
        n_sq += sq
    assert 0 < n_sq < 64


def test_margin_matches_mpmath():
    rng = np.random.default_rng(11)
    pts = [(tuple(rng.uniform(-20, 20, 2)), tuple(rng.uniform(-20, 20, 2))) for _ in range(300)]
    pts += [(c[2], c[3]) for c in O.BOUNDARY_CASES if math.isfinite(c[1]) and c[1] > 0]
    pts += [((0.0, 0.0), p) for p in O.circle_points(16)]
    for thres in (10.0, 0.1, 25.5):
        for a, b in pts:
            with mpmath.workprec(400):
                d = mpmath.sqrt((mpmath.mpf(b[0]) - mpmath.mpf(a[0])) ** 2 + (mpmath.mpf(b[1]) - mpmath.mpf(a[1])) ** 2)
                t = mpmath.mpf(thres)
                want = abs(d - t) / max(d, t)
            got = O.exact_margin(a, b, thres)
            assert abs(got - float(want)) <= 1e-15 * float(want) + 1e-300, (a, b, thres, got, want)
    assert O.exact_margin((1.0, 1.0), (1.0, 1.0), 0.0) == 0.0
    assert O.exact_margin((1.0, 1.0), (1.0, 2.0), 0.0) == 1.0
    assert O.exact_margin((1.0, 1.0), (1e300, 2.0), math.inf) == 1.0


def test_smallest_margin_sees_every_same_image_pair_of_a_track():
    """Only pixels of one image inside one component count, including pairs that are not adjacent in gid order."""
    P = T.ImagePairMatches
    feats = {1: np.array([[0.0, 0.0], [5.0, 0.0], [10.0, 0.0], [40.0, 0.0]]), 2: np.zeros((3, 2))}
    # (1,0), (1,1), (1,2) in one track: the pair (0, 2) is exactly 10 apart; (1,3) is in another track
    pairs = [P(1, 2, np.array([[0, 0], [1, 0], [2, 0], [3, 1]]), np.arange(4))]
    assert O.smallest_margin(pairs, feats, 10.0) == 0.0
    assert O.smallest_margin(pairs, feats, 20.0) == 0.5
    assert O.smallest_margin(pairs[:0], feats, 10.0) == math.inf


@pytest.mark.parametrize("batch", [1, 7, 1 << 24])
def test_host_pair_scan_is_exhaustive_in_any_batch(batch):
    """The host's per-group check (bounding box, then every pair in batches) against a plain double loop, on groups of
    1-40 pixels whose boxes exceed the bound while most pairs do not."""
    rng = np.random.default_rng(21)
    sizes = rng.integers(1, 41, 300)
    gstart = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    gend = gstart + sizes
    xy = rng.uniform(0.0, 9.0, (int(sizes.sum()), 2))
    far_pt = rng.uniform(size=len(xy)) < 0.01
    xy[far_pt] += 8.0
    got = T._far_groups(xy, gstart, gend, 10.0, pairs_per_batch=batch)
    want = [any(O.norm_exceeds(xy[i], xy[j], 10.0) for i in range(s, e) for j in range(i + 1, e)) for s, e in zip(gstart, gend)]
    assert got.tolist() == want and 0 < sum(want) < len(want)
