"""Device track establishment (b200sfm_tracks_establish) at the shapes where a union-find and a per-image scan go wrong,
compared exactly (track ids, begin, observations, discarded count) with the canonicalised transcription of
TrackEngine::EstablishFullTracks (oracle/track_oracle.py) on small and medium cases and with the host restatement
(glomap_b200.track_establishment) on large ones.  Every comparison that is not a deliberate boundary case first requires
the scene's smallest distance margin to the inconsistency bound to exceed 1e-12; the boundary cases assert the side the
oracle's FP64 form (sqrt(fl(fl(dx*dx) + fl(dy*dy))) > thres) puts them on.  Every device call is made twice and the two
results must be byte-identical."""
import importlib.util
import math
import os
import time

import numpy as np
import pytest

from glomap_b200 import synthetic as S, track_establishment as T
from oracle import track_oracle as O

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("_track_oracle_cpu", os.path.join(os.path.dirname(__file__), "test_track_oracle_cpu.py"))
_cpu = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_cpu)
same = _cpu.same

MARGIN = 1e-12


def _gid(image, feature):
    return (np.asarray(image, np.uint64) << np.uint64(32)) | np.asarray(feature, np.uint64)


def device(g1, g2, xy1, xy2, thres=10.0):
    """The device result, from two calls that must agree byte for byte."""
    a, da = T.establish_tracks_from_matches_device(g1, g2, xy1, xy2, thres)
    b, db = T.establish_tracks_from_matches_device(g1, g2, xy1, xy2, thres)
    same(a, b)
    assert da == db
    return a, da


def device_pairs(pairs, features, thres=10.0):
    """``device`` on the inlier matches of ``pairs``; ``features[image][feature]`` may be a dict of dicts."""
    g, xy = [], []
    for g1, g2 in O._inlier_matches(pairs):
        g.append((g1, g2))
        xy.append((O._pixel(features, g1 >> 32, g1 & 0xFFFFFFFF), O._pixel(features, g2 >> 32, g2 & 0xFFFFFFFF)))
    g = np.array(g, np.uint64).reshape(-1, 2)
    xy = np.array(xy, np.float64).reshape(-1, 2, 2)
    return device(g[:, 0], g[:, 1], xy[:, 0], xy[:, 1], thres)


def against_oracle(pairs, features, thres=10.0, boundary=False):
    if not boundary:
        assert O.smallest_margin(pairs, features, thres) > MARGIN
    want, dis_w = O.establish_canonical(pairs, features, thres)
    got, dis_g = device_pairs(pairs, features, thres)
    same(got, want)
    assert dis_g == dis_w
    return got, dis_g


def one_track(nodes):
    """The Tracks of one consistent component over the global ids ``nodes``."""
    s = np.sort(np.asarray(nodes, np.uint64))
    return T.Tracks(s[:1], np.array([0, len(s)], np.int64), (s >> np.uint64(32)).astype(np.uint32),
                    (s & np.uint64(0xFFFFFFFF)).astype(np.uint32))


def fp64_smallest_margin(g1, g2, xy1, xy2, thres):
    """The smallest margin of a large scene in FP64 (every same-image pair of every component; the FP64 distance is within
    1e-15 relative of the exact one, so a result above 1e-9 puts the exact margin far above MARGIN)."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    nodes, first, inv = np.unique(np.concatenate([g1, g2]), return_index=True, return_inverse=True)
    xy = np.concatenate([xy1, xy2])[first]
    n = len(nodes)
    _, lab = connected_components(sp.coo_matrix((np.ones(len(g1), np.int8), (inv[:len(g1)], inv[len(g1):])), shape=(n, n)),
                                  directed=False)
    order = np.lexsort((nodes >> np.uint64(32), lab))
    key = lab[order].astype(np.uint64) << np.uint64(32) | (nodes[order] >> np.uint64(32))
    gs = np.concatenate([[0], np.nonzero(np.diff(key))[0] + 1])
    ge = np.concatenate([gs[1:], [n]])
    sizes = ge - gs
    out = np.inf
    for k in np.unique(sizes[sizes > 1]):                     # all pairs of the groups of size k at once
        st = gs[sizes == k]
        i, j = np.triu_indices(k, 1)
        a, b = xy[order[st[:, None] + i]], xy[order[st[:, None] + j]]
        d = np.hypot(a[..., 0] - b[..., 0], a[..., 1] - b[..., 1])
        out = min(out, float((np.abs(d - thres) / np.maximum(d, thres)).min()))
    return out


# ---- small and medium cases against the transcription ----------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("thres", [10.0, 25.0, 0.0, math.inf])
def test_random_degenerate_scenes_equal_the_transcription(seed, thres):
    rng = np.random.default_rng(100 + seed)
    features, pairs = _cpu.random_pairs(rng, n_images=4 + 2 * seed, n_feat=1000, n_pairs=250, spread=30.0 + 5 * seed)
    got, dis = against_oracle(pairs, features, thres)
    want_pub, dis_pub = T.establish_full_tracks_device(pairs, features, T.TrackEstablishmentOptions(thres_inconsistency=thres))
    same(want_pub, got)
    assert dis_pub == dis
    if thres == 10.0:
        assert 0 < dis < len(got)


def test_degenerate_matches():
    P = T.ImagePairMatches
    feats = {3: np.array([[0.0, 0.0], [2.0, 0.0], [50.0, 0.0], [1.0, 1.0]]), 9: np.array([[5.0, 5.0], [6.0, 5.0], [7.0, 5.0]])}
    # a self match alone: a one-observation track
    got, dis = against_oracle([P(3, 3, np.array([[1, 1]]), np.array([0]))], feats)
    assert dis == 0 and got.track_ids.tolist() == [3 << 32 | 1] and got.begin.tolist() == [0, 1]
    # a pair inside one image (2 px: kept; 50 px: discarded) and a reversed pair (image_id1 > image_id2)
    got, dis = against_oracle([P(3, 3, np.array([[0, 1], [2, 3]]), np.array([0, 1])), P(9, 3, np.array([[0, 1]]), np.array([0]))],
                              feats)
    assert dis == 1 and got.track_ids.tolist() == [3 << 32 | 0, 3 << 32 | 2]
    assert got.begin.tolist() == [0, 3, 3] and got.obs_image.tolist() == [3, 3, 9]
    # an inlier list that repeats an index, a duplicate and a reversed duplicate match, an invalid pair, no inliers
    pairs = [P(3, 9, np.array([[0, 0], [3, 2], [0, 0]]), np.array([0, 0, 2, 1, 1])), P(9, 3, np.array([[0, 0]]), np.array([0])),
             P(3, 9, np.array([[2, 1]]), np.array([0]), is_valid=False), P(3, 9, np.array([[2, 2]]), np.zeros(0, np.int64))]
    got, dis = against_oracle(pairs, feats)
    assert dis == 0 and got.begin.tolist() == [0, 2, 4]
    got_pub, _ = T.establish_full_tracks_device(pairs, feats)
    same(got_pub, got)
    got, dis = against_oracle(pairs[2:], feats)
    assert dis == 0 and len(got) == 0 and got.begin.tolist() == [0]


def test_id_extremes_sort_as_unsigned():
    """Image ids 0, 1, 2^31 - 1, 2^31, 2^32 - 1 and feature ids 0, 2^32 - 1: the global id reaches the top bit, so the
    track ids and the observations must sort as unsigned 64-bit values."""
    P = T.ImagePairMatches
    F = 0xFFFFFFFF
    imgs = [0, 1, 2**31 - 1, 2**31, 2**32 - 1]
    rng = np.random.default_rng(3)
    feats = {i: {0: tuple(rng.uniform(0, 3, 2)), F: tuple(rng.uniform(0, 3, 2)), 7: tuple(rng.uniform(0, 3, 2))} for i in imgs}
    pairs = [P(2**32 - 1, 2**31, np.array([[7, 0]]), np.array([0])),
             P(2**31 - 1, 0, np.array([[F, F]]), np.array([0])),
             P(0, 2**32 - 1, np.array([[F, 0]]), np.array([0])),            # joins (0, F) to (2^32 - 1, 0)
             P(1, 1, np.array([[0, F]]), np.array([0])),                    # two features of image 1, both extremes
             P(2**31, 2**31, np.array([[7, 7]]), np.array([0])),           # a self match with the top bit set
             P(2**32 - 1, 2**32 - 1, np.array([[F, F]]), np.array([0]))]    # the largest global id, alone
    got, dis = against_oracle(pairs, feats)
    assert dis == 0
    assert got.track_ids.tolist() == [F, 1 << 32, 2**31 << 32, 2**31 << 32 | 7, 2**64 - 1]
    for t in range(len(got)):
        im, ft = got.observations(t)
        g = [int(i) << 32 | int(f) for i, f in zip(im, ft)]
        assert g == sorted(g) and g[0] == int(got.track_ids[t])
    # joining (2^32 - 1, 7) to (0, F) puts features 0 and 7 of image 2^32 - 1 into one track; 100 px apart, it goes
    far = {i: dict(v) for i, v in feats.items()}
    far[2**32 - 1][0] = (100.0, 0.0)
    pairs.append(P(2**32 - 1, 0, np.array([[7, F]]), np.array([0])))
    got, dis = against_oracle(pairs, far)
    assert dis == 1 and got.track_ids.tolist() == [F, 1 << 32, 2**31 << 32 | 7, 2**64 - 1]
    assert got.begin.tolist() == [0, 0, 2, 3, 4]


def test_dense_graph_listed_twice():
    """K_256, every edge listed twice (the second time reversed, in reverse order), over 16 images with 16 features each."""
    rng = np.random.default_rng(8)
    k = np.arange(256)
    img, ft = 1 + k % 16, 3 * (k // 16)
    feats = {int(i): rng.uniform(0.0, 6.0, (64, 2)) for i in range(1, 17)}
    i, j = np.triu_indices(256, 1)
    P = T.ImagePairMatches
    pairs = [P(int(img[a]), int(img[b]), np.array([[ft[a], ft[b]]]), np.array([0])) for a, b in zip(i, j)]
    pairs += [P(p.image_id2, p.image_id1, p.matches[:, ::-1].copy(), p.inliers) for p in pairs[::-1]]
    got, dis = against_oracle(pairs, feats)
    same(got, one_track(_gid(img, ft)))
    assert dis == 0
    feats[5][3 * 7] = (40.0, 40.0)                            # one far feature discards the whole component
    got, dis = against_oracle(pairs, feats)
    assert dis == 1 and got.begin.tolist() == [0, 0]


def test_inconsistency_layout():
    """Two features of one image; three where only the first and third are far apart (not adjacent in gid order);
    33 with the only far pair (0, 32); and a track over 1000 images with one far feature pair in image 500."""
    P = T.ImagePairMatches
    for xs, discard in (([0.0, 9.0], False), ([0.0, 11.0], True), ([0.0, 6.0, 12.0], True), ([0.0, 5.0, 9.5], False),
                        ([0.0] + [5.0] * 31 + [10.5], True), ([0.0] + [5.0] * 31 + [9.5], False)):
        m = len(xs)
        feats = {4: np.array([[x, 2.0] for x in xs]), 8: np.zeros((m, 2))}
        pairs = [P(4, 8, np.array([[f, 0] for f in range(m)]), np.arange(m))]
        got, dis = against_oracle(pairs, feats)
        assert dis == int(discard) and got.begin[-1] == (0 if discard else m + 1), xs
    rng = np.random.default_rng(12)
    feats = {i: rng.uniform(0, 5, (2, 2)) for i in range(1, 1001)}
    chain = [P(i, i + 1, np.array([[0, 0]]), np.array([0])) for i in range(1, 1000)]
    got, dis = against_oracle(chain, feats)
    assert dis == 0 and got.begin.tolist() == [0, 1000]
    chain.append(P(500, 500, np.array([[0, 1]]), np.array([0])))
    got, dis = against_oracle(chain, feats)
    assert dis == 0 and got.begin.tolist() == [0, 1001]
    feats[500][1] = (60.0, 0.0)
    got, dis = against_oracle(chain, feats)
    assert dis == 1 and got.begin.tolist() == [0, 0]


def test_twenty_thousand_features_in_one_image(record_property):
    """20 000 features of one image in one track, all within the threshold: the per-image scan is O(m^2)."""
    m = 20000
    rng = np.random.default_rng(13)
    xy = rng.uniform(0.0, 7.0, (m, 2))                        # diagonal of the box < 9.9: every pair within 10
    assert math.hypot(*(xy.max(0) - xy.min(0))) < 9.9
    g1 = _gid(np.full(m, 6), np.arange(m))
    g2 = _gid(np.full(m, 7), np.zeros(m))
    xy2 = np.zeros((m, 2))
    T.establish_tracks_from_matches_device(g1[:64], g2[:64], xy[:64], xy2[:64])   # warm-up
    t0 = time.perf_counter()
    got, dis = device(g1, g2, xy, xy2)
    ms = (time.perf_counter() - t0) * 1e3 / 2
    record_property("ms_20000_features_one_image", ms)
    print(f"20000 features in one image: {ms:.1f} ms per call")
    same(got, one_track(np.concatenate([g1, g2[:1]])))
    want, dis_w = T.establish_tracks_from_matches(g1, g2, xy, xy2)
    same(got, want)
    assert dis == dis_w == 0


# ---- the inconsistency bound ------------------------------------------------------------------------------------------
def _bound_scene(cases):
    """One track per case k: features 2k (pixel a) and 2k + 1 (pixel b) of image 1, both matched to feature k of image 2."""
    n = len(cases)
    f1 = np.array([p for _, a, b in cases for p in (a, b)], np.float64).reshape(-1, 2)
    feats = {1: f1, 2: np.zeros((n, 2))}
    m = np.array([[2 * k + s, k] for k in range(n) for s in (0, 1)])
    return [T.ImagePairMatches(1, 2, m, np.arange(len(m)))], feats


@pytest.mark.parametrize("thres", [0.0, 0.1, 10.0, math.inf])
def test_inconsistency_bound(thres):
    """Integer offsets exactly at the bound, one ulp either side, (10, 1.2e-7), coordinates near 1e6 and, at 10, 64
    points on the circle where a fused multiply-add decides differently: the device keeps or discards each track as the
    reference's FP64 norm does.  With thres 0 equal pixels stay and distinct ones go."""
    cases = [(c[0], c[2], c[3]) for c in O.BOUNDARY_CASES if c[1] == thres]
    if thres == 10.0:
        cases += [(f"circle {i}", (0.0, 0.0), p) for i, p in enumerate(O.circle_points(64))]
    want_discard = [O.norm_exceeds(a, b, thres) for _, a, b in cases]
    claimed = {c[0]: c[4] for c in O.BOUNDARY_CASES}
    assert all(w == claimed.get(name, False) for (name, _, _), w in zip(cases, want_discard))
    pairs, feats = _bound_scene(cases)
    got, dis = against_oracle(pairs, feats, thres, boundary=True)
    kept = np.diff(got.begin) > 0
    wrong = [name for (name, _, _), k, w in zip(cases, kept, want_discard) if k == w]
    assert not wrong, f"decided against the FP64 norm: {wrong}"
    assert dis == sum(want_discard)


# ---- large cases against the host restatement and closed forms --------------------------------------------------------
@pytest.mark.parametrize("hub_first", [True, False])
@pytest.mark.parametrize("hub_smallest", [True, False])
def test_star_contention(hub_first, hub_smallest):
    """One feature matched to 2^20 features over 1000 images: every hook contends for the hub's root."""
    n = 1 << 20
    k = np.arange(n)
    leaves = _gid(1 + k % 1000, k // 1000)
    hub = _gid(0, 5) if hub_smallest else _gid(1001, 0)
    rng = np.random.default_rng(14)
    xy_leaf = rng.uniform(0.0, 7.0, (n, 2))
    xy_hub = np.zeros((n, 2))
    g_hub = np.full(n, hub, np.uint64)
    args = (g_hub, leaves, xy_hub, xy_leaf) if hub_first else (leaves, g_hub, xy_leaf, xy_hub)
    got, dis = device(*args)
    same(got, one_track(np.concatenate([leaves, [hub]])))
    assert dis == 0
    if hub_first and hub_smallest:
        want, dis_w = T.establish_tracks_from_matches(*args)
        same(got, want)
        assert dis_w == 0


@pytest.mark.parametrize("order", ["ascending", "descending", "random", "interleaved"])
def test_chain_depth(order):
    """A chain of 2^21 nodes (one per image, so no per-image scan), its links listed in four orders; the links alternate
    which end is gid1."""
    n = 1 << 21
    nodes = _gid(np.arange(1, n + 1), 5)
    links = np.arange(n - 1)
    if order == "descending":
        links = links[::-1]
    elif order == "random":
        links = np.random.default_rng(15).permutation(links)
    elif order == "interleaved":
        links = np.concatenate([links[1::2], links[0::2]])
    a, b = nodes[links], nodes[links + 1]
    flip = links % 2 == 1
    a, b = np.where(flip, b, a), np.where(flip, a, b)
    xy = np.zeros((n - 1, 2))
    got, dis = device(a, b, xy, xy)
    same(got, one_track(nodes))
    assert dis == 0
    if order == "random":
        want, _ = T.establish_tracks_from_matches(a, b, xy, xy)
        same(got, want)


def test_breadth():
    """2^20 two-node components, listed in random order with the larger id as gid1 half of the time."""
    n = 1 << 20
    rng = np.random.default_rng(16)
    perm = rng.permutation(n)
    g1, g2 = _gid(2, np.arange(n)), _gid(1, perm)
    swap = rng.uniform(size=n) < 0.5
    g1, g2 = np.where(swap, g2, g1), np.where(swap, g1, g2)
    xy1, xy2 = rng.uniform(0, 1000, (n, 2)), rng.uniform(0, 1000, (n, 2))
    got, dis = device(g1, g2, xy1, xy2)
    want, dis_w = T.establish_tracks_from_matches(g1, g2, xy1, xy2)
    same(got, want)
    assert dis == dis_w == 0 and len(got) == n
    assert np.array_equal(got.track_ids, _gid(1, np.arange(n))) and np.array_equal(np.diff(got.begin), np.full(n, 2))


def test_ten_million_matches_with_wrong_matches(record_property):
    """make_scene with 2.6 M tracks: the consecutive observations of every track matched (10.4 M matches), 1 % of them
    re-pointed at a random observation, which glues tracks together and puts distant features of one image into one
    track.  Device and host restatement must agree exactly."""
    sc = S.make_scene(1000, 2_600_000, mean_track_len=5, seed=17)
    order = np.argsort(sc.obs_cam, kind="stable")
    counts = np.bincount(sc.obs_cam, minlength=sc.C)
    feat = np.empty(sc.N, np.int64)
    feat[order] = np.arange(sc.N) - np.repeat(np.concatenate([[0], np.cumsum(counts)[:-1]]), counts)
    gid = _gid(sc.obs_cam.astype(np.int64) + 1, feat)
    last = np.zeros(sc.N, bool)
    last[sc.pt_obs_begin[1:] - 1] = True
    u = np.nonzero(~last)[0]
    v = u + 1
    rng = np.random.default_rng(18)
    wrong = rng.uniform(size=len(u)) < 0.01
    v[wrong] = rng.integers(0, sc.N, int(wrong.sum()))
    g1, g2, xy1, xy2 = gid[u], gid[v], sc.obs_xy[u], sc.obs_xy[v]
    assert len(g1) >= 10_000_000
    assert fp64_smallest_margin(g1, g2, xy1, xy2, 10.0) > 1e-9
    t0 = time.perf_counter()
    got, dis = device(g1, g2, xy1, xy2)
    t_dev = (time.perf_counter() - t0) / 2
    t0 = time.perf_counter()
    want, dis_w = T.establish_tracks_from_matches(g1, g2, xy1, xy2)
    t_host = time.perf_counter() - t0
    record_property("s_device_10M", t_dev)
    record_property("s_host_10M", t_host)
    print(f"10 M matches: device {t_dev:.2f} s per call, host restatement {t_host:.2f} s, {dis} of {len(got)} discarded")
    same(got, want)
    assert dis == dis_w and 0 < dis
