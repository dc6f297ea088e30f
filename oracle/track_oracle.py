"""ORACLE (test infrastructure, NOT product code) -- literal loop-and-dict
transcription of glomap::TrackEngine::EstablishFullTracks
(glomap/controllers/track_establishment.cc:5-150): BlindConcatenation
(:19-63) and TrackCollection (:65-150), in the reference's loop order.

UPSTREAM-UNVERIFIED: COLMAP's ``UnionFind`` is not in the reference tree.  It
is restated as the reference calls it: ``Union(x, y)`` sets
``parent[Find(x)] = Find(y)``, ``Find`` adds an unseen element as its own
root.  The reference's track id is the root its union-find ends with, which
depends on the order of the pairs and matches.  ``canonical`` renames every
track by the smallest global id of its component, sorts its observations by
global id and the tracks by id: the convention of
``glomap_b200.track_establishment``.

The inconsistency decision is the reference's ``(feature - other).norm() >
thres`` in FP64 with two roundings: ``sqrt(fl(fl(dx*dx) + fl(dy*dy))) >
thres`` (``norm_exceeds``; CPython rounds every operation).  The squared form
and both fused multiply-add forms are here too, for the boundary cases
(``squared_exceeds``, ``fma_exceeds``).  ``exact_margin`` is
|dist - thres| / max(thres, dist) of one pair from the exact distance of its
two pixels; ``smallest_margin`` is its minimum over every same-image pair of
every track of a scene.  A device comparison at a scene whose smallest margin
is far above the FP64 rounding cannot flip on rounding."""
import math
from fractions import Fraction

import numpy as np


class UnionFind:
    """colmap::UnionFind<uint64_t> as TrackEngine uses it (UPSTREAM-UNVERIFIED, see the module docstring)."""

    def __init__(self):
        self.parent = {}

    def find(self, x):
        if x not in self.parent:
            self.parent[x] = x
            return x
        root = x
        while self.parent[root] != root:
            root = self.parent[root]
        while self.parent[x] != root:        # path compression: changes no component and no root
            self.parent[x], x = root, self.parent[x]
        return root

    def union(self, x, y):
        rx, ry = self.find(x), self.find(y)
        if rx != ry:
            self.parent[rx] = ry


def _inlier_matches(pairs):
    """(global id 1, global id 2) of every inlier match of the valid pairs, in the reference's loop order (:23-53)."""
    for p in pairs:
        if not p.is_valid:
            continue
        for idx in p.inliers:
            idx = int(idx)
            point1_idx = int(p.matches[idx][0]) & 0xFFFFFFFF
            point2_idx = int(p.matches[idx][1]) & 0xFFFFFFFF
            yield (int(p.image_id1) & 0xFFFFFFFF) << 32 | point1_idx, (int(p.image_id2) & 0xFFFFFFFF) << 32 | point2_idx


def blind_concatenation(pairs):
    """:19-63 -- link the two features of every inlier match, the smaller global id as the second argument."""
    uf = UnionFind()
    for point_global_id1, point_global_id2 in _inlier_matches(pairs):
        if point_global_id2 < point_global_id1:
            uf.union(point_global_id1, point_global_id2)
        else:
            uf.union(point_global_id2, point_global_id1)
    return uf


def _pixel(features, image_id, feature_id):
    v = features[image_id][feature_id]
    return float(v[0]), float(v[1])


def norm_exceeds(a, b, thres):
    """(a - b).norm() > thres in FP64: dx, dy, both squares and the sum each rounded, then a correctly rounded sqrt."""
    dx, dy = float(a[0]) - float(b[0]), float(a[1]) - float(b[1])
    return math.sqrt(dx * dx + dy * dy) > thres


def squared_exceeds(a, b, thres):
    """dx*dx + dy*dy > thres*thres with every operation rounded: the form the device used before."""
    dx, dy = float(a[0]) - float(b[0]), float(a[1]) - float(b[1])
    return dx * dx + dy * dy > thres * thres


def fma_exceeds(a, b, thres):
    """(fma(dx, dx, fl(dy*dy)) > fl(thres^2), fma(dy, dy, fl(dx*dx)) > fl(thres^2)): the squared form as a compiler
    may contract it.  float(Fraction) rounds correctly, so each fma is rounded once."""
    dx, dy = float(a[0]) - float(b[0]), float(a[1]) - float(b[1])
    t2 = thres * thres

    def fma(x, y, z):
        if math.isinf(z):
            return z
        try:
            return float(Fraction(x) * Fraction(y) + Fraction(z))
        except OverflowError:
            return math.inf
    return fma(dx, dx, dy * dy) > t2, fma(dy, dy, dx * dx) > t2


def track_collection(pairs, features, uf, thres_inconsistency=10.0):
    """:65-150.  Returns (tracks {root: [(image_id, feature_id), ...]}, track_map {root: {global ids}}, discarded)."""
    track_map, track_counter = {}, {}
    for point_global_id1, point_global_id2 in _inlier_matches(pairs):
        track_id = uf.find(point_global_id1)
        track_map.setdefault(track_id, set()).update((point_global_id1, point_global_id2))
        track_counter[track_id] = track_counter.get(track_id, 0) + 1
    tracks = {}
    discarded_counter = 0
    for track_id, correspondence_set in track_map.items():
        image_id_set = {}
        for point_global_id in correspondence_set:
            image_id = point_global_id >> 32
            feature_id = point_global_id & 0xFFFFFFFF
            if image_id in image_id_set:
                for feature in image_id_set[image_id]:
                    if norm_exceeds(feature, _pixel(features, image_id, feature_id), thres_inconsistency):
                        tracks.setdefault(track_id, []).clear()
                        break
                if len(tracks.setdefault(track_id, [])) == 0:
                    discarded_counter += 1
                    break
            else:
                image_id_set[image_id] = []
            image_id_set[image_id].append(_pixel(features, image_id, feature_id))
            tracks.setdefault(track_id, []).append((image_id, feature_id))
    return tracks, track_map, discarded_counter


def establish_full_tracks(pairs, features, thres_inconsistency=10.0):
    """EstablishFullTracks (:5-17): (tracks, track_map, discarded) keyed by the union-find's roots."""
    uf = blind_concatenation(pairs)
    return track_collection(pairs, features, uf, thres_inconsistency)


def canonical(tracks, track_map):
    """The reference's result in the project's layout: a ``Tracks`` with id = smallest global id of the component,
    observations sorted by global id, tracks in ascending id (a discarded track keeps its id and has no observation)."""
    from glomap_b200.track_establishment import Tracks
    rows = sorted((min(track_map[r]), sorted((i << 32) | f for i, f in obs)) for r, obs in tracks.items())
    ids = np.array([r[0] for r in rows], np.uint64)
    begin = np.concatenate([[0], np.cumsum([len(r[1]) for r in rows], dtype=np.int64)]).astype(np.int64)
    gids = [g for r in rows for g in r[1]]
    img = np.array([g >> 32 for g in gids], np.uint32)
    feat = np.array([g & 0xFFFFFFFF for g in gids], np.uint32)
    return Tracks(ids, begin, img, feat)


def establish_canonical(pairs, features, thres_inconsistency=10.0):
    """(canonical Tracks, discarded) of the transcription."""
    tracks, track_map, discarded = establish_full_tracks(pairs, features, thres_inconsistency)
    return canonical(tracks, track_map), discarded


# ---- distance to the bound -------------------------------------------------------------------------------------------
_SQRT_BITS = 256


def _sqrt_fraction(D):
    """sqrt of the non-negative Fraction D to a relative 2^-_SQRT_BITS (exact when D is a square)."""
    if D == 0:
        return Fraction(0)
    p, q = D.numerator, D.denominator
    N = p * q
    k = max(0, (2 * _SQRT_BITS - N.bit_length()) // 2 + 1)
    return Fraction(math.isqrt(N << (2 * k)), q << k)


def exact_distance(a, b):
    """|a - b| of two FP64 pixels, from the exact difference (a Fraction to a relative 2^-256)."""
    dx = Fraction(float(a[0])) - Fraction(float(b[0]))
    dy = Fraction(float(a[1])) - Fraction(float(b[1]))
    return _sqrt_fraction(dx * dx + dy * dy)


def exact_margin(a, b, thres):
    """|dist - thres| / max(thres, dist) with dist the exact distance of the pixels a and b: 0 on the bound, 1 for any
    finite distance at thres = inf."""
    if math.isinf(thres):
        return 1.0
    d, t = exact_distance(a, b), Fraction(thres)
    if max(d, t) == 0:
        return 0.0
    return float(abs(d - t) / max(d, t))


def same_image_pairs(pairs, features):
    """Every pair of pixels (a, b) of one image inside one component of the matches (each unordered pair once)."""
    uf = blind_concatenation(pairs)
    comp = {}
    for g in uf.parent:
        comp.setdefault(uf.find(g), []).append(g)
    for members in comp.values():
        by_image = {}
        for g in sorted(members):
            by_image.setdefault(g >> 32, []).append(g & 0xFFFFFFFF)
        for image_id, feats in by_image.items():
            xy = [_pixel(features, image_id, f) for f in feats]
            for i in range(len(xy)):
                for j in range(i + 1, len(xy)):
                    yield xy[i], xy[j]


def smallest_margin(pairs, features, thres_inconsistency=10.0):
    """min ``exact_margin`` over ``same_image_pairs`` (inf for a scene without one)."""
    return min((exact_margin(a, b, thres_inconsistency) for a, b in same_image_pairs(pairs, features)), default=math.inf)


# ---- boundary constructions ------------------------------------------------------------------------------------------
_NX = math.nextafter
_X6 = 1e6 - 3.3                                  # near 1e6 the difference of two coordinates cancels exactly (Sterbenz)
_X6B = _X6 + 10.0

# (name, thres, a, b, norm_exceeds(a, b), squared_exceeds(a, b)): the side each construction is claimed to fall on
BOUNDARY_CASES = [
    ("(6, 8) at 10", 10.0, (0.0, 0.0), (6.0, 8.0), False, False),
    ("(8, 6) at 10", 10.0, (3.0, 5.0), (11.0, 11.0), False, False),
    ("(10, 0) at 10", 10.0, (0.0, 0.0), (10.0, 0.0), False, False),
    ("(0, -10) at 10", 10.0, (1.0, 2.0), (1.0, -8.0), False, False),
    ("(10 + ulp, 0) at 10", 10.0, (0.0, 0.0), (_NX(10.0, math.inf), 0.0), True, True),
    ("(10 - ulp, 0) at 10", 10.0, (0.0, 0.0), (_NX(10.0, 0.0), 0.0), False, False),
    ("(6, 8 + ulp) at 10", 10.0, (0.0, 0.0), (6.0, _NX(8.0, math.inf)), True, True),
    ("(6, 8 - ulp) at 10", 10.0, (0.0, 0.0), (6.0, _NX(8.0, 0.0)), False, False),
    ("(10, 1.2e-7) at 10", 10.0, (0.0, 0.0), (10.0, 1.2e-7), False, True),
    ("(-10, -1.2e-7) at 10", 10.0, (0.0, 0.0), (-10.0, -1.2e-7), False, True),
    ("(0.1, 0) at 0.1", 0.1, (0.0, 0.0), (0.1, 0.0), False, False),
    ("(0.1 + ulp, 0) at 0.1", 0.1, (0.0, 0.0), (_NX(0.1, 1.0), 0.0), True, True),
    ("(0.1 - ulp, 0) at 0.1", 0.1, (0.0, 0.0), (_NX(0.1, 0.0), 0.0), False, False),
    ("(0.06, 0.08) at 0.1", 0.1, (0.0, 0.0), (0.06, 0.08), False, False),
    ("equal pixels at 0", 0.0, (4.5, 7.25), (4.5, 7.25), False, False),
    ("(1e-3, 0) at 0", 0.0, (4.5, 7.25), (4.501, 7.25), True, True),
    ("(0, 1e-150) at 0", 0.0, (0.0, 0.0), (0.0, 1e-150), True, True),
    ("(1e200, 0) at inf", math.inf, (0.0, 0.0), (1e200, 0.0), False, False),
    ("(3, 4) at inf", math.inf, (0.0, 0.0), (3.0, 4.0), False, False),
    ("(10, 0) near 1e6", 10.0, (_X6, 1e6), (_X6B, 1e6), False, False),
    ("(10 + ulp(1e6), 0) near 1e6", 10.0, (_X6, 1e6), (_NX(_X6B, math.inf), 1e6), True, True),
    ("(10 - ulp(1e6), 0) near 1e6", 10.0, (_X6, 1e6), (_NX(_X6B, 0.0), 1e6), False, False),
]


def circle_points(n=64, seed=3):
    """n pixels b near the 10-px circle around a = (0, 0) (y moved by at most one ulp) where a fused multiply-add form of
    the squared distance decides differently from the two-rounding form (``fma_exceeds`` vs ``squared_exceeds``)."""
    import random
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        th = rng.uniform(0.0, 2.0 * math.pi)
        x, y = 10.0 * math.cos(th), 10.0 * math.sin(th)
        y += rng.choice((-1, 0, 1)) * math.ulp(y)
        sq = squared_exceeds((x, y), (0.0, 0.0), 10.0)
        if any(f != sq for f in fma_exceeds((x, y), (0.0, 0.0), 10.0)):
            out.append((x, y))
    return out
