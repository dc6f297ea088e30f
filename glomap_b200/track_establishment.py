"""Track establishment on the host (SURVEY.md 8(f) item 4) -- a vectorised restatement of
``glomap::TrackEngine`` (glomap/controllers/track_establishment.{h,cc}):

* ``establish_full_tracks``  = EstablishFullTracks (:5-17): union-find over the inlier matches of the valid image
  pairs (BlindConcatenation :19-63; here connected components of the match graph), then TrackCollection (:65-150):
  a track whose features inside ONE image are further apart than ``thres_inconsistency`` pixels is discarded (its
  observation list is cleared, the track id stays, as in the reference).
* ``find_tracks_for_problem`` = FindTracksForProblem (:153-234): tracks sorted by (length, id) descending, too short /
  too long ones skipped, observations restricted to registered images, greedy per-camera quota
  ``min_num_tracks_per_view`` -- compared as an UNSIGNED 64-bit value exactly like the reference (``track_t`` counters
  against an ``int``), so the default -1 means "no quota" -- and the ``max_num_tracks`` cut-off.

Both run on the GPU as well, with the same result: ``establish_full_tracks_device`` (b200sfm_tracks_establish) and
``find_tracks_for_problem_device`` (b200sfm_tracks_select, the greedy loop in its exact data-parallel form).

Global feature id = image_id << 32 | feature_id (:48-53); a track is identified by the smallest global id of its
component (the reference roots the union at the smaller id).  Observations inside a track are sorted by global id
(the reference iterates an unordered_set; the order is immaterial to the solvers).
The GPU solvers consume the result through ``tracks_to_scene`` (``tracks_to_rig_scene`` for rigs)."""
from __future__ import annotations

import dataclasses

import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components


@dataclasses.dataclass
class TrackEstablishmentOptions:
    """track_establishment.h:9-25 (defaults identical)."""
    thres_inconsistency: float = 10.0
    min_num_tracks_per_view: int = -1
    min_num_view_per_track: int = 3
    max_num_view_per_track: int = 100
    max_num_tracks: int = 10_000_000


@dataclasses.dataclass
class ImagePairMatches:
    """The fields of glomap::ImagePair the track engine and the inlier count read (scene/image_pair.h:13-40)."""
    image_id1: int
    image_id2: int
    matches: np.ndarray          # [m,2] feature indices (image 1, image 2)
    inliers: np.ndarray          # [k] row indices into ``matches``
    is_valid: bool = True
    config: int = 0              # colmap::TwoViewGeometry::ConfigurationType (image_pair_inliers.TWO_VIEW_*)
    quat_xyzw: np.ndarray = dataclasses.field(default_factory=lambda: np.array([0.0, 0.0, 0.0, 1.0]))   # cam2_from_cam1
    trans: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros(3))
    F: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros((3, 3)))
    H: np.ndarray = dataclasses.field(default_factory=lambda: np.zeros((3, 3)))


@dataclasses.dataclass
class Tracks:
    """CSR over tracks: observations = (image_id, feature_id)."""
    track_ids: np.ndarray        # [T] uint64
    begin: np.ndarray            # [T+1]
    obs_image: np.ndarray        # [n] uint32
    obs_feature: np.ndarray      # [n] uint32

    def __len__(self):
        return len(self.track_ids)

    def observations(self, t: int):
        a, b = int(self.begin[t]), int(self.begin[t + 1])
        return self.obs_image[a:b], self.obs_feature[a:b]


def _global_ids(pairs):
    g1, g2 = [], []
    for p in pairs:
        if not p.is_valid or len(p.inliers) == 0:
            continue
        m = np.asarray(p.matches)[np.asarray(p.inliers, dtype=np.int64)]
        g1.append((np.uint64(p.image_id1) << np.uint64(32)) | m[:, 0].astype(np.uint64))
        g2.append((np.uint64(p.image_id2) << np.uint64(32)) | m[:, 1].astype(np.uint64))
    if not g1:
        return np.zeros(0, np.uint64), np.zeros(0, np.uint64)
    return np.concatenate(g1), np.concatenate(g2)


def establish_full_tracks(pairs, features: dict, options: TrackEstablishmentOptions | None = None):
    """Returns (Tracks, number of tracks discarded for inconsistency).  ``features[image_id]`` is the [n,2] pixel table
    (Image::features)."""
    o = options or TrackEstablishmentOptions()
    g1, g2 = _global_ids(pairs)
    nodes, inv = np.unique(np.concatenate([g1, g2]), return_inverse=True)
    n = len(nodes)
    if n == 0:
        return Tracks(np.zeros(0, np.uint64), np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32)), 0
    a, b = inv[:len(g1)], inv[len(g1):]
    ncomp, lab = connected_components(sp.coo_matrix((np.ones(len(a), np.int8), (a, b)), shape=(n, n)), directed=False)
    order = np.lexsort((nodes, lab))                       # by component, then by global id
    lab_s, nodes_s = lab[order], nodes[order]
    starts = np.concatenate([[0], np.nonzero(np.diff(lab_s))[0] + 1, [n]])
    track_ids = nodes_s[starts[:-1]]                        # smallest global id of each component
    img = (nodes_s >> np.uint64(32)).astype(np.uint32)
    feat = (nodes_s & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    # consistency: inside a track, features of one image must lie within thres_inconsistency of each other (:118-131)
    keep = np.ones(ncomp, bool)
    same = (lab_s[1:] == lab_s[:-1]) & (img[1:] == img[:-1])        # (sorted by gid => same-image features are adjacent)
    discarded = 0
    comp_label = lab_s[starts[:-1]]                         # ascending (lexsort by label)
    for t in np.unique(lab_s[1:][same]):
        ti = int(np.searchsorted(comp_label, t))
        s, e = int(starts[ti]), int(starts[ti + 1])
        im_t, ft_t = img[s:e], feat[s:e]
        bad = False
        for im in np.unique(im_t[np.concatenate([[False], im_t[1:] == im_t[:-1]])]):
            xy = np.asarray(features[int(im)], dtype=np.float64)[ft_t[im_t == im]]
            d = np.linalg.norm(xy[:, None, :] - xy[None, :, :], axis=-1)
            if (d > o.thres_inconsistency).any():
                bad = True
                break
        if bad:
            keep[ti] = False
            discarded += 1
    lens = np.diff(starts)
    lens_kept = np.where(keep, lens, 0)
    sel = np.repeat(keep, lens)
    # component order above is by label; present the tracks in ascending track id
    perm = np.argsort(track_ids, kind="stable")
    begin = np.concatenate([[0], np.cumsum(lens_kept[perm])]).astype(np.int64)
    pos = np.concatenate([np.arange(starts[t], starts[t + 1]) for t in perm if keep[t]]) if sel.any() else np.zeros(0, np.int64)
    return Tracks(track_ids[perm], begin, img[pos], feat[pos]), discarded


def establish_full_tracks_device(pairs, features: dict, options: TrackEstablishmentOptions | None = None, ctx=None):
    """EstablishFullTracks on the GPU (b200sfm_tracks_establish: union-find, track collection, inconsistency rule); same
    return value as ``establish_full_tracks``.  The host only concatenates the inlier matches of the valid pairs."""
    import ctypes as ct

    from . import _lib, estimators as E
    o = options or TrackEstablishmentOptions()
    ctx = ctx or E.default_context()
    g1, g2 = _global_ids(pairs)
    M = len(g1)
    xy1, xy2 = np.empty((M, 2)), np.empty((M, 2))
    pos = 0
    for p in pairs:
        if not p.is_valid or len(p.inliers) == 0:
            continue
        m = np.asarray(p.matches)[np.asarray(p.inliers, dtype=np.int64)]
        k = len(m)
        xy1[pos:pos + k] = np.asarray(features[int(p.image_id1)], dtype=np.float64)[m[:, 0]]
        xy2[pos:pos + k] = np.asarray(features[int(p.image_id2)], dtype=np.float64)[m[:, 1]]
        pos += k
    g1, g2 = np.ascontiguousarray(g1, np.uint64), np.ascontiguousarray(g2, np.uint64)
    h = ct.c_void_p()
    nt, nobs, ndis = ct.c_int64(), ct.c_int64(), ct.c_int64()
    ptr = lambda a: a.ctypes.data_as(ct.c_void_p) if len(a) else None   # noqa: E731
    _lib.check(ctx.handle, ctx.lib.b200sfm_tracks_establish(ctx.handle, M, ptr(g1), ptr(g2), ptr(xy1), ptr(xy2),
                                                            float(o.thres_inconsistency), ct.byref(h), ct.byref(nt), ct.byref(nobs),
                                                            ct.byref(ndis)))
    try:
        T, n = nt.value, nobs.value
        ids, begin = np.zeros(T, np.uint64), np.zeros(T + 1, np.int64)
        img, feat = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        _lib.check(ctx.handle, ctx.lib.b200sfm_tracks_get(h, ptr(ids), begin.ctypes.data_as(ct.c_void_p), ptr(img), ptr(feat)))
    finally:
        ctx.lib.b200sfm_tracks_free(h)
    return Tracks(ids, begin, img, feat), int(ndis.value)


def find_tracks_for_problem(tracks: Tracks, registered_images, options: TrackEstablishmentOptions | None = None) -> Tracks:
    """FindTracksForProblem on the host, a loop over the tracks.  Only ``min_num_tracks_per_view`` is compared as an
    unsigned value here; the reference also converts ``min_num_view_per_track``, ``max_num_view_per_track`` and
    ``max_num_tracks`` to unsigned, so for a NEGATIVE value of one of those three this loop differs from the reference
    (and from ``find_tracks_for_problem_device``, which follows the reference).  Non-negative values agree."""
    o = options or TrackEstablishmentOptions()
    reg = np.asarray(sorted(int(i) for i in registered_images), np.int64)
    lens = np.diff(tracks.begin)
    cand = np.nonzero((lens >= o.min_num_view_per_track) & (lens <= o.max_num_view_per_track))[0]
    # std::sort(rbegin, rend) on (length, track_id): descending by length, then by id (:166)
    cand = cand[np.lexsort((tracks.track_ids[cand], lens[cand]))[::-1]]
    quota = o.min_num_tracks_per_view & 0xFFFFFFFFFFFFFFFF       # int -> uint64 conversion of the comparison (:209)
    counter = {int(i): 0 for i in reg}
    cameras_left = len(counter)
    out_ids, out_img, out_feat, out_begin = [], [], [], [0]
    for t in cand:
        im, ft = tracks.observations(int(t))
        m = np.isin(im, reg)
        im, ft = im[m], ft[m]
        if len(np.unique(im)) < o.min_num_view_per_track:
            continue
        added = False
        for i in im:
            c = counter[int(i)]
            if c > quota:
                continue
            counter[int(i)] = c + 1
            if c + 1 > quota:
                cameras_left -= 1
            if not added:
                out_ids.append(tracks.track_ids[t]); out_img.append(im); out_feat.append(ft)
                out_begin.append(out_begin[-1] + len(im))
                added = True
        if cameras_left == 0 or len(out_ids) > o.max_num_tracks:
            break
    if not out_ids:
        return Tracks(np.zeros(0, np.uint64), np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32))
    return Tracks(np.asarray(out_ids, np.uint64), np.asarray(out_begin, np.int64), np.concatenate(out_img).astype(np.uint32),
                  np.concatenate(out_feat).astype(np.uint32))


def restrict_to_images(tracks: Tracks, image_ids) -> Tracks:
    """Observations restricted to ``image_ids`` (track_temp of FindTracksForProblem, :181-190); tracks keep their order."""
    m = np.isin(tracks.obs_image, np.asarray([int(i) for i in image_ids], np.uint32))
    t = np.repeat(np.arange(len(tracks)), np.diff(tracks.begin))
    lens = np.bincount(t[m], minlength=len(tracks))
    return Tracks(tracks.track_ids.copy(), np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), tracks.obs_image[m],
                  tracks.obs_feature[m])


def _subset(tracks: Tracks, idx: np.ndarray) -> Tracks:
    lens = np.diff(tracks.begin)[idx]
    out_begin = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    pos = np.repeat(np.asarray(tracks.begin, np.int64)[idx] - out_begin[:-1], lens) + np.arange(out_begin[-1])
    return Tracks(tracks.track_ids[idx], np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), tracks.obs_image[pos],
                  tracks.obs_feature[pos])


def find_tracks_for_problem_device(tracks: Tracks, registered_images, options: TrackEstablishmentOptions | None = None,
                                   ctx=None) -> Tracks:
    """FindTracksForProblem on the GPU (b200sfm_tracks_select).  Same result and layout as ``find_tracks_for_problem``:
    the selected tracks in descending (length, id) order, observations restricted to the registered images.  The four
    options are compared as unsigned values, as in the reference (see ``find_tracks_for_problem``).  Two tracks with one
    id raise ``_lib.B200Error`` (INVALID_ARG)."""
    import ctypes as ct

    from . import _lib, estimators as E
    o = options or TrackEstablishmentOptions()
    for f in ("min_num_tracks_per_view", "min_num_view_per_track", "max_num_view_per_track", "max_num_tracks"):
        v = int(getattr(o, f))
        if not -2**31 <= v < 2**31:
            raise ValueError(f"{f} = {v} is outside the range of int")
    ctx = ctx or E.default_context()
    T = len(tracks)
    ids = np.ascontiguousarray(tracks.track_ids, np.uint64)
    begin = np.ascontiguousarray(tracks.begin, np.int64)
    img = np.ascontiguousarray(tracks.obs_image, np.uint32)
    if len(begin) != T + 1 or len(img) != int(begin[-1]):
        raise ValueError("tracks.begin must have len(tracks) + 1 entries and end at len(tracks.obs_image)")
    reg = np.ascontiguousarray([int(i) for i in registered_images], np.uint32)
    keep = np.zeros(T, np.uint8)
    num = ct.c_int64()
    ptr = lambda a: a.ctypes.data_as(ct.c_void_p) if len(a) else None   # noqa: E731
    _lib.check(ctx.handle, ctx.lib.b200sfm_tracks_select(ctx.handle, T, ptr(ids), begin.ctypes.data_as(ct.c_void_p), ptr(img),
                                                         len(reg), ptr(reg), int(o.min_num_tracks_per_view),
                                                         int(o.min_num_view_per_track), int(o.max_num_view_per_track),
                                                         int(o.max_num_tracks), ptr(keep), ct.byref(num)))
    sel = np.nonzero(keep)[0]
    assert len(sel) == num.value
    lens = np.diff(begin)[sel]
    sel = sel[np.lexsort((ids[sel], lens))[::-1]]            # descending (length, id), the reference's processing order
    return restrict_to_images(_subset(tracks, sel), reg)


def tracks_to_rig_scene(tracks: Tracks, features: dict, image_ids, rig_scene):
    """The rig counterpart of ``tracks_to_scene``: ``rig_scene`` (a ``synthetic.RigScene``) with its tracks replaced by
    ``tracks`` -- in ascending track id, each observation as (frame, sensor, pixel), points zero.  The image of the k-th
    smallest of ``image_ids`` is image k of the scene's table.  Frames, sensors and intrinsics are shared with
    ``rig_scene``."""
    import dataclasses as dc
    begin, fr, se, xy = _rig_observations(tracks, features, image_ids, rig_scene.image_frame, rig_scene.image_sensor)
    return dc.replace(rig_scene, points=np.zeros((len(begin) - 1, 3)), pt_obs_begin=begin, obs_frame=fr, obs_sensor=se,
                      obs_xy=xy)


def _rig_observations(tracks: Tracks, features: dict, image_ids, image_frame, image_sensor):
    """(pt_obs_begin, obs_frame, obs_sensor, obs_xy) of ``tracks_to_rig_scene``, without a loop over observations."""
    image_ids = np.asarray(sorted(int(i) for i in image_ids), np.int64)
    order = np.argsort(tracks.track_ids, kind="stable")
    lens = np.diff(tracks.begin)[order]
    begin = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    src = np.repeat(np.asarray(tracks.begin, np.int64)[order] - begin[:-1], lens) + np.arange(begin[-1])
    img = np.searchsorted(image_ids, tracks.obs_image[src].astype(np.int64))
    if len(img) and (img.max() >= len(image_ids) or (image_ids[img] != tracks.obs_image[src]).any()):
        raise ValueError("a track observes an image that image_ids does not name")
    feats = [np.asarray(features[int(i)], np.float64).reshape(-1, 2) for i in image_ids]
    feat_begin = np.concatenate([[0], np.cumsum([len(f) for f in feats])]).astype(np.int64)
    all_xy = np.concatenate(feats) if feats else np.zeros((0, 2))
    xy = all_xy[feat_begin[img] + tracks.obs_feature[src].astype(np.int64)]
    return (begin, np.asarray(image_frame, np.int32)[img], np.asarray(image_sensor)[img].astype(np.uint16), xy)


def tracks_to_scene(tracks: Tracks, features: dict, image_ids, cam_intr, intr_model, intr_params):
    """Flat ``synthetic.Scene`` (poses identity, points zero) over ``image_ids`` (sorted-id order = camera index) --
    the input of GlobalPositioner / BundleAdjuster."""
    from . import synthetic as S
    image_ids = np.asarray(sorted(int(i) for i in image_ids), np.int64)
    idx = {int(i): k for k, i in enumerate(image_ids)}
    order = np.argsort(tracks.track_ids, kind="stable")
    obs_cam, obs_xy, begin = [], [], [0]
    for t in order:
        im, ft = tracks.observations(int(t))
        for i, f in zip(im, ft):
            obs_cam.append(idx[int(i)]); obs_xy.append(np.asarray(features[int(i)])[int(f)])
        begin.append(len(obs_cam))
    C, P = len(image_ids), len(order)
    quat = np.tile(np.array([0.0, 0.0, 0.0, 1.0]), (C, 1))
    return S.Scene(quat, np.zeros((C, 3)), np.zeros((P, 3)), np.asarray(begin, np.int64), np.asarray(obs_cam, np.int32),
                   np.asarray(obs_xy, np.float64).reshape(-1, 2), np.asarray(cam_intr, np.int32), np.asarray(intr_model, np.int32),
                   np.asarray(intr_params, np.float64))
