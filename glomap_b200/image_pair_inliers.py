"""Inlier matches of the image pairs (stage 2 of ``GlobalMapper::Solve``, glomap/controllers/global_mapper.cc:64-70):

* ``image_pairs_inlier_count``  = ImagePairsInlierCount (processors/image_pair_inliers.cc:200-213) with the scorers
  ScoreErrorEssential / Fundamental / Homography (:20-198) and the two-view arithmetic of math/two_view_geometry.cc --
  a vectorised host restatement, the reference the device path is tested against;
* ``image_pairs_inlier_count_device`` -- the same through ``b200sfm_image_pairs_inlier_count`` (pair_kernels.cuh);
* ``filter_inlier_num`` / ``filter_inlier_ratio`` = RelPoseFilter::FilterInlierNum / FilterInlierRatio
  (processors/relpose_filter.cc:35-65), O(pairs) host loops as in the reference.

Pairs are ``track_establishment.ImagePairMatches`` (config, cam2_from_cam1, F, H, matches); ``features[image_id]`` is the
[n,2] pixel table (Image::features) and ``cameras[image_id]`` the ``Camera`` of the image.  CALIBRATED pairs are scored
on the unit bearings of the features (Image::features_undist, UndistortImages), computed here from the camera.  The
result inliers are written back to the pairs, as the reference rewrites ImagePair::inliers, and returned."""
from __future__ import annotations

import ctypes as ct
import dataclasses

import numpy as np

from . import geometry as geo, synthetic as S
from .mapper import InlierThresholdOptions  # noqa: F401  (the options of this stage live on the mapper's struct)

# colmap::TwoViewGeometry::ConfigurationType (colmap/estimators/two_view_geometry.h, un-vendored; UPSTREAM-UNVERIFIED)
TWO_VIEW_UNDEFINED, TWO_VIEW_DEGENERATE, TWO_VIEW_CALIBRATED, TWO_VIEW_UNCALIBRATED = 0, 1, 2, 3
TWO_VIEW_PLANAR, TWO_VIEW_PANORAMIC, TWO_VIEW_PLANAR_OR_PANORAMIC, TWO_VIEW_WATERMARK, TWO_VIEW_MULTIPLE = 4, 5, 6, 7, 8
_HOMOGRAPHY_CONFIGS = (TWO_VIEW_PLANAR, TWO_VIEW_PANORAMIC, TWO_VIEW_PLANAR_OR_PANORAMIC)

EPS = 1e-12                                                          # glomap/types.h:14
COS_EPIPOLE_THR = float(np.cos(3.0 * 0.0174532925199432954743716805978692718953)) + 1e-6   # cos(DegToRad(3)) + 1e-6
ANGLE_THR = 1.0 + 1e-6                                               # image_pair_inliers.cc:55-56


@dataclasses.dataclass
class Camera:
    """The camera of an image: COLMAP model id (0-3 for CALIBRATED pairs) and its parameters."""
    model: int
    params: np.ndarray

    def focal(self) -> float:
        """Camera::Focal() = (fx + fy) / 2 (glomap/scene/camera.h:28)."""
        p = np.asarray(self.params, np.float64)
        return float((p[0] + p[1]) / 2.0) if self.model == S.PINHOLE else float((p[0] + p[0]) / 2.0)


@dataclasses.dataclass
class InlierCount:
    """Per pair (in the order given): inlier rows in ascending order, the scorer's return value (0 for a pair that was not
    scored) and whether it was scored; ``r2`` (host restatement only) is each match's squared error, None when not scored."""
    inliers: list
    scores: np.ndarray
    scored: np.ndarray
    r2: list | None = None


def _seq_sum(v) -> float:
    """Left-to-right sum, the order the reference's loop adds its terms in."""
    return float(np.add.accumulate(v)[-1]) if len(v) else 0.0


def _mv(M, x0, x1, x2):
    """(M x) for [n] component arrays, summed left to right as the device does."""
    return [M[i, 0] * x0 + M[i, 1] * x1 + M[i, 2] * x2 for i in range(3)]


def score_image_pair(pair, features: dict, cameras: dict, options: InlierThresholdOptions | None = None,
                     bearings: dict | None = None) -> dict:
    """One pair, as ImagePairInliers::ScoreError: {'inlier' [m] bool, 'score', 'r2' [m], 'thr2'} plus the quantities the
    decision compares -- E: 'lambda1', 'lambda2', 'min_depth', 'max_depth', 'diff_angle', 'diff_epipole1', 'diff_epipole2';
    F: 'signum', 'signum_scale', 'tie'.  ``bearings`` caches the unit bearings per image."""
    o = options or InlierThresholdOptions()
    m = np.asarray(pair.matches, np.int64).reshape(-1, 2)
    n = len(m)
    c = int(pair.config)
    out = {"inlier": np.zeros(n, bool), "score": 0.0, "r2": np.full(n, np.nan), "thr2": np.nan}
    if c == TWO_VIEW_CALIBRATED:
        bearings = {} if bearings is None else bearings
        for i in (pair.image_id1, pair.image_id2):
            if i not in bearings:
                cam = cameras[i]
                if int(cam.model) not in S.MODEL_NUM_PARAMS:
                    raise ValueError(f"camera model {cam.model} of a CALIBRATED pair is not supported")
                bearings[i] = S.bearings_from_pixels(int(cam.model), np.asarray(cam.params, np.float64),
                                                     np.asarray(features[i], np.float64).reshape(-1, 2))
        x1, x2 = bearings[pair.image_id1][m[:, 0]], bearings[pair.image_id2][m[:, 1]]
        R = geo.quat_xyzw_to_rotmat(np.asarray(pair.quat_xyzw, np.float64))
        t = np.asarray(pair.trans, np.float64)
        tx = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])
        Em = np.array([[tx[i, 0] * R[0, j] + tx[i, 1] * R[1, j] + tx[i, 2] * R[2, j] for j in range(3)] for i in range(3)])
        e12 = -t if t[2] < 0 else t
        e21 = np.array([-(R[0, i] * t[0] + R[1, i] * t[1] + R[2, i] * t[2]) for i in range(3)])
        e21 = -e21 if e21[2] < 0 else e21
        thr = o.max_epipolar_error_E * 0.5 * (1. / cameras[pair.image_id1].focal() + 1. / cameras[pair.image_id2].focal())
        thr2 = thr * thr
        d1, d2 = EPS + x1[:, 2], EPS + x2[:, 2]
        Ex1 = [v / d1 for v in _mv(Em, x1[:, 0], x1[:, 1], x1[:, 2])]
        Etx2 = [v / d2 for v in _mv(Em.T, x2[:, 0], x2[:, 1], x2[:, 2])]
        C = Ex1[0] * x2[:, 0] + Ex1[1] * x2[:, 1] + Ex1[2] * x2[:, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            r2 = C * C / ((Ex1[0] * Ex1[0] + Ex1[1] * Ex1[1]) + (Etx2[0] * Etx2[0] + Etx2[1] * Etx2[1]))
        # CheckCheirality(cam2_from_cam1, x1, x2, 1e-2, 100) (two_view_geometry.cc:5-29)
        Rx1 = _mv(R, x1[:, 0], x1[:, 1], x1[:, 2])
        Rtx2 = _mv(R.T, x2[:, 0], x2[:, 1], x2[:, 2])
        a = -(Rx1[0] * x2[:, 0] + Rx1[1] * x2[:, 1] + Rx1[2] * x2[:, 2])
        b1 = -(Rx1[0] * t[0] + Rx1[1] * t[1] + Rx1[2] * t[2])
        b2 = x2[:, 0] * t[0] + x2[:, 1] * t[1] + x2[:, 2] * t[2]
        l1, l2 = b1 - a * b2, -a * b1 + b2
        min_d, max_d = 1e-2 * (1 - a * a), 100. * (1 - a * a)
        cheir = (l1 > min_d) & (l2 > min_d) & (l1 < max_d) & (l2 < max_d)
        diff_angle = x1[:, 0] * Rtx2[0] + x1[:, 1] * Rtx2[1] + x1[:, 2] * Rtx2[2]
        dep1 = x1[:, 0] * e21[0] + x1[:, 1] * e21[1] + x1[:, 2] * e21[2]
        dep2 = x2[:, 0] * e12[0] + x2[:, 1] * e12[1] + x2[:, 2] * e12[2]
        inl = (r2 < thr2) & cheir & (diff_angle < ANGLE_THR) & (dep1 < COS_EPIPOLE_THR) & (dep2 < COS_EPIPOLE_THR)
        out.update(inlier=inl, r2=r2, thr2=thr2, score=_seq_sum(np.where(inl, r2, thr2)), lambda1=l1, lambda2=l2,
                   min_depth=min_d, max_depth=max_d, diff_angle=diff_angle, diff_epipole1=dep1, diff_epipole2=dep2)
    elif c == TWO_VIEW_UNCALIBRATED or c in _HOMOGRAPHY_CONFIGS:
        x1 = np.asarray(features[pair.image_id1], np.float64).reshape(-1, 2)[m[:, 0]]
        x2 = np.asarray(features[pair.image_id2], np.float64).reshape(-1, 2)[m[:, 1]]
        one = np.ones(n)
        if c == TWO_VIEW_UNCALIBRATED:
            F = np.asarray(pair.F, np.float64).reshape(3, 3)
            thr2 = o.max_epipolar_error_F * o.max_epipolar_error_F
            Fx1 = _mv(F, x1[:, 0], x1[:, 1], one)
            Ftx2 = _mv(F.T, x2[:, 0], x2[:, 1], one)
            C = Fx1[0] * x2[:, 0] + Fx1[1] * x2[:, 1] + Fx1[2]
            with np.errstate(divide="ignore", invalid="ignore"):
                r2 = C * C / ((Fx1[0] * Fx1[0] + Fx1[1] * Fx1[1]) + (Ftx2[0] * Ftx2[0] + Ftx2[1] * Ftx2[1]))
            ep = np.cross(F[0], F[2])
            if not ((ep > EPS) | (ep < -EPS)).any():
                ep = np.cross(F[1], F[2])
            signum = (F[0, 0] * x2[:, 0] + F[1, 0] * x2[:, 1] + F[2, 0]) * (ep[1] - ep[2] * x1[:, 1])
            pre = r2 < thr2
            pos = pre & (signum > 0)
            npos, nneg = int(pos.sum()), int((pre & ~(signum > 0)).sum())
            tie = npos == nneg
            inl = np.zeros(n, bool) if tie else (pre & ((signum > 0) == (npos > nneg)))
            # the first loop adds the threshold of every other match, the second the kept pre-inliers' r2 (:128-163)
            score = 0.0 if tie else _seq_sum(np.concatenate([np.full(int((~pre).sum()), thr2), np.where(inl, r2, thr2)[pre]]))
            # magnitude of the terms the signum is made of: the scale its rounding error is relative to
            signum_scale = (np.abs(F[0, 0] * x2[:, 0]) + np.abs(F[1, 0] * x2[:, 1]) + abs(F[2, 0])) * \
                (abs(ep[1]) + np.abs(ep[2] * x1[:, 1]))
            out.update(inlier=inl, r2=r2, thr2=thr2, score=score, signum=signum, signum_scale=signum_scale, tie=tie)
        else:
            Hm = np.asarray(pair.H, np.float64).reshape(3, 3)
            thr2 = o.max_epipolar_error_H * o.max_epipolar_error_H
            h = _mv(Hm, x1[:, 0], x1[:, 1], one)
            with np.errstate(divide="ignore", invalid="ignore"):
                dx, dy = h[0] / (EPS + h[2]) - x2[:, 0], h[1] / (EPS + h[2]) - x2[:, 1]
            r2 = dx * dx + dy * dy
            inl = r2 < thr2
            out.update(inlier=inl, r2=r2, thr2=thr2, score=_seq_sum(np.where(inl, r2, thr2)))
    return out


def _to_score(pairs, clean_inliers):
    """The reference's loop head (image_pair_inliers.cc:205-211): pairs whose inliers are cleared, and of those the
    valid ones, which are scored."""
    cleared = [k for k, p in enumerate(pairs) if clean_inliers or len(p.inliers) == 0]
    return cleared, [k for k in cleared if pairs[k].is_valid]


def image_pairs_inlier_count(pairs, features: dict, cameras: dict, options: InlierThresholdOptions | None = None,
                             clean_inliers: bool = True) -> InlierCount:
    cleared, scored = _to_score(pairs, clean_inliers)
    res = InlierCount([np.asarray(p.inliers, np.int64) for p in pairs], np.zeros(len(pairs)), np.zeros(len(pairs), bool),
                      [None] * len(pairs))
    bearings = {}
    for k in cleared:
        res.inliers[k] = np.zeros(0, np.int64)
    for k in scored:
        d = score_image_pair(pairs[k], features, cameras, options, bearings)
        res.inliers[k], res.scores[k], res.scored[k], res.r2[k] = np.flatnonzero(d["inlier"]), d["score"], True, d["r2"]
    for p, inl in zip(pairs, res.inliers):
        p.inliers = inl
    return res


def image_pairs_inlier_count_device(pairs, features: dict, cameras: dict, options: InlierThresholdOptions | None = None,
                                    clean_inliers: bool = True, ctx=None) -> InlierCount:
    """``image_pairs_inlier_count`` on the GPU; ``r2`` is None.  The host only concatenates the arrays and turns the
    inlier mask back into ascending row lists."""
    from . import _lib, estimators as E
    o = options or InlierThresholdOptions()
    cleared, scored = _to_score(pairs, clean_inliers)
    res = InlierCount([np.asarray(p.inliers, np.int64) for p in pairs], np.zeros(len(pairs)), np.zeros(len(pairs), bool))
    for k in cleared:
        res.inliers[k] = np.zeros(0, np.int64)
    if scored:
        ctx = ctx or E.default_context()
        image_ids = sorted(features)
        idx = {int(i): k for k, i in enumerate(image_ids)}
        tables = [np.asarray(features[i], np.float64).reshape(-1, 2) for i in image_ids]
        feature_begin = np.concatenate([[0], np.cumsum([len(t) for t in tables])]).astype(np.int64)
        feats = np.ascontiguousarray(np.concatenate(tables) if tables else np.zeros((0, 2)))
        blocks, image_intr = {}, np.full(len(image_ids), -1, np.int32)   # cameras shared by several images: one block
        for k, i in enumerate(image_ids):
            cam = cameras.get(i)
            if cam is not None:
                image_intr[k] = blocks.setdefault(id(cam), (len(blocks), cam))[0]
        intr_model = np.array([int(c.model) for _, c in blocks.values()], np.int32)
        intr_params = np.zeros((len(blocks), _lib.INTR_STRIDE))
        for b, c in blocks.values():
            p = np.asarray(c.params, np.float64)
            intr_params[b, :len(p)] = p
        ps = [pairs[k] for k in scored]
        Ep = len(ps)
        m_list = [np.asarray(p.matches, np.int64).reshape(-1, 2) for p in ps]
        match_begin = np.concatenate([[0], np.cumsum([len(m) for m in m_list])]).astype(np.int64)
        matches = np.ascontiguousarray(np.concatenate(m_list).astype(np.int32)) if Ep else np.zeros((0, 2), np.int32)
        img1 = np.array([idx[int(p.image_id1)] for p in ps], np.int32)
        img2 = np.array([idx[int(p.image_id2)] for p in ps], np.int32)
        config = np.array([int(p.config) for p in ps], np.int32)
        quat = np.array([np.asarray(p.quat_xyzw, np.float64) for p in ps]).reshape(Ep, 4)
        trans = np.array([np.asarray(p.trans, np.float64) for p in ps]).reshape(Ep, 3)
        Fs = np.array([np.asarray(p.F, np.float64).reshape(9) for p in ps]).reshape(Ep, 9)
        Hs = np.array([np.asarray(p.H, np.float64).reshape(9) for p in ps]).reshape(Ep, 9)
        M = int(match_begin[-1])
        mask, n_inl, score = np.zeros(M, np.uint8), np.zeros(Ep, np.int32), np.zeros(Ep)
        ptr = lambda a: a.ctypes.data_as(ct.c_void_p) if a.size else None   # noqa: E731
        _lib.check(ctx.handle, ctx.lib.b200sfm_image_pairs_inlier_count(
            ctx.handle, len(image_ids), ptr(feature_begin), ptr(feats), ptr(image_intr), len(intr_model), ptr(intr_model),
            ptr(intr_params), Ep, ptr(img1), ptr(img2), ptr(config), ptr(quat), ptr(trans), ptr(Fs), ptr(Hs), ptr(match_begin),
            ptr(matches), float(o.max_epipolar_error_E), float(o.max_epipolar_error_F), float(o.max_epipolar_error_H), ptr(mask),
            ptr(n_inl), ptr(score)))
        rows = np.flatnonzero(mask)
        cut = np.searchsorted(rows, match_begin)
        for j, k in enumerate(scored):
            res.inliers[k] = rows[cut[j]:cut[j + 1]] - match_begin[j]
            res.scores[k], res.scored[k] = score[j], True
        assert all(len(res.inliers[k]) == n_inl[j] for j, k in enumerate(scored))
    for p, inl in zip(pairs, res.inliers):
        p.inliers = inl
    return res


def filter_inlier_num(pairs, min_inlier_num) -> int:
    """RelPoseFilter::FilterInlierNum (relpose_filter.cc:35-48): invalidates valid pairs with fewer inliers than
    ``int(min_inlier_num)``, compared as an unsigned 64-bit value like the reference (``size()`` against an ``int``);
    returns the number invalidated."""
    n, thr = 0, int(min_inlier_num) & 0xFFFFFFFFFFFFFFFF
    for p in pairs:
        if p.is_valid and len(p.inliers) < thr:
            p.is_valid = False
            n += 1
    return n


def filter_inlier_ratio(pairs, min_inlier_ratio: float) -> int:
    """RelPoseFilter::FilterInlierRatio (relpose_filter.cc:50-65).  A pair without matches gives 0 / 0 = NaN, which is not
    below the threshold: it stays valid, as in the reference."""
    n = 0
    for p in pairs:
        m = len(np.asarray(p.matches).reshape(-1, 2))
        ratio = len(p.inliers) / m if m else float("nan")
        if p.is_valid and ratio < min_inlier_ratio:
            p.is_valid = False
            n += 1
    return n
