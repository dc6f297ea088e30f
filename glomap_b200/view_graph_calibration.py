"""View-graph calibration (stage 1 of ``GlobalMapper::Solve``, glomap/controllers/global_mapper.cc:41-50) on the GPU:
``ViewGraphCalibrator.Solve`` = ViewGraphCalibrator::Solve (glomap/estimators/view_graph_calibration.cc:11-185) through
``b200sfm_view_graph_calibrate`` (vgc_kernels.cuh / vgc_solver.cuh).  One focal length per camera is refined from the
fundamental matrices of the valid CALIBRATED / UNCALIBRATED pairs; cameras whose estimate stays within the ratio bounds
get it (``has_refined_focal_length``), and pairs whose Fetzer residual exceeds ``thres_two_view_error`` are invalidated.

Pairs are ``track_establishment.ImagePairMatches`` (image ids, ``config``, ``F``, ``is_valid``), cameras
``image_pair_inliers.Camera`` objects (models 0-3) keyed by camera id, and ``image_camera`` maps an image id to its camera
id.  ``CalibCamera`` adds the two flags the reference's Camera carries.  The CPU restatement is oracle/vgc_oracle.py."""
from __future__ import annotations

import ctypes as ct
import dataclasses

import numpy as np

from . import synthetic as S
from .image_pair_inliers import TWO_VIEW_CALIBRATED, TWO_VIEW_UNCALIBRATED, Camera

TERMINATION = {0: "none", 1: "function tolerance", 2: "parameter tolerance", 3: "gradient tolerance",
               4: "max iterations", 5: "min trust region radius", 6: "too many invalid steps"}


@dataclasses.dataclass
class ViewGraphCalibratorOptions:
    """ViewGraphCalibratorOptions (view_graph_calibration.h:10-29), the OptimizationBaseOptions solver settings
    (optimization_base.h:18-23, Ceres defaults otherwise) and the PCG knobs of the device solver."""
    thres_lower_ratio: float = 0.1
    thres_higher_ratio: float = 10.0
    thres_two_view_error: float = 2.0
    thres_loss_function: float = 1e-2
    max_num_iterations: int = 100
    max_num_line_search_step_size_iterations: int = 20
    function_tolerance: float = 1e-5
    gradient_tolerance: float = 1e-10
    parameter_tolerance: float = 1e-8
    pcg_max_iterations: int = 1000
    pcg_min_iterations: int = 0
    pcg_rel_tolerance: float = 1e-12
    profile_kernels: bool = False

    def to_c(self):
        from . import _lib
        o = _lib.VGCOpts()
        for name, _ in o._fields_:
            if hasattr(self, name):
                setattr(o, name, type(getattr(o, name))(getattr(self, name)))
        return o


@dataclasses.dataclass
class CalibCamera(Camera):
    """A ``Camera`` with glomap's focal flags: a prior focal is held constant; a refined one was set by the calibrator."""
    has_prior_focal_length: bool = False
    has_refined_focal_length: bool = False


def focal_length_idxs(model: int) -> list:
    """Camera::FocalLengthIdxs() of COLMAP models 0-3 (PINHOLE: fx, fy)."""
    return [0, 1] if int(model) == S.PINHOLE else [0]


def principal_point(cam: Camera) -> np.ndarray:
    p = np.asarray(cam.params, np.float64)
    return p[2:4] if int(cam.model) == S.PINHOLE else p[1:3]


def calibrate_arrays(principal_point, focal, focal_constant, cam1, cam2, F, options: ViewGraphCalibratorOptions | None = None,
                     ctx=None, want_residual: bool = False) -> dict:
    """Flat form of ``b200sfm_view_graph_calibrate``: K cameras (principal_point [K, 2], focal [K] = Camera::Focal(),
    focal_constant [K] or None), E qualifying pairs (cam1, cam2 [E], F [E, 9]).  Returns focal [K] (estimates of the
    cameras used by a pair), cam_accepted [K] bool, pair_valid [E] bool, residual [E, 2] or None, stats (dict of
    b200sfm_lm_stats).  On the reference's early return (no pair or no variable camera) nothing is written: focal as
    given, cam_accepted all False, pair_valid all True."""
    from . import _lib, estimators as E_
    o = options or ViewGraphCalibratorOptions()
    ctx = ctx or E_.default_context()
    K = len(focal)
    pp = np.ascontiguousarray(np.asarray(principal_point, np.float64).reshape(K, 2))
    f = np.ascontiguousarray(np.asarray(focal, np.float64).copy())
    fc = None if focal_constant is None else np.ascontiguousarray(np.asarray(focal_constant, np.uint8))
    c1 = np.ascontiguousarray(np.asarray(cam1, np.int32))
    c2 = np.ascontiguousarray(np.asarray(cam2, np.int32))
    Ep = len(c1)
    Fm = np.ascontiguousarray(np.asarray(F, np.float64).reshape(Ep, 9))
    valid = np.ones(Ep, np.uint8)
    acc = np.zeros(K, np.uint8)
    res = np.zeros((Ep, 2)) if want_residual else None
    st = _lib.LMStats()
    ptr = lambda a: a.ctypes.data_as(ct.c_void_p) if a is not None and a.size else None   # noqa: E731
    copts = o.to_c()
    _lib.check(ctx.handle, ctx.lib.b200sfm_view_graph_calibrate(
        ctx.handle, ct.byref(copts), K, ptr(pp), ptr(f), ptr(fc), Ep, ptr(c1), ptr(c2), ptr(Fm), ptr(valid), ptr(acc),
        ptr(res), ct.byref(st)))
    return dict(focal=f, cam_accepted=acc.astype(bool), pair_valid=valid.astype(bool), residual=res, stats=st.as_dict())


class ViewGraphCalibrator:
    """ViewGraphCalibrator (view_graph_calibration.h:31-73) on the device."""

    def __init__(self, options: ViewGraphCalibratorOptions | None = None, ctx=None):
        self.options = options or ViewGraphCalibratorOptions()
        self.ctx = ctx
        self.summary = None

    def Solve(self, pairs, cameras: dict, image_camera: dict) -> bool:
        """Refines the focal of every camera used by a valid CALIBRATED / UNCALIBRATED pair (in place: ``params`` at
        FocalLengthIdxs and ``has_refined_focal_length``), invalidates the pairs with a large residual and returns
        summary.IsSolutionUsable().  Pairs are taken in the order given."""
        o = self.options
        qual = [p for p in pairs if int(p.config) in (TWO_VIEW_CALIBRATED, TWO_VIEW_UNCALIBRATED) and p.is_valid]
        cam_ids = sorted(cameras)
        idx = {c: k for k, c in enumerate(cam_ids)}
        cams = [cameras[c] for c in cam_ids]
        K = len(cams)
        pp = np.array([principal_point(c) for c in cams]).reshape(K, 2)
        focal = np.array([c.focal() for c in cams], np.float64)
        prior = np.array([bool(getattr(c, "has_prior_focal_length", False)) for c in cams], np.uint8)
        c1 = np.array([idx[image_camera[p.image_id1]] for p in qual], np.int32)
        c2 = np.array([idx[image_camera[p.image_id2]] for p in qual], np.int32)
        F = np.array([np.asarray(p.F, np.float64).reshape(9) for p in qual]).reshape(len(qual), 9)
        out = calibrate_arrays(pp, focal, prior, c1, c2, F, o, self.ctx)
        self.summary = out["stats"]
        for k in np.flatnonzero(out["cam_accepted"]):
            cam = cams[k]
            cam.has_refined_focal_length = True
            for i in focal_length_idxs(cam.model):
                cam.params[i] = out["focal"][k]
        for p, v in zip(qual, out["pair_valid"]):
            if not v:
                p.is_valid = False
        return bool(out["stats"]["usable"])
