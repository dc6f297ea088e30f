"""Gravity refinement (``GravityRefiner::RefineGravity``, glomap/estimators/gravity_refinement.cc:9-181, run by
``glomap rotation_averager --refine_gravity 1``) on the GPU through ``b200sfm_gravity_refine`` (gravity_kernels.cuh).

Frames whose gravity prior disagrees with too many neighbours (IdentifyErrorProneGravity) get a new gravity from their
neighbours' priors carried across the relative rotations: AverageGravity, then an LM on the unit sphere under
ArctanLoss, kept when it agrees with more than half of them.  Every error-prone frame is refined against the priors as
they were on entry; the other rules where the reference depends on hash order are stated in include/b200sfm.h.  The CPU
restatement is oracle/gravity_oracle.py."""
from __future__ import annotations

import ctypes as ct
import dataclasses

import numpy as np


@dataclasses.dataclass
class GravityRefinerOptions:
    """gravity_refinement.h:12-26 + the solver options of optimization_base.h:18-23 (defaults identical)."""
    max_outlier_ratio: float = 0.5
    max_gravity_error: float = 1.0     # degrees
    min_num_neighbors: int = 7
    max_num_iterations: int = 100
    function_tolerance: float = 1e-5
    gradient_tolerance: float = 1e-10
    parameter_tolerance: float = 1e-8

    def to_c(self):
        from . import _lib
        o = _lib.GravityOpts()
        _lib.load().b200sfm_gravity_default_opts(ct.byref(o))
        for f in ("max_outlier_ratio", "max_gravity_error", "min_num_neighbors", "max_num_iterations", "function_tolerance",
                  "gradient_tolerance", "parameter_tolerance"):
            setattr(o, f, getattr(self, f))
        return o


def get_align_rot_householder(gravity) -> np.ndarray:
    """GetAlignRot (math/gravity.cc:11-24) with Eigen's completion: column 1 is the unit gravity, columns 0 and 2 are the
    last two columns of the Householder reflector of HouseholderQR, column 2 negated when the determinant is negative.
    ``gravity`` [..., 3] -> [..., 3, 3]; a zero or non-finite gravity gives a non-finite matrix."""
    g = np.asarray(gravity, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        v = g / np.linalg.norm(g, axis=-1, keepdims=True)
        c0, tail = v[..., 0], v[..., 1:]
        tsq = (tail * tail).sum(-1)
        trivial = tsq <= np.finfo(np.float64).tiny                  # Eigen makeHouseholder: tau = 0, H = I
        beta = np.sqrt(c0 * c0 + tsq)
        beta = np.where(c0 >= 0, -beta, beta)
        ess = tail / (c0 - beta)[..., None]
        tau = (beta - c0) / beta
        w = np.concatenate([np.ones(c0.shape + (1,)), ess], axis=-1)
        H = np.eye(3) - tau[..., None, None] * w[..., :, None] * w[..., None, :]
        H = np.where(trivial[..., None, None], np.eye(3), H)
        R = np.stack([H[..., :, 1], v, H[..., :, 2]], axis=-1)
        flip = np.linalg.det(np.where(np.isfinite(R), R, 0.0)) < 0
        R[..., :, 2] = np.where(flip[..., None], -R[..., :, 2], R[..., :, 2])
    return R


def frame_pairs(vg, img_frame=None, img_sensor=None, sensor_quat=None):
    """Frame-level pairs of the view graph ``vg`` (every pair valid): (frame1, frame2, M [E,3,3]) with
    M = R_c2^T R_rel R_c1 (rig2_from_rig1), as ``estimators.rig_view_graph`` composes it; pairs inside one frame are
    kept.  Without rig inputs image i is frame i and M = R_rel."""
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    R_rel = np.asarray(vg.R_rel, dtype=np.float64).reshape(-1, 3, 3)
    if img_frame is None:
        return ei, ej, R_rel
    from . import geometry as geo
    img_frame = np.asarray(img_frame)
    if img_sensor is None or sensor_quat is None:
        return img_frame[ei], img_frame[ej], R_rel
    Rs = geo.quat_xyzw_to_rotmat(np.asarray(sensor_quat, dtype=np.float64))
    img_sensor = np.asarray(img_sensor)
    M = np.einsum("nji,njk,nkl->nil", Rs[img_sensor[ej]], R_rel, Rs[img_sensor[ei]])
    return img_frame[ei], img_frame[ej], M


class GravityRefiner:
    """glomap::GravityRefiner (gravity_refinement.h:28-43)."""

    def __init__(self, options: GravityRefinerOptions | None = None, ctx=None):
        self.options_ = options or GravityRefinerOptions()
        self.ctx = ctx
        self.stats: dict | None = None

    def RefineGravity(self, vg, gravity, img_frame=None, img_sensor=None, sensor_quat=None):
        """``gravity`` [F,3] per frame, NaN rows = no prior (F = vg.n_images without ``img_frame``).  Optional rig inputs:
        ``img_frame`` [n_images], ``img_sensor`` [n_images] and ``sensor_quat`` [S,4] xyzw (cam_from_rig).
        Returns (gravity [F,3] with the accepted frames replaced, status [F] uint8 as in include/b200sfm.h, stats)."""
        g = np.asarray(gravity, dtype=np.float64)
        nimg = int(vg.n_images)
        if img_frame is not None:
            img_frame = _as_index(img_frame, "img_frame")
            if img_frame.shape != (nimg,):
                raise ValueError(f"img_frame must have n_images = {nimg} entries, not {img_frame.shape}")
            if img_frame.size and (img_frame.min() < 0 or img_frame.max() >= len(g)):
                raise ValueError("img_frame outside [0, F)")
        if img_sensor is not None:
            img_sensor = _as_index(img_sensor, "img_sensor")
            if img_sensor.shape != (nimg,):
                raise ValueError(f"img_sensor must have n_images = {nimg} entries, not {img_sensor.shape}")
            if sensor_quat is None or img_sensor.size and (img_sensor.min() < 0 or img_sensor.max() >= len(sensor_quat)):
                raise ValueError("img_sensor outside the sensors of sensor_quat")
        ei, ej = _as_index(vg.ei, "vg.ei"), _as_index(vg.ej, "vg.ej")
        if ei.shape != ej.shape or ei.ndim != 1:
            raise ValueError("vg.ei and vg.ej must be 1-D of equal length")
        if ei.size and (min(ei.min(), ej.min()) < 0 or max(ei.max(), ej.max()) >= nimg):
            raise ValueError("vg.ei / vg.ej outside [0, n_images)")
        if img_frame is None and len(g) != nimg:
            raise ValueError(f"gravity must have n_images = {nimg} rows without img_frame, not {len(g)}")
        f1, f2, M = frame_pairs(vg, img_frame, img_sensor, sensor_quat)
        return self.refine_frames(g, f1, f2, M)

    def refine_frames(self, gravity, frame1, frame2, M):
        """The flat call: ``gravity`` [F,3] (NaN rows = no prior), frames of the valid pairs and their M [E,3,3]."""
        from . import _lib, estimators as E_
        g = np.asarray(gravity, dtype=np.float64)
        if g.ndim != 2 or g.shape[1] != 3:
            raise ValueError(f"gravity must be [F,3], not {g.shape}")
        F = len(g)
        nan_row = np.isnan(g).all(axis=1)
        if not np.isfinite(g[~nan_row]).all():
            raise ValueError("gravity rows must be finite or all NaN (no prior)")
        f1, f2 = _as_index(frame1, "frame1"), _as_index(frame2, "frame2")
        M = np.ascontiguousarray(np.asarray(M, dtype=np.float64).reshape(-1, 9))
        if f1.shape != f2.shape or f1.ndim != 1 or len(M) != len(f1):
            raise ValueError("frame1, frame2 and M must have one entry per pair")
        if f1.size and (min(f1.min(), f2.min()) < 0 or max(f1.max(), f2.max()) >= F):
            raise ValueError("frame1 / frame2 outside [0, F)")
        has = ~nan_row
        keep = has[f1] & has[f2]                                  # .cc:62-64,149
        f1, f2, M = np.ascontiguousarray(f1[keep]), np.ascontiguousarray(f2[keep]), np.ascontiguousarray(M[keep])
        R_align = np.tile(np.eye(3), (F, 1, 1))
        if has.any():
            R_align[has] = get_align_rot_householder(g[has])
        R_align = np.ascontiguousarray(R_align.reshape(F, 9))
        has8 = np.ascontiguousarray(has.astype(np.uint8))
        out = np.zeros((F, 3))
        status = np.zeros(F, np.uint8)
        ctx = self.ctx or E_.default_context()
        st = _lib.GravityStats()
        ptr = lambda a: a.ctypes.data_as(ct.c_void_p) if a.size else None   # noqa: E731
        _lib.check(ctx.handle, ctx.lib.b200sfm_gravity_refine(
            ctx.handle, ct.byref(self.options_.to_c()), F, ptr(R_align), ptr(has8), len(f1), ptr(f1), ptr(f2), ptr(M), ptr(out),
            ptr(status), ct.byref(st)))
        self.stats = st.as_dict()
        g_new = g.copy()
        g_new[status == 2] = out[status == 2]
        return g_new, status, self.stats


def _as_index(a, name):
    """int32 index array; integers that do not fit raise instead of wrapping."""
    a = np.asarray(a)
    if a.size == 0:
        return np.zeros(a.shape, np.int32)
    if a.dtype.kind not in "iu":
        raise ValueError(f"{name} must be an integer array, not {a.dtype}")
    info = np.iinfo(np.int32)
    if a.min() < info.min or a.max() > info.max:
        raise ValueError(f"{name} has entries outside the range of int32")
    return np.ascontiguousarray(a.astype(np.int32, copy=False))
