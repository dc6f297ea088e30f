"""``ConvertRotationsFromImageToRig`` (glomap/estimators/rotation_initializer.cc:7-125) on the device
(b200sfm_rig_rotations_from_images): per-image cam_from_world rotations -> the cam_from_rig rotations of the cameras
that are not calibrated yet and the frames' rig_from_world rotations.  The rules are stated in include/b200sfm.h."""
from __future__ import annotations

import ctypes as ct

import numpy as np

from . import _lib
from .estimators import Context, _c, _ptr, default_context


def convert_rotations_from_image_to_rig(image_frame, image_camera, cam_from_world, frame_ref_camera, camera_known,
                                        cam_from_rig, rig_from_world, image_estimated=None, ctx: Context | None = None,
                                        stats: _lib.RigInitStats | None = None):
    """Quaternions xyzw.  image_frame [I] (-1: not registered), image_camera [I], cam_from_world [I,4],
    frame_ref_camera [F], camera_known [K] (pass the reference cameras as known, with the identity), cam_from_rig [K,4],
    rig_from_world [F,4] (kept where a frame gets no sample), image_estimated [I] or None (every image).  Returns
    (cam_from_rig [K,4], cam_samples [K], rig_from_world [F,4], frame_samples [F]); ``stats``, when given, receives the
    call's b200sfm_rig_init_stats."""
    ctx = ctx or default_context()
    fr, cam = _c(image_frame, np.int32), _c(image_camera, np.int32)
    q = _c(np.reshape(cam_from_world, (-1, 4)), np.float64)
    ref, known = _c(frame_ref_camera, np.int32), _c(camera_known, np.uint8)
    est = None if image_estimated is None else _c(image_estimated, np.uint8)
    cq = np.array(np.reshape(cam_from_rig, (-1, 4)), dtype=np.float64, order="C", copy=True)
    fq = np.array(np.reshape(rig_from_world, (-1, 4)), dtype=np.float64, order="C", copy=True)
    I, F, K = len(fr), len(ref), len(known)
    if len(cam) != I or len(q) != I or (est is not None and len(est) != I) or len(cq) != K or len(fq) != F:
        raise ValueError("inconsistent array lengths")
    cn, fn = np.empty(K, np.int32), np.empty(F, np.int32)
    st = stats if stats is not None else _lib.RigInitStats()
    _lib.check(ctx.handle, ctx.lib.b200sfm_rig_rotations_from_images(
        ctx.handle, I, F, K, _ptr(fr), _ptr(cam), _ptr(est), _ptr(q), _ptr(ref), _ptr(known), _ptr(cq), _ptr(cn), _ptr(fq),
        _ptr(fn), ct.byref(st)))
    return cq, cn, fq, fn
