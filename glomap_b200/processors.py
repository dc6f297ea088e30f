"""Host-side steps on either side of the solvers (SURVEY.md 8(f) item 2), on the flat SoA scene:

* ``normalize_reconstruction`` -- glomap/processors/reconstruction_normalizer.cc:5-104: robust (p0..p1 percentile, float32
  coordinates as in the reference) bounding box of the projection centres of the registered images (on rigs: the image
  table, not every frame-sensor combination) -> Sim3 with identity rotation that moves the
  trimmed mean to the origin and scales the box diagonal to ``extent``; applied to the frame poses
  (colmap::TransformCameraWorld), the non-reference cam_from_rig translations and the points.  It runs between the BA
  solves of the mapper (controllers/global_mapper.cc:185,232,336) and fixes the gauge / scale BA leaves free.
* ``undistort_images`` -- glomap/processors/image_undistorter.cc:7-53: pixel -> unit bearing per feature
  (``CamFromImg(xy).homogeneous().normalized()``), the input of global positioning and of the angle filter; radial
  models are inverted on the radius by a safeguarded Newton iteration (``synthetic.undistort_radius_scale``).

Both are O(N) host work in the reference as well; the device-resident versions are a later row."""
from __future__ import annotations

import numpy as np

from . import geometry as geo
from . import synthetic as S


def normalize_reconstruction(scene, fixed_scale: bool = False, extent: float = 10.0, p0: float = 0.1, p1: float = 0.9):
    """In place on a ``Scene`` or ``RigScene``; returns the applied Sim3 as (scale, translation): X' = scale * X + t."""
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    if hasattr(scene, "obs_sensor"):      # centres of the images of the table, the registered ones (reconstruction_normalizer.cc:23-29)
        Ri, ti = scene.image_poses()
        centers = geo.centers_from_pose(Ri, ti)
    else:
        centers = geo.centers_from_pose(R, scene.trans)
    c32 = np.sort(centers.astype(np.float32), axis=0)          # per-axis sort of float coordinates (.cc:26-34)
    n = len(c32)
    i0 = int(p0 * (n - 1)) if n > 3 else 0
    i1 = int(p1 * (n - 1)) if n > 3 else n - 1
    bbox_min, bbox_max = c32[i0].astype(np.float64), c32[i1].astype(np.float64)
    mean = c32[i0:i1 + 1].astype(np.float64).sum(0) / (i1 - i0 + 1)
    scale = 1.0
    if not fixed_scale:
        old = float(np.linalg.norm(bbox_max - bbox_min))
        if old >= np.finfo(np.float64).eps:
            scale = extent / old
    t = -scale * mean
    # TransformCameraWorld: rotation unchanged, translation' = scale * t_old - R t
    scene.trans = scale * scene.trans - np.einsum("nij,j->ni", R, t)
    if hasattr(scene, "obs_sensor"):
        scene.sensor_trans = scene.sensor_trans * scale                                   # .cc:89-97
    scene.points = scale * scene.points + t                                               # .cc:99-101
    return scale, t


def undistort_images(scene) -> np.ndarray:
    """Unit bearing of every observation, [N,3] (``Image::features_undist``); rig scenes use the sensor's camera."""
    if hasattr(scene, "obs_sensor"):
        return S.bearings_from_scene(scene.images_scene())
    return S.bearings_from_scene(scene)
