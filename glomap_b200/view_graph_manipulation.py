"""Stage 0 of ``GlobalMapper::Solve`` (glomap/controllers/global_mapper.cc:22-34), its first half:
``ViewGraphManipulater::UpdateImagePairsConfig`` (processors/view_graph_manipulation.cc:178-237).

Every camera counts the valid CALIBRATED and UNCALIBRATED pairs it takes part in, over the pairs whose two cameras both
have a prior focal length (a pair inside one camera counts twice for it).  A camera is valid when more than half of its
pairs are CALIBRATED (``calibrated * 1. / total > 0.5``); a camera no pair counted is not valid.  A valid UNCALIBRATED pair
whose two cameras are valid then becomes CALIBRATED, with F = K2^-T [t]x R K1^-1 of its cam2_from_cam1
(FundamentalFromMotionAndCameras, math/two_view_geometry.cc:38-55; K = Camera::GetK, scene/camera.h:34-39, with fx = fy
for the SIMPLE_* models; R is Eigen's toRotationMatrix of the quaternion as given).  F is computed from whatever
cam2_from_cam1 the pair carries: the reference runs this pass before DecomposeRelPose, on the identity pose its database
converter gives every pair, so a promoted pair's F is the zero matrix there.  DecomposeRelPose, the second half of
stage 0, calls COLMAP's EstimateTwoViewGeometryPose and is not part of this package: pairs keep the pose they have.

``update_image_pairs_config`` is a host restatement written as loops in the reference's form;
``update_image_pairs_config_device`` runs ``b200sfm_view_graph_update_pairs_config`` (pair_config_kernels.cuh) and is
tested against it.  ``UpdateImagePairsConfig`` takes ``track_establishment.ImagePairMatches`` lists and camera objects,
as ``view_graph_calibration.ViewGraphCalibrator.Solve`` does."""
from __future__ import annotations

import ctypes as ct

import numpy as np

from . import synthetic as S
from .image_pair_inliers import TWO_VIEW_CALIBRATED, TWO_VIEW_UNCALIBRATED


def _pinhole(model: int, p) -> tuple:
    """fx, fy, cx, cy of Camera::GetK for models 0-3."""
    model = int(model)
    if model == S.PINHOLE:
        return float(p[0]), float(p[1]), float(p[2]), float(p[3])
    if model in (S.SIMPLE_PINHOLE, S.SIMPLE_RADIAL, S.RADIAL):
        return float(p[0]), float(p[0]), float(p[1]), float(p[2])
    raise ValueError(f"camera model {model} is not supported (models 0-3)")


def fundamental_from_motion_and_cameras(model1, params1, model2, params2, quat_xyzw, trans) -> np.ndarray:
    """F [3, 3] = K2^-T [t]x R K1^-1, R = Eigen's toRotationMatrix of ``quat_xyzw`` (not normalised).  Scalar FP64 in the
    device kernel's operation order (pc_promote), so the two agree bit for bit; K^-1 is taken in closed form."""
    x, y, z, w = (float(v) for v in quat_xyzw)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    R = [1.0 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.0 - (txx + tzz), tyz - twx, txz - twy, tyz + twx,
         1.0 - (txx + tyy)]
    t0, t1, t2 = (float(v) for v in trans)
    T = [0.0, -t2, t1, t2, 0.0, -t0, -t1, t0, 0.0]                                   # EssentialFromMotion: [t]x R
    E = [T[3 * r] * R[c] + T[3 * r + 1] * R[3 + c] + T[3 * r + 2] * R[6 + c] for r in range(3) for c in range(3)]
    fx1, fy1, cx1, cy1 = _pinhole(model1, params1)
    fx2, fy2, cx2, cy2 = _pinhole(model2, params2)
    ia, ib, ua, ub = 1.0 / fx1, 1.0 / fy1, -cx1 / fx1, -cy1 / fy1                    # M = E K1^-1
    M = []
    for r in range(3):
        M += [E[3 * r] * ia, E[3 * r + 1] * ib, E[3 * r] * ua + E[3 * r + 1] * ub + E[3 * r + 2]]
    ja, jb, va, vb = 1.0 / fx2, 1.0 / fy2, -cx2 / fx2, -cy2 / fy2                    # F = K2^-T M
    F = [M[c] * ja for c in range(3)] + [M[3 + c] * jb for c in range(3)] + \
        [M[c] * va + M[3 + c] * vb + M[6 + c] for c in range(3)]
    return np.array(F).reshape(3, 3)


def update_image_pairs_config(intr_model, intr_params, has_prior_focal, pair_cam1, pair_cam2, pair_valid, pair_quat,
                              pair_trans, pair_config, pair_F):
    """Host restatement.  K cameras (intr_model [K], intr_params [K, >= 4], has_prior_focal [K]), E pairs (pair_cam1 /
    pair_cam2 [E] camera of each image, pair_valid [E], pair_quat [E, 4] xyzw / pair_trans [E, 3] cam2_from_cam1,
    pair_config [E], pair_F [E, 9]).  Returns (config [E] int32, F [E, 9], number of pairs promoted); the inputs are not
    changed.  A camera index outside [0, K) raises ValueError."""
    models = np.asarray(intr_model).tolist()
    params = np.asarray(intr_params, np.float64)
    prior = np.asarray(has_prior_focal, bool).tolist()
    c1, c2 = np.asarray(pair_cam1).tolist(), np.asarray(pair_cam2).tolist()
    valid = np.asarray(pair_valid, bool).tolist()
    quat = np.asarray(pair_quat, np.float64).reshape(-1, 4)
    trans = np.asarray(pair_trans, np.float64).reshape(-1, 3)
    config = np.array(pair_config, np.int32)
    F = np.array(pair_F, np.float64).reshape(-1, 9)
    K = len(models)
    for a, b in zip(c1, c2):
        if not (0 <= a < K and 0 <= b < K):
            raise ValueError("pair camera index outside [0, K)")
    camera_counter: dict = {}                                      # camera -> [total, calibrated]
    for e in range(len(c1)):
        if not valid[e]:
            continue
        a, b = c1[e], c2[e]
        if not prior[a] or not prior[b]:
            continue
        if config[e] == TWO_VIEW_CALIBRATED:
            camera_counter.setdefault(a, [0, 0])
            camera_counter[a][0] += 1
            camera_counter.setdefault(b, [0, 0])
            camera_counter[b][0] += 1
            camera_counter[a][1] += 1
            camera_counter[b][1] += 1
        elif config[e] == TWO_VIEW_UNCALIBRATED:
            camera_counter.setdefault(a, [0, 0])
            camera_counter[a][0] += 1
            camera_counter.setdefault(b, [0, 0])
            camera_counter[b][0] += 1
    camera_validity: dict = {}
    for cam, (total, calibrated) in camera_counter.items():
        camera_validity[cam] = calibrated * 1. / total > 0.5
    promoted = 0
    for e in range(len(c1)):
        if not valid[e] or config[e] != TWO_VIEW_UNCALIBRATED:
            continue
        a, b = c1[e], c2[e]
        if camera_validity.get(a, False) and camera_validity.get(b, False):
            config[e] = TWO_VIEW_CALIBRATED
            F[e] = fundamental_from_motion_and_cameras(models[a], params[a], models[b], params[b], quat[e], trans[e]).ravel()
            promoted += 1
    return config, F, promoted


def _ptr(a):
    return a.ctypes.data_as(ct.c_void_p) if a is not None and a.size else None


def update_image_pairs_config_device(intr_model, intr_params, has_prior_focal, pair_cam1, pair_cam2, pair_valid, pair_quat,
                                     pair_trans, pair_config, pair_F, ctx=None):
    """``update_image_pairs_config`` on the GPU; same arguments and return value.  A camera index outside [0, K) raises
    ``_lib.B200Error`` (B200SFM_ERR_INVALID_ARG), and so does a promoted pair's camera model outside 0-3
    (B200SFM_ERR_UNSUPPORTED)."""
    from . import _lib, estimators as E_
    from .view_graph import _index_array
    model = _index_array(intr_model, "intr_model")
    K = len(model)
    params = np.zeros((K, S.INTR_STRIDE))
    p = np.asarray(intr_params, np.float64).reshape(K, -1)
    params[:, :min(p.shape[1], S.INTR_STRIDE)] = p[:, :S.INTR_STRIDE]
    prior = np.ascontiguousarray(np.asarray(has_prior_focal, bool).astype(np.uint8))
    c1, c2 = _index_array(pair_cam1, "pair_cam1"), _index_array(pair_cam2, "pair_cam2")
    E = len(c1)
    valid = np.ascontiguousarray(np.asarray(pair_valid, bool).astype(np.uint8))
    quat = np.ascontiguousarray(np.asarray(pair_quat, np.float64).reshape(-1, 4))
    trans = np.ascontiguousarray(np.asarray(pair_trans, np.float64).reshape(-1, 3))
    config = np.ascontiguousarray(np.array(pair_config, np.int32))
    F = np.ascontiguousarray(np.array(pair_F, np.float64).reshape(-1, 9))
    if prior.shape != (K,):
        raise ValueError("has_prior_focal must have one entry per camera")
    if len(c2) != E or valid.shape != (E,) or len(quat) != E or len(trans) != E or config.shape != (E,) or len(F) != E:
        raise ValueError("pair_cam2, pair_valid, pair_quat, pair_trans, pair_config and pair_F must have one entry per pair")
    ctx = ctx or E_.default_context()
    n = ct.c_int64(0)
    _lib.check(ctx.handle, ctx.lib.b200sfm_view_graph_update_pairs_config(
        ctx.handle, K, _ptr(model), _ptr(params), _ptr(prior), E, _ptr(c1), _ptr(c2), _ptr(valid), _ptr(quat), _ptr(trans),
        _ptr(config), _ptr(F), ct.byref(n)))
    return config, F, int(n.value)


def pair_arrays(pairs, cameras: dict, image_camera: dict):
    """Flat arrays of ``ImagePairMatches`` ``pairs`` over ``cameras`` ({camera id: ``image_pair_inliers.Camera``, with
    ``has_prior_focal_length`` as ``view_graph_calibration.CalibCamera`` has it; absent means False}) and
    ``image_camera`` ({image id: camera id}): a dict of the arguments of ``update_image_pairs_config``, the cameras in
    ascending id order."""
    cam_ids = sorted(cameras)
    idx = {c: k for k, c in enumerate(cam_ids)}
    cams = [cameras[c] for c in cam_ids]
    K, E = len(cams), len(pairs)
    params = np.zeros((K, S.INTR_STRIDE))
    for k, c in enumerate(cams):
        p = np.asarray(c.params, np.float64)
        params[k, :len(p)] = p
    return dict(intr_model=np.array([int(c.model) for c in cams], np.int32), intr_params=params,
                has_prior_focal=np.array([bool(getattr(c, "has_prior_focal_length", False)) for c in cams], bool),
                pair_cam1=np.array([idx[image_camera[p.image_id1]] for p in pairs], np.int32).reshape(E),
                pair_cam2=np.array([idx[image_camera[p.image_id2]] for p in pairs], np.int32).reshape(E),
                pair_valid=np.array([bool(p.is_valid) for p in pairs], bool).reshape(E),
                pair_quat=np.array([np.asarray(p.quat_xyzw, np.float64) for p in pairs]).reshape(E, 4),
                pair_trans=np.array([np.asarray(p.trans, np.float64) for p in pairs]).reshape(E, 3),
                pair_config=np.array([int(p.config) for p in pairs], np.int32).reshape(E),
                pair_F=np.array([np.asarray(p.F, np.float64).reshape(9) for p in pairs]).reshape(E, 9))


def UpdateImagePairsConfig(pairs, cameras: dict, image_camera: dict, device: bool = True, ctx=None) -> int:
    """ViewGraphManipulater::UpdateImagePairsConfig over ``ImagePairMatches`` objects (see ``pair_arrays``): sets
    ``config`` and ``F`` of the promoted pairs in place and returns their number.  ``device`` selects the GPU or the
    host restatement; both give the same configs."""
    if not pairs:
        return 0
    a = pair_arrays(pairs, cameras, image_camera)
    if device:
        config, F, n = update_image_pairs_config_device(**a, ctx=ctx)
    else:
        config, F, n = update_image_pairs_config(**a)
    for e in np.flatnonzero(config != a["pair_config"]):
        pairs[e].config = int(config[e])
        pairs[e].F = F[e].reshape(3, 3).copy()
    return n
