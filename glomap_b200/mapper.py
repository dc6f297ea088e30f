"""Host driver over the three estimators: stages 0, 1, 3, 5 and 6 of ``glomap::GlobalMapper::Solve``
(glomap/controllers/global_mapper.cc:19-276) on the flat SoA scene -- rotation averaging (run twice, with
``RelPoseFilter::FilterRotations`` and the largest connected component in between), global positioning followed by the
three track filters and ``NormalizeReconstruction``, then the staged bundle adjustment loop (positions only, then
rotations too; normalise; reprojection filters with the tightening threshold ``max(3 - ite, 1) * thr``), and, with
``skip_pruning = False``, stage 8: ``PruneWeaklyConnectedImages`` over the final tracks (``frame_cluster_id`` /
``frame_registered`` of the mapper; ``colmap_io.write_clustered_model`` writes one model per cluster).

After each rotation averaging run, ``RelPoseFilter::FilterRotations`` and ``ViewGraph::KeepLargestConnectedComponents``
(view_graph.py; on the GPU from ``VIEW_GRAPH_DEVICE_MIN_PAIRS`` pairs up) invalidate pairs and may leave images outside
the largest component.  Those images are unregistered (``image_registered`` of the mapper): the second run and the stages
after it see only the registered images (track establishment is given their ids; global positioning and bundle
adjustment run on the scene compacted to their cameras, and the results are scattered back), and an unregistered camera
keeps its input pose, as in the reference, where its frame is simply not optimised.

It mirrors the reference's control flow so that the GPU solvers are exercised in the order, and with the option
mutations, the real mapper uses; it is host glue (as in the reference) and owns no numerics: every solve and every
filter goes through ``libb200sfm.so``.  Stage 4, track establishment (``TrackEngine``: EstablishFullTracks, then
FindTracksForProblem, both on the device), runs when ``Solve`` is given the image pairs and features.

Given the image pairs and ``camera_prior_focal`` (Camera::has_prior_focal_length of every intrinsics block), stage 0's
``ViewGraphManipulater::UpdateImagePairsConfig`` (view_graph_manipulation.py; on the GPU from
``UPDATE_PAIRS_CONFIG_DEVICE_MIN_PAIRS`` pairs up) and stage 1's ``ViewGraphCalibrator`` run first: the focals without a
prior are refined and written into ``intr_params`` (so undistortion, global positioning and bundle adjustment use them),
and a view-graph edge whose pair stage 1 invalidated starts stage 3 invalid.  Global positioning then gives the cameras
without a prior the down-weighted loss and the angle filter the doubled threshold, as the reference does from the prior
flag (not from has_refined_focal_length).  Without ``camera_prior_focal`` every camera is calibrated and stages 0 and 1
do not run.

Not covered here: stage 0's DecomposeRelPose and stage 2, relative-pose estimation (COLMAP's
EstimateTwoViewGeometryPose and PoseLib in the reference; the pairs keep the cam2_from_cam1 they are given), and
retriangulation (COLMAP code).

``Solve`` takes trivial frames (``synthetic.Scene``, one camera = one frame) or camera rigs (``synthetic.RigScene``: several
rigs, each frame seen through the sensors of its rig, cam_from_rig known or not).  On rigs, stage 3 runs
``rotation_averager.solve_rotation_averaging_rig`` (which estimates the unknown cam_from_rig rotations; they get a NaN
translation) and filters the image rotations cam_from_rig * rig_from_world; the largest component is taken in frame
space, and an image is registered when its frame is (``frame_in_component`` / ``image_registered``).  Stages 4-6 run on
the problem compacted to the registered frames and the sensors they use: the selected tracks become (frame, sensor)
observations (``track_establishment.tracks_to_rig_scene``), global positioning uses the known cam_from_rig as offsets
and solves the NaN translations as RigUnknownBATA centres, then the filters, the normalisation and the staged bundle
adjustment run on the rig problem (with ``opt_ba.optimize_rig_poses`` every non-reference cam_from_rig is refined).
An unregistered frame keeps its input pose, a sensor without a registered image its input cam_from_rig.

Given gravity priors (``Solve(..., gravity=...)``: Frame::gravity_info, one row per camera on trivial frames, per frame
on rigs) and ``opt_ra.use_gravity``, both stage-3 paths run the gravity-aligned, stratified SolveRotationAveraging
(rotation_averager.py): the frames with a prior are 1-DoF about their gravity and, unless there are none or they make up
more than 95 % of the pairs, the pairs between two of them are solved first.  On trivial frames each run is
``solve_rotation_averaging`` on the registered pairs; on rigs, ``solve_rotation_averaging_rig`` folds the image pairs onto
the frames with the known cam_from_rig, and a sensor without one fails the solve, as in the reference.  The frames with a
prior start from R_align, as the reference's ReadGravity sets them.  Stages 4-8 do not read gravity."""
from __future__ import annotations

import dataclasses
from typing import TYPE_CHECKING

import numpy as np

from . import estimators as E, geometry as geo, processors as PR, reconstruction_pruning as RP, synthetic as S
from . import track_establishment as TE, view_graph as VG

if TYPE_CHECKING:
    from .view_graph_calibration import ViewGraphCalibratorOptions


@dataclasses.dataclass
class InlierThresholdOptions:
    """glomap/types.h:18-33."""
    max_angle_error: float = 1.0            # degrees, global positioning
    max_reprojection_error: float = 1e-2    # normalised image plane, bundle adjustment
    min_triangulation_angle: float = 1.0    # degrees
    max_rotation_error: float = 10.0        # degrees, rotation averaging
    # image pairs (image_pair_inliers.py)
    max_epipolar_error_E: float = 1.0       # pixels, converted with the mean focal of the two cameras
    max_epipolar_error_F: float = 4.0       # pixels
    max_epipolar_error_H: float = 4.0       # pixels
    min_inlier_num: float = 30              # RelPoseFilter::FilterInlierNum (takes it as an int)
    min_inlier_ratio: float = 0.25          # RelPoseFilter::FilterInlierRatio


def _vgc_options():
    # imported here: view_graph_calibration imports image_pair_inliers, which takes InlierThresholdOptions from this module
    from .view_graph_calibration import ViewGraphCalibratorOptions
    return ViewGraphCalibratorOptions()


@dataclasses.dataclass
class GlobalMapperOptions:
    """controllers/global_mapper.h:14-44 (the fields of the stages implemented here)."""
    opt_ra: E.RotationEstimatorOptions = dataclasses.field(default_factory=E.RotationEstimatorOptions)
    opt_gp: E.GlobalPositionerOptions = dataclasses.field(default_factory=E.GlobalPositionerOptions)
    opt_ba: E.BundleAdjusterOptions = dataclasses.field(default_factory=E.BundleAdjusterOptions)
    inlier_thresholds: InlierThresholdOptions = dataclasses.field(default_factory=InlierThresholdOptions)
    num_iteration_bundle_adjustment: int = 3
    skip_rotation_averaging: bool = False
    skip_global_positioning: bool = False
    skip_bundle_adjustment: bool = False
    skip_pruning: bool = True                # global_mapper.h:41; --skip_pruning 0 turns stage 8 on
    opt_track: TE.TrackEstablishmentOptions = dataclasses.field(default_factory=TE.TrackEstablishmentOptions)
    skip_track_establishment: bool = False   # stage 4 runs only when Solve is given the image pairs and features
    # stages 0 and 1 run only when Solve is given the image pairs and the cameras' prior-focal flags
    skip_preprocessing: bool = False         # global_mapper.h:33
    skip_view_graph_calibration: bool = False   # global_mapper.h:34
    opt_vgcalib: ViewGraphCalibratorOptions = dataclasses.field(default_factory=_vgc_options)


def compact_observations(scene: S.Scene, keep: np.ndarray) -> S.Scene:
    """Drop the observations with keep == False (what the filters do to ``Track::observations``); ``scene`` may be a
    ``Scene`` or a ``RigScene``."""
    keep = np.asarray(keep, bool)
    pt = np.repeat(np.arange(scene.P), np.diff(scene.pt_obs_begin))
    lens = np.bincount(pt[keep], minlength=scene.P)
    out = scene.copy()
    if isinstance(scene, S.RigScene):
        out.obs_frame, out.obs_sensor = scene.obs_frame[keep], scene.obs_sensor[keep]
    else:
        out.obs_cam = scene.obs_cam[keep]
    out.obs_xy = scene.obs_xy[keep]
    out.pt_obs_begin = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return out


def drop_tracks(scene: S.Scene, keep_track: np.ndarray) -> S.Scene:
    """FilterTrackTriangulationAngle clears the observations of the removed tracks (track_filter.cc:118-121)."""
    pt = np.repeat(np.arange(scene.P), np.diff(scene.pt_obs_begin))
    return compact_observations(scene, np.asarray(keep_track, bool)[pt])


def filter_rotations(vg: S.ViewGraph, R: np.ndarray, max_angle_deg: float) -> np.ndarray:
    """RelPoseFilter::FilterRotations (processors/relpose_filter.cc:7-33): valid-edge mask."""
    R_calc = R[vg.ej] @ np.swapaxes(R[vg.ei], -1, -2)
    return geo.rotation_angle_deg(R_calc, vg.R_rel) <= max_angle_deg


def largest_connected_component(n: int, ei, ej) -> np.ndarray:
    """ViewGraph::KeepLargestConnectedComponents (scene/view_graph.cc:56): image mask."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    g = sp.coo_matrix((np.ones(len(ei)), (ei, ej)), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    return lab == np.bincount(lab).argmax()


def _sub_view_graph(vg: S.ViewGraph, edge_mask) -> S.ViewGraph:
    return S.ViewGraph(vg.n_images, vg.ei[edge_mask], vg.ej[edge_mask], vg.R_rel[edge_mask], np.asarray(vg.weight)[edge_mask],
                       vg.R_gt)


# Below this many pairs the two view-graph passes of stage 3 run as the host restatements (view_graph.py), which give
# the same masks: a device call costs a few allocations, copies and synchronisations, more than the host loops over a
# handful of pairs (profiles/view_graph_filter_bench.py).
VIEW_GRAPH_DEVICE_MIN_PAIRS = 100
# Below this many pairs stage 0's UpdateImagePairsConfig runs as the host restatement (view_graph_manipulation.py), which
# gives the same configs and F to 1e-13 (profiles/update_pairs_config_bench.py).
UPDATE_PAIRS_CONFIG_DEVICE_MIN_PAIRS = 100


def registered_view_graph(vg: S.ViewGraph, pair_valid, image_registered):
    """The valid pairs between registered images, the images renumbered in ascending order: (view graph, image ids)."""
    idx = np.flatnonzero(image_registered)
    if len(idx) == vg.n_images:
        return _sub_view_graph(vg, np.asarray(pair_valid, bool)), idx
    remap = np.full(vg.n_images, -1, np.int64)
    remap[idx] = np.arange(len(idx))
    ei, ej = np.asarray(vg.ei), np.asarray(vg.ej)
    k = np.asarray(pair_valid, bool) & image_registered[ei] & image_registered[ej]
    R_gt = None if vg.R_gt is None else np.asarray(vg.R_gt)[idx]
    return S.ViewGraph(len(idx), remap[ei[k]].astype(np.int32), remap[ej[k]].astype(np.int32), np.asarray(vg.R_rel)[k],
                       np.asarray(vg.weight)[k], R_gt), idx


def compact_cameras(scene: S.Scene, idx: np.ndarray) -> S.Scene:
    """The scene over the cameras ``idx`` (ascending), renumbered in that order; the observations of the other cameras
    are dropped, every point is kept."""
    keep = np.zeros(scene.C, bool)
    keep[idx] = True
    out = compact_observations(scene, keep[scene.obs_cam])
    remap = np.full(scene.C, -1, np.int64)
    remap[idx] = np.arange(len(idx))
    out.obs_cam = remap[out.obs_cam].astype(np.int32)
    out.quat, out.trans, out.cam_intr = scene.quat[idx].copy(), scene.trans[idx].copy(), scene.cam_intr[idx].copy()
    return out


def scatter_cameras(full: S.Scene, part: S.Scene, idx: np.ndarray) -> S.Scene:
    """Inverse of ``compact_cameras``: ``full`` with the poses of the cameras ``idx``, the points, tracks and intrinsics of
    ``part``; the other cameras keep their poses."""
    out = full.copy()
    out.quat[idx], out.trans[idx] = part.quat, part.trans
    out.points, out.pt_obs_begin = part.points.copy(), part.pt_obs_begin.copy()
    out.obs_cam, out.obs_xy = np.asarray(idx)[part.obs_cam].astype(np.int32), part.obs_xy.copy()
    out.intr_model, out.intr_params = part.intr_model.copy(), part.intr_params.copy()
    return out


def compact_frames(scene: S.RigScene, frames: np.ndarray):
    """The rig problem over the frames ``frames`` (ascending), renumbered in that order: their images (in table order),
    the sensors those images use (ascending, renumbered; a rig whose reference sensor is dropped gets -1), the
    observations of those images; every point and intrinsics block is kept.  Returns (scene, sensor ids)."""
    frames = np.asarray(frames, np.int64)
    fmap = np.full(scene.F, -1, np.int64)
    fmap[frames] = np.arange(len(frames))
    img = fmap[scene.image_frame] >= 0
    sensors = np.unique(scene.image_sensor[img]).astype(np.int64)
    smap = np.full(scene.S, -1, np.int64)
    smap[sensors] = np.arange(len(sensors))
    out = compact_observations(scene, fmap[scene.obs_frame] >= 0)
    out.obs_frame = fmap[out.obs_frame].astype(np.int32)
    out.obs_sensor = smap[out.obs_sensor].astype(np.uint16)
    out.quat, out.trans = scene.quat[frames].copy(), scene.trans[frames].copy()
    out.sensor_quat, out.sensor_trans = scene.sensor_quat[sensors].copy(), scene.sensor_trans[sensors].copy()
    out.sensor_intr, out.sensor_known = scene.sensor_intr[sensors].copy(), scene.sensor_known[sensors].copy()
    out.sensor_rig, out.frame_rig = scene.sensor_rig[sensors].copy(), scene.frame_rig[frames].copy()
    out.rig_ref_sensor = smap[scene.rig_ref_sensor].astype(np.int32)
    out.image_frame = fmap[scene.image_frame[img]].astype(np.int32)
    out.image_sensor = smap[scene.image_sensor[img]].astype(np.int32)
    return out, sensors


def scatter_frames(full: S.RigScene, part: S.RigScene, frames: np.ndarray, sensors: np.ndarray) -> S.RigScene:
    """Inverse of ``compact_frames``: ``full`` with the poses of the frames ``frames`` and the cam_from_rig (and known
    flag) of the sensors ``sensors`` from ``part``, and its points, tracks and intrinsics; the other frames and sensors
    keep theirs."""
    frames, sensors = np.asarray(frames, np.int64), np.asarray(sensors, np.int64)
    out = full.copy()
    out.quat[frames], out.trans[frames] = part.quat, part.trans
    out.sensor_quat[sensors], out.sensor_trans[sensors] = part.sensor_quat, part.sensor_trans
    out.sensor_known[sensors] = part.sensor_known
    out.points, out.pt_obs_begin = part.points.copy(), part.pt_obs_begin.copy()
    out.obs_frame = frames[part.obs_frame].astype(np.int32)
    out.obs_sensor = sensors[part.obs_sensor.astype(np.int64)].astype(np.uint16)
    out.obs_xy = part.obs_xy.copy()
    out.intr_model, out.intr_params = part.intr_model.copy(), part.intr_params.copy()
    return out


def _ra_options(o: E.RotationEstimatorOptions):
    from . import rotation_averager as RA
    return RA.RotationAveragerOptions(**dataclasses.asdict(o))


class GlobalMapper:
    def __init__(self, options: GlobalMapperOptions | None = None, ctx: E.Context | None = None):
        self.options_ = options or GlobalMapperOptions()
        self.ctx = ctx
        self.log: list[str] = []
        self.frame_cluster_id: np.ndarray | None = None   # stage 8: cluster of every frame (-1: none)
        self.frame_registered: np.ndarray | None = None   # stage 8: frames of the largest visibility component
        self.image_registered: np.ndarray | None = None   # stage 3: images of the view graph's largest component
        self.frame_in_component: np.ndarray | None = None  # stage 3, rigs: frames of the view graph's largest component
        self.pair_valid_after_calibration: np.ndarray | None = None   # stage 1: is_valid of every image pair after it
        self.focal_refined: np.ndarray | None = None      # stage 1: intrinsics blocks whose focal the calibrator set
        self._prior_focal: np.ndarray | None = None       # [K] has_prior_focal_length per intrinsics block, or None
        self._gravity: np.ndarray | None = None           # [C,3] (trivial frames) / [F,3] (rigs) gravity priors, or None
        self._keep_input_state = False                     # global positioning starts from the input reconstruction

    # -- helpers ------------------------------------------------------------------------------------
    def _filters(self, scene: S.Scene, what) -> S.Scene:
        """Run a list of (kind, threshold) filters on ONE resident problem per filter (the observation set changes
        after each, as in the reference where every filter rewrites Track::observations)."""
        ctx = self.ctx or E.default_context()
        for kind, thr in what:
            prob = E.BAProblem(ctx, scene, self.options_.opt_ba.min_num_view_per_track)
            try:
                prob.set_state(scene.intr_params, scene.quat, scene.trans, scene.points)
                if kind == "angle":                                               # bearings: the device's own UndistortImages
                    keep, n = prob.filter_angle("resident", thr, self._calibrated_flags(scene))
                    scene = compact_observations(scene, keep)
                elif kind == "reprojection":
                    keep, n = prob.filter_reprojection(thr, "resident")
                    scene = compact_observations(scene, keep)
                else:
                    keep_t, n = prob.filter_triangulation_angle(thr)
                    scene = drop_tracks(scene, keep_t)
            finally:
                prob.free()
            self.log.append(f"filter {kind} thr={thr:g}: {n} tracks changed, {scene.N} observations left")
            self.last_filtered = n
        return scene

    def _filter_rotations(self, vg: S.ViewGraph, q_rel, R, valid, registered, max_angle):
        """RelPoseFilter::FilterRotations: (valid, pairs invalidated)."""
        return self._filter_rotations_q(vg, q_rel, geo.rotmat_to_quat_xyzw_fast(R), valid, registered, max_angle)

    def _filter_rotations_q(self, vg: S.ViewGraph, q_rel, q_img, valid, registered, max_angle):
        if vg.E >= VIEW_GRAPH_DEVICE_MIN_PAIRS:
            return VG.filter_rotations_device(q_img, vg.ei, vg.ej, q_rel, max_angle, valid, registered,
                                              self.ctx or E.default_context())
        return VG.filter_rotations(q_img, vg.ei, vg.ej, q_rel, max_angle, valid, registered)

    def _largest_component(self, vg: S.ViewGraph, valid, registered, image_frame=None):
        """ViewGraph::KeepLargestConnectedComponents in frame space (frames = images unless ``image_frame`` [I] is
        given, with ``registered`` then one flag per frame): (valid, registered, registered images)."""
        if image_frame is None:
            frame, F = np.arange(vg.n_images, dtype=np.int32), vg.n_images
        else:
            frame, F = image_frame, len(registered)
        if vg.E >= VIEW_GRAPH_DEVICE_MIN_PAIRS:
            return VG.keep_largest_connected_components_device(F, frame, vg.ei, vg.ej, valid, registered,
                                                               self.ctx or E.default_context())
        return VG.keep_largest_connected_components(F, frame, vg.ei, vg.ej, valid, registered)

    def _calibrated_flags(self, scene):
        """has_prior_focal_length of every camera (trivial frames) or sensor (rigs) of ``scene``, from the prior flags of
        their intrinsics blocks; None without prior flags, or when all are set (every camera calibrated: the solvers'
        default)."""
        if self._prior_focal is None or self._prior_focal.all():
            return None
        blocks = scene.sensor_intr if isinstance(scene, S.RigScene) else scene.cam_intr
        return self._prior_focal[np.asarray(blocks, np.int64)]

    def _calibrate_cameras(self, view_graph: S.ViewGraph, scene, image_pairs, features):
        """Stages 0 and 1 (:22-50): UpdateImagePairsConfig on the image pairs, then ViewGraphCalibrator.  The camera of
        an image is the intrinsics block of its camera (trivial frames) or sensor (rigs); image k is the k-th smallest id
        of ``features`` (image ids 0, 1, ... without features).  The pairs are copies: the caller's are not changed.
        Writes the accepted focals into ``scene.intr_params``.  Returns (ok, pairs, the view-graph edges that start stage
        3 valid): an edge whose pair (either orientation) stage 1 invalidated starts invalid."""
        from . import view_graph_calibration as VGC, view_graph_manipulation as VGM
        o = self.options_
        rig = isinstance(scene, S.RigScene)
        n_img = scene.I if rig else scene.C
        image_ids = sorted(int(i) for i in features) if features is not None else list(range(n_img))
        if len(image_ids) != n_img:
            raise ValueError(f"features name {len(image_ids)} images, the scene has {n_img}")
        image_intr = scene.sensor_intr[scene.image_sensor] if rig else scene.cam_intr
        image_camera = {iid: int(image_intr[k]) for k, iid in enumerate(image_ids)}
        K = len(scene.intr_model)
        prior = self._prior_focal
        if prior.shape != (K,):
            raise ValueError(f"camera_prior_focal has {prior.shape[0]} flags, the scene has {K} intrinsics blocks")
        cameras = {k: VGC.CalibCamera(int(scene.intr_model[k]),
                                      scene.intr_params[k, :S.MODEL_NUM_PARAMS[int(scene.intr_model[k])]].copy(),
                                      has_prior_focal_length=bool(prior[k])) for k in range(K)}
        pairs = [dataclasses.replace(p) for p in image_pairs]
        edge_valid = np.ones(view_graph.E, bool)
        if not o.skip_preprocessing:
            n = VGM.UpdateImagePairsConfig(pairs, cameras, image_camera,
                                           device=len(pairs) >= UPDATE_PAIRS_CONFIG_DEVICE_MIN_PAIRS, ctx=self.ctx)
            self.log.append(f"preprocessing: {n} pairs promoted to CALIBRATED")
        if not o.skip_view_graph_calibration:
            before = np.array([bool(p.is_valid) for p in pairs], bool)
            if not VGC.ViewGraphCalibrator(o.opt_vgcalib, self.ctx).Solve(pairs, cameras, image_camera):
                self.log.append("view graph calibration: the solution is not usable")
                return False, pairs, edge_valid
            self.pair_valid_after_calibration = np.array([bool(p.is_valid) for p in pairs], bool)
            self.focal_refined = np.array([cameras[k].has_refined_focal_length for k in range(K)], bool)
            for k in np.flatnonzero(self.focal_refined):
                for i in VGC.focal_length_idxs(scene.intr_model[k]):
                    scene.intr_params[k, i] = cameras[k].params[i]
            cut = before & ~self.pair_valid_after_calibration
            if cut.any():
                idx = {iid: k for k, iid in enumerate(image_ids)}
                a = np.array([idx[pairs[e].image_id1] for e in np.flatnonzero(cut)], np.int64)
                b = np.array([idx[pairs[e].image_id2] for e in np.flatnonzero(cut)], np.int64)
                key = np.minimum(a, b) * n_img + np.maximum(a, b)
                ei, ej = np.asarray(view_graph.ei, np.int64), np.asarray(view_graph.ej, np.int64)
                edge_valid = ~np.isin(np.minimum(ei, ej) * n_img + np.maximum(ei, ej), key)
            self.log.append(f"view graph calibration: {int(self.focal_refined.sum())} / {K} focals refined, "
                            f"{int(cut.sum())} pairs invalidated")
        return True, pairs, edge_valid

    # -- controllers/global_mapper.cc:19-355 (stages 0, 1, 3, 5, 6) ----------------------------------
    def Solve(self, view_graph: S.ViewGraph, scene: S.Scene, image_pairs=None, features: dict | None = None,
              camera_prior_focal=None, gravity=None, registered=None, keep_input_state: bool = False):
        """Returns (ok, scene): poses / points / intrinsics of ``scene`` estimated from the relative rotations of
        ``view_graph`` and the tracks of ``scene`` (its poses and points are only used when a stage is skipped).
        Given ``image_pairs`` (``track_establishment.ImagePairMatches``) and ``features`` ({image_id: [n,2] pixels}; camera k
        of ``scene`` is the k-th smallest image id), stage 4 builds the tracks on the device instead and the tracks of
        ``scene`` are not used.

        ``scene`` may be a ``synthetic.RigScene`` instead: ``view_graph`` is then over its images (image k = row k of the
        image table, and the k-th smallest id of ``features``), the poses are the frames' rig_from_world, and the
        sensors whose cam_from_rig is not known are estimated (see ``_solve_rig``).

        ``camera_prior_focal`` [K] flags the intrinsics blocks whose focal length is known (Camera::
        has_prior_focal_length).  Given it and ``image_pairs``, stages 0 (UpdateImagePairsConfig) and 1
        (ViewGraphCalibrator: the focals without a prior are refined and written into ``intr_params``, pairs with a large
        residual are invalidated) run first (see ``_calibrate_cameras``); stage 1's unusable solution fails the solve.
        Global positioning and the angle filter then treat the cameras without a prior as uncalibrated.  Without it,
        every camera is calibrated and stages 0 and 1 do not run.

        ``gravity``: the gravity priors (Frame::gravity_info), one row per camera of a ``Scene`` or per frame of a
        ``RigScene``, NaN rows for none.  With ``opt_ra.use_gravity`` stage 3 runs the gravity-aligned, stratified
        SolveRotationAveraging (see ``_rotation_averaging`` / ``_rotation_averaging_rig``); without it the priors are not
        read.  As in the reference, use_gravity with a sensor whose cam_from_rig is not known fails the solve.

        ``registered``: the input registration, [C] images of a ``Scene`` or [F] frames of a ``RigScene`` (all by
        default).  Only the registered images or frames reach stages 4-8, through the same compaction as stage 3's
        component cut (which can only unregister more of them); the others keep their input poses and lose their
        observations.

        ``keep_input_state``: the poses and points of ``scene`` are a reconstruction (a resumed model), so global
        positioning starts from them and randomises only what the reference randomises (global_positioning.cc:145-151,
        258-263): the frames observed by a track of >= min_num_view_per_track views and those tracks, and only with
        generate_random_* and optimize_* on; the other centres and points keep their input.  Without it every centre
        and point starts random, as before."""
        self._keep_input_state = bool(keep_input_state)
        self._prior_focal = None if camera_prior_focal is None else np.asarray(camera_prior_focal, bool).reshape(-1)
        self._gravity = None if gravity is None else np.asarray(gravity, np.float64)
        self.pair_valid_after_calibration = self.focal_refined = None
        n = scene.F if isinstance(scene, S.RigScene) else scene.C
        registered = np.ones(n, bool) if registered is None else np.asarray(registered, bool).reshape(-1)
        if registered.shape != (n,):
            raise ValueError(f"registered has {registered.shape[0]} flags, the scene has {n} "
                             f"{'frames' if isinstance(scene, S.RigScene) else 'images'}")
        if isinstance(scene, S.RigScene):
            return self._solve_rig(view_graph, scene, image_pairs, features, registered)
        o, thr = self.options_, self.options_.inlier_thresholds
        scene = scene.copy()
        edge_valid = np.ones(view_graph.E, bool)
        if image_pairs is not None and self._prior_focal is not None:
            ok, image_pairs, edge_valid = self._calibrate_cameras(view_graph, scene, image_pairs, features)
            if not ok:
                return False, scene
        track_stage = image_pairs is not None and features is not None and not o.skip_track_establishment
        # 3. rotation averaging: first run for filtering, second for the estimate, each followed by FilterRotations and
        # KeepLargestConnectedComponents (:84-116)
        self.image_registered = reg = registered
        if not o.skip_rotation_averaging:
            if not self._rotation_averaging(view_graph, scene, edge_valid):
                return False, scene
            self.image_registered = reg = self.image_registered & registered
        # cameras of the registered images: the problem of stages 4-6 (all of them unless stage 3 cut some off)
        cams = np.flatnonzero(reg)
        full = scene
        if len(cams) < scene.C:
            scene = compact_cameras(scene, cams)
        # 4. track establishment (:119-137) over the registered images
        if track_stage:
            image_ids = sorted(int(i) for i in features)
            if len(image_ids) != full.C:
                raise ValueError(f"features name {len(image_ids)} images, the scene has {full.C} cameras")
            reg_ids = [image_ids[k] for k in cams]
            full_tracks, discarded = TE.establish_full_tracks_device(image_pairs, features, o.opt_track, self.ctx)
            sel = TE.find_tracks_for_problem_device(full_tracks, reg_ids, o.opt_track, self.ctx)
            flat = TE.tracks_to_scene(sel, features, reg_ids, scene.cam_intr, scene.intr_model, scene.intr_params)
            flat.quat, flat.trans = scene.quat, scene.trans
            scene = flat
            self.log.append(f"track establishment: {len(full_tracks)} tracks ({discarded} discarded), {len(sel)} selected")
        ok, scene = self._solve_positions(scene)
        if len(cams) < full.C:
            scene = scatter_cameras(full, scene, cams)
        if not ok:
            return False, scene
        # 8. reconstruction pruning (:340-353): trivial frames, so the tracks' frames are their images
        if not o.skip_pruning:
            out = RP.prune_weakly_connected_images(scene.pt_obs_begin, scene.obs_cam, scene.C, ctx=self.ctx)
            self.frame_cluster_id, self.frame_registered = out["cluster_id"], out["is_registered"]
            self.log.append(f"pruning: {out['num_clusters']} clusters, threshold {out['stats']['strong_threshold']:g}")
        return True, scene

    def _gravity_start(self, R: np.ndarray) -> np.ndarray:
        """The rotations rotation averaging starts from with gravity: R_align for the frames with a prior, as
        ``ReadGravity`` sets them (io/pose_io.cc:170-175), ``R`` elsewhere."""
        from .gravity_refinement import get_align_rot_householder
        R = np.array(R, dtype=np.float64, copy=True)
        has = ~np.isnan(self._gravity).any(axis=1)
        R[has] = get_align_rot_householder(self._gravity[has])
        return R

    def _check_gravity(self, n: int, what: str):
        """The gravity rotation averaging is given: one row per ``what`` with use_gravity, None otherwise."""
        if self._gravity is None or not self.options_.opt_ra.use_gravity:
            return None
        if self._gravity.shape != (n, 3):
            raise ValueError(f"gravity must be [{n},3], one row per {what}, got {self._gravity.shape}")
        return self._gravity

    def _log_gravity(self, run: int, info: dict):
        if "gravity_pairs" in info:
            self.log.append(f"rotation averaging run {run + 1}: {info['gravity_pairs']} / {info['total_pairs']} pairs with "
                            f"gravity, 1-DoF pass {'run' if info.get('stratified') else 'skipped'}")
        self.log.extend(info.get("log", []))

    def _rotation_averaging(self, vg: S.ViewGraph, scene: S.Scene, edge_valid) -> bool:
        """Stage 3 on trivial frames (:84-116): rotation averaging twice, each run followed by FilterRotations and
        KeepLargestConnectedComponents.  Sets ``image_registered`` and, in ``scene``, the rotations of the registered
        cameras.  With gravity (one row per camera) and ``opt_ra.use_gravity`` each run is
        ``rotation_averager.solve_rotation_averaging`` on the registered pairs: the gravity-aligned, stratified
        SolveRotationAveraging.  The first run starts from R_align for the cameras with a prior and the identity
        elsewhere, the second from the first's rotations."""
        o, thr = self.options_, self.options_.inlier_thresholds
        gravity = self._check_gravity(scene.C, "camera")
        q_rel = geo.rotmat_to_quat_xyzw_fast(vg.R_rel)
        valid, reg = edge_valid.copy(), np.ones(vg.n_images, bool)
        R_all = None
        R_start = None if gravity is None else self._gravity_start(np.tile(np.eye(3), (vg.n_images, 1, 1)))
        for run in range(2):
            # SolveRotationAveraging solves on the largest component (rotation_averager.cc:13)
            valid, reg, num_img = self._largest_component(vg, valid, reg)
            self.image_registered = reg
            if num_img == 0:
                self.log.append(f"rotation averaging run {run + 1}: no pair is left")
                return False
            sub, idx = registered_view_graph(vg, valid, reg)
            if gravity is None:
                ra = E.RotationEstimator(o.opt_ra, self.ctx)
                ok, R = ra.EstimateRotations(sub)
            else:
                from . import rotation_averager as RA
                info = {}
                ok, R, _ = RA.solve_rotation_averaging(sub, gravity[idx], _ra_options(o.opt_ra), R_init=R_start[idx],
                                                       ctx=self.ctx, info=info)
                self._log_gravity(run, info)
            if not ok:
                if run == 1:
                    return False
                continue
            if gravity is None:
                R_all = np.tile(np.eye(3), (vg.n_images, 1, 1))
            else:
                R_all = R_start                        # the second run starts from the first's rotations
            R_all[idx] = R
            valid, cut = self._filter_rotations(vg, q_rel, R_all, valid, reg, thr.max_rotation_error)
            valid, reg, num_img = self._largest_component(vg, valid, reg)
            self.image_registered = reg
            if num_img == 0:
                self.log.append(f"rotation averaging run {run + 1}: no connected component is left")
                return False
            self.log.append(f"rotation averaging run {run + 1}: {cut} edges filtered, {num_img} / {vg.n_images} images "
                            "in the largest component")
        scene.quat = np.where(reg[:, None], geo.rotmat_to_quat_xyzw_fast(R_all), scene.quat)
        return True

    def _rotation_averaging_rig(self, vg: S.ViewGraph, scene: S.RigScene, edge_valid=None) -> bool:
        """Stage 3 on rigs (:84-116): SolveRotationAveraging twice, each run followed by FilterRotations on the image
        rotations cam_from_rig * rig_from_world and KeepLargestConnectedComponents in frame space.  Sets
        ``frame_in_component`` / ``image_registered`` and, in ``scene``, the rotations of the frames in the component
        and those of the sensors it estimated (with a NaN translation, global_rotation_averaging.cc:800-813).  With
        gravity (one row per frame) and ``opt_ra.use_gravity`` the driver runs gravity-aligned and stratified, the
        frames with a prior starting from R_align; a sensor without a known cam_from_rig then fails the run."""
        from . import rotation_averager as RA
        o, thr = self.options_, self.options_.inlier_thresholds
        fr, sen = scene.image_frame.astype(np.int64), scene.image_sensor.astype(np.int64)
        ref_sensor = scene.rig_ref_sensor[scene.frame_rig]
        known = scene.sensor_known.copy()
        known[scene.rig_ref_sensor] = True
        q_cam = scene.sensor_quat.copy()
        q_rel = geo.rotmat_to_quat_xyzw_fast(vg.R_rel)
        valid = np.ones(vg.E, bool) if edge_valid is None else edge_valid.copy()
        freg = np.ones(scene.F, bool)
        R = geo.quat_xyzw_to_rotmat(scene.quat)
        gravity = self._check_gravity(scene.F, "frame")
        if gravity is not None:
            R = self._gravity_start(R)
        estimated = np.zeros(scene.S, bool)
        ra_opts = _ra_options(o.opt_ra)
        for run in range(2):
            valid, freg, num_img = self._largest_component(vg, valid, freg, fr)
            self.frame_in_component, self.image_registered = freg, freg[fr]
            if num_img == 0:
                self.log.append(f"rotation averaging run {run + 1}: no pair is left")
                return False
            info = {}
            ok, R_run, R_cam, solved = RA.solve_rotation_averaging_rig(_sub_view_graph(vg, valid), fr, sen, known, q_cam,
                                                                       ref_sensor, ra_opts, R_init=R, ctx=self.ctx, info=info,
                                                                       gravity=gravity)
            self._log_gravity(run, info)
            if not ok:
                if run == 1:
                    return False
                continue
            R = R_run
            seen = np.zeros(scene.S, bool)
            seen[sen[solved[fr]]] = True
            new = seen & ~known                        # these cam_from_rig have a value from now on (.cc:800-813)
            q_cam[new] = geo.rotmat_to_quat_xyzw_fast(R_cam[new])
            known |= new
            estimated |= new
            # the image rotations; an image whose sensor has no rotation yet is NaN and keeps its pairs
            q_img = geo.rotmat_to_quat_xyzw_fast(np.einsum("nij,njk->nik", geo.quat_xyzw_to_rotmat(q_cam)[sen], R[fr]))
            q_img[~known[sen]] = np.nan
            valid, cut = self._filter_rotations_q(vg, q_rel, q_img, valid, freg[fr], thr.max_rotation_error)
            valid, freg, num_img = self._largest_component(vg, valid, freg, fr)
            self.frame_in_component, self.image_registered = freg, freg[fr]
            if num_img == 0:
                self.log.append(f"rotation averaging run {run + 1}: no connected component is left")
                return False
            self.log.append(f"rotation averaging run {run + 1}: {cut} edges filtered, {num_img} / {scene.I} images in "
                            f"the largest component ({int(freg.sum())} / {scene.F} frames)")
        scene.quat = np.where(freg[:, None], geo.rotmat_to_quat_xyzw_fast(R), scene.quat)
        has_image = np.zeros(scene.S, bool)
        has_image[sen[freg[fr]]] = True
        estimated &= has_image                         # a sensor without a registered image keeps its input
        scene.sensor_quat[estimated] = q_cam[estimated]
        scene.sensor_trans[estimated] = np.nan
        return True

    def _solve_rig(self, view_graph: S.ViewGraph, scene: S.RigScene, image_pairs=None, features: dict | None = None,
                   registered=None):
        """``Solve`` on rigs (global_mapper.cc:82-353).  Stage 3 (``_rotation_averaging_rig``) registers the images of
        the frames in the view graph's largest component.  Stages 4-6 run on the problem compacted to those frames and
        the sensors their images use: tracks over the registered images, global positioning with the known
        cam_from_rig as offsets and the sensors with a NaN translation as RigUnknownBATA centres (ConvertResults turns
        them into translations), the filters and normalisation on the rig problem, then the staged bundle adjustment
        (with ``opt_ba.optimize_rig_poses`` every non-reference sensor is a variable).  The results are scattered back:
        an unregistered frame keeps its input pose, a sensor without a registered image its input cam_from_rig.
        Stage 8 prunes in frame space."""
        o = self.options_
        full = scene.copy()
        edge_valid = None
        if image_pairs is not None and self._prior_focal is not None:
            ok, image_pairs, edge_valid = self._calibrate_cameras(view_graph, full, image_pairs, features)
            if not ok:
                return False, scene
        track_stage = image_pairs is not None and features is not None and not o.skip_track_establishment
        registered = np.ones(full.F, bool) if registered is None else registered
        if not o.skip_rotation_averaging and not self._rotation_averaging_rig(view_graph, full, edge_valid):
            return False, scene
        self.frame_in_component = registered if o.skip_rotation_averaging else self.frame_in_component & registered
        self.image_registered = self.frame_in_component[full.image_frame]
        frames = np.flatnonzero(self.frame_in_component)
        part, sensors = compact_frames(full, frames)
        # 4. track establishment (:119-137) over the registered images
        if track_stage:
            image_ids = sorted(int(i) for i in features)
            if len(image_ids) != full.I:
                raise ValueError(f"features name {len(image_ids)} images, the scene has {full.I}")
            reg_ids = [image_ids[k] for k in np.flatnonzero(self.image_registered)]
            full_tracks, discarded = TE.establish_full_tracks_device(image_pairs, features, o.opt_track, self.ctx)
            sel = TE.find_tracks_for_problem_device(full_tracks, reg_ids, o.opt_track, self.ctx)
            part = TE.tracks_to_rig_scene(sel, features, reg_ids, part)
            self.log.append(f"track establishment: {len(full_tracks)} tracks ({discarded} discarded), {len(sel)} selected")
        ok, part = self._solve_positions(part)
        out = scatter_frames(full, part, frames, sensors)
        if not ok:
            return False, out
        # 8. reconstruction pruning (:340-353) over the frames of the observations
        if not o.skip_pruning:
            images = np.bincount(out.image_frame[self.image_registered], minlength=out.F)
            res = RP.prune_weakly_connected_images(out.pt_obs_begin, out.obs_frame, out.F, frame_self_loop=images >= 2,
                                                   ctx=self.ctx)
            self.frame_cluster_id, self.frame_registered = res["cluster_id"], res["is_registered"]
            self.log.append(f"pruning: {res['num_clusters']} clusters, threshold {res['stats']['strong_threshold']:g}")
        return True, out

    def _solve_positions(self, scene: S.Scene):
        """Stages 5 and 6 on the registered cameras (or frames, for a ``RigScene``): (ok, scene)."""
        o, thr = self.options_, self.options_.inlier_thresholds
        # 5. global positioning (:143-189)
        if not o.skip_global_positioning:
            bear = PR.undistort_images(scene)
            gp = E.GlobalPositioner(o.opt_gp, self.ctx)
            # with keep_input_state the input centres and points, kept where the positioner does not randomise
            centers = points = None
            if self._keep_input_state:
                centers = geo.centers_from_pose(geo.quat_xyzw_to_rotmat(scene.quat), scene.trans)
                points = np.array(scene.points, np.float64, copy=True)
            if isinstance(scene, S.RigScene):
                # RigBATA with the known cam_from_rig; a NaN translation (rotation averaging's estimate) is unknown
                unk = np.isnan(scene.sensor_trans).any(axis=1)
                prob = E.PositioningProblem(scene.quat, scene.pt_obs_begin, scene.obs_frame, bear, obs_sensor=scene.obs_sensor,
                                            sensor_quat=scene.sensor_quat, sensor_trans=scene.sensor_trans,
                                            sensor_calibrated=self._calibrated_flags(scene),
                                            sensor_unknown=unk if unk.any() else None, centers=centers, points=points)
            else:
                prob = E.PositioningProblem(scene.quat, scene.pt_obs_begin, scene.obs_cam, bear,
                                            cam_calibrated=self._calibrated_flags(scene), centers=centers, points=points)
            if not gp.Solve(prob):
                return False, scene
            scene.trans, scene.points = prob.trans, prob.points
            if isinstance(scene, S.RigScene) and prob.sensor_unknown is not None:
                scene.sensor_trans = prob.sensor_trans                   # ConvertResults (.cc:578-582)
                scene.sensor_known = scene.sensor_known | prob.sensor_unknown
            scene = self._filters(scene, [("angle", thr.max_angle_error), ("triangulation", thr.min_triangulation_angle),
                                          ("reprojection", 10 * thr.max_reprojection_error)])
            PR.normalize_reconstruction(scene)
        # 6. bundle adjustment (:191-280)
        if not o.skip_bundle_adjustment:
            ite = 0
            while ite < o.num_iteration_bundle_adjustment:
                ba = E.BundleAdjuster(o.opt_ba, self.ctx)
                inner = ba.GetOptions()
                inner.optimize_rotations = False                          # 6.1 positions only (:207-211)
                if not ba.Solve(scene):
                    return False, scene
                inner.optimize_rotations = o.opt_ba.optimize_rotations    # 6.2 (:217-222)
                if inner.optimize_rotations and not ba.Solve(scene):
                    return False, scene
                self.log.append(f"bundle adjustment iteration {ite + 1}: cost {ba.summary.final_cost:.6g}")
                PR.normalize_reconstruction(scene)
                status, filtered = True, 0                                 # 6.3 (:236-262)
                while status and ite < o.num_iteration_bundle_adjustment:
                    scaling = max(3 - ite, 1)
                    scene = self._filters(scene, [("reprojection", scaling * thr.max_reprojection_error)])
                    filtered += self.last_filtered
                    if filtered > 1e-3 * scene.P:
                        status = False
                    else:
                        ite += 1
                if status:
                    self.log.append("fewer than 0.1% tracks are filtered, stop the iteration")
                    break
                ite += 1
            scene = self._filters(scene, [("reprojection", thr.max_reprojection_error),
                                          ("triangulation", thr.min_triangulation_angle)])
        return True, scene
