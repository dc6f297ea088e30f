"""Host-side mirror of the reference estimator classes over the C ABI.

Same class / option / method names and error behaviour as
  glomap::BundleAdjuster      glomap/estimators/bundle_adjustment.h:12-51
  glomap::GlobalPositioner    glomap/estimators/global_positioning.h:9-70
  glomap::RotationEstimator   glomap/estimators/global_rotation_averaging.h:39-87
but operating on the flat SoA containers of ``glomap_b200.synthetic`` (what the
C++ shim builds from the reference's unordered_maps in sorted-id order,
INTEGRATION.md).  ``Solve`` mutates the container in place and returns a bool
like the reference.  All arithmetic happens in libb200sfm.so on the GPU.
"""
from __future__ import annotations

import ctypes as ct
import dataclasses

import numpy as np

from . import _lib
from ._lib import BAOpts, B200Error, LMStats


def _ptr(a: np.ndarray | None):
    return None if a is None else a.ctypes.data_as(ct.c_void_p)


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


class Context:
    """One per process and GPU (b200sfm_create / b200sfm_create_dist)."""

    def __init__(self, device: int = 0, rank: int = 0, world_size: int = 1, nccl_id: bytes | None = None):
        self.lib = _lib.load()
        h = ct.c_void_p()
        if world_size > 1:
            buf = ct.create_string_buffer(nccl_id, _lib.NCCL_ID_BYTES)
            rc = self.lib.b200sfm_create_dist(device, rank, world_size, buf, ct.byref(h))
        else:
            rc = self.lib.b200sfm_create(device, ct.byref(h))
        if rc != 0:
            raise B200Error(rc, "b200sfm_create failed (is a CUDA device visible? there is no CPU fallback)")
        self.handle = h
        self.rank, self.world_size = rank, world_size

    @staticmethod
    def nccl_unique_id() -> bytes:
        buf = ct.create_string_buffer(_lib.NCCL_ID_BYTES)
        rc = _lib.load().b200sfm_nccl_unique_id(buf)
        if rc != 0:
            raise B200Error(rc, "b200sfm_nccl_unique_id failed")
        return buf.raw

    def close(self):
        if self.handle:
            self.lib.b200sfm_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(0)
    return _default_ctx


# ---------------------------------------------------------------------------
# Bundle adjustment
# ---------------------------------------------------------------------------
@dataclasses.dataclass
class SolverOptions:
    """The ceres::Solver::Options fields the reference sets
    (optimization_base.h:18-23) + the PCG knobs of this implementation."""
    max_num_iterations: int = 100
    function_tolerance: float = 1e-5
    gradient_tolerance: float = 1e-10
    parameter_tolerance: float = 1e-8
    pcg_max_iterations: int = 500
    pcg_min_iterations: int = 0
    pcg_rel_tolerance: float = 1e-2
    preconditioner: int = 1


@dataclasses.dataclass
class BundleAdjusterOptions:
    """bundle_adjustment.h:12-37 (defaults identical)."""
    optimize_rig_poses: bool = False
    optimize_rotations: bool = True
    optimize_translation: bool = True
    optimize_intrinsics: bool = True
    optimize_principal_point: bool = False
    optimize_points: bool = True
    use_gpu: bool = True
    gpu_index: str = "-1"
    min_num_images_gpu_solver: int = 50
    min_num_view_per_track: int = 3
    thres_loss_function: float = 1.0
    solver_options: SolverOptions = dataclasses.field(default_factory=lambda: SolverOptions(max_num_iterations=200))
    # implementation extras
    profile_kernels: bool = False
    fixed_num_iterations: int = 0
    design: int = 0          # 0 auto, 1 = v1 (W blocks + atomics), 2 = v2 (compact rows, two passes)

    def to_c(self) -> BAOpts:
        o = BAOpts()
        _lib.load().b200sfm_ba_default_opts(ct.byref(o))
        for f in ("optimize_rig_poses", "optimize_rotations", "optimize_translation", "optimize_intrinsics",
                  "optimize_principal_point", "optimize_points", "profile_kernels"):
            setattr(o, f, int(getattr(self, f)))
        o.min_num_view_per_track = self.min_num_view_per_track
        o.thres_loss_function = self.thres_loss_function
        o.fixed_num_iterations = self.fixed_num_iterations
        o.design = self.design
        so = self.solver_options
        for f in ("max_num_iterations", "function_tolerance", "gradient_tolerance", "parameter_tolerance",
                  "pcg_max_iterations", "pcg_min_iterations", "pcg_rel_tolerance", "preconditioner"):
            setattr(o, f, getattr(so, f))
        return o


def first_frame_mask(C: int) -> np.ndarray:
    """The reference holds the first frame (in its map order) constant,
    bundle_adjustment.cc:261-266; the shim orders frames by id, so index 0."""
    m = np.zeros(C, dtype=np.uint8)
    if C:
        m[0] = 3
    return m


class BAProblem:
    """Device-resident BA problem (b200sfm_ba_problem_*)."""

    def __init__(self, ctx: Context, scene, min_num_view_per_track: int = 3, cam_const_mask: np.ndarray | None = None):
        self.ctx, self.lib = ctx, ctx.lib
        self.C, self.P, self.N, self.K = scene.C, scene.P, scene.N, len(scene.intr_model)
        mask = first_frame_mask(self.C) if cam_const_mask is None else _c(cam_const_mask, np.uint8)
        h = ct.c_void_p()
        if hasattr(scene, "obs_sensor"):
            # known rigs (synthetic.RigScene): the pose blocks are frames, the images carry a constant cam_from_rig
            self._keep = [_c(scene.pt_obs_begin, np.int64), _c(scene.obs_frame, np.int32), _c(scene.obs_sensor, np.uint16),
                          _c(scene.obs_xy, np.float64), _c(scene.sensor_quat, np.float64), _c(scene.sensor_trans, np.float64),
                          _c(scene.sensor_intr, np.int32), _c(scene.intr_model, np.int32)]
            rc = self.lib.b200sfm_ba_problem_create_rig(ctx.handle, self.C, self.P, self.N, self.K, scene.S,
                                                        *[_ptr(a) for a in self._keep], _ptr(mask), min_num_view_per_track,
                                                        ct.byref(h))
            _lib.check(ctx.handle, rc)
            self.handle = h
            self.S = scene.S
            # the image table, unless it is the dense layout the problem assumes without it (normalize() reads it)
            fr, se = np.asarray(scene.image_frame), np.asarray(scene.image_sensor)
            dense = len(fr) == scene.F * scene.S and np.array_equal(fr, np.arange(len(fr)) // scene.S) \
                and np.array_equal(se, np.arange(len(se)) % scene.S)
            if not dense:
                self._keep += [_c(fr, np.int32), _c(se, np.int32)]
                _lib.check(ctx.handle, self.lib.b200sfm_ba_problem_set_images(h, len(fr), _ptr(self._keep[-2]),
                                                                              _ptr(self._keep[-1])))
            return
        self.S = 0
        self._keep = [_c(scene.pt_obs_begin, np.int64), _c(scene.obs_cam, np.int32), _c(scene.obs_xy, np.float64),
                      _c(scene.cam_intr, np.int32), _c(scene.intr_model, np.int32)]
        rc = self.lib.b200sfm_ba_problem_create(ctx.handle, self.C, self.P, self.N, self.K, *[_ptr(a) for a in self._keep],
                                                _ptr(mask), min_num_view_per_track, ct.byref(h))
        _lib.check(ctx.handle, rc)
        self.handle = h

    def set_state(self, intr_params, quat, trans, points):
        a = [_c(intr_params, np.float64), _c(quat, np.float64), _c(trans, np.float64), _c(points, np.float64)]
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_set_state(self.handle, *[_ptr(x) for x in a]))

    def get_state(self):
        intr = np.empty((self.K, _lib.INTR_STRIDE)); quat = np.empty((self.C, 4)); trans = np.empty((self.C, 3))
        pts = np.empty((self.P, 3))
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_get_state(self.handle, _ptr(intr), _ptr(quat), _ptr(trans), _ptr(pts)))
        return intr, quat, trans, pts

    def set_sensor_variable(self, sensor_variable):
        """optimize_rig_poses: the sensors whose cam_from_rig is an unknown (bundle_adjustment.cc:296-308: every
        non-reference camera sensor); effective when options.optimize_rig_poses is set."""
        v = _c(sensor_variable, np.uint8)
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_set_sensor_variable(self.handle, _ptr(v)))

    def get_sensor_poses(self):
        q = np.empty((self.S, 4)); t = np.empty((self.S, 3))
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_get_sensor_poses(self.handle, _ptr(q), _ptr(t)))
        return q, t

    def save_state(self):
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_save_state(self.handle))

    def restore_state(self):
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_restore_state(self.handle))

    def solve(self, options: BundleAdjusterOptions) -> LMStats:
        st = LMStats()
        o = options.to_c()
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_solve(self.handle, ct.byref(o), ct.byref(st)))
        return st

    def cost(self, options: BundleAdjusterOptions) -> float:
        o = options.to_c()
        c = ct.c_double()
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_cost(self.handle, ct.byref(o), ct.byref(c)))
        return c.value

    # -- processors on the resident state -------------------------------------------
    def normalize(self, fixed_scale: bool = False, extent: float = 10.0, p0: float = 0.1, p1: float = 0.9):
        """NormalizeReconstruction (glomap/processors/reconstruction_normalizer.cc:5-104) on the device state: returns
        (scale, translation[3]) of the applied similarity X' = scale X + t."""
        sc = ct.c_double()
        t = np.zeros(3)
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_normalize(self.handle, int(fixed_scale), extent, p0, p1, ct.byref(sc), _ptr(t)))
        return sc.value, t

    def undistort(self, download: bool = True):
        """UndistortImages (glomap/processors/image_undistorter.cc:7-53): unit bearings [N,3] of all observations from the
        current intrinsics; they stay resident for the bearing-based filters (``bearings="resident"``)."""
        out = np.empty((self.N, 3)) if download else None
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_undistort(self.handle, _ptr(out)))
        return out

    # -- track filters on the resident state (glomap/processors/track_filter.cc) --
    def filter_reprojection(self, max_reprojection_error: float, bearings=None):
        """TrackFilter::FilterTracksByReprojection: (keep [N] bool, #tracks changed).  Pixel space by default
        (in_normalized_image = false); with ``bearings`` (features_undist) the normalised-image-plane variant the
        mapper uses (track_filter.cc:24-31)."""
        keep = np.empty(self.N, np.uint8)
        cnt = ct.c_int64()
        if bearings is not None:
            b = None if isinstance(bearings, str) else _c(bearings, np.float64)   # "resident": the device's own bearings
            _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_filter_reprojection_normalized(
                self.handle, _ptr(b), max_reprojection_error, _ptr(keep), ct.byref(cnt)))
            return keep.astype(bool), cnt.value
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_filter_reprojection(self.handle, max_reprojection_error, _ptr(keep), ct.byref(cnt)))
        return keep.astype(bool), cnt.value

    def filter_angle(self, bearings, max_angle_error_deg: float, cam_calibrated=None):
        """TrackFilter::FilterTracksByAngle."""
        keep = np.empty(self.N, np.uint8)
        cnt = ct.c_int64()
        b = None if isinstance(bearings, str) else _c(bearings, np.float64)       # "resident": the device's own bearings
        cal = None if cam_calibrated is None else _c(cam_calibrated, np.uint8)
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_filter_angle(self.handle, _ptr(b), _ptr(cal), max_angle_error_deg, _ptr(keep), ct.byref(cnt)))
        return keep.astype(bool), cnt.value

    def filter_triangulation_angle(self, min_angle_deg: float):
        """TrackFilter::FilterTrackTriangulationAngle: (keep_track [P] bool, #tracks removed)."""
        keep = np.empty(self.P, np.uint8)
        cnt = ct.c_int64()
        _lib.check(self.ctx.handle, self.lib.b200sfm_ba_problem_filter_triangulation_angle(self.handle, min_angle_deg, _ptr(keep), ct.byref(cnt)))
        return keep.astype(bool), cnt.value

    def free(self):
        if self.handle:
            self.lib.b200sfm_ba_problem_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class BundleAdjuster:
    """glomap::BundleAdjuster (bundle_adjustment.h:38-51): options are copied
    at construction and may be mutated through GetOptions() between Solve calls
    (controllers/global_mapper.cc:204-219)."""

    def __init__(self, options: BundleAdjusterOptions | None = None, ctx: Context | None = None):
        self.options_ = dataclasses.replace(options) if options else BundleAdjusterOptions()
        self.ctx = ctx
        self.summary: LMStats | None = None

    def GetOptions(self) -> BundleAdjusterOptions:
        return self.options_

    def Solve(self, scene, cam_const_mask: np.ndarray | None = None) -> bool:
        """One-shot b200sfm_ba_solve with host buffers; poses, points (and
        intrinsics) of ``scene`` are updated in place.  Returns False on empty
        input (bundle_adjustment.cc:17-24) or an unusable solution (.cc:105)."""
        if scene.C == 0 or scene.P == 0 or scene.N == 0:
            return False
        ctx = self.ctx or default_context()
        lib = ctx.lib
        if hasattr(scene, "obs_sensor"):
            # known rigs (bundle_adjustment.cc:147-161): resident-problem path, pose blocks = frames
            prob = BAProblem(ctx, scene, self.options_.min_num_view_per_track, cam_const_mask)
            try:
                prob.set_state(scene.intr_params, scene.quat, scene.trans, scene.points)
                if self.options_.optimize_rig_poses:
                    # bundle_adjustment.cc:296-308: the cam_from_rig of every non-reference sensor is an unknown
                    ref = getattr(scene, "sensor_is_ref", np.arange(scene.S) == 0)
                    prob.set_sensor_variable((~np.asarray(ref, bool)).astype(np.uint8))
                self.summary = prob.solve(self.options_)
                scene.intr_params, scene.quat, scene.trans, scene.points = prob.get_state()
                if self.options_.optimize_rig_poses:
                    scene.sensor_quat, scene.sensor_trans = prob.get_sensor_poses()
            finally:
                prob.free()
            return bool(self.summary.usable)
        o = self.options_.to_c()
        st = LMStats()
        ptb, cam, xy = _c(scene.pt_obs_begin, np.int64), _c(scene.obs_cam, np.int32), _c(scene.obs_xy, np.float64)
        ci, im = _c(scene.cam_intr, np.int32), _c(scene.intr_model, np.int32)
        intr, quat = _c(scene.intr_params, np.float64), _c(scene.quat, np.float64)
        trans, pts = _c(scene.trans, np.float64), _c(scene.points, np.float64)
        mask = first_frame_mask(scene.C) if cam_const_mask is None else _c(cam_const_mask, np.uint8)
        rc = lib.b200sfm_ba_solve(ctx.handle, ct.byref(o), scene.C, scene.P, scene.N, len(im), _ptr(ptb), _ptr(cam),
                                  _ptr(xy), _ptr(ci), _ptr(im), _ptr(intr), _ptr(quat), _ptr(trans), _ptr(mask),
                                  _ptr(pts), ct.byref(st))
        self.summary = st
        if rc == 4:   # B200SFM_ERR_EMPTY
            return False
        _lib.check(ctx.handle, rc)
        scene.intr_params, scene.quat, scene.trans, scene.points = intr, quat, trans, pts
        return bool(st.usable)


# ---------------------------------------------------------------------------
# Global positioning (BATA)
# ---------------------------------------------------------------------------
@dataclasses.dataclass
class GlobalPositionerOptions:
    """global_positioning.h:9-54 (defaults identical).  Only ONLY_POINTS is
    implemented -- the constraint type the mapper enforces
    (controllers/global_mapper.cc:145-149)."""
    ONLY_POINTS = 0
    generate_random_positions: bool = True
    generate_random_points: bool = True
    generate_scales: bool = True
    optimize_positions: bool = True
    optimize_points: bool = True
    optimize_scales: bool = True
    use_gpu: bool = True
    gpu_index: str = "-1"
    min_num_images_gpu_solver: int = 50
    min_num_view_per_track: int = 3
    seed: int = 1
    constraint_type: int = 0
    thres_loss_function: float = 1e-1
    solver_options: SolverOptions = dataclasses.field(default_factory=lambda: SolverOptions(max_num_iterations=100, pcg_max_iterations=1000))
    profile_kernels: bool = False
    fixed_num_iterations: int = 0

    def to_c(self) -> _lib.GPOpts:
        o = _lib.GPOpts()
        _lib.load().b200sfm_gp_default_opts(ct.byref(o))
        for f in ("optimize_positions", "optimize_points", "optimize_scales", "profile_kernels"):
            setattr(o, f, int(getattr(self, f)))
        o.min_num_view_per_track = self.min_num_view_per_track
        o.thres_loss_function = self.thres_loss_function
        o.fixed_num_iterations = self.fixed_num_iterations
        so = self.solver_options
        for f in ("max_num_iterations", "function_tolerance", "gradient_tolerance", "parameter_tolerance",
                  "pcg_max_iterations", "pcg_min_iterations", "pcg_rel_tolerance", "preconditioner"):
            setattr(o, f, getattr(so, f))
        return o


@dataclasses.dataclass
class PositioningProblem:
    """Flat GP input (what the shim builds from frames/images/tracks):
    rotations are known (from rotation averaging), bearings are
    Image::features_undist (scene/image.h:31)."""
    quat: np.ndarray           # [C,4] cam_from_world rotations (fixed during GP)
    pt_obs_begin: np.ndarray   # [P+1]
    obs_cam: np.ndarray        # [N]
    bearings: np.ndarray       # [N,3] unit bearings in the camera frame
    cam_calibrated: np.ndarray | None = None   # [C] has_prior_focal_length
    centers: np.ndarray | None = None          # [C,3] filled by Solve (or initial values)
    points: np.ndarray | None = None           # [P,3]
    scales: np.ndarray | None = None           # [N]
    trans: np.ndarray | None = None            # [C,3] cam_from_world translations, written by Solve
    # known rigs (global_positioning.cc:325-346): quat/obs_cam/centers then refer to FRAMES (rig_from_world)
    obs_sensor: np.ndarray | None = None       # [N] sensor of the observing image
    sensor_quat: np.ndarray | None = None      # [S,4] cam_from_rig rotations
    sensor_trans: np.ndarray | None = None     # [S,3] cam_from_rig translations (rig scale 1)
    sensor_calibrated: np.ndarray | None = None  # [S] has_prior_focal_length of the sensor's camera
    # unknown cam_from_rig translations (global_positioning.cc:347-364, RigUnknownBATA): the camera centre in the rig
    # frame of these sensors is an unknown shared by their images; sensor_trans is ignored for them on input and holds
    # the estimated cam_from_rig translation (-R_cr c_cr, ConvertResults .cc:578-582) on return
    sensor_unknown: np.ndarray | None = None     # [S] bool
    rig_centers: np.ndarray | None = None        # [S,3] initial / estimated centres (rows of known sensors unused)

    @property
    def C(self):
        return len(self.quat)

    @property
    def P(self):
        return len(self.pt_obs_begin) - 1

    @property
    def N(self):
        return len(self.obs_cam)


def world_bearings(quat, bearings_cam, obs_cam):
    """t_obs = R_cw^T * bearing (global_positioning.cc:294-296) -- host-side input prep."""
    from . import geometry as geo
    R = geo.quat_xyzw_to_rotmat(np.asarray(quat, dtype=np.float64))[np.asarray(obs_cam)]
    return np.einsum("nji,nj->ni", R, bearings_cam)


def rig_world_terms(quat_frames, sensor_quat, sensor_trans, bearings_cam, obs_frame, obs_sensor):
    """Known rigs: (t_obs, t_rig) per observation with R_cw = R_cam_from_rig R_rig_from_world --
    t_obs = R_cw^T bearing (.cc:294-296), t_rig = R_cw^T t_cam_from_rig (.cc:339-345)."""
    from . import geometry as geo
    Rf = geo.quat_xyzw_to_rotmat(np.asarray(quat_frames, dtype=np.float64))[np.asarray(obs_frame)]
    Rs = geo.quat_xyzw_to_rotmat(np.asarray(sensor_quat, dtype=np.float64))[np.asarray(obs_sensor)]
    Rcw = np.einsum("nij,njk->nik", Rs, Rf)
    t_obs = np.einsum("nji,nj->ni", Rcw, bearings_cam)
    t_rig = np.einsum("nji,nj->ni", Rcw, np.asarray(sensor_trans, dtype=np.float64)[np.asarray(obs_sensor)])
    return t_obs, t_rig


class GlobalPositioner:
    """glomap::GlobalPositioner (global_positioning.h:56-70)."""

    def __init__(self, options: GlobalPositionerOptions | None = None, ctx: Context | None = None):
        self.options_ = dataclasses.replace(options) if options else GlobalPositionerOptions()
        self.ctx = ctx
        self.rng = np.random.default_rng(self.options_.seed)    # reference: std::mt19937(seed), .cc:23-26
        self.summary: LMStats | None = None

    def GetOptions(self) -> GlobalPositionerOptions:
        return self.options_

    def Solve(self, prob: PositioningProblem) -> bool:
        """Returns False on empty input (global_positioning.cc:37-50) or an
        unusable solution; on success ``prob.centers/points/scales`` hold the
        optimum and ``prob.trans = -R c`` (ConvertResults, .cc:562-572)."""
        o = self.options_
        if o.constraint_type != GlobalPositionerOptions.ONLY_POINTS:
            raise NotImplementedError("only ONLY_POINTS is implemented (controllers/global_mapper.cc:145-149)")
        if prob.C == 0 or prob.P == 0 or prob.N == 0:
            return False
        ctx = self.ctx or default_context()
        lib = ctx.lib
        # InitializeRandomPositions (.cc:123-165) / random points (.cc:261-264): 100 * U(-1,1)^3
        if o.generate_random_positions and o.optimize_positions or prob.centers is None:
            prob.centers = 100.0 * self.rng.uniform(-1, 1, size=(prob.C, 3))
        if o.generate_random_points and o.optimize_points or prob.points is None:
            prob.points = 100.0 * self.rng.uniform(-1, 1, size=(prob.P, 3))
        if o.generate_scales or prob.scales is None:
            prob.scales = np.ones(prob.N)                               # .cc:298
        ptb, cam = _c(prob.pt_obs_begin, np.int64), _c(prob.obs_cam, np.int32)
        cal = None if prob.cam_calibrated is None else _c(prob.cam_calibrated, np.uint8)
        cen, pts, sc = _c(prob.centers, np.float64), _c(prob.points, np.float64), _c(prob.scales, np.float64)
        co = o.to_c()
        st = LMStats()
        if prob.obs_sensor is not None:
            # RigBATA with constant rig scale: resident-problem path + per-observation rig terms
            unk = None if prob.sensor_unknown is None else np.asarray(prob.sensor_unknown, bool)
            st_in = np.array(prob.sensor_trans, dtype=np.float64, copy=True)
            if unk is not None and unk.any():
                st_in[unk] = 0.0                                         # no known offset for these images
            t_obs, t_rig = rig_world_terms(prob.quat, prob.sensor_quat, st_in, prob.bearings, prob.obs_cam, prob.obs_sensor)
            t_obs, t_rig = _c(t_obs, np.float64), _c(t_rig, np.float64)
            ocal = None if prob.sensor_calibrated is None else _c(
                np.asarray(prob.sensor_calibrated)[np.asarray(prob.obs_sensor)], np.uint8)
            h = ct.c_void_p()
            rc = lib.b200sfm_gp_problem_create(ctx.handle, prob.C, prob.P, prob.N, _ptr(ptb), _ptr(cam), _ptr(t_obs), None,
                                               None, o.min_num_view_per_track, ct.byref(h))
            if rc == 4:
                return False
            _lib.check(ctx.handle, rc)
            try:
                _lib.check(ctx.handle, lib.b200sfm_gp_problem_set_rig_terms(h, _ptr(t_rig), _ptr(ocal)))
                ucen = None
                if unk is not None and unk.any():
                    from . import geometry as geo
                    uidx = np.full(len(unk), -1, np.int32)
                    uidx[unk] = np.arange(int(unk.sum()), dtype=np.int32)
                    obs_us = _c(uidx[np.asarray(prob.obs_sensor)], np.int32)
                    frot = _c(geo.quat_xyzw_to_rotmat(np.asarray(prob.quat, np.float64)).reshape(-1, 9), np.float64)
                    if prob.rig_centers is None or (o.generate_random_positions and o.optimize_positions):
                        rc0 = np.zeros((len(unk), 3))
                        rc0[unk] = self.rng.uniform(-1, 1, size=(int(unk.sum()), 3))       # .cc:440-453
                        prob.rig_centers = rc0
                    ucen = _c(np.asarray(prob.rig_centers, np.float64)[unk], np.float64)
                    _lib.check(ctx.handle, lib.b200sfm_gp_problem_set_rig_unknown(h, int(unk.sum()), _ptr(obs_us), _ptr(frot), _ptr(ucen)))
                _lib.check(ctx.handle, lib.b200sfm_gp_problem_set_state(h, _ptr(cen), _ptr(pts), _ptr(sc)))
                _lib.check(ctx.handle, lib.b200sfm_gp_problem_solve(h, ct.byref(co), ct.byref(st)))
                _lib.check(ctx.handle, lib.b200sfm_gp_problem_get_state(h, _ptr(cen), _ptr(pts), _ptr(sc)))
                if ucen is not None:
                    from . import geometry as geo
                    _lib.check(ctx.handle, lib.b200sfm_gp_problem_get_rig_unknown(h, _ptr(ucen)))
                    prob.rig_centers = np.array(prob.rig_centers, dtype=np.float64, copy=True)
                    prob.rig_centers[unk] = ucen
                    Rs = geo.quat_xyzw_to_rotmat(np.asarray(prob.sensor_quat, np.float64))
                    prob.sensor_trans = np.array(prob.sensor_trans, dtype=np.float64, copy=True)
                    prob.sensor_trans[unk] = -np.einsum("sij,sj->si", Rs[unk], ucen)    # ConvertResults .cc:578-582
            finally:
                lib.b200sfm_gp_problem_free(h)
            self.summary = st
            prob.centers, prob.points, prob.scales = cen, pts, sc
            from . import geometry as geo
            prob.trans = -np.einsum("nij,nj->ni", geo.quat_xyzw_to_rotmat(prob.quat), cen)   # ConvertResults .cc:566-570
            return bool(st.usable)
        t_obs = _c(world_bearings(prob.quat, prob.bearings, prob.obs_cam), np.float64)
        rc = lib.b200sfm_gp_solve(ctx.handle, ct.byref(co), prob.C, prob.P, prob.N, _ptr(ptb), _ptr(cam), _ptr(t_obs),
                                  _ptr(cal), None, _ptr(cen), _ptr(pts), _ptr(sc), ct.byref(st))
        self.summary = st
        if rc == 4:
            return False
        _lib.check(ctx.handle, rc)
        prob.centers, prob.points, prob.scales = cen, pts, sc
        from . import geometry as geo
        R = geo.quat_xyzw_to_rotmat(prob.quat)
        prob.trans = -np.einsum("nij,nj->ni", R, cen)                   # ConvertResults .cc:566-568
        return bool(st.usable)


# ---------------------------------------------------------------------------
# Rotation averaging
# ---------------------------------------------------------------------------
@dataclasses.dataclass
class RotationEstimatorOptions:
    """global_rotation_averaging.h:39-75 (defaults identical)."""
    GEMAN_MCCLURE = 0
    HALF_NORM = 1
    max_num_l1_iterations: int = 5
    l1_step_convergence_threshold: float = 0.001
    max_num_irls_iterations: int = 100
    irls_step_convergence_threshold: float = 0.001
    irls_loss_parameter_sigma: float = 5.0
    weight_type: int = 0
    skip_initialization: bool = False
    use_weight: bool = False
    use_gravity: bool = False
    pcg_max_iterations: int = 5000
    pcg_rel_tolerance: float = 1e-8

    def to_c(self) -> _lib.RAOpts:
        o = _lib.RAOpts()
        _lib.load().b200sfm_ra_default_opts(ct.byref(o))
        for f in ("max_num_l1_iterations", "l1_step_convergence_threshold", "max_num_irls_iterations",
                  "irls_step_convergence_threshold", "irls_loss_parameter_sigma", "weight_type", "pcg_max_iterations",
                  "pcg_rel_tolerance"):
            setattr(o, f, getattr(self, f))
        o.use_weight = int(self.use_weight)
        return o


def initialize_from_maximum_spanning_tree(vg, R_init: np.ndarray | None = None) -> np.ndarray:
    """Host-side InitializeFromMaximumSpanningTree
    (global_rotation_averaging.cc:87-138 + math/tree.cc:78-170): Kruskal on
    (max_weight - weight), BFS from index 0, compose R_child from the parent
    along tree edges.  O(E log E); the reference that initialize_from_maximum_spanning_tree_device is tested against."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import breadth_first_order, minimum_spanning_tree
    n = vg.n_images
    wmax = float(vg.weight.max()) if vg.E else 0.0
    cost = (wmax - vg.weight) + 1e-9 * (1 + np.arange(vg.E) / max(vg.E, 1))   # strictly positive, stable tie order
    G = sp.coo_matrix((cost, (vg.ei, vg.ej)), shape=(n, n)).tocsr()
    G = G.maximum(G.T)
    T = minimum_spanning_tree(G)
    T = T.maximum(T.T).tocsr()
    order, pred = breadth_first_order(T, 0, directed=False)
    R = np.tile(np.eye(3), (n, 1, 1)) if R_init is None else np.array(R_init, copy=True)
    lut = {}
    for e in range(vg.E):
        lut[(int(vg.ei[e]), int(vg.ej[e]))] = e
    for node in order[1:]:
        par = int(pred[node])
        if (int(node), par) in lut:          # image_id1 == curr: R_curr = R_rel^T R_parent   (.cc:125-129)
            R[node] = vg.R_rel[lut[(int(node), par)]].T @ R[par]
        else:                                # R_curr = R_rel R_parent                          (.cc:130-134)
            R[node] = vg.R_rel[lut[(par, int(node))]] @ R[par]
    return R


# EstimateRotations initialises on the device from this many edges up (single-rank contexts).  On an H100 the device
# call (about 0.6 ms of fixed cost: copies, launches, a few synchronisations) was faster than the host function at every
# size measured, down to 45 edges, but by no more than about 0.2 ms below 200 edges (profiles/mst_init_bench.py, DESIGN.md 6.w);
# the smallest graphs stay on the host, where the two cost the same to within that margin.
MST_DEVICE_MIN_EDGES = 100


def initialize_from_maximum_spanning_tree_device(vg, R_init: np.ndarray | None = None, ctx: Context | None = None,
                                                 root: int = 0, stats: _lib.MSTStats | None = None):
    """InitializeFromMaximumSpanningTree on the device (b200sfm_ra_mst_init): the same tree and composition as
    initialize_from_maximum_spanning_tree, rooted at ``root``, which starts from R_init[root] (the identity without
    R_init).  Unreached nodes keep R_init.  Returns (R [n,3,3], parent [n]: parent[root] = root, unreached -1);
    ``stats``, when given, receives the call's b200sfm_mst_stats."""
    ctx = ctx or default_context()
    n = vg.n_images
    R = np.tile(np.eye(3), (n, 1, 1)) if R_init is None else np.array(R_init, dtype=np.float64, order="C", copy=True)
    if R.shape != (n, 3, 3):
        raise ValueError(f"R_init must be [{n},3,3], got {R.shape}")
    parent = np.empty(n, np.int32)
    st = stats if stats is not None else _lib.MSTStats()
    ei, ej = _c(vg.ei, np.int32), _c(vg.ej, np.int32)
    Rr, w = _c(np.reshape(vg.R_rel, (-1, 9)), np.float64), _c(vg.weight, np.float64)
    _lib.check(ctx.handle, ctx.lib.b200sfm_ra_mst_init(ctx.handle, n, len(ei), _ptr(ei), _ptr(ej), _ptr(Rr), _ptr(w), root,
                                                       _ptr(R), _ptr(parent), ct.byref(st)))
    return R, parent


def rig_view_graph(vg, img_frame, img_sensor, sensor_quat, R_gt_frames=None):
    """Known rigs in rotation averaging (global_rotation_averaging.cc:274-309): the unknowns are the
    FRAME rotations, an image pair (i, j) contributes
        R_rel(frames) = R_cam2_from_rig2^T * R_cam2_from_cam1 * R_cam1_from_rig1
    and pairs inside one frame are skipped (self loops).  Returns a ViewGraph over the frames."""
    from . import geometry as geo
    from .synthetic import ViewGraph
    img_frame, img_sensor = np.asarray(img_frame), np.asarray(img_sensor)
    Rs = geo.quat_xyzw_to_rotmat(np.asarray(sensor_quat, dtype=np.float64))
    fi, fj = img_frame[vg.ei], img_frame[vg.ej]
    keep = fi != fj
    R1 = Rs[img_sensor[vg.ei[keep]]]
    R2 = Rs[img_sensor[vg.ej[keep]]]
    R_rel = np.einsum("nji,njk,nkl->nil", R2, vg.R_rel[keep], R1)
    n_frames = int(img_frame.max()) + 1
    R_gt = np.tile(np.eye(3), (n_frames, 1, 1)) if R_gt_frames is None else np.asarray(R_gt_frames)
    return ViewGraph(n_frames, fi[keep].astype(np.int32), fj[keep].astype(np.int32), R_rel,
                     np.asarray(vg.weight)[keep].copy(), R_gt)


def rig_view_graph_unknown(vg, img_frame, img_sensor, sensor_quat, sensor_known):
    """Rigs with sensors whose cam_from_rig is NOT known yet (global_rotation_averaging.cc:173-245,274-309,425-440): the
    unknowns are the frame rotations followed by one rotation per uncalibrated sensor.  An image pair contributes
    R_rel = R_c2r2^T R_21 R_c1r1 with the identity for an uncalibrated sensor, -I / +I blocks on its frames and on the
    uncalibrated cameras; a pair inside one frame is dropped only when both sensors are calibrated (.cc:300-304).
    Returns dict(n_frames, n_cams, ei, ej, eci, ecj, R_rel, weight, cam_of_sensor [S] (-1 or node index),
    cam_frames_begin, cam_frames)."""
    from . import geometry as geo
    img_frame, img_sensor = np.asarray(img_frame), np.asarray(img_sensor)
    known = np.asarray(sensor_known, bool)
    n_frames = int(img_frame.max()) + 1
    cam_idx = np.full(len(known), -1, np.int64)
    cam_idx[~known] = n_frames + np.arange(int((~known).sum()))
    Rs = geo.quat_xyzw_to_rotmat(np.asarray(sensor_quat, dtype=np.float64)).copy()
    Rs[~known] = np.eye(3)
    fi, fj = img_frame[vg.ei], img_frame[vg.ej]
    si, sj = img_sensor[vg.ei], img_sensor[vg.ej]
    keep = ~((fi == fj) & known[si] & known[sj])
    R_rel = np.einsum("nji,njk,nkl->nil", Rs[sj[keep]], vg.R_rel[keep], Rs[si[keep]])
    frames_of = [np.unique(img_frame[img_sensor == s_]) for s_ in np.nonzero(~known)[0]]
    cfb = np.concatenate([[0], np.cumsum([len(f) for f in frames_of])]).astype(np.int32)
    return dict(n_frames=n_frames, n_cams=int((~known).sum()), ei=fi[keep].astype(np.int32), ej=fj[keep].astype(np.int32),
                eci=cam_idx[si[keep]].astype(np.int32), ecj=cam_idx[sj[keep]].astype(np.int32), R_rel=R_rel,
                weight=np.asarray(vg.weight)[keep].copy(), cam_of_sensor=cam_idx, cam_frames_begin=cfb,
                cam_frames=(np.concatenate(frames_of) if frames_of else np.zeros(0)).astype(np.int32))


class RotationEstimator:
    """glomap::RotationEstimator (global_rotation_averaging.h:77-87)."""

    def __init__(self, options: RotationEstimatorOptions | None = None, ctx: Context | None = None):
        self.options_ = options or RotationEstimatorOptions()     # the reference keeps a const& (.h:140)
        self.ctx = ctx
        self.summary: _lib.RAStats | None = None

    def EstimateRotations(self, vg, R_init: np.ndarray | None = None, fixed: int = 0, gravity: np.ndarray | None = None):
        """Returns (ok, R [n,3,3] cam_from_world rotations).  False on a NaN
        step/weight (.cc:508-512,590-593).  ``gravity`` [n,3] (NaN rows = no
        gravity prior) is used when options.use_gravity: those frames become
        1-DoF (.cc:207-217) and the initialisation is skipped (.cc:61-63)."""
        from . import geometry as geo
        o = self.options_
        n = vg.n_images
        use_grav = o.use_gravity and gravity is not None
        ctx = self.ctx or default_context()
        if not o.skip_initialization and not o.use_gravity:
            if ctx.world_size == 1 and vg.E >= MST_DEVICE_MIN_EDGES:
                R0, _ = initialize_from_maximum_spanning_tree_device(vg, R_init, ctx)
            else:
                R0 = initialize_from_maximum_spanning_tree(vg, R_init)
        else:
            R0 = np.tile(np.eye(3), (n, 1, 1)) if R_init is None else np.asarray(R_init, dtype=np.float64)
        co = o.to_c()
        st = _lib.RAStats()
        ei, ej = _c(vg.ei, np.int32), _c(vg.ej, np.int32)
        w = _c(vg.weight, np.float64)
        if not use_grav:
            theta = _c(geo.so3_log(R0), np.float64)
            Rr = _c(vg.R_rel.reshape(-1, 9), np.float64)
            rc = ctx.lib.b200sfm_ra_solve(ctx.handle, ct.byref(co), n, vg.E, _ptr(ei), _ptr(ej), _ptr(Rr), _ptr(w), fixed,
                                          _ptr(theta), ct.byref(st))
            self.summary = st
            if rc == 4:
                return False, None
            _lib.check(ctx.handle, rc)
            return bool(st.usable), geo.so3_exp(theta)
        hg, R_align, theta, Rr, g_fixed = gravity_aligned_inputs(vg, R0, gravity)
        fixed = fixed if g_fixed is None else g_fixed
        theta = _c(theta, np.float64)
        Rr = _c(Rr.reshape(-1, 9), np.float64)
        hg8 = _c(hg, np.uint8)
        rc = ctx.lib.b200sfm_ra_solve_gravity(ctx.handle, ct.byref(co), n, vg.E, _ptr(ei), _ptr(ej), _ptr(Rr), _ptr(w),
                                              _ptr(hg8), fixed, _ptr(theta), ct.byref(st))
        self.summary = st
        if rc == 4:
            return False, None
        _lib.check(ctx.handle, rc)
        R = geo.so3_exp(theta)
        R[hg] = R_align[hg] @ R[hg]                                                       # ConvertResults .cc:787-793
        return bool(st.usable), R


def gravity_aligned_inputs(vg, R0, gravity):
    """The host preparation of the gravity-aligned solve (SetupLinearSystem, global_rotation_averaging.cc:207-217,
    311-326) over the frame graph ``vg``: the frames with a prior (non-NaN rows of ``gravity`` [n,3]) carry
    theta = (0, RotUpToAngle(R_align^T R0), 0), the others the angle-axis of R0; a pair's R_rel is multiplied by
    R_align1 on the right when frame 1 has a prior and by R_align2^T on the left when frame 2 has one.  Returns
    (has_gravity [n], R_align [n,3,3] (identity without a prior), theta [n,3], aligned R_rel [E,3,3], the gauge: the
    first frame with a prior, or None without one)."""
    from . import geometry as geo
    n = vg.n_images
    g = np.asarray(gravity, dtype=np.float64)
    hg = ~np.isnan(g).any(axis=1)
    R_align = np.tile(np.eye(3), (n, 1, 1))
    for i in np.nonzero(hg)[0]:
        R_align[i] = get_align_rot(g[i])
    theta = geo.so3_log(R0)
    for i in np.nonzero(hg)[0]:
        theta[i] = [0.0, geo.so3_log((R_align[i].T @ R0[i])[None])[0, 1], 0.0]     # RotUpToAngle
    Rr = np.array(vg.R_rel, dtype=np.float64, copy=True)
    gi, gj = hg[vg.ei], hg[vg.ej]
    Rr[gi] = Rr[gi] @ R_align[vg.ei[gi]]
    Rr[gj] = np.swapaxes(R_align[vg.ej[gj]], -1, -2) @ Rr[gj]
    fixed = int(np.nonzero(hg)[0][0]) if hg.any() else None                            # .cc:213-217
    return hg, R_align, theta, Rr, fixed


def estimate_rotations_rig_unknown(est: "RotationEstimator", g: dict, R_frames0, R_cams0, fixed: int = 0):
    """RotationEstimator::EstimateRotations over the flattening of rig_view_graph_unknown: returns
    (ok, R_frames [F,3,3], R_cams [n_cams,3,3] = the estimated cam_from_rig rotations, .cc:805-813)."""
    from . import geometry as geo
    ctx = est.ctx or default_context()
    co = est.options_.to_c()
    st = _lib.RAStats()
    theta = _c(np.concatenate([geo.so3_log(np.asarray(R_frames0, np.float64)), geo.so3_log(np.asarray(R_cams0, np.float64))]), np.float64)
    a = [_c(g["ei"], np.int32), _c(g["ej"], np.int32), _c(g["eci"], np.int32), _c(g["ecj"], np.int32),
         _c(g["R_rel"].reshape(-1, 9), np.float64), _c(g["weight"], np.float64), _c(g["cam_frames_begin"], np.int32),
         _c(g["cam_frames"], np.int32)]
    rc = ctx.lib.b200sfm_ra_solve_rig(ctx.handle, ct.byref(co), g["n_frames"], g["n_cams"], len(a[0]), *[_ptr(x) for x in a], fixed,
                                      _ptr(theta), ct.byref(st))
    est.summary = st
    if rc == 4:
        return False, None, None
    _lib.check(ctx.handle, rc)
    R = geo.so3_exp(theta)
    return bool(st.usable), R[:g["n_frames"]], R[g["n_frames"]:]


def get_align_rot(gravity) -> np.ndarray:
    """GetAlignRot (math/gravity.cc:11-24): rotation whose second column is the
    gravity direction (any orthonormal completion; the 1-DoF angle absorbs the choice)."""
    v = np.asarray(gravity, dtype=np.float64)
    v = v / np.linalg.norm(v)
    a = np.array([1.0, 0, 0]) if abs(v[0]) < 0.9 else np.array([0, 0, 1.0])
    x = np.cross(v, a)
    x /= np.linalg.norm(x)
    z = np.cross(x, v)
    R = np.stack([x, v, z], axis=1)
    if np.linalg.det(R) < 0:
        R[:, 2] = -R[:, 2]
    return R
