/* b200sfm.h -- C ABI of the H100-native global-SfM solver core.
 *
 * This is the drop-in boundary for the three numeric hot loops of
 * colmap/glomap's estimators.  The reference has no FFI layer: the seam is the
 * public surface of its estimator classes, and each entry point below replaces
 * the arithmetic behind one of them (paths relative to the reference root):
 *
 *   b200sfm_ba_*   <-  glomap::BundleAdjuster::Solve
 *                      glomap/estimators/bundle_adjustment.h:38-51, .cc:11-106
 *   b200sfm_gp_*   <-  glomap::GlobalPositioner::Solve
 *                      glomap/estimators/global_positioning.h:56-70, .cc:28-93
 *   b200sfm_ra_*   <-  glomap::RotationEstimator::EstimateRotations
 *                      glomap/estimators/global_rotation_averaging.h:77-87, .cc:40-85
 *
 * Conventions: plain pointers and sizes only (no C++/torch types), caller-owned
 * HOST buffers unless a parameter is documented as a device pointer, FP64
 * values, int32 indices (int64 CSR offsets), return 0 on success or a
 * b200sfm_status code; b200sfm_last_error() gives the message.  A context is
 * thread-compatible (one thread at a time), distinct contexts are independent
 * -- the same contract as the reference estimators (SURVEY.md 8(b)).
 * There is no CPU fallback behind any of these calls.
 */
#ifndef B200SFM_H_
#define B200SFM_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200SFM_VERSION 100
/* doubles reserved per intrinsics block (colmap Camera::params, un-vendored) */
#define B200SFM_INTR_STRIDE 12
#define B200SFM_NCCL_ID_BYTES 128

typedef enum {
  B200SFM_OK = 0,
  B200SFM_ERR_INVALID_ARG = 1,
  B200SFM_ERR_CUDA = 2,
  B200SFM_ERR_NCCL = 3,
  B200SFM_ERR_EMPTY = 4,        /* reference returns false: no images / no tracks */
  B200SFM_ERR_UNSUPPORTED = 5,
  B200SFM_ERR_NUMERIC = 6       /* NaN encountered (reference: LOG(ERROR) + false) */
} b200sfm_status;

/* COLMAP camera model ids supported on the device (colmap/sensor/models.h). */
typedef enum {
  B200SFM_SIMPLE_PINHOLE = 0,   /* f, cx, cy */
  B200SFM_PINHOLE = 1,          /* fx, fy, cx, cy */
  B200SFM_SIMPLE_RADIAL = 2,    /* f, cx, cy, k */
  B200SFM_RADIAL = 3            /* f, cx, cy, k1, k2 */
} b200sfm_camera_model;

typedef enum {
  B200SFM_TERM_NONE = 0,
  B200SFM_TERM_FUNCTION_TOLERANCE = 1,
  B200SFM_TERM_PARAMETER_TOLERANCE = 2,
  B200SFM_TERM_GRADIENT_TOLERANCE = 3,
  B200SFM_TERM_MAX_ITERATIONS = 4,
  B200SFM_TERM_MIN_RADIUS = 5,
  B200SFM_TERM_INVALID_STEPS = 6
} b200sfm_termination;

typedef struct b200sfm_ctx b200sfm_ctx;

/* ---- context ------------------------------------------------------------ */
int b200sfm_version(void);
/* One context per process and GPU.  `device` is the CUDA ordinal
 * (reference: colmap::SetBestCudaDevice(gpu_indices[0]),
 * bundle_adjustment.cc:79-84). */
int b200sfm_create(int device, b200sfm_ctx** out);
/* Multi-GPU: one process per GPU; rank 0 obtains an id with
 * b200sfm_nccl_unique_id and the host distributes it (torch.distributed /
 * MPI / file).  Points (with all their observations) or edges are sharded
 * across ranks by the caller; camera-sized vectors are replicated and
 * all-reduced over NCCL inside the solver (SURVEY.md 8(e)). */
int b200sfm_nccl_unique_id(void* out_id /* B200SFM_NCCL_ID_BYTES */);
int b200sfm_create_dist(int device, int rank, int world_size, const void* nccl_id, b200sfm_ctx** out);
void b200sfm_destroy(b200sfm_ctx* ctx);
const char* b200sfm_last_error(const b200sfm_ctx* ctx);
int b200sfm_rank(const b200sfm_ctx* ctx);
int b200sfm_world_size(const b200sfm_ctx* ctx);
/* the cudaStream_t every kernel of this context is launched on (for CUDA-event timing by the host) */
void* b200sfm_cuda_stream(const b200sfm_ctx* ctx);
/* kernels launched by this context so far */
int64_t b200sfm_kernel_launches(const b200sfm_ctx* ctx);

/* ---- statistics common to the LM-based solvers (BA, GP) ------------------ */
typedef struct {
  int32_t iterations;            /* LM iterations (successful + unsuccessful) == ceres summary.iterations - 1 */
  int32_t num_successful_steps;
  int32_t termination;           /* b200sfm_termination */
  int32_t usable;                /* summary.IsSolutionUsable() */
  double initial_cost;
  double final_cost;
  int64_t num_observations;      /* residual blocks actually used (this rank) */
  int64_t pcg_iterations;        /* total PCG iterations (mat-vecs) */
  int64_t kernel_launches;       /* kernels of this library launched by the call */
  double ms_total;               /* device time of the whole solve (CUDA events) */
  double ms_linearize;           /* accumulated time of the Jacobian+Schur kernel */
  int64_t n_linearize;
  double ms_matvec;              /* accumulated time of the implicit-Schur mat-vec kernel */
  int64_t n_matvec;
  double ms_h2d;                 /* host->device copies inside the call */
  double ms_d2h;
  int64_t h2d_bytes;
  int64_t d2h_bytes;
} b200sfm_lm_stats;

/* ---- (iii) bundle adjustment --------------------------------------------- */
/* Field-for-field mirror of BundleAdjusterOptions (bundle_adjustment.h:12-37)
 * + the inherited ceres::Solver::Options the reference sets
 * (optimization_base.h:18-23), + the PCG knobs of this implementation. */
typedef struct {
  int32_t optimize_rig_poses;        /* unknown cam_from_rig of the sensors marked with b200sfm_ba_problem_set_sensor_variable */
  int32_t optimize_rotations;        /* default 1 */
  int32_t optimize_translation;      /* default 1 */
  int32_t optimize_intrinsics;       /* default 1 in the reference; shared blocks, <= 12 variable parameters in total */
  int32_t optimize_principal_point;  /* default 0 */
  int32_t optimize_points;           /* default 1 */
  int32_t min_num_view_per_track;    /* default 3 */
  int32_t max_num_iterations;        /* default 200 */
  double thres_loss_function;        /* Huber threshold, default 1.0 px */
  double function_tolerance;         /* default 1e-5 */
  double gradient_tolerance;         /* Ceres default 1e-10 */
  double parameter_tolerance;        /* Ceres default 1e-8 */
  /* implementation knobs (no reference counterpart: the reference factors
   * the reduced camera system with CHOLMOD, bundle_adjustment.cc:94-96) */
  int32_t pcg_max_iterations;        /* default 500 */
  int32_t pcg_min_iterations;        /* default 0 */
  double pcg_rel_tolerance;          /* ||r_k|| <= tol * ||r_0||, default 1e-2 */
  int32_t preconditioner;            /* 0 = block-Jacobi on U, 1 = Schur-Jacobi (default) */
  int32_t profile_kernels;           /* 1: time linearize / mat-vec kernels with CUDA events */
  int32_t fixed_num_iterations;      /* >0: run exactly this many LM iterations (bench), ignore tolerances */
  int32_t design;                    /* data layout of the Schur passes: 0 = auto, 1 = v1 (stored 6x3 W blocks, atomics per
                                        observation), 2 = v2 (compact J rows in both orders, camera-order second pass).
                                        Identical arithmetic; auto picks v2 unless intrinsics are optimised. */
} b200sfm_ba_opts;

void b200sfm_ba_default_opts(b200sfm_ba_opts* opts);

/* One-shot solve with host buffers: uploads, solves, writes the results back
 * in place (the estimator mutates frames/tracks/cameras in place,
 * bundle_adjustment.cc:140-146).
 *   C cameras (frames with trivial rigs), P points (tracks), N observations,
 *   K intrinsics blocks.
 *   pt_obs_begin [P+1]  CSR by point over the observation arrays
 *   obs_cam      [N]    camera index of each observation
 *   obs_xy       [N][2] observed (distorted) pixel, Image::features
 *   cam_intr     [C]    intrinsics block of each camera
 *   intr_model   [K]    b200sfm_camera_model
 *   intr_params  [K][B200SFM_INTR_STRIDE]   in/out
 *   quat_xyzw    [C][4] cam_from_world rotation, Eigen coeffs order, in/out
 *   trans        [C][3] cam_from_world translation, in/out
 *   cam_const_mask [C]  bit0: rotation constant, bit1: translation constant.
 *                       The shim sets 3 on the first frame
 *                       (bundle_adjustment.cc:261-266).  May be NULL.
 *   points       [P][3] in/out
 * In a distributed context every rank passes its own shard of points and
 * observations and the same cameras/intrinsics. */
int b200sfm_ba_solve(b200sfm_ctx* ctx, const b200sfm_ba_opts* opts, int32_t C, int32_t P, int64_t N, int32_t K,
                     const int64_t* pt_obs_begin, const int32_t* obs_cam, const double* obs_xy,
                     const int32_t* cam_intr, const int32_t* intr_model, double* intr_params,
                     double* quat_xyzw, double* trans, const uint8_t* cam_const_mask, double* points,
                     b200sfm_lm_stats* stats);

/* Resident problem: upload once, solve many times (GlobalMapper re-solves the
 * same BundleAdjuster after flipping GetOptions().optimize_rotations,
 * controllers/global_mapper.cc:204-221). */
typedef struct b200sfm_ba_problem b200sfm_ba_problem;
int b200sfm_ba_problem_create(b200sfm_ctx* ctx, int32_t C, int32_t P, int64_t N, int32_t K,
                              const int64_t* pt_obs_begin, const int32_t* obs_cam, const double* obs_xy,
                              const int32_t* cam_intr, const int32_t* intr_model, const uint8_t* cam_const_mask,
                              int32_t min_num_view_per_track, b200sfm_ba_problem** out);
/* Known (constant) camera rigs -- the `!optimize_rig_poses` branch of
 * BundleAdjuster::AddPointToCameraConstraints (glomap/estimators/bundle_adjustment.cc:147-161,
 * colmap::RigReprojErrorConstantRigCostFunctor): the unknown pose blocks are the F FRAMES
 * (rig_from_world); every observation is made by an image = (frame, sensor) whose cam_from_rig is a
 * constant and whose intrinsics block belongs to the sensor:
 *     r = ImgFromCam(intr[sensor_intr[s]], R_cr[s] (R_f X + t_f) + t_cr[s]) - xy.
 * obs_frame[N] indexes the frames (state arrays quat/trans are [F]), obs_sensor[N] the S sensors
 * (S <= 65535; reference sensors carry the identity transform).  Everything else -- masks, state
 * calls, solve, filters -- is b200sfm_ba_problem_*; the angle filter's `cam_calibrated` is then [S]. */
int b200sfm_ba_problem_create_rig(b200sfm_ctx* ctx, int32_t F, int32_t P, int64_t N, int32_t K, int32_t S,
                                  const int64_t* pt_obs_begin, const int32_t* obs_frame, const uint16_t* obs_sensor,
                                  const double* obs_xy, const double* sensor_quat_xyzw /*[S][4] cam_from_rig*/,
                                  const double* sensor_trans /*[S][3]*/, const int32_t* sensor_intr /*[S]*/,
                                  const int32_t* intr_model, const uint8_t* frame_const_mask,
                                  int32_t min_num_view_per_track, b200sfm_ba_problem** out);
/* The image table of a rig problem: image i is frame image_frame[i] seen through sensor image_sensor[i] (I > 0 images,
 * frames in [0, F), sensors in [0, S)).  Only b200sfm_ba_problem_normalize reads it: its box and mean run over these
 * images, the registered ones, as reconstruction_normalizer.cc:23-29 does.  Without the call the problem assumes the
 * dense layout, every frame through every sensor (F * S images). */
int b200sfm_ba_problem_set_images(b200sfm_ba_problem* p, int32_t I, const int32_t* image_frame, const int32_t* image_sensor);
/* optimize_rig_poses (bundle_adjustment.cc:162-180,296-308, colmap::RigReprojErrorCostFunctor): mark the sensors whose
 * cam_from_rig is an UNKNOWN of the following solves (the reference: every non-reference camera sensor); takes effect
 * when b200sfm_ba_opts::optimize_rig_poses is set.  sensor_variable[S]: 1 = unknown.  The optimised poses are read
 * back with b200sfm_ba_problem_get_sensor_poses (quat_xyzw [S][4] / trans [S][3], either may be NULL). */
int b200sfm_ba_problem_set_sensor_variable(b200sfm_ba_problem* p, const uint8_t* sensor_variable);
int b200sfm_ba_problem_get_sensor_poses(b200sfm_ba_problem* p, double* sensor_quat_xyzw, double* sensor_trans);
int b200sfm_ba_problem_set_state(b200sfm_ba_problem* p, const double* intr_params, const double* quat_xyzw,
                                 const double* trans, const double* points);
int b200sfm_ba_problem_get_state(b200sfm_ba_problem* p, double* intr_params, double* quat_xyzw, double* trans,
                                 double* points);
/* device-side snapshot / restore of the state (benchmark loops) */
int b200sfm_ba_problem_save_state(b200sfm_ba_problem* p);
int b200sfm_ba_problem_restore_state(b200sfm_ba_problem* p);
int b200sfm_ba_problem_solve(b200sfm_ba_problem* p, const b200sfm_ba_opts* opts, b200sfm_lm_stats* stats);
/* robust cost 1/2 sum rho(|r|^2) of the current state (all ranks) */
int b200sfm_ba_problem_cost(b200sfm_ba_problem* p, const b200sfm_ba_opts* opts, double* cost);
/* Track filters on the resident problem (SURVEY.md 8(f) item 1): the mapper runs them between the
 * BA solves (controllers/global_mapper.cc:164-186,243-276,309-337) on the arrays the problem already
 * holds.  Reference: glomap/processors/track_filter.cc:7-52 (pixel reprojection), :54-90 (angle),
 * :92-127 (triangulation angle).  They evaluate the CURRENT state and return a keep-mask (1 = keep)
 * per observation / per track plus the reference's return value (number of tracks changed / removed);
 * the caller compacts Track::observations. */
int b200sfm_ba_problem_filter_reprojection(b200sfm_ba_problem* p, double max_reprojection_error, uint8_t* keep /*[N]*/,
                                           int64_t* num_tracks_changed);
int b200sfm_ba_problem_filter_angle(b200sfm_ba_problem* p, const double* bearings /*[N][3] features_undist, or NULL = resident*/,
                                    const uint8_t* cam_calibrated /*[C] or NULL*/, double max_angle_error_deg,
                                    uint8_t* keep /*[N]*/, int64_t* num_tracks_changed);
/* FilterTracksByReprojection with in_normalized_image = true (track_filter.cc:24-31) -- the variant the mapper
 * calls (controllers/global_mapper.cc:176-181,254-259,289-294): error = |X_c.xy / X_c.z - b.xy / (b.z + EPS)|
 * against the undistorted feature b (Image::features_undist), threshold 1e-2 by default (types.h:21). */
int b200sfm_ba_problem_filter_reprojection_normalized(b200sfm_ba_problem* p, const double* bearings /*[N][3] or NULL = resident*/,
                                                      double max_reprojection_error, uint8_t* keep /*[N]*/,
                                                      int64_t* num_tracks_changed);
/* The two per-element processors the mapper runs between the solvers, on the resident problem (SURVEY.md 8(f) item 2).
 * b200sfm_ba_problem_normalize -- glomap/processors/reconstruction_normalizer.cc:5-104 (NormalizeReconstruction): robust
 * p0..p1 percentile box and trimmed mean of the image centres (float coordinates, sorted per axis; on rigs the images of
 * b200sfm_ba_problem_set_images, or all F * S frame-sensor combinations without it), similarity with
 * identity rotation X' = scale X + t applied to the frame poses, the cam_from_rig translations and the points of the
 * CURRENT state; returns the similarity (either pointer may be NULL).
 * b200sfm_ba_problem_undistort -- glomap/processors/image_undistorter.cc:7-53 (UndistortImages): unit bearing
 * CamFromImg(xy).homogeneous().normalized() of every observation from the current intrinsics, kept on the device;
 * bearings_out [N][3] may be NULL.  The two bearing-based filters below accept bearings == NULL and then use the resident
 * bearings (computing them first if needed), which saves the 24 N-byte upload per call. */
int b200sfm_ba_problem_normalize(b200sfm_ba_problem* p, int32_t fixed_scale, double extent, double p0, double p1,
                                 double* scale_out, double* translation_out /*[3]*/);
int b200sfm_ba_problem_undistort(b200sfm_ba_problem* p, double* bearings_out /*[N][3] or NULL*/);
int b200sfm_ba_problem_filter_triangulation_angle(b200sfm_ba_problem* p, double min_angle_deg, uint8_t* keep_track /*[P]*/,
                                                  int64_t* num_tracks_removed);
void b200sfm_ba_problem_free(b200sfm_ba_problem* p);

/* ---- track establishment (SURVEY.md 8(f) item 4) ---------------------------------------------------------------------
 * TrackEngine::EstablishFullTracks (glomap/controllers/track_establishment.cc:5-17): the union-find over all inlier
 * matches of the valid image pairs (BlindConcatenation, :19-63) and the collection of the components into tracks with the
 * inconsistency rule (TrackCollection, :65-150) on the device.  Input: the M inlier matches as global feature ids
 * gid = image_id << 32 | feature_id (:48-53) with the pixel of both features (Image::features).  Result: tracks in
 * ascending track id (= smallest global id of the component, the reference's root rule :56-60), observations of a track
 * in ascending global id; a track with two features of ONE image further apart than thres_inconsistency pixels keeps its
 * id but loses its observations (:118-131) and is counted in num_discarded.  The selection FindTracksForProblem is
 * b200sfm_tracks_select below. */
typedef struct b200sfm_tracks b200sfm_tracks;
int b200sfm_tracks_establish(b200sfm_ctx* ctx, int64_t num_matches, const uint64_t* gid1, const uint64_t* gid2,
                             const double* xy1 /*[M][2]*/, const double* xy2 /*[M][2]*/, double thres_inconsistency,
                             b200sfm_tracks** out, int64_t* num_tracks, int64_t* num_observations, int64_t* num_discarded);
int b200sfm_tracks_get(b200sfm_tracks* t, uint64_t* track_ids /*[T]*/, int64_t* begin /*[T+1]*/, uint32_t* obs_image /*[n]*/,
                       uint32_t* obs_feature /*[n]*/);
void b200sfm_tracks_free(b200sfm_tracks* t);
/* TrackEngine::FindTracksForProblem (track_establishment.cc:153-227) on the device, through its exact data-parallel form
 * (a per-image counter saturates, so an observation counts iff its rank among the registered observations of its image in
 * processing order is <= the quota).  Input: T tracks as host arrays, a CSR over the image ids of their observations in any
 * order, and the registered images (any order, repeats allowed).  The reference's rules:
 *   - candidates: L >= min_num_view_per_track and L <= max_num_view_per_track, L = number of observations (registered or
 *     not), processed in descending (L, track id) order;
 *   - a candidate with fewer than min_num_view_per_track DISTINCT registered images is skipped;
 *   - a registered observation increments its image's counter while the counter is <= min_num_tracks_per_view; a track
 *     with an increment is selected;
 *   - the walk stops once more than max_num_tracks tracks are selected (so at most max_num_tracks + 1 are).
 * The four options are ints compared with unsigned values, as in the reference: min_num_tracks_per_view < 0 (the default
 * -1) means no quota, min_num_view_per_track < 0 selects nothing, max_num_view_per_track < 0 removes the upper length
 * bound, max_num_tracks < 0 removes the cap.
 * Output: keep[t] = 1 for a selected track and num_selected; the caller restricts the selected tracks' observations to the
 * registered images.  Two tracks with one id, begin[0] != 0, a decreasing begin, null arrays for T > 0 or n > 0, and more
 * than 2^31 - 2 tracks or observations give B200SFM_ERR_INVALID_ARG (checked before the device is touched, except the
 * duplicate ids).  T == 0 returns num_selected = 0.  Runs on the context's device without a collective: on a
 * distributed context each rank selects from the tracks it is given. */
int b200sfm_tracks_select(b200sfm_ctx* ctx, int64_t num_tracks, const uint64_t* track_ids /*[T]*/,
                          const int64_t* begin /*[T+1] CSR over obs_image*/, const uint32_t* obs_image /*[n]*/,
                          int32_t num_registered, const uint32_t* registered_image_ids /*[R]*/,
                          int32_t min_num_tracks_per_view, int32_t min_num_view_per_track, int32_t max_num_view_per_track,
                          int32_t max_num_tracks, uint8_t* keep /*[T] out, 1 = selected*/, int64_t* num_selected);

/* ---- image pair inliers ------------------------------------------------------------------------------------------------
 * ImagePairsInlierCount (glomap/processors/image_pair_inliers.cc:200-213), the scorers ScoreErrorEssential / Fundamental /
 * Homography (:20-198) and the two-view arithmetic they call (glomap/math/two_view_geometry.cc:5-93), run by
 * GlobalMapper::Solve after the relative poses (controllers/global_mapper.cc:64-65).  Every pair passed in is scored by
 * its config: PLANAR / PANORAMIC / PLANAR_OR_PANORAMIC against H (max_epipolar_error_H px), UNCALIBRATED against F
 * (max_epipolar_error_F px, orientation-signum majority), CALIBRATED against E = [t]x R of cam2_from_cam1 on the unit
 * bearings of the features (features_undist; computed here once per feature from the image's camera, as UndistortImages
 * does), with threshold max_epipolar_error_E * (1/f1 + 1/f2) / 2, cheirality and the 3-degree epipole cones; any other
 * config gives no inliers.  The caller selects the pairs (valid pairs, minus those it keeps under clean_inliers = false).
 *   feature_begin [I+1]   CSR over the features of the I images (int64); features [nf][2] distorted pixels
 *   image_intr [I]        camera block of each image; intr_model [K] / intr_params [K][B200SFM_INTR_STRIDE] -- only the
 *                         cameras of CALIBRATED pairs are read (models 0-3, else B200SFM_ERR_UNSUPPORTED)
 *   pair_image1/2 [E]     image indices; pair_config [E] b200sfm_two_view_config; pair_quat_xyzw [E][4] / pair_trans [E][3]
 *                         cam2_from_cam1; pair_F / pair_H [E][9] row-major
 *   match_begin [E+1]     CSR over matches [M][2] (feature index in image 1, in image 2); an index outside its image's
 *                         features gives B200SFM_ERR_INVALID_ARG (checked on the device, never dereferenced)
 *   is_inlier [M]         1 = inlier (ImagePair::inliers are its set rows in ascending order); num_inliers [E]; score [E]
 *                         the scorer's return value (the reference's caller discards it).
 * num_pairs == 0 returns B200SFM_OK and writes nothing.  No collectives: on a distributed context each rank scores the
 * pairs it is given. */
/* colmap::TwoViewGeometry::ConfigurationType (colmap/estimators/two_view_geometry.h, un-vendored; UPSTREAM-UNVERIFIED) */
typedef enum {
  B200SFM_TWO_VIEW_UNDEFINED = 0,
  B200SFM_TWO_VIEW_DEGENERATE = 1,
  B200SFM_TWO_VIEW_CALIBRATED = 2,
  B200SFM_TWO_VIEW_UNCALIBRATED = 3,
  B200SFM_TWO_VIEW_PLANAR = 4,
  B200SFM_TWO_VIEW_PANORAMIC = 5,
  B200SFM_TWO_VIEW_PLANAR_OR_PANORAMIC = 6,
  B200SFM_TWO_VIEW_WATERMARK = 7,
  B200SFM_TWO_VIEW_MULTIPLE = 8
} b200sfm_two_view_config;
int b200sfm_image_pairs_inlier_count(b200sfm_ctx* ctx, int32_t num_images, const int64_t* feature_begin, const double* features,
                                     const int32_t* image_intr, int32_t K, const int32_t* intr_model, const double* intr_params,
                                     int64_t num_pairs, const int32_t* pair_image1, const int32_t* pair_image2,
                                     const int32_t* pair_config, const double* pair_quat_xyzw, const double* pair_trans,
                                     const double* pair_F, const double* pair_H, const int64_t* match_begin, const int32_t* matches,
                                     double max_epipolar_error_E, double max_epipolar_error_F, double max_epipolar_error_H,
                                     uint8_t* is_inlier, int32_t* num_inliers, double* score);

/* ---- view-graph passes of stage 3 ---------------------------------------------------------------------------------------
 * GlobalMapper::Solve runs both after each rotation averaging (controllers/global_mapper.cc:91-115), and
 * SolveRotationAveraging takes the largest component before and between its solves (controllers/rotation_averager.cc).
 *
 * b200sfm_view_graph_filter_rotations: RelPoseFilter::FilterRotations (glomap/processors/relpose_filter.cc:7-33).  A pair
 * with pair_valid[e] != 0 whose two images are registered (image_registered NULL: all are) is invalidated when the angle
 * between q2 * q1^-1 (cam_from_world_quat_xyzw [I][4] of its images) and its cam2_from_cam1 rotation pair_quat_xyzw [E][4]
 * is larger than max_angle_deg.  The angle is Eigen's angularDistance (math/rigid3d.cc:7-9, the Rigid3d overload of
 * CalcAngle): d = q_calc * conj(q_rel), 2 atan2(|d.vec|, |d.w|), in degrees.  An angle equal to max_angle_deg keeps the
 * pair, and so does a NaN angle.  num_invalidated counts the pairs this call invalidated.
 *
 * b200sfm_view_graph_keep_largest_component: ViewGraph::KeepLargestConnectedComponents (glomap/scene/view_graph.cc:56-97)
 * in frame space.  image_frame [I] names each image's frame in [0, F).  The nodes are the frames of the valid pairs
 * (CreateFrameAdjacencyList, :140-150; a valid pair inside one frame makes that frame a node).  Of the connected
 * components the largest is kept; between equally large ones, the one holding the smallest frame index (the reference's
 * choice depends on hash-map order).  Then frame_registered [F] is 1 exactly for the frames of that component, every pair
 * with an image outside it gets pair_valid 0, and num_registered_images is the number of images whose frame is registered.
 * Without a valid pair nothing is written and num_registered_images is 0 (:71).
 *
 * Both: host buffers.  A pair image index outside [0, num_images), or an image_frame outside [0, num_frames), gives
 * B200SFM_ERR_INVALID_ARG; it is checked on the device, never dereferenced, and the outputs are then untouched.
 * num_pairs == 0 returns B200SFM_OK with a zero count.  No collectives: on a distributed context each rank works on the
 * graph it is given. */
int b200sfm_view_graph_filter_rotations(b200sfm_ctx* ctx, int32_t num_images, const double* cam_from_world_quat_xyzw,
                                        const uint8_t* image_registered, int64_t num_pairs, const int32_t* pair_image1,
                                        const int32_t* pair_image2, const double* pair_quat_xyzw, double max_angle_deg,
                                        uint8_t* pair_valid, int64_t* num_invalidated);
int b200sfm_view_graph_keep_largest_component(b200sfm_ctx* ctx, int32_t num_frames, int32_t num_images, const int32_t* image_frame,
                                              int64_t num_pairs, const int32_t* pair_image1, const int32_t* pair_image2,
                                              uint8_t* pair_valid, uint8_t* frame_registered, int32_t* num_registered_images);

/* ---- stage 0: image pair configurations --------------------------------------------------------------------------------
 * b200sfm_view_graph_update_pairs_config: ViewGraphManipulater::UpdateImagePairsConfig
 * (glomap/processors/view_graph_manipulation.cc:178-237), the first half of stage 0 of GlobalMapper::Solve
 * (controllers/global_mapper.cc:22-34).  K cameras: intr_model [K] / intr_params [K][B200SFM_INTR_STRIDE] and
 * has_prior_focal [K] (Camera::has_prior_focal_length); E pairs: pair_cam1 / pair_cam2 [E] the camera of each image,
 * pair_valid [E], pair_quat_xyzw [E][4] / pair_trans [E][3] cam2_from_cam1, pair_config [E] (b200sfm_two_view_config,
 * in/out) and pair_F [E][9] row-major (in/out).
 *   Counting: a pair with pair_valid[e] != 0 whose two cameras both have a prior focal adds 1 to `total` of both cameras
 *   when it is CALIBRATED or UNCALIBRATED, and 1 to `calibrated` of both when it is CALIBRATED (a pair inside one camera
 *   counts twice for it).  A camera is valid when calibrated * 1. / total > 0.5 (FP64, strict); a camera no pair counted
 *   is not valid.
 *   Promotion: a valid UNCALIBRATED pair whose two cameras are valid becomes CALIBRATED, and its F becomes
 *   K2^-T [t]x R K1^-1 (FundamentalFromMotionAndCameras, math/two_view_geometry.cc:38-55; K = Camera::GetK with fx = fy =
 *   f for the SIMPLE_* models; R = Eigen's toRotationMatrix of the quaternion as given).  F is computed from the
 *   cam2_from_cam1 the pair carries: the reference runs this pass before DecomposeRelPose, when a pair read from the
 *   database still has the converter's identity pose, so its promoted F is the zero matrix there too.
 * num_promoted counts the promoted pairs; pair_valid is not changed.  Host buffers.  A camera index outside [0, K) gives
 * B200SFM_ERR_INVALID_ARG (checked on the device, never dereferenced); a pair to be promoted whose camera model is
 * outside 0-3 gives B200SFM_ERR_UNSUPPORTED; the outputs are then untouched.  num_pairs == 0 returns B200SFM_OK with a
 * zero count.  No collectives: on a distributed context each rank works on the pairs it is given. */
int b200sfm_view_graph_update_pairs_config(b200sfm_ctx* ctx, int32_t K, const int32_t* intr_model, const double* intr_params,
                                           const uint8_t* has_prior_focal, int64_t num_pairs, const int32_t* pair_cam1,
                                           const int32_t* pair_cam2, const uint8_t* pair_valid, const double* pair_quat_xyzw,
                                           const double* pair_trans, int32_t* pair_config, double* pair_F, int64_t* num_promoted);

/* ---- (ii) global positioning (BATA) ----------------------------------------- */
/* Mirror of GlobalPositionerOptions (global_positioning.h:9-54) + inherited
 * solver options (optimization_base.h:18-23) + PCG knobs.  Only the
 * ONLY_POINTS constraint type is implemented (the mapper enforces it,
 * controllers/global_mapper.cc:145-149); random initialisation
 * (generate_random_positions / points, seed) is done by the host shim. */
typedef struct {
  int32_t optimize_positions;        /* default 1 */
  int32_t optimize_points;           /* default 1 */
  int32_t optimize_scales;           /* default 1 */
  int32_t min_num_view_per_track;    /* default 3 */
  int32_t max_num_iterations;        /* default 100 */
  int32_t max_num_line_search_step_size_iterations;  /* Ceres default 20 (bounded problems) */
  double thres_loss_function;        /* Huber threshold, default 0.1 */
  double function_tolerance;         /* 1e-5 */
  double gradient_tolerance;         /* 1e-10 */
  double parameter_tolerance;        /* 1e-8 */
  int32_t pcg_max_iterations;        /* default 1000 */
  int32_t pcg_min_iterations;
  double pcg_rel_tolerance;          /* default 1e-2 */
  int32_t preconditioner;            /* 0 block-Jacobi, 1 Schur-Jacobi (default) */
  int32_t profile_kernels;
  int32_t fixed_num_iterations;
  int32_t reserved0;
} b200sfm_gp_opts;

void b200sfm_gp_default_opts(b200sfm_gp_opts* opts);

/* One-shot solve with host buffers (results written back in place):
 *   pt_obs_begin [P+1], obs_cam [N]  as for BA
 *   obs_dir      [N][3]  unit bearing rotated into the world frame,
 *                        R_cw^T * features_undist (global_positioning.cc:294-296)
 *   cam_calibrated [C]   1: Huber loss, 0: ScaledLoss(Huber, 0.5) (.cc:313-316); NULL = all calibrated
 *   cam_const_mask [C]   nonzero: centre held constant; may be NULL
 *   centers [C][3]       camera centres (the reference keeps them in
 *                        RigFromWorld().translation during the solve), in/out
 *   points  [P][3]       in/out
 *   scales  [N]          one per observation, in/out (initialise to 1, .cc:298);
 *                        lower bound 1e-5 (.cc:373); the first scale of rank 0 is constant (.cc:484-489) */
int b200sfm_gp_solve(b200sfm_ctx* ctx, const b200sfm_gp_opts* opts, int32_t C, int32_t P, int64_t N,
                     const int64_t* pt_obs_begin, const int32_t* obs_cam, const double* obs_dir,
                     const uint8_t* cam_calibrated, const uint8_t* cam_const_mask, double* centers, double* points,
                     double* scales, b200sfm_lm_stats* stats);

typedef struct b200sfm_gp_problem b200sfm_gp_problem;
int b200sfm_gp_problem_create(b200sfm_ctx* ctx, int32_t C, int32_t P, int64_t N, const int64_t* pt_obs_begin,
                              const int32_t* obs_cam, const double* obs_dir, const uint8_t* cam_calibrated,
                              const uint8_t* cam_const_mask, int32_t min_num_view_per_track, b200sfm_gp_problem** out);
/* Known rigs in global positioning -- RigBATAPairwiseDirectionError with the rig scale held at 1
 * (glomap/estimators/cost_function.h:49-82, global_positioning.cc:325-346,493-497):
 *     r = t_obs - s (X - c_frame + obs_offset),   obs_offset = R_cam_from_world^T t_cam_from_rig.
 * obs_cam then indexes FRAMES (c = rig centre).  obs_calibrated[N] (optional) is the prior-focal flag
 * of the observing camera and replaces the per-frame cam_calibrated (the loss is chosen per camera,
 * .cc:313-316).  NULL/NULL restores the trivial-frame behaviour. */
int b200sfm_gp_problem_set_rig_terms(b200sfm_gp_problem* p, const double* obs_offset /*[N][3]*/,
                                     const uint8_t* obs_calibrated /*[N] or NULL*/);
/* Unknown cam_from_rig in global positioning -- RigUnknownBATAPairwiseDirectionError (glomap/estimators/cost_function.h:
 * 90-136, call site global_positioning.cc:347-364): for the images of a sensor whose cam_from_rig translation is not
 * known yet,  r = t_obs - s (X - c_frame - R_rw^T u_s)  with u_s (3 doubles, "cam_from_rig_center") an unknown shared by
 * all images of the sensor.  obs_unknown_sensor[N]: index in [0, S_u) or -1 for observations of reference / calibrated
 * sensors; frame_rot[C][9]: rig_from_world rotations, row-major; centers[S_u][3]: initial values (the reference draws
 * U(-1,1)^3, global_positioning.cc:440-453) -- read back with b200sfm_gp_problem_get_rig_unknown. */
int b200sfm_gp_problem_set_rig_unknown(b200sfm_gp_problem* p, int32_t num_unknown_sensors, const int32_t* obs_unknown_sensor,
                                       const double* frame_rot, const double* centers);
int b200sfm_gp_problem_get_rig_unknown(b200sfm_gp_problem* p, double* centers);
int b200sfm_gp_problem_set_state(b200sfm_gp_problem* p, const double* centers, const double* points, const double* scales);
int b200sfm_gp_problem_get_state(b200sfm_gp_problem* p, double* centers, double* points, double* scales);
int b200sfm_gp_problem_save_state(b200sfm_gp_problem* p);
int b200sfm_gp_problem_restore_state(b200sfm_gp_problem* p);
int b200sfm_gp_problem_solve(b200sfm_gp_problem* p, const b200sfm_gp_opts* opts, b200sfm_lm_stats* stats);
void b200sfm_gp_problem_free(b200sfm_gp_problem* p);

/* ---- (i) rotation averaging --------------------------------------------------- */
/* Mirror of RotationEstimatorOptions (global_rotation_averaging.h:39-75) for
 * 3-DoF frames with trivial rigs.  skip_initialization / use_gravity / axis are
 * host-side concerns (the maximum-spanning-tree initialisation they switch off
 * runs on the device through b200sfm_ra_mst_init below).  The l1_* fields are
 * the colmap::LeastAbsoluteDeviationSolver options the reference uses
 * (global_rotation_averaging.cc:483-486 + COLMAP defaults). */
typedef struct {
  int32_t max_num_l1_iterations;           /* 5 */
  int32_t max_num_irls_iterations;         /* 100 */
  int32_t weight_type;                     /* 0 GEMAN_MCCLURE (default), 1 HALF_NORM */
  int32_t use_weight;                      /* 0 */
  double l1_step_convergence_threshold;    /* 1e-3 */
  double irls_step_convergence_threshold;  /* 1e-3 */
  double irls_loss_parameter_sigma;        /* 5 degrees */
  int32_t l1_max_admm_iterations;          /* 10 (.cc:484) */
  int32_t reserved0;
  double l1_rho;                           /* 1.0 */
  double l1_absolute_tolerance;            /* 1e-4 */
  double l1_relative_tolerance;            /* 1e-2 */
  /* PCG replaces the reference's CHOLMOD factorisations (.cc:491,547-611) */
  int32_t pcg_max_iterations;              /* 5000 */
  int32_t reserved1;
  double pcg_rel_tolerance;                /* 1e-8 */
} b200sfm_ra_opts;

typedef struct {
  int32_t l1_iterations;
  int32_t irls_iterations;
  int32_t admm_iterations;
  int32_t usable;                 /* 0: NaN encountered -> EstimateRotations returns false */
  int64_t num_edges;
  int64_t pcg_iterations;         /* Laplacian mat-vecs */
  int64_t kernel_launches;
  double ms_total;
} b200sfm_ra_stats;

void b200sfm_ra_default_opts(b200sfm_ra_opts* opts);

/*   n_frames          registered frames (unknown blocks of 3)
 *   ei, ej [E]        image/frame indices of each valid pair (image_id1, image_id2)
 *   R_rel  [E][9]     row-major cam2_from_cam1 rotation (ImagePairTempInfo::R_rel, .h:29)
 *   edge_w [E]        ImagePair::weight (used when use_weight; <0 -> 1); may be NULL
 *   fixed_frame       gauge frame (fixed_camera_id_, .cc:248-256)
 *   theta  [n][3]     angle-axis of every frame: in = initial estimate, out = result.
 * In a distributed context every rank passes its own shard of edges and the
 * same theta. */
int b200sfm_ra_solve(b200sfm_ctx* ctx, const b200sfm_ra_opts* opts, int32_t n_frames, int64_t n_edges,
                     const int32_t* ei, const int32_t* ej, const double* R_rel, const double* edge_w,
                     int32_t fixed_frame, double* theta, b200sfm_ra_stats* stats);

/* use_gravity variant (global_rotation_averaging.cc:207-217,311-340,386-421): frames flagged in
 * frame_has_gravity carry ONE unknown, the angle about the gravity axis, passed as theta = (0, phi, 0)
 * with phi = RotUpToAngle(R_align^T R) (.cc:208-210); R_rel must already be gravity-aligned by the host
 * (R_align2^T R_rel R_align1, .cc:311-326); fixed_frame must be the first frame with gravity if any
 * (.cc:213-217).  Pairs of two gravity frames contribute one row; the rand() jitter of RelAngleError
 * near +-pi (.cc:28-33) is not reproduced.  frame_has_gravity == NULL is b200sfm_ra_solve. */
int b200sfm_ra_solve_gravity(b200sfm_ctx* ctx, const b200sfm_ra_opts* opts, int32_t n_frames, int64_t n_edges,
                             const int32_t* ei, const int32_t* ej, const double* R_rel, const double* edge_w,
                             const uint8_t* frame_has_gravity, int32_t fixed_frame, double* theta,
                             b200sfm_ra_stats* stats);

/* Rotation averaging with UNKNOWN cam_from_rig rotations (glomap/estimators/global_rotation_averaging.cc:173-245 the
 * unknown layout, :425-440 the extra -I / +I blocks, :646-693 the update with colmap::AverageQuaternions over the frames
 * of each camera, :726-736 residuals with R_k = R_cam R_frame, :805-813 the estimated rotations).
 *   theta [n_frames + n_cams][3]: frame rotations followed by the cam_from_rig rotations of the sensors that are not
 *   calibrated (initial values in, result out);  eci/ecj [E]: node index (>= n_frames) of the camera of image 1 / 2 or -1;
 *   R_rel carries the calibrated cam_from_rig factors (:305-309);  cam_frames (CSR over the n_cams cameras): the frames that
 *   hold an image of the camera.  A pair inside one frame is kept when a camera of it is unknown (:300-304). */
int b200sfm_ra_solve_rig(b200sfm_ctx* ctx, const b200sfm_ra_opts* opts, int32_t n_frames, int32_t n_cams, int64_t n_edges,
                         const int32_t* ei, const int32_t* ej, const int32_t* eci, const int32_t* ecj, const double* R_rel,
                         const double* edge_w, const int32_t* cam_frames_begin, const int32_t* cam_frames,
                         int32_t fixed_frame, double* theta, b200sfm_ra_stats* stats);

typedef struct {
  int32_t num_reached;     /* nodes in the root's component, root included */
  int32_t num_tree_edges;  /* edges of the whole spanning forest */
  int32_t boruvka_rounds;
  int32_t max_depth;       /* deepest reached node below the root */
  int64_t kernel_launches;
  double ms_total;         /* host wall clock of the call */
} b200sfm_mst_stats;

/* InitializeFromMaximumSpanningTree (global_rotation_averaging.cc:87-138 + math/tree.cc:78-153).
 *   ei, ej [E], R_rel [E][9]: as b200sfm_ra_solve (row-major cam2_from_cam1)
 *   weight [E]: #inliers (INLIER_NUM); key max_w - w (max_w the maximum over the E edges), ties by edge index -- a total
 *               order, so the maximum spanning forest is unique: the one Kruskal gives with a stable sort of the edges
 *   R [n][9]: in = R[root] is the starting rotation; out = every reached node, others untouched.  A node v of the root's
 *             component gets R_v = A_v R_parent(v), A_v = R_rel of its tree edge when v is that edge's ej, R_rel^T when
 *             it is its ei
 *   parent [n] or NULL: parent[root] = root, unreached = -1 (the parents any BFS of the tree from root gives);
 *   stats may be NULL.
 * Self loops never enter the tree; of parallel edges only the lowest-ranked can.  Repeated calls give bit-identical
 * outputs.  A null context, R or edge array, n_nodes < 1, n_edges < 0 or > INT32_MAX, root or an endpoint out of range
 * and a non-finite weight give B200SFM_ERR_INVALID_ARG before the device is touched; a context with more than one rank
 * gives B200SFM_ERR_UNSUPPORTED (the tree needs every edge, ranks hold shards). */
int b200sfm_ra_mst_init(b200sfm_ctx* ctx, int32_t n_nodes, int64_t n_edges, const int32_t* ei, const int32_t* ej,
                        const double* R_rel, const double* weight, int32_t root, double* R, int32_t* parent,
                        b200sfm_mst_stats* stats);

typedef struct {
  int32_t num_ref_frames;       /* frames with a registered reference image */
  int32_t num_cam_samples;      /* samples over all cameras (rule 2) */
  int32_t num_cams_averaged;    /* unknown cameras that got an average (rule 3) */
  int32_t num_frame_samples;    /* samples over all frames (rule 4) */
  int32_t num_frames_averaged;  /* frames that got an average */
  int32_t reserved0;
  int64_t kernel_launches;
  double ms_total;              /* host wall clock of the call */
} b200sfm_rig_init_stats;

/* ConvertRotationsFromImageToRig (glomap/estimators/rotation_initializer.cc:7-125) on flat arrays in sorted-id order:
 * per-image cam_from_world rotations -> the cam_from_rig rotations of the unknown cameras and the frames' rig_from_world
 * rotations.  Quaternions are xyzw (Eigen's coeffs() order) and need not be normalised.
 *   image_frame [I]        frame index of the image, -1 when it is not registered
 *   image_camera [I]       camera index
 *   image_estimated [I]    1 when cam_from_world holds an estimate for the image (the reference's cam_from_worlds map);
 *                          NULL: every image
 *   cam_from_world [I][4]
 *   frame_ref_camera [F]   the reference camera of the frame's rig
 *   camera_known [K]       1 when the camera's cam_from_rig is known (MaybeSensorFromRig has a value); pass the reference
 *                          cameras as known, with the identity
 *   cam_from_rig [K][4]    in: the known rotations; out: the averaged ones (rows of other cameras untouched)
 *   cam_samples [K]        out, or NULL: the number of samples of each camera (0 for a known one)
 *   rig_from_world [F][4]  in/out: a frame without a sample keeps its input
 *   frame_samples [F]      out, or NULL
 * Rules (images in ascending index; the reference's order is Frame::ImageIds()):
 *   1. the reference image of frame f is its registered image of smallest index whose camera is frame_ref_camera[f]
 *      (.cc:24-43, the first in ImageIds()); a frame without one gives no camera sample
 *   2. every registered image i of a frame with reference image r whose camera is neither the frame's reference camera
 *      nor known gives its camera the sample q_i conj(q_r) (.cc:45-73); the reference .at()-throws when i or r has no
 *      estimate, here such a sample is skipped
 *   3. an unknown camera with at least one sample gets their average (.cc:79-88; the caller sets its translation to NaN);
 *      a camera without a sample stays unknown
 *   4. every frame averages over its registered, estimated images (.cc:91-122): the reference image contributes q_i,
 *      another image whose camera is known or was averaged in rule 3 contributes conj(q_cam_from_rig) q_i, any other
 *      is skipped.  The reference re-averages inside the image loop; its final value is the average over all samples
 *   5. the average is colmap::AverageQuaternions with unit weights (UPSTREAM-UNVERIFIED restatement): the dominant
 *      eigenvector of sum q q^T over the normalised samples, by the power iteration ra_update_cams uses (200 steps from
 *      the first sample: exact to rounding when the samples estimate one rotation, as they do here; samples spread
 *      over very different rotations converge more slowly); a single sample is returned as it is (normalised).  The
 *      sign is canonical: w >= 0
 *   6. sums run in a fixed order without floating-point atomics: repeated calls give bit-identical outputs
 * A null context or array (but image_estimated, cam_samples, frame_samples, stats), n_images < 1 or > INT32_MAX,
 * n_frames < 1, n_cameras < 1, and a frame or camera index out of range give B200SFM_ERR_INVALID_ARG before the device is
 * touched; a context with more than one rank gives B200SFM_ERR_UNSUPPORTED. */
int b200sfm_rig_rotations_from_images(b200sfm_ctx* ctx, int64_t n_images, int32_t n_frames, int32_t n_cameras,
                                      const int32_t* image_frame, const int32_t* image_camera,
                                      const uint8_t* image_estimated, const double* cam_from_world,
                                      const int32_t* frame_ref_camera, const uint8_t* camera_known, double* cam_from_rig,
                                      int32_t* cam_samples, double* rig_from_world, int32_t* frame_samples,
                                      b200sfm_rig_init_stats* stats);

/* ---- view-graph calibration ---------------------------------------------------------------------------------------
 * ViewGraphCalibrator::Solve (glomap/estimators/view_graph_calibration.cc:11-185), stage 1 of GlobalMapper::Solve
 * (controllers/global_mapper.cc:41-50): one focal length per camera refined from the fundamental matrices of the image
 * pairs with FetzerFocalLengthCost / FetzerFocalLengthSameCameraCost (glomap/estimators/cost_function.h:138-310) under
 * CauchyLoss(thres_loss_function), lower bound 1e-3 on every focal (.cc:105-120).  Field-for-field mirror of
 * ViewGraphCalibratorOptions (view_graph_calibration.h:10-29) + the inherited solver options (optimization_base.h:18-23)
 * + the PCG knobs of this implementation (the reference factors the normal matrix exactly, .cc:21-24). */
typedef struct {
  int32_t max_num_iterations;                        /* 100 */
  int32_t max_num_line_search_step_size_iterations;  /* Ceres default 20 (bounded problem) */
  double thres_loss_function;                        /* Cauchy scale, 1e-2 (view_graph_calibration.h:23) */
  double function_tolerance;                         /* 1e-5 */
  double gradient_tolerance;                         /* Ceres default 1e-10 */
  double parameter_tolerance;                        /* Ceres default 1e-8 */
  double thres_lower_ratio;                          /* 0.1 */
  double thres_higher_ratio;                         /* 10 */
  double thres_two_view_error;                       /* 2 */
  int32_t pcg_max_iterations;                        /* default 1000 */
  int32_t pcg_min_iterations;                        /* default 0 */
  double pcg_rel_tolerance;                          /* ||r_k|| <= tol * ||r_0||, default 1e-12 */
  int32_t profile_kernels;                           /* 1: time the linearisation / mat-vec kernels with CUDA events */
  int32_t reserved0;
} b200sfm_vgc_opts;

void b200sfm_vgc_default_opts(b200sfm_vgc_opts* opts);

/* The caller passes the qualifying pairs only: valid pairs whose config is CALIBRATED or UNCALIBRATED (.cc:71-79).
 *   principal_point [K][2]   Camera::PrincipalPoint()
 *   focal [K]                in: Camera::Focal() = (fx + fy) / 2; out: the estimate of every camera used by a pair
 *                            (those of the others are left as they are)
 *   focal_constant [K]       nonzero: has_prior_focal_length, the focal is held constant (.cc:113-116); may be NULL
 *   cam1, cam2 [E]           camera of image_id1 / image_id2; cam1 == cam2 uses the same-camera cost
 *   F [E][9]                 ImagePair::F (i1_F_i0), row-major
 *   pair_valid [E]           out: 0 = |r|^2 > thres_two_view_error^2 at the final focals (FilterImagePairs, .cc:150-185),
 *                            the unlossed residuals evaluated with the estimate even where the ratio test rejected it
 *   cam_accepted [K]         out: 1 = a camera used by a pair whose estimate lies within [thres_lower_ratio,
 *                            thres_higher_ratio] times its initial focal: CopyBackResults (.cc:122-148) sets
 *                            has_refined_focal_length and every FocalLengthIdxs() entry to the estimate; 0 otherwise
 *   pair_residual [E][2]     out: the unlossed residuals at the final focals; may be NULL
 * E == 0 or no variable camera: B200SFM_OK with stats->usable = 1 and nothing written (the early return, .cc:30-35).
 * stats->num_observations is E.  A non-finite F leaves the focals as they were and gives usable = 0, as the failed
 * evaluation makes Ceres' solution unusable.  A camera index outside [0, K) gives B200SFM_ERR_INVALID_ARG; a context with
 * more than one rank B200SFM_ERR_UNSUPPORTED. */
int b200sfm_view_graph_calibrate(b200sfm_ctx* ctx, const b200sfm_vgc_opts* opts, int32_t K, const double* principal_point,
                                 double* focal, const uint8_t* focal_constant, int64_t E, const int32_t* cam1,
                                 const int32_t* cam2, const double* F, uint8_t* pair_valid, uint8_t* cam_accepted,
                                 double* pair_residual, b200sfm_lm_stats* stats);

/* ---- reconstruction pruning ---------------------------------------------------------------------------------------
 * PruneWeaklyConnectedImages (glomap/processors/reconstruction_pruning.cc:6-131), stage 8 of GlobalMapper::Solve
 * (controllers/global_mapper.cc:340-353, on with --skip_pruning 0), in frame space: frames 0..F-1 in sorted frame-id
 * order, a track is the frame index of each of its observations.
 *   1. covisibility (:14-36): tracks of <= 2 observations are skipped; every observation of another track adds 1 to its
 *      frame's observation count, every index pair i < j of it whose frames differ adds 1 to the unordered frame pair
 *      (multiplicities count: frames [a, a, b] add 2 to (a, b))
 *   2. visibility edges (:38-61): a pair counted >= 5 times (pairs_min5) is an edge of weight = count unless either frame's
 *      observation count is below min_num_observations
 *   3. intra-frame edges (:63-104) join the first image of a frame to its other images: in frame space they are
 *      self-loops, whose only effect is that such a frame belongs to the frame adjacency list (and so is a component of
 *      its own) even without another edge.  frame_self_loop[f] != 0 marks a frame with >= 2 images present
 *   4. threshold (:106-127): median = w[E / 2] of the sorted weights, MAD = the same of |w - median|,
 *      strong_threshold = max(median - MAD, 20)
 *   5. EstablishStrongClusters (processors/view_graph_manipulation.cc:70-176): KeepLargestConnectedComponents
 *      (scene/view_graph.cc:56-97) sets is_registered; frames of the edges with weight > thr are united; then up to 10
 *      passes count the edges with weight >= 0.75 thr between two sets and unite every pair of sets counted >= 2 times,
 *      repeating while a pass found such a pair (clustering_iterations is the reference's `iteration` at exit, 1..11);
 *      edges between sets are dropped and MarkConnectedComponents (view_graph.cc:99-126, min_num_img = -1: every
 *      component gets an id) numbers the components of the rest by size, descending.
 * Where the reference depends on hash-map order or is undefined:
 *   (i)   between equally large components in 5a, the one with the smallest frame index is kept;
 *   (ii)  equally large clusters are numbered by their smallest frame index, ascending;
 *   (iii) with no visibility edge (the reference indexes an empty vector) the call returns B200SFM_OK with num_clusters = 0,
 *         every cluster_id = -1 and is_registered as it was.
 *   track_begin [T + 1]         CSR of the tracks over obs_frame; track_begin[0] = 0, non-decreasing
 *   obs_frame [track_begin[T]]  frame of every observation; outside [0, F) gives B200SFM_ERR_INVALID_ARG (checked on the
 *                               device, never dereferenced)
 *   frame_self_loop [F]         may be NULL (trivial frames)
 *   max_pair_keys_per_pass      covisibility keys sorted at once (8 B each, ~36 B of device memory per key); <= 0: 2^27,
 *                               at most 2^30.  The distinct frame pairs of all passes together must stay below 2^31
 *                               (B200SFM_ERR_INVALID_ARG otherwise; a larger pass size gives fewer)
 *   cluster_id [F]              out: component of every frame, -1 outside every component
 *   is_registered [F]           in/out: 1 = in the largest component of the visibility graph
 *   num_clusters                out: the return value of PruneWeaklyConnectedImages
 *   stats                       may be NULL
 * All counting is integer work on the device; the result does not depend on the pass size.  A context with more than one
 * rank gives B200SFM_ERR_UNSUPPORTED; a kernel launch that fails gives B200SFM_ERR_CUDA (checked before the call returns). */
typedef struct {
  int64_t covisible_pairs;           /* distinct frame pairs seen together in a track longer than 2 */
  int64_t pairs_min5;                /* of these, counted >= 5 times (the reference's `counter`) */
  int64_t visibility_edges;          /* of these, passing the min_num_observations filter */
  double strong_threshold;           /* max(median - MAD, 20); 0 when there is no visibility edge */
  int32_t clustering_iterations;     /* 0 when there is no visibility edge */
  int32_t largest_component_frames;  /* frames registered by KeepLargestConnectedComponents */
} b200sfm_prune_stats;

int b200sfm_prune_weakly_connected(b200sfm_ctx* ctx, int32_t num_frames, int64_t num_tracks, const int64_t* track_begin,
                                   const int32_t* obs_frame, const uint8_t* frame_self_loop, int32_t min_num_observations,
                                   int64_t max_pair_keys_per_pass, int32_t* cluster_id, uint8_t* is_registered,
                                   int32_t* num_clusters, b200sfm_prune_stats* stats);

/* ---- gravity refinement -------------------------------------------------------------------------------------------
 * GravityRefiner::RefineGravity (glomap/estimators/gravity_refinement.cc:9-181), run by `glomap rotation_averager
 * --refine_gravity 1`, in frame space: frames 0..F-1, and per pair the frame-level relative rotation
 * M = R_c2^T R_rel R_c1 (rig2_from_rig1; R_c is the image's cam_from_rig rotation, the identity for a trivial frame).
 *   1. IdentifyErrorProneGravity (.cc:129-181): a pair is a mistake when CalcAngle(R, AngleToRotUp(RotUpToAngle(R))) >
 *      max_gravity_error for R = Ra2^T M Ra1; it counts once toward the (mistakes, total) of each of its two frames (twice
 *      for a pair inside one frame).  A frame is error-prone when total >= min_num_neighbors and
 *      mistakes / total >= max_outlier_ratio
 *   2. per error-prone frame (.cc:42-124): the observed gravities are M^T g2 for the frame of image 1 and M g1 for the
 *      frame of image 2 (g = column 1 of R_align; a pair inside the frame is one term, of the first kind).  With fewer
 *      than min_num_neighbors terms the frame is skipped (status 1); otherwise AverageGravity (math/gravity.cc:37-91) starts
 *      an LM on SphereManifold<3> with residual g - g_obs under ArctanLoss(1 - cos(max_gravity_error)), and the result is
 *      accepted (status 2) when fewer than max_outlier_ratio of the terms lie more than 2 max_gravity_error away, else
 *      rejected (status 3)
 * Rules where the reference depends on hash order or a library convention:
 *   (i)   every error-prone frame is refined against the gravities as they were on entry (the reference refines in
 *         unordered_set order and later frames see earlier results)
 *   (ii)  when exactly half of the terms point against the principal direction, its sign is the one whose dot product
 *         with the frame's prior gravity is >= 0 (the reference leaves it to the SVD)
 *   (iii) the error test depends on the completion of R_align around its gravity column; the reference completes it with
 *         Eigen's Householder QR (GetAlignRot, math/gravity.cc:11-24), and callers that want its decisions pass that one.
 *   R_align [F][9]       row-major; column 1 = unit gravity.  Frames with gravity must have finite entries and a non-zero
 *                        column 1 (B200SFM_ERR_INVALID_ARG otherwise)
 *   has_gravity [F]      nonzero: the frame has a gravity prior; pairs with a frame without one are ignored
 *   frame1, frame2 [E]   frames of image 1 / image 2 of the valid pairs whose two images have gravity (.cc:62-64,149);
 *                        outside [0, F) gives B200SFM_ERR_INVALID_ARG (checked on the device, never dereferenced); E < 2^30
 *   M [E][9]             row-major; a non-finite entry gives B200SFM_ERR_INVALID_ARG
 *   gravity [F][3]       out: the refined gravity, written for the frames of status 2 only
 *   status [F]           out: 0 = not error-prone, 1 = error-prone with too few terms, 2 = refined and accepted,
 *                        3 = refined and rejected; written for every frame when a frame is error-prone
 *   stats                may be NULL
 * E == 0, or no error-prone frame, gives B200SFM_OK with nothing written.  A context with more than one rank gives
 * B200SFM_ERR_UNSUPPORTED; a kernel launch that fails gives B200SFM_ERR_CUDA (checked before the call returns). */
typedef struct {
  double max_outlier_ratio;    /* 0.5 (gravity_refinement.h:14) */
  double max_gravity_error;    /* degrees, 1 (gravity_refinement.h:16) */
  int32_t min_num_neighbors;   /* 7 (gravity_refinement.h:18) */
  int32_t max_num_iterations;  /* 100 (optimization_base.h:20) */
  double function_tolerance;   /* 1e-5 (optimization_base.h:22) */
  double gradient_tolerance;   /* Ceres default 1e-10 */
  double parameter_tolerance;  /* Ceres default 1e-8 */
  int32_t reserved[4];
} b200sfm_gravity_opts;

void b200sfm_gravity_default_opts(b200sfm_gravity_opts* opts);

typedef struct {
  int32_t error_prone_frames;
  int32_t rectified_frames;    /* status 2 */
  int32_t too_few_terms;       /* status 1 */
  int32_t max_lm_iterations;
  int64_t lm_iterations;       /* summed over the refined frames */
  double ms_total;             /* host wall clock of the call */
  double ms_h2d, ms_error_test, ms_csr, ms_refine;   /* device events */
} b200sfm_gravity_stats;

int b200sfm_gravity_refine(b200sfm_ctx* ctx, const b200sfm_gravity_opts* opts, int32_t F, const double* R_align,
                           const uint8_t* has_gravity, int64_t E, const int32_t* frame1, const int32_t* frame2,
                           const double* M, double* gravity, uint8_t* status, b200sfm_gravity_stats* stats);

#ifdef __cplusplus
}
#endif
#endif /* B200SFM_H_ */
