/* b200sfm_testing.h -- test-only probes into resident bundle-adjustment, rotation-averaging and global-positioning
 * problems, the gravity refiner's stages and the solvers' small device helpers.
 *
 * NOT part of the drop-in ABI of b200sfm.h: these entry points exist so that the
 * test suite can compare every quantity one Levenberg-Marquardt step forms on the
 * device (the linearisation, the damping, the preconditioner, the right-hand side,
 * the PCG iterate, the candidate state and the step scalars) with an FP64 sparse
 * reference (oracle/ba_system.py), and apply the reduced camera operator to an
 * arbitrary vector through the production mat-vec kernels.  Single-rank contexts
 * only: a multi-rank context returns B200SFM_ERR_INVALID_ARG.
 *
 * Device layout of the camera-side vectors: nbk blocks of 6 doubles, block order
 * frame f | C + intrinsics k | C + K + sensor s (the last two only on the extended
 * paths).  A frame block holds rotation (slots 0-2) and translation (3-5); an
 * intrinsics block holds its variable parameters in ascending parameter index; a
 * sensor block holds the cam_from_rig rotation (0-2) and translation (3-5).
 * Symmetric 6x6 blocks are packed as 21 doubles, upper triangle, row by row.
 */
#ifndef B200SFM_TESTING_H_
#define B200SFM_TESTING_H_

#include "b200sfm.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Outputs of b200sfm_test_ba_step.  Every array pointer is caller-owned and may be NULL (not downloaded).
 * Sizes: U, Minv [nbk*21]; g_c, jscale_c, Dc, b, px [nbk*6] (allocate (C+K+S)*6 / *21 when nbk is not known
 * yet); V [P*6]; g_p, jscale_p, cand_points [P*3]; cand_quat [C*4]; cand_trans [C*3];
 * cand_intr [K*B200SFM_INTR_STRIDE]; cand_sensor_quat [S*4]; cand_sensor_trans [S*3] (rig problems only). */
typedef struct {
  double* U;                 /* camera-block Gauss-Newton blocks J_c^T J_c after finalisation (identity on non-variable dofs) */
  double* g_c;               /* camera-side gradient J_c^T r */
  double* jscale_c;          /* Jacobi scales 1/(1+sqrt(U_ii)); -1 marks a non-variable dof */
  double* V;                 /* point blocks J_p^T J_p, packed 3x3 upper triangle (6) */
  double* g_p;               /* point gradient J_p^T r */
  double* jscale_p;          /* point Jacobi scales */
  double* Dc;                /* camera-side LM damping diagonal */
  double* Minv;              /* preconditioner blocks (inverses) */
  double* b;                 /* right-hand side of the reduced camera system */
  double* px;                /* camera step: the PCG iterate */
  double* cand_points;       /* candidate state (the step is not accepted) */
  double* cand_quat;
  double* cand_trans;
  double* cand_intr;
  double* cand_sensor_quat;
  double* cand_sensor_trans;
  double cost;               /* robust cost at the current state */
  double gmax;               /* max |g| over the variable dofs */
  double model_cost_change;  /* decrease predicted by the linear model for the step */
  double cand_cost;          /* robust cost of the candidate state */
  double step_norm;
  double x_norm;
  int32_t pcg_iterations;
  /* the paths the solve selected */
  int32_t use_v2, use_ell, kfast, nk, ext, ext_k, ext_s, schur_jacobi, nbk;
} b200sfm_test_ba_step_out;

/* At the problem's current state (b200sfm_ba_problem_set_state): select the paths as b200sfm_ba_problem_solve does,
 * linearise as its first LM iteration, run one trust-region step at `radius` with the PCG settings of `opts`, and
 * download into `out`.  With first_radius > 0 a step at first_radius comes first and is rejected, as the solve does
 * after a step it does not accept; the step at `radius` then reuses that linearisation.  The candidate is not
 * accepted: the current state is unchanged afterwards. */
int b200sfm_test_ba_step(b200sfm_ba_problem* problem, const b200sfm_ba_opts* opts, double first_radius, double radius,
                         b200sfm_test_ba_step_out* out);

/* y = (S + D) x over the nbk*6 camera-side dofs, with the linearisation and damping of the last
 * b200sfm_test_ba_step, through the mat-vec kernels of the selected path.  x, y: host arrays [nbk*6]. */
int b200sfm_test_ba_apply(b200sfm_ba_problem* problem, const double* x, double* y);

/* ---- rotation averaging ----------------------------------------------------------------------------------------
 * A resident rotation-averaging problem, built by the constructor b200sfm_ra_solve_gravity / b200sfm_ra_solve_rig use
 * (path selection, environment included, is the production one), and probes that run the solver's own stages on it.
 *
 * Node vectors hold n = n_frames + n_cams nodes of 3 doubles: the frames' angle-axis rotations, then the unknown
 * cam_from_rig rotations.  A gravity frame's unknown is its y slot.  Edge vectors hold E = n_edges + 1 edges: the
 * n_edges pairs, then the gauge pseudo-edge (identity -> fixed frame).  Jacobi blocks are packed 3x3 upper triangles
 * (6 doubles per node). */
typedef struct b200sfm_test_ra_problem b200sfm_test_ra_problem;

/* The paths the problem selected.  fused: the fused two-level PCG iteration, read as a solve reads it. */
typedef struct {
  int32_t n, n_frames, n_cams, has_grav;
  int32_t use_csr, use_2lvl, fused, nc;
  int64_t rows_total, E_total;
} b200sfm_test_ra_info;

/* Outputs of b200sfm_test_ra_system.  Caller-owned, each may be NULL.  Sizes: res, b [3E]; w [E]; rhs, deg [3n];
 * Minv [6n]; Ac [nc*nc] (two-level paths only). */
typedef struct {
  double* res;      /* residuals at theta */
  double* w;        /* edge weights of the system (before squaring) */
  double* b;        /* square = 1 only: the L1 stage's W r */
  double* rhs;      /* A^T W^p r, p = 1 + square */
  double* deg;      /* the Laplacian diagonal as the preconditioner sees it */
  double* Minv;     /* Jacobi blocks */
  double* Ac;       /* the inverted coarse matrix (P^T L P)^-1 */
  double b_norm2;   /* square = 1 only: |W r|^2 */
} b200sfm_test_ra_system_out;

/* Arguments as b200sfm_ra_solve_rig (eci, ecj, cam_frames_begin, cam_frames: NULL when n_cams == 0) plus the gravity
 * mask of b200sfm_ra_solve_gravity (NULL: none); theta [n*3] is the initial state.  Only opts->use_weight is read. */
int b200sfm_test_ra_problem_create(b200sfm_ctx* ctx, const b200sfm_ra_opts* opts, int32_t n_frames, int32_t n_cams,
                                   int64_t n_edges, const int32_t* ei, const int32_t* ej, const int32_t* eci,
                                   const int32_t* ecj, const double* R_rel, const double* edge_w,
                                   const uint8_t* frame_has_gravity, const int32_t* cam_frames_begin,
                                   const int32_t* cam_frames, int32_t fixed_frame, const double* theta,
                                   b200sfm_test_ra_problem** out);
void b200sfm_test_ra_problem_free(b200sfm_test_ra_problem* problem);

/* The selected paths; agg_of [n] (may be NULL) receives each node's aggregate on two-level paths. */
int b200sfm_test_ra_problem_info(b200sfm_test_ra_problem* problem, b200sfm_test_ra_info* info, int32_t* agg_of);

/* Residuals and weights at the current theta (mode 0: the L1 rows' weights, 1: Geman-McClure, 2: half-norm, with
 * sigma2 = sigma^2 in radians^2), then the linear system as a solve prepares it: square = 1 as the L1 stage does (b = W r,
 * z = u = 0, the coarse inverse kept while it holds the L1 weights), square = 0 as an IRLS iteration does. */
int b200sfm_test_ra_system(b200sfm_test_ra_problem* problem, int32_t mode, double sigma2, int32_t square,
                           b200sfm_test_ra_system_out* out);

/* y = L x through the mat-vec of a PCG iteration on the selected path, with the weights of the last system.
 * x, y [3n]. */
int b200sfm_test_ra_apply(b200sfm_test_ra_problem* problem, const double* x, double* y);

/* z = M^-1 r: the Jacobi blocks and, on two-level paths, the coarse correction, as a PCG iteration applies them.
 * r, z [3n]. */
int b200sfm_test_ra_precond(b200sfm_test_ra_problem* problem, const double* r, double* z);

/* Exactly k PCG iterations (tolerance 0) on the last system's rhs: cold from x = 0, or warm-started from warm_x [3n]
 * as the L1 stage's ADMM solves after the first.  x_out [3n]; iterations (may be NULL) receives the count. */
int b200sfm_test_ra_pcg(b200sfm_test_ra_problem* problem, int32_t k, const double* warm_x, double* x_out,
                        int32_t* iterations);

/* One ADMM iteration of the L1 stage with the last system's weights after the x-update x [3n]: b [3E], z and u [3E]
 * (updated in place), rsu [9n] receives rhs | svec | uvec, norms [5] |A_w x - z - b|^2, |A_w x|^2, |z|^2, |svec|^2,
 * |uvec|^2. */
int b200sfm_test_ra_admm_step(b200sfm_test_ra_problem* problem, double rho, const double* x, const double* b, double* z,
                              double* u, double* rsu, double* norms);

/* theta <- theta (+) step, the frames' update and the unknown cameras' quaternion average, as a solve applies a step.
 * step, theta_out [3n]; sums [3] = average frame step, |step|, NaN flag. */
int b200sfm_test_ra_update(b200sfm_test_ra_problem* problem, const double* step, double* theta_out, double* sums);

/* ---- global positioning ----------------------------------------------------------------------------------------
 * A resident global-positioning problem (b200sfm_gp_problem_create, _set_rig_terms, _set_rig_unknown, _set_state).
 * Block vectors hold CB = C + S_u blocks of 3 doubles: the C frame centres, then the S_u unknown cam_from_rig centres.
 * Symmetric 3x3 blocks are packed as 6 doubles, upper triangle, row by row.  Observation arrays are in the problem's
 * observation order, short tracks included (zero rows). */

/* Outputs of b200sfm_test_gp_step.  Every array pointer is caller-owned and may be NULL (not downloaded).
 * Sizes: M [N*6]; bw [N*4]; jscale_s, ds, cand_scales [N]; Vinv [P*6]; gX, dX, cand_points [P*3]; Dp, jscale_p [P];
 * U, Minv [CB*6]; gc, Dc, b, px, resid [CB*3]; jscale_c [CB]; cand_centers [C*3]; cand_ucen [S_u*3]. */
typedef struct {
  double* M;            /* per observation: the 3x3 block with the scale eliminated, w s^2 (I - w d d^T / h) */
  double* bw;           /* per observation: (b_o, w s^2), b_o = w s (r - (w / h) d (d.r)) */
  double* jscale_s;     /* Jacobi scale of each variable scale (0 on constant scales) */
  double* ds;           /* scale step from the back-substitution */
  double* Vinv;         /* per point: (V + D_p I)^-1 (0 on constant points) */
  double* gX;           /* per point: -sum b_o */
  double* Dp;           /* point damping */
  double* jscale_p;     /* point Jacobi scales (variable points only) */
  double* dX;           /* point step from the back-substitution */
  double* U;            /* per block: sum M_o (R M_o R^T for an unknown sensor); identity on constant blocks */
  double* gc;           /* per block: sum b_o (R b_o); 0 on constant blocks */
  double* Dc;           /* block damping */
  double* Minv;         /* preconditioner blocks */
  double* jscale_c;     /* block Jacobi scales; -1 marks a constant block */
  double* b;            /* right-hand side of the reduced system */
  double* px;           /* the PCG iterate: the block step */
  double* resid;        /* the PCG residual b - (S + D) px */
  double* cand_centers; /* candidate state Project(x + alpha delta) (not accepted) */
  double* cand_points;
  double* cand_scales;
  double* cand_ucen;
  double cost;          /* robust cost at the current state */
  double gmax;          /* max |g| for the gradient tolerance */
  double g_dot_delta;   /* g . delta over the full step */
  double model_cost_change;
  double cand_cost;     /* robust cost of the candidate */
  double step_norm;     /* |candidate - x| over the variable blocks */
  double x_norm;        /* |x| over the variable blocks */
  int32_t pcg_iterations;
  /* the paths the step took */
  int32_t schur_jacobi, CB, n_us, pcg_depth;
} b200sfm_test_gp_step_out;

/* At the problem's current state: apply the option masks as b200sfm_gp_problem_solve does, linearise as its first LM
 * iteration and solve one step at `radius` with the PCG settings of `opts`, then form the candidate at step length
 * `alpha` without accepting it, and download into `out`.  With first_radius > 0 a step at first_radius comes first; the
 * step at `radius` then reuses its Jacobi scales, as every step of a solve after the first does. */
int b200sfm_test_gp_step(b200sfm_gp_problem* problem, const b200sfm_gp_opts* opts, double first_radius, double radius,
                         double alpha, b200sfm_test_gp_step_out* out);

/* y = (S + D) x over the CB*3 block dofs with the linearisation of the last b200sfm_test_gp_step, through the kernels
 * of one PCG iteration.  x, y: host arrays [CB*3]. */
int b200sfm_test_gp_apply(b200sfm_gp_problem* problem, const double* x, double* y);

/* ---- gravity refinement ----------------------------------------------------------------------------------------
 * b200sfm_test_gravity runs b200sfm_gravity_refine's stages (gravity_kernels.cuh) on its arguments and downloads what
 * each stage leaves.  Every array pointer is caller-owned and may be NULL (not downloaded).  E is the number of pairs
 * given, k indexes the error-prone frames in the order of ep.  Sizes: mistake, angle [E]; offs [F+1]; inc [2E];
 * total, mistakes, error_prone, ep [F]; gobs [2E*3]; x [F*3], status, iterations [F] (the first n_error_prone rows);
 * trace [F * (5 + 5 trace_cap)]. */
typedef struct {
  uint8_t* mistake;      /* per pair: CalcAngle > max_gravity_error (0 for a pair with a frame without gravity) */
  double* angle;         /* per pair: the angle in degrees (unwritten for a pair with a frame without gravity) */
  int32_t* offs;         /* frame f's incidences are inc[offs[f] .. offs[f+1]) */
  int32_t* inc;          /* the incidences 2 pair + side sorted by frame, ascending inside a frame */
  int32_t* total;        /* per frame: counted incidences */
  int32_t* mistakes;     /* per frame: incidences of pairs with a mistake */
  uint8_t* error_prone;  /* per frame: the error-prone flag */
  int32_t* ep;           /* the error-prone frames, ascending (n_error_prone entries) */
  double* gobs;          /* per incidence of an error-prone frame: its observed gravity (NaN: not a term); NaN elsewhere */
  double* x;             /* per k: the LM result before the consistency check */
  uint8_t* status;       /* per k: 1 too few terms, 2 accepted, 3 rejected */
  int32_t* iterations;   /* per k: LM iterations */
  double* trace;         /* per k, stride 5 + 5 trace_cap: the AverageGravity start x0 [3] (after the sign rule), the
                            termination (-1 too few terms, 0 gradient tolerance at x0, 1 max iterations, 2 min radius,
                            3 too many invalid steps, 4 parameter tolerance, 5 function tolerance, 6 gradient tolerance),
                            the number of recorded iterations, then per iteration up to trace_cap: cost, radius, model
                            cost change, candidate cost (NaN for an invalid step) and a code (-1 invalid step, 0 rejected,
                            1 accepted, 2 stopped by the parameter tolerance, 3 stopped by the function tolerance) */
  int32_t trace_cap;     /* in: iterations recorded per frame */
  int32_t n_error_prone; /* out */
} b200sfm_test_gravity_out;

/* Arguments and return codes as b200sfm_gravity_refine (gravity and status are not written).  Single-rank only. */
int b200sfm_test_gravity(b200sfm_ctx* ctx, const b200sfm_gravity_opts* opts, int32_t F, const double* R_align,
                         const uint8_t* has_gravity, int64_t E, const int32_t* frame1, const int32_t* frame2,
                         const double* M, b200sfm_test_gravity_out* out);

/* The solvers' per-warp device helpers on n inputs, one thread each, through the production __device__ functions.
 * Row widths in -> out per op:
 *   0 grv_householder      x [3]                      -> v [3], beta
 *   1 grv_plus             x [3], d [2]               -> x [+] d [3]
 *   2 grv_plus_jacobian    x [3]                      -> P [3x2 row-major]
 *   3 grv_principal        A [3x3 row-major, symmetric] -> its principal eigenvector [3]
 *   4 quat_avg_eig         M [10 packed 4x4 upper triangle], q0 [4] -> the dominant eigenvector [4] (q0 picks its sign)
 *   5 grv_pair_angle       R [3x3 row-major]          -> RotUpToAngle(R), CalcAngle(R, AngleToRotUp(.)) in degrees */
int b200sfm_test_device_helpers(b200sfm_ctx* ctx, int32_t op, int64_t n, const double* in, double* out);

#ifdef __cplusplus
}
#endif
#endif /* B200SFM_TESTING_H_ */
