/* b200sfm_testing.h -- test-only probe into a resident bundle-adjustment problem.
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

#ifdef __cplusplus
}
#endif
#endif /* B200SFM_TESTING_H_ */
