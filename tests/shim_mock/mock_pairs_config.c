/* TEST DOUBLE (tests only, never shipped): the stage-0 entry of the C ABI, linked beside mock_b200sfm.c.  Records what
 * the shim's ViewGraphManipulater::UpdateImagePairsConfig passes ("name n v0 v1 ..." lines appended to $MOCK_DUMP) and
 * returns a recognisable result: every UNCALIBRATED pair e is promoted, with F[e][k] = 100 * e + k. */
#include <stdio.h>
#include <stdlib.h>

#include "b200sfm.h"
#include "mock_dump.h"


int b200sfm_view_graph_update_pairs_config(b200sfm_ctx* ctx, int32_t K, const int32_t* intr_model, const double* intr_params,
                                           const uint8_t* has_prior_focal, int64_t num_pairs, const int32_t* pair_cam1,
                                           const int32_t* pair_cam2, const uint8_t* pair_valid, const double* pair_quat_xyzw,
                                           const double* pair_trans, int32_t* pair_config, double* pair_F, int64_t* num_promoted) {
  (void)ctx;
  FILE* f = mock_dump_open();
  fprintf(f, "call view_graph_update_pairs_config\n");
  dump_i32(f, "intr_model", intr_model, K);
  dump_f64(f, "intr_params", intr_params, (long long)K * B200SFM_INTR_STRIDE);
  dump_u8(f, "has_prior_focal", has_prior_focal, K);
  dump_i32(f, "pair_cam1", pair_cam1, num_pairs);
  dump_i32(f, "pair_cam2", pair_cam2, num_pairs);
  dump_u8(f, "pair_valid", pair_valid, num_pairs);
  dump_i32(f, "pair_config", pair_config, num_pairs);
  dump_f64(f, "pair_quat", pair_quat_xyzw, 4 * num_pairs);
  dump_f64(f, "pair_trans", pair_trans, 3 * num_pairs);
  dump_f64(f, "pair_F", pair_F, 9 * num_pairs);
  fclose(f);
  int64_t n = 0;
  for (int64_t e = 0; e < num_pairs; ++e) {
    if (pair_config[e] != B200SFM_TWO_VIEW_UNCALIBRATED) continue;
    pair_config[e] = B200SFM_TWO_VIEW_CALIBRATED;
    for (int k = 0; k < 9; ++k) pair_F[9 * e + k] = 100.0 * (double)e + k;
    ++n;
  }
  *num_promoted = n;
  return B200SFM_OK;
}
