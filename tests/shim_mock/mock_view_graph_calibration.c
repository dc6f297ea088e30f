/* TEST DOUBLE (tests only, never shipped): the view-graph calibration entries of the C ABI, linked beside mock_b200sfm.c.
 * Records what the shim's ViewGraphCalibrator passes ("name n v0 v1 ..." lines appended to $MOCK_DUMP) and returns a
 * recognisable result: focal[k] = 1000 + k, camera k accepted when k is even, pair e invalidated when e is even,
 * usable = 1. */
#include <stdio.h>
#include <stdlib.h>

#include "b200sfm.h"

static FILE* dump_file(void) {
  const char* p = getenv("MOCK_DUMP");
  return fopen(p ? p : "/dev/null", "a");
}
static void dump_i32(FILE* f, const char* name, const int32_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %d", v[i]);
  fprintf(f, "\n");
}
static void dump_u8(FILE* f, const char* name, const uint8_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %d", (int)v[i]);
  fprintf(f, "\n");
}
static void dump_f64(FILE* f, const char* name, const double* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %.17g", v[i]);
  fprintf(f, "\n");
}

void b200sfm_vgc_default_opts(b200sfm_vgc_opts* o) {
  b200sfm_vgc_opts d = {100, 20, 1e-2, 1e-5, 1e-10, 1e-8, 0.1, 10.0, 2.0, 1000, 0, 1e-12, 0, 0};
  *o = d;
}

int b200sfm_view_graph_calibrate(b200sfm_ctx* ctx, const b200sfm_vgc_opts* o, int32_t K, const double* pp, double* focal,
                                 const uint8_t* focal_constant, int64_t E, const int32_t* cam1, const int32_t* cam2,
                                 const double* F, uint8_t* pair_valid, uint8_t* cam_accepted, double* pair_residual,
                                 b200sfm_lm_stats* stats) {
  (void)ctx;
  (void)pair_residual;
  FILE* f = dump_file();
  fprintf(f, "call view_graph_calibrate\n");
  const double opts[9] = {o->max_num_iterations, o->max_num_line_search_step_size_iterations, o->thres_loss_function,
                          o->function_tolerance, o->thres_lower_ratio, o->thres_higher_ratio, o->thres_two_view_error,
                          o->pcg_max_iterations, o->pcg_rel_tolerance};
  dump_f64(f, "opts", opts, 9);
  dump_f64(f, "principal_point", pp, 2 * (long long)K);
  dump_f64(f, "focal", focal, K);
  dump_u8(f, "focal_constant", focal_constant, K);
  dump_i32(f, "cam1", cam1, E);
  dump_i32(f, "cam2", cam2, E);
  dump_f64(f, "F", F, 9 * E);
  fclose(f);
  for (int32_t k = 0; k < K; ++k) {
    focal[k] = 1000.0 + k;
    cam_accepted[k] = (k % 2) == 0;
  }
  for (int64_t e = 0; e < E; ++e) pair_valid[e] = (e % 2) != 0;
  if (stats) {
    b200sfm_lm_stats s = {0};
    s.usable = 1;
    s.num_observations = E;
    *stats = s;
  }
  return B200SFM_OK;
}
