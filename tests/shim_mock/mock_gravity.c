/* TEST DOUBLE (tests only, never shipped): the gravity-refinement entries of the C ABI, linked beside mock_b200sfm.c.
 * Records what the shim's GravityRefiner passes ("name n v0 v1 ..." lines appended to $MOCK_DUMP) and returns a
 * recognisable result: every frame with gravity gets status 2 and gravity (0, 1, f) when its index f is even, status 3
 * otherwise. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "b200sfm.h"
#include "mock_dump.h"


void b200sfm_gravity_default_opts(b200sfm_gravity_opts* o) {
  memset(o, 0, sizeof(*o));
  o->max_outlier_ratio = 0.5;
  o->max_gravity_error = 1.0;
  o->min_num_neighbors = 7;
  o->max_num_iterations = 100;
}

int b200sfm_gravity_refine(b200sfm_ctx* ctx, const b200sfm_gravity_opts* opts, int32_t F, const double* R_align,
                           const uint8_t* has_gravity, int64_t E, const int32_t* frame1, const int32_t* frame2,
                           const double* M, double* gravity, uint8_t* status, b200sfm_gravity_stats* stats) {
  (void)ctx;
  FILE* f = mock_dump_open();
  fprintf(f, "call gravity_refine\n");
  const double scalars[6] = {opts->max_outlier_ratio, opts->max_gravity_error, opts->min_num_neighbors,
                             opts->max_num_iterations, (double)F, (double)E};
  dump_f64(f, "scalars", scalars, 6);
  dump_f64(f, "R_align", R_align, 9LL * F);
  fprintf(f, "has_gravity %d", F);
  for (int32_t k = 0; k < F; ++k) fprintf(f, " %d", (int)has_gravity[k]);
  fprintf(f, "\n");
  dump_i32(f, "frame1", frame1, E);
  dump_i32(f, "frame2", frame2, E);
  dump_f64(f, "M", M, 9 * E);
  fclose(f);
  if (stats) memset(stats, 0, sizeof(*stats));
  for (int32_t k = 0; k < F; ++k) {
    status[k] = has_gravity[k] ? (k % 2 == 0 ? 2 : 3) : 0;
    if (status[k] == 2) { gravity[3 * k] = 0; gravity[3 * k + 1] = 1; gravity[3 * k + 2] = k; }
  }
  return B200SFM_OK;
}
