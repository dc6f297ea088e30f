/* TEST DOUBLE (tests only, never shipped): the image-pair entry of the C ABI, linked beside mock_b200sfm.c.  Records what
 * the shim's ImagePairsInlierCount passes ("name n v0 v1 ..." lines appended to $MOCK_DUMP) and returns a recognisable
 * result: every match row k of the call with k % 3 != 1 is an inlier, the score of pair e is e + 0.5. */
#include <stdio.h>
#include <stdlib.h>

#include "b200sfm.h"
#include "mock_dump.h"


int b200sfm_image_pairs_inlier_count(b200sfm_ctx* ctx, int32_t I, const int64_t* fb, const double* feat, const int32_t* image_intr,
                                     int32_t K, const int32_t* intr_model, const double* intr, int64_t E, const int32_t* i1,
                                     const int32_t* i2, const int32_t* cfg, const double* q, const double* t, const double* F,
                                     const double* H, const int64_t* mb, const int32_t* m, double eE, double eF, double eH,
                                     uint8_t* inl, int32_t* n_inl, double* score) {
  (void)ctx;
  const long long M = E > 0 ? mb[E] : 0;
  FILE* f = mock_dump_open();
  fprintf(f, "call image_pairs_inlier_count\n");
  const int64_t dims[4] = {I, K, E, M};
  const double thr[3] = {eE, eF, eH};
  dump_i64(f, "dims", dims, 4); dump_f64(f, "thresholds", thr, 3);
  dump_i64(f, "feature_begin", fb, I + 1); dump_f64(f, "features", feat, 2 * (fb ? fb[I] : 0)); dump_i32(f, "image_intr", image_intr, I);
  dump_i32(f, "intr_model", intr_model, K); dump_f64(f, "intr", intr, (long long)K * B200SFM_INTR_STRIDE);
  dump_i32(f, "image1", i1, E); dump_i32(f, "image2", i2, E); dump_i32(f, "config", cfg, E);
  dump_f64(f, "quat", q, 4 * E); dump_f64(f, "trans", t, 3 * E); dump_f64(f, "F", F, 9 * E); dump_f64(f, "H", H, 9 * E);
  dump_i64(f, "match_begin", mb, E + 1); dump_i32(f, "matches", m, 2 * M);
  fclose(f);
  for (int64_t e = 0; e < E; ++e) {
    n_inl[e] = 0;
    for (int64_t k = mb[e]; k < mb[e + 1]; ++k) {
      inl[k] = k % 3 != 1;
      n_inl[e] += inl[k];
    }
    score[e] = (double)e + 0.5;
  }
  return B200SFM_OK;
}
