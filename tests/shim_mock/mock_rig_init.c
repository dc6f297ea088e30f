/* TEST DOUBLE (tests only, never shipped): the entries of the C ABI that the shim's rig pre-pass adds, linked beside
 * mock_b200sfm.c.  Records what RigRotationPrePass passes ("name n v0 v1 ..." lines appended to $MOCK_DUMP) and returns
 * a recognisable result: the spanning tree reaches every node with the rotations left as passed; every unknown camera
 * with a registered, estimated image gets 0.25 rad about x (one sample), every frame one sample, its rotation unchanged. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "b200sfm.h"
#include "mock_dump.h"


int b200sfm_ra_mst_init(b200sfm_ctx* ctx, int32_t n, int64_t E, const int32_t* ei, const int32_t* ej, const double* R,
                        const double* w, int32_t root, double* Rout, int32_t* parent, b200sfm_mst_stats* st) {
  (void)ctx; (void)Rout;
  FILE* f = mock_dump_open();
  fprintf(f, "call ra_mst_init\n");
  const int32_t dims[3] = {n, (int32_t)E, root};
  dump_i32(f, "dims", dims, 3);
  dump_i32(f, "ei", ei, E); dump_i32(f, "ej", ej, E); dump_f64(f, "R_rel", R, 9 * E); dump_f64(f, "weight", w, E);
  fclose(f);
  for (int32_t v = 0; parent && v < n; ++v) parent[v] = root;
  if (st) memset(st, 0, sizeof(*st));
  return B200SFM_OK;
}

int b200sfm_rig_rotations_from_images(b200sfm_ctx* ctx, int64_t I, int32_t F, int32_t K, const int32_t* fr, const int32_t* cam,
                                      const uint8_t* est, const double* q, const int32_t* ref, const uint8_t* known, double* cq,
                                      int32_t* cn, double* fq, int32_t* fn, b200sfm_rig_init_stats* st) {
  (void)ctx; (void)fq;
  FILE* f = mock_dump_open();
  fprintf(f, "call rig_rotations_from_images\n");
  const int32_t dims[3] = {(int32_t)I, F, K};
  dump_i32(f, "dims", dims, 3);
  dump_i32(f, "image_frame", fr, I); dump_i32(f, "image_camera", cam, I); dump_u8(f, "image_estimated", est, I);
  dump_f64(f, "cam_from_world", q, 4 * I); dump_i32(f, "frame_ref_camera", ref, F); dump_u8(f, "camera_known", known, K);
  fclose(f);
  for (int32_t c = 0; cn && c < K; ++c) cn[c] = 0;
  for (int64_t i = 0; i < I; ++i) {
    const int32_t c = cam[i];
    if (fr[i] < 0 || known[c] || (est && !est[i])) continue;
    cq[4 * c] = 0.12467473338522769; cq[4 * c + 1] = 0; cq[4 * c + 2] = 0; cq[4 * c + 3] = 0.99219766722932900;
    if (cn) cn[c] = 1;
  }
  for (int32_t k = 0; fn && k < F; ++k) fn[k] = 1;
  if (st) memset(st, 0, sizeof(*st));
  return B200SFM_OK;
}
