/* TEST DOUBLE (tests only, never shipped): the two view-graph entries of the C ABI, linked beside mock_b200sfm.c.
 * Records what the shim's RelPoseFilter::FilterRotations and KeepLargestConnectedComponentsDevice pass ("name n v0 v1 ..."
 * lines appended to $MOCK_DUMP) and returns a recognisable result:
 *   filter_rotations: every pair at an odd index is invalidated;
 *   keep_largest_component: every frame but the last stays registered, the pair at index 0 is invalidated and
 *   num_registered_images = 100 + num_images. */
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

int b200sfm_view_graph_filter_rotations(b200sfm_ctx* ctx, int32_t num_images, const double* cam_from_world_quat_xyzw,
                                        const uint8_t* image_registered, int64_t num_pairs, const int32_t* pair_image1,
                                        const int32_t* pair_image2, const double* pair_quat_xyzw, double max_angle_deg,
                                        uint8_t* pair_valid, int64_t* num_invalidated) {
  (void)ctx;
  FILE* f = dump_file();
  fprintf(f, "call view_graph_filter_rotations\n");
  dump_f64(f, "max_angle", &max_angle_deg, 1);
  dump_f64(f, "cam_from_world", cam_from_world_quat_xyzw, 4LL * num_images);
  dump_u8(f, "image_registered", image_registered, num_images);
  dump_i32(f, "pair_image1", pair_image1, num_pairs);
  dump_i32(f, "pair_image2", pair_image2, num_pairs);
  dump_f64(f, "pair_quat", pair_quat_xyzw, 4 * num_pairs);
  dump_u8(f, "pair_valid", pair_valid, num_pairs);
  fclose(f);
  int64_t n = 0;
  for (int64_t e = 1; e < num_pairs; e += 2) {
    pair_valid[e] = 0;
    ++n;
  }
  *num_invalidated = n;
  return B200SFM_OK;
}

int b200sfm_view_graph_keep_largest_component(b200sfm_ctx* ctx, int32_t num_frames, int32_t num_images, const int32_t* image_frame,
                                              int64_t num_pairs, const int32_t* pair_image1, const int32_t* pair_image2,
                                              uint8_t* pair_valid, uint8_t* frame_registered, int32_t* num_registered_images) {
  (void)ctx;
  FILE* f = dump_file();
  fprintf(f, "call view_graph_keep_largest_component\n");
  dump_i32(f, "image_frame", image_frame, num_images);
  dump_i32(f, "pair_image1", pair_image1, num_pairs);
  dump_i32(f, "pair_image2", pair_image2, num_pairs);
  dump_u8(f, "pair_valid", pair_valid, num_pairs);
  dump_u8(f, "frame_registered", frame_registered, num_frames);
  fclose(f);
  for (int32_t k = 0; k < num_frames; ++k) frame_registered[k] = k != num_frames - 1;
  if (num_pairs > 0) pair_valid[0] = 0;
  *num_registered_images = 100 + num_images;
  return B200SFM_OK;
}
