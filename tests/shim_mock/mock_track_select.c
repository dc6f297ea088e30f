/* TEST DOUBLE (tests only, never shipped): the track entries of the C ABI with the context calls the shim's TrackEngine
 * needs, linked on their own (not beside mock_b200sfm.c, whose establishment entries record nothing).  Records what
 * TrackEngine passes ("name n v0 v1 ..." lines appended to $MOCK_DUMP) and returns recognisable results:
 *   b200sfm_tracks_establish / _get: two tracks, id 7 with observations (1, 0) (2, 5), and id 3 with none (discarded);
 *   b200sfm_tracks_select: keep[t] = 1 for every even t; num_selected = their count. */
#include <stdio.h>
#include <stdlib.h>

#include "b200sfm.h"

static int g_ctx_storage;

static FILE* dump_file(void) {
  const char* p = getenv("MOCK_DUMP");
  return fopen(p ? p : "/dev/null", "a");
}
static void dump_u64(FILE* f, const char* name, const uint64_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %llu", (unsigned long long)v[i]);
  fprintf(f, "\n");
}
static void dump_i64(FILE* f, const char* name, const int64_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %lld", (long long)v[i]);
  fprintf(f, "\n");
}
static void dump_u32(FILE* f, const char* name, const uint32_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %u", v[i]);
  fprintf(f, "\n");
}
static void dump_d(FILE* f, const char* name, const double* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %.17g", v[i]);
  fprintf(f, "\n");
}

int b200sfm_create(int device, b200sfm_ctx** o) {
  (void)device;
  *o = (b200sfm_ctx*)&g_ctx_storage;
  return B200SFM_OK;
}
const char* b200sfm_last_error(const b200sfm_ctx* c) {
  (void)c;
  return "mock";
}

int b200sfm_tracks_establish(b200sfm_ctx* ctx, int64_t m, const uint64_t* g1, const uint64_t* g2, const double* xy1, const double* xy2,
                             double thr, b200sfm_tracks** out, int64_t* nt, int64_t* no, int64_t* nd) {
  (void)ctx;
  FILE* f = dump_file();
  fprintf(f, "call tracks_establish\n");
  dump_d(f, "thres", &thr, 1);
  dump_u64(f, "gid1", g1, m);
  dump_u64(f, "gid2", g2, m);
  dump_d(f, "xy1", xy1, 2 * m);
  dump_d(f, "xy2", xy2, 2 * m);
  fclose(f);
  *out = (b200sfm_tracks*)&g_ctx_storage;
  *nt = 2;
  *no = 2;
  *nd = 1;
  return B200SFM_OK;
}
int b200sfm_tracks_get(b200sfm_tracks* t, uint64_t* ids, int64_t* begin, uint32_t* im, uint32_t* ft) {
  (void)t;
  ids[0] = 3; ids[1] = 7;
  begin[0] = 0; begin[1] = 0; begin[2] = 2;
  im[0] = 1; im[1] = 2;
  ft[0] = 0; ft[1] = 5;
  return B200SFM_OK;
}
void b200sfm_tracks_free(b200sfm_tracks* t) { (void)t; }

int b200sfm_tracks_select(b200sfm_ctx* ctx, int64_t num_tracks, const uint64_t* track_ids, const int64_t* begin,
                          const uint32_t* obs_image, int32_t num_registered, const uint32_t* registered_image_ids,
                          int32_t min_num_tracks_per_view, int32_t min_num_view_per_track, int32_t max_num_view_per_track,
                          int32_t max_num_tracks, uint8_t* keep, int64_t* num_selected) {
  (void)ctx;
  FILE* f = dump_file();
  fprintf(f, "call tracks_select\n");
  const int64_t opts[4] = {min_num_tracks_per_view, min_num_view_per_track, max_num_view_per_track, max_num_tracks};
  dump_i64(f, "options", opts, 4);
  dump_u64(f, "track_ids", track_ids, num_tracks);
  dump_i64(f, "begin", begin, num_tracks + 1);
  dump_u32(f, "obs_image", obs_image, begin[num_tracks]);
  dump_u32(f, "registered", registered_image_ids, num_registered);
  fclose(f);
  int64_t n = 0;
  for (int64_t t = 0; t < num_tracks; ++t) {
    keep[t] = t % 2 == 0;
    n += keep[t];
  }
  *num_selected = n;
  return B200SFM_OK;
}
