/* TEST DOUBLE (tests only, never shipped): the reconstruction-pruning entry of the C ABI, linked beside mock_b200sfm.c.
 * Records what the shim's PruneWeaklyConnectedImages passes ("name n v0 v1 ..." lines appended to $MOCK_DUMP) and
 * returns a recognisable result: frame f gets cluster f % 3 and stays registered, except every third frame (f % 3 == 2),
 * which gets -1 and is deregistered; 2 clusters. */
#include <stdio.h>
#include <stdlib.h>

#include "b200sfm.h"

static void dump_i64(FILE* f, const char* name, const int64_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %lld", (long long)v[i]);
  fprintf(f, "\n");
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

int b200sfm_prune_weakly_connected(b200sfm_ctx* ctx, int32_t num_frames, int64_t num_tracks, const int64_t* track_begin,
                                   const int32_t* obs_frame, const uint8_t* frame_self_loop, int32_t min_num_observations,
                                   int64_t max_pair_keys_per_pass, int32_t* cluster_id, uint8_t* is_registered,
                                   int32_t* num_clusters, b200sfm_prune_stats* stats) {
  (void)ctx;
  (void)stats;
  const char* p = getenv("MOCK_DUMP");
  FILE* f = fopen(p ? p : "/dev/null", "a");
  fprintf(f, "call prune_weakly_connected\n");
  const int64_t scalars[3] = {min_num_observations, max_pair_keys_per_pass, num_frames};
  dump_i64(f, "scalars", scalars, 3);
  dump_i64(f, "track_begin", track_begin, num_tracks + 1);
  dump_i32(f, "obs_frame", obs_frame, track_begin[num_tracks]);
  dump_u8(f, "frame_self_loop", frame_self_loop, num_frames);
  dump_u8(f, "is_registered", is_registered, num_frames);
  fclose(f);
  for (int32_t k = 0; k < num_frames; ++k) {
    cluster_id[k] = k % 3 == 2 ? -1 : k % 3;
    is_registered[k] = k % 3 != 2;
  }
  *num_clusters = 2;
  return B200SFM_OK;
}
