/* TEST DOUBLE (tests only, never shipped): the entries of the C ABI the shim's TrackFilter, UndistortImages and
 * NormalizeReconstruction call, linked on their own.  Records what the shim passes ("name n v0 v1 ..." lines appended to
 * $MOCK_DUMP) and returns recognisable results:
 *   _create / _create_rig: B200SFM_ERR_UNSUPPORTED for a camera model outside 0-3, as the library;
 *   the observation filters: keep[o] = (o % 3 != 1), 7 tracks changed; the triangulation filter: keep[p] = (p % 2 == 0),
 *   5 tracks removed;
 *   _normalize: scale 2, translation (1, 2, 3); _get_state: trans[i] = 100 + i, points[i] = 200 + i;
 *   b200sfm_undistort_features: bearing i = (i, 0.5, -i), B200SFM_ERR_UNSUPPORTED for a used model outside 0-3. */
#include <stdio.h>
#include <stdlib.h>

#include "b200sfm.h"

static int g_ctx_storage;
static struct { int rig; int32_t C, P, K, S; int64_t N; } g_prob;

static FILE* dump_file(void) {
  const char* p = getenv("MOCK_DUMP");
  return fopen(p ? p : "/dev/null", "a");
}
static void dump_i(FILE* f, const char* name, const int32_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %d", v[i]);
  fprintf(f, "\n");
}
static void dump_u16(FILE* f, const char* name, const uint16_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %u", v[i]);
  fprintf(f, "\n");
}
static void dump_u8(FILE* f, const char* name, const uint8_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %u", v[i]);
  fprintf(f, "\n");
}
static void dump_i64(FILE* f, const char* name, const int64_t* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %lld", (long long)v[i]);
  fprintf(f, "\n");
}
static void dump_d(FILE* f, const char* name, const double* v, long long n) {
  fprintf(f, "%s %lld", name, v ? n : 0);
  for (long long i = 0; v && i < n; ++i) fprintf(f, " %.17g", v[i]);
  fprintf(f, "\n");
}
static int bad_model(const int32_t* m, int32_t K) {
  for (int32_t k = 0; k < K; ++k)
    if (m[k] < 0 || m[k] > 3) return 1;
  return 0;
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

int b200sfm_ba_problem_create(b200sfm_ctx* ctx, int32_t C, int32_t P, int64_t N, int32_t K, const int64_t* ptb,
                              const int32_t* obs_cam, const double* obs_xy, const int32_t* cam_intr, const int32_t* intr_model,
                              const uint8_t* mask, int32_t min_views, b200sfm_ba_problem** out) {
  (void)ctx;
  FILE* f = dump_file();
  fprintf(f, "call create\n");
  const int32_t dims[5] = {C, P, (int32_t)N, K, min_views};
  dump_i(f, "dims", dims, 5);
  dump_i64(f, "ptb", ptb, P + 1);
  dump_i(f, "obs_cam", obs_cam, N);
  dump_d(f, "obs_xy", obs_xy, 2 * N);
  dump_i(f, "cam_intr", cam_intr, C);
  dump_i(f, "intr_model", intr_model, K);
  dump_u8(f, "mask", mask, C);
  fclose(f);
  if (bad_model(intr_model, K)) return B200SFM_ERR_UNSUPPORTED;
  g_prob.rig = 0; g_prob.C = C; g_prob.P = P; g_prob.K = K; g_prob.S = 0; g_prob.N = N;
  *out = (b200sfm_ba_problem*)&g_prob;
  return B200SFM_OK;
}

int b200sfm_ba_problem_create_rig(b200sfm_ctx* ctx, int32_t F, int32_t P, int64_t N, int32_t K, int32_t S, const int64_t* ptb,
                                  const int32_t* obs_frame, const uint16_t* obs_sensor, const double* obs_xy, const double* sq,
                                  const double* st, const int32_t* sensor_intr, const int32_t* intr_model, const uint8_t* mask,
                                  int32_t min_views, b200sfm_ba_problem** out) {
  (void)ctx;
  FILE* f = dump_file();
  fprintf(f, "call create_rig\n");
  const int32_t dims[6] = {F, P, (int32_t)N, K, S, min_views};
  dump_i(f, "dims", dims, 6);
  dump_i64(f, "ptb", ptb, P + 1);
  dump_i(f, "obs_frame", obs_frame, N);
  dump_u16(f, "obs_sensor", obs_sensor, N);
  dump_d(f, "obs_xy", obs_xy, 2 * N);
  dump_d(f, "sensor_q", sq, 4 * S);
  dump_d(f, "sensor_t", st, 3 * S);
  dump_i(f, "sensor_intr", sensor_intr, S);
  dump_i(f, "intr_model", intr_model, K);
  dump_u8(f, "mask", mask, F);
  fclose(f);
  if (bad_model(intr_model, K)) return B200SFM_ERR_UNSUPPORTED;
  g_prob.rig = 1; g_prob.C = F; g_prob.P = P; g_prob.K = K; g_prob.S = S; g_prob.N = N;
  *out = (b200sfm_ba_problem*)&g_prob;
  return B200SFM_OK;
}

int b200sfm_ba_problem_set_images(b200sfm_ba_problem* p, int32_t I, const int32_t* image_frame, const int32_t* image_sensor) {
  (void)p;
  FILE* f = dump_file();
  fprintf(f, "call set_images\n");
  dump_i(f, "image_frame", image_frame, I);
  dump_i(f, "image_sensor", image_sensor, I);
  fclose(f);
  return B200SFM_OK;
}

int b200sfm_ba_problem_set_state(b200sfm_ba_problem* p, const double* intr, const double* quat, const double* trans,
                                 const double* points) {
  (void)p;
  FILE* f = dump_file();
  fprintf(f, "call set_state\n");
  dump_d(f, "intr", intr, (long long)g_prob.K * B200SFM_INTR_STRIDE);
  dump_d(f, "quat", quat, 4LL * g_prob.C);
  dump_d(f, "trans", trans, 3LL * g_prob.C);
  dump_d(f, "points", points, 3LL * g_prob.P);
  fclose(f);
  return B200SFM_OK;
}

int b200sfm_ba_problem_get_state(b200sfm_ba_problem* p, double* intr, double* quat, double* trans, double* points) {
  (void)p; (void)intr; (void)quat;
  for (int64_t i = 0; trans && i < 3LL * g_prob.C; ++i) trans[i] = 100.0 + (double)i;
  for (int64_t i = 0; points && i < 3LL * g_prob.P; ++i) points[i] = 200.0 + (double)i;
  return B200SFM_OK;
}

void b200sfm_ba_problem_free(b200sfm_ba_problem* p) { (void)p; }

static int observation_filter(const char* name, double thr, const double* bearings, const uint8_t* calibrated, uint8_t* keep,
                              int64_t* n) {
  FILE* f = dump_file();
  fprintf(f, "call %s\n", name);
  dump_d(f, "threshold", &thr, 1);
  dump_d(f, "bearings", bearings, 3 * g_prob.N);
  dump_u8(f, "calibrated", calibrated, g_prob.rig ? g_prob.S : g_prob.C);
  fclose(f);
  for (int64_t o = 0; o < g_prob.N; ++o) keep[o] = o % 3 != 1;
  *n = 7;
  return B200SFM_OK;
}
int b200sfm_ba_problem_filter_reprojection(b200sfm_ba_problem* p, double thr, uint8_t* keep, int64_t* n) {
  (void)p;
  return observation_filter("filter_reprojection", thr, NULL, NULL, keep, n);
}
int b200sfm_ba_problem_filter_reprojection_normalized(b200sfm_ba_problem* p, const double* bearings, double thr, uint8_t* keep,
                                                      int64_t* n) {
  (void)p;
  return observation_filter("filter_reprojection_normalized", thr, bearings, NULL, keep, n);
}
int b200sfm_ba_problem_filter_angle(b200sfm_ba_problem* p, const double* bearings, const uint8_t* calibrated, double thr,
                                    uint8_t* keep, int64_t* n) {
  (void)p;
  return observation_filter("filter_angle", thr, bearings, calibrated, keep, n);
}
int b200sfm_ba_problem_filter_triangulation_angle(b200sfm_ba_problem* p, double thr, uint8_t* keep, int64_t* n) {
  (void)p;
  FILE* f = dump_file();
  fprintf(f, "call filter_triangulation_angle\n");
  dump_d(f, "threshold", &thr, 1);
  fclose(f);
  for (int32_t t = 0; t < g_prob.P; ++t) keep[t] = t % 2 == 0;
  *n = 5;
  return B200SFM_OK;
}

int b200sfm_ba_problem_normalize(b200sfm_ba_problem* p, int32_t fixed_scale, double extent, double p0, double p1, double* scale,
                                 double* t) {
  (void)p;
  FILE* f = dump_file();
  fprintf(f, "call normalize\n");
  const double args[4] = {(double)fixed_scale, extent, p0, p1};
  dump_d(f, "args", args, 4);
  fclose(f);
  *scale = 2.0;
  t[0] = 1.0; t[1] = 2.0; t[2] = 3.0;
  return B200SFM_OK;
}

int b200sfm_undistort_features(b200sfm_ctx* ctx, int32_t K, const int32_t* intr_model, const double* intr_params, int64_t n,
                               const int32_t* feat_intr, const double* xy, double* out) {
  (void)ctx;
  FILE* f = dump_file();
  fprintf(f, "call undistort_features\n");
  dump_i(f, "intr_model", intr_model, K);
  dump_d(f, "intr", intr_params, (long long)K * B200SFM_INTR_STRIDE);
  dump_i(f, "feat_intr", feat_intr, n);
  dump_d(f, "xy", xy, 2 * n);
  fclose(f);
  for (int64_t i = 0; i < n; ++i)
    if (intr_model[feat_intr[i]] < 0 || intr_model[feat_intr[i]] > 3) return B200SFM_ERR_UNSUPPORTED;
  for (int64_t i = 0; i < n; ++i) {
    out[3 * i] = (double)i;
    out[3 * i + 1] = 0.5;
    out[3 * i + 2] = -(double)i;
  }
  return B200SFM_OK;
}
