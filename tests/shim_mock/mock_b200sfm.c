/* TEST DOUBLE (tests only, never shipped): records what the C++ estimator shim passes across the C ABI so that
 * the shim's host-side flattening (sorted-id order, rig sensor tables, per-observation rig terms, frame folding of
 * the view graph) can be checked on a box without a GPU.  Every call appends "name n v0 v1 ..." lines to $MOCK_DUMP
 * and leaves the state untouched (stats.usable = 1). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "b200sfm.h"
#include "mock_dump.h"

struct b200sfm_ctx { int dummy; };
struct b200sfm_ba_problem { b200sfm_ctx* ctx; };
/* structure of the last BA problem (for the filter stubs) */
static long long g_ba_n = 0, g_ba_p = 0;
static long long* g_ba_ptb = NULL;
static void remember_ba(int32_t P, int64_t N, const int64_t* ptb) {
  g_ba_n = N; g_ba_p = P;
  free(g_ba_ptb);
  g_ba_ptb = (long long*)malloc(sizeof(long long) * (size_t)(P + 1));
  for (int32_t i = 0; i <= P; ++i) g_ba_ptb[i] = ptb[i];
}
/* filter stub: keeps everything, or drops every m-th observation when $MOCK_DROP_EVERY = m > 0 */
static long long stub_filter(const char* name, double thr, uint8_t* keep) {
  FILE* f = mock_dump_open();
  fprintf(f, "call %s\nthreshold 1 %.17g\nnobs 1 %lld\n", name, thr, g_ba_n);
  fclose(f);
  const char* e = getenv("MOCK_DROP_EVERY");
  const long long m = e ? atoll(e) : 0;
  long long changed = 0;
  for (long long p = 0; p < g_ba_p; ++p) {
    int any = 0;
    for (long long o = g_ba_ptb[p]; o < g_ba_ptb[p + 1]; ++o) {
      keep[o] = (m > 0 && o % m == 0) ? 0 : 1;
      any |= !keep[o];
    }
    changed += any;
  }
  return changed;
}
struct b200sfm_gp_problem { b200sfm_ctx* ctx; };
static struct b200sfm_ctx g_ctx;
static long long g_gp_n = 0;
static int g_ba_S = 0;   /* sensors of the last rig problem */

int b200sfm_version(void) { return B200SFM_VERSION; }
int b200sfm_create(int device, b200sfm_ctx** o) { (void)device; *o = &g_ctx; return B200SFM_OK; }
void b200sfm_destroy(b200sfm_ctx* c) { (void)c; }
const char* b200sfm_last_error(const b200sfm_ctx* c) { (void)c; return "mock"; }

void b200sfm_ba_default_opts(b200sfm_ba_opts* o) { memset(o, 0, sizeof(*o)); o->min_num_view_per_track = 3; }
void b200sfm_gp_default_opts(b200sfm_gp_opts* o) { memset(o, 0, sizeof(*o)); o->min_num_view_per_track = 3; }
void b200sfm_ra_default_opts(b200sfm_ra_opts* o) { memset(o, 0, sizeof(*o)); }

int b200sfm_ba_solve(b200sfm_ctx* ctx, const b200sfm_ba_opts* o, int32_t C, int32_t P, int64_t N, int32_t K,
                     const int64_t* ptb, const int32_t* obs_cam, const double* obs_xy, const int32_t* cam_intr,
                     const int32_t* intr_model, double* intr, double* quat, double* trans, const uint8_t* mask, double* points,
                     b200sfm_lm_stats* st) {
  (void)ctx;
  FILE* f = mock_dump_open();
  fprintf(f, "call ba_solve\n");
  int32_t dims[4] = {C, P, (int32_t)N, K};
  dump_i32(f, "dims", dims, 4);
  int32_t flags[3] = {o->optimize_rotations, o->optimize_intrinsics, o->optimize_rig_poses};
  dump_i32(f, "flags", flags, 3);
  dump_i64(f, "pt_obs_begin", ptb, P + 1); dump_i32(f, "obs_cam", obs_cam, N); dump_f64(f, "obs_xy", obs_xy, 2 * N);
  dump_i32(f, "cam_intr", cam_intr, C); dump_i32(f, "intr_model", intr_model, K); dump_f64(f, "intr", intr, (long long)K * B200SFM_INTR_STRIDE);
  dump_f64(f, "quat", quat, 4ll * C); dump_f64(f, "trans", trans, 3ll * C); dump_u8(f, "mask", mask, C); dump_f64(f, "points", points, 3ll * P);
  fclose(f);
  memset(st, 0, sizeof(*st)); st->usable = 1;
  return B200SFM_OK;
}
int b200sfm_ba_problem_create_rig(b200sfm_ctx* ctx, int32_t F, int32_t P, int64_t N, int32_t K, int32_t S, const int64_t* ptb,
                                  const int32_t* obs_frame, const uint16_t* obs_sensor, const double* obs_xy,
                                  const double* sq, const double* stv, const int32_t* sintr, const int32_t* intr_model,
                                  const uint8_t* mask, int32_t minv, b200sfm_ba_problem** o) {
  FILE* f = mock_dump_open();
  fprintf(f, "call ba_problem_create_rig\n");
  int32_t dims[6] = {F, P, (int32_t)N, K, S, minv};
  dump_i32(f, "dims", dims, 6);
  dump_i64(f, "pt_obs_begin", ptb, P + 1); dump_i32(f, "obs_frame", obs_frame, N); dump_u16(f, "obs_sensor", obs_sensor, N);
  dump_f64(f, "obs_xy", obs_xy, 2 * N); dump_f64(f, "sensor_quat", sq, 4ll * S); dump_f64(f, "sensor_trans", stv, 3ll * S);
  dump_i32(f, "sensor_intr", sintr, S); dump_i32(f, "intr_model", intr_model, K); dump_u8(f, "mask", mask, F);
  fclose(f);
  remember_ba(P, N, ptb);
  g_ba_S = S;
  static struct b200sfm_ba_problem p; p.ctx = ctx; *o = &p;
  return B200SFM_OK;
}
int b200sfm_ba_problem_set_state(b200sfm_ba_problem* p, const double* intr, const double* q, const double* t, const double* pts) {
  (void)p; (void)intr; (void)q; (void)t; (void)pts;
  dump_call("ba_problem_set_state");
  return B200SFM_OK;
}
int b200sfm_ba_problem_set_sensor_variable(b200sfm_ba_problem* p, const uint8_t* v) {
  (void)p;
  FILE* f = mock_dump_open();
  fprintf(f, "call ba_problem_set_sensor_variable\n");
  dump_u8(f, "sensor_variable", v, g_ba_S);
  fclose(f);
  return B200SFM_OK;
}
/* a recognisable "optimised" cam_from_rig for every sensor: rotation 90 deg about z, translation (7 + s, 8, 9) */
int b200sfm_ba_problem_get_sensor_poses(b200sfm_ba_problem* p, double* q, double* t) {
  (void)p;
  for (int s = 0; s < g_ba_S; ++s) {
    if (q) { q[4 * s] = 0; q[4 * s + 1] = 0; q[4 * s + 2] = 0.70710678118654757; q[4 * s + 3] = 0.70710678118654757; }
    if (t) { t[3 * s] = 7.0 + s; t[3 * s + 1] = 8; t[3 * s + 2] = 9; }
  }
  return B200SFM_OK;
}
int b200sfm_ba_problem_set_images(b200sfm_ba_problem* p, int32_t I, const int32_t* image_frame, const int32_t* image_sensor) {
  (void)p;
  FILE* f = mock_dump_open();
  fprintf(f, "call ba_problem_set_images\n");
  dump_i32(f, "image_frame", image_frame, I); dump_i32(f, "image_sensor", image_sensor, I);
  fclose(f);
  return B200SFM_OK;
}
int b200sfm_ba_problem_normalize(b200sfm_ba_problem* p, int32_t fixed_scale, double extent, double p0, double p1, double* sc,
                                 double* t) {
  (void)p; (void)fixed_scale; (void)extent; (void)p0; (void)p1;
  dump_call("ba_problem_normalize");
  if (sc) *sc = 1.0;
  if (t) t[0] = t[1] = t[2] = 0.0;
  return B200SFM_OK;
}
int b200sfm_ba_problem_undistort(b200sfm_ba_problem* p, double* out) {
  (void)p; (void)out;
  dump_call("ba_problem_undistort");
  return B200SFM_OK;
}
int b200sfm_ba_problem_get_state(b200sfm_ba_problem* p, double* intr, double* q, double* t, double* pts) {
  (void)p; (void)intr; (void)q; (void)t; (void)pts;
  return B200SFM_OK;
}
int b200sfm_ba_problem_solve(b200sfm_ba_problem* p, const b200sfm_ba_opts* o, b200sfm_lm_stats* st) {
  (void)p; (void)o; dump_call("ba_problem_solve"); memset(st, 0, sizeof(*st)); st->usable = 1; return B200SFM_OK;
}
void b200sfm_ba_problem_free(b200sfm_ba_problem* p) { (void)p; }

int b200sfm_gp_solve(b200sfm_ctx* ctx, const b200sfm_gp_opts* o, int32_t C, int32_t P, int64_t N, const int64_t* ptb,
                     const int32_t* obs_cam, const double* obs_dir, const uint8_t* cal, const uint8_t* mask, double* cen,
                     double* pts, double* sc, b200sfm_lm_stats* st) {
  (void)ctx; (void)o; (void)mask; (void)cen; (void)pts; (void)sc;
  FILE* f = mock_dump_open();
  fprintf(f, "call gp_solve\n");
  dump_i64(f, "pt_obs_begin", ptb, P + 1); dump_i32(f, "obs_cam", obs_cam, N); dump_f64(f, "obs_dir", obs_dir, 3 * N); dump_u8(f, "calibrated", cal, C);
  fclose(f);
  memset(st, 0, sizeof(*st)); st->usable = 1;
  return B200SFM_OK;
}
int b200sfm_gp_problem_create(b200sfm_ctx* ctx, int32_t C, int32_t P, int64_t N, const int64_t* ptb, const int32_t* obs_cam,
                              const double* obs_dir, const uint8_t* cal, const uint8_t* mask, int32_t minv, b200sfm_gp_problem** o) {
  (void)mask; (void)minv;
  FILE* f = mock_dump_open();
  fprintf(f, "call gp_problem_create\n");
  int32_t dims[3] = {C, P, (int32_t)N};
  dump_i32(f, "dims", dims, 3);
  dump_i64(f, "pt_obs_begin", ptb, P + 1); dump_i32(f, "obs_cam", obs_cam, N); dump_f64(f, "obs_dir", obs_dir, 3 * N); dump_u8(f, "calibrated", cal, C);
  fclose(f);
  static struct b200sfm_gp_problem p; p.ctx = ctx; *o = &p;
  g_gp_n = N;
  return B200SFM_OK;
}
int b200sfm_gp_problem_set_rig_terms(b200sfm_gp_problem* p, const double* off, const uint8_t* cal) {
  (void)p;
  FILE* f = mock_dump_open();
  fprintf(f, "call gp_problem_set_rig_terms\n");
  dump_f64(f, "obs_offset", off, 3 * g_gp_n); dump_u8(f, "obs_calibrated", cal, g_gp_n);
  fclose(f);
  return B200SFM_OK;
}
static int g_gp_su = 0;
int b200sfm_gp_problem_set_rig_unknown(b200sfm_gp_problem* p, int32_t su, const int32_t* os, const double* fr, const double* c) {
  (void)p; (void)fr;
  FILE* f = mock_dump_open();
  fprintf(f, "call gp_problem_set_rig_unknown\n");
  int32_t dims[1] = {su};
  dump_i32(f, "dims", dims, 1);
  dump_i32(f, "obs_unknown_sensor", os, g_gp_n);
  dump_f64(f, "centers", c, 3ll * su);
  fclose(f);
  g_gp_su = su;
  return B200SFM_OK;
}
/* a recognisable "estimated" centre for every unknown sensor: (1 + s, 2, 3) */
int b200sfm_gp_problem_get_rig_unknown(b200sfm_gp_problem* p, double* c) {
  (void)p;
  for (int s = 0; s < g_gp_su; ++s) { c[3 * s] = 1.0 + s; c[3 * s + 1] = 2; c[3 * s + 2] = 3; }
  return B200SFM_OK;
}
int b200sfm_gp_problem_set_state(b200sfm_gp_problem* p, const double* c, const double* x, const double* s) { (void)p; (void)c; (void)x; (void)s; return B200SFM_OK; }
int b200sfm_gp_problem_get_state(b200sfm_gp_problem* p, double* c, double* x, double* s) { (void)p; (void)c; (void)x; (void)s; return B200SFM_OK; }
int b200sfm_gp_problem_solve(b200sfm_gp_problem* p, const b200sfm_gp_opts* o, b200sfm_lm_stats* st) {
  (void)p; (void)o; dump_call("gp_problem_solve"); memset(st, 0, sizeof(*st)); st->usable = 1; return B200SFM_OK;
}
void b200sfm_gp_problem_free(b200sfm_gp_problem* p) { (void)p; }

int b200sfm_ra_solve(b200sfm_ctx* ctx, const b200sfm_ra_opts* o, int32_t n, int64_t E, const int32_t* ei, const int32_t* ej,
                     const double* R, const double* w, int32_t fixed, double* theta, b200sfm_ra_stats* st) {
  (void)ctx; (void)o; (void)fixed;
  FILE* f = mock_dump_open();
  fprintf(f, "call ra_solve\n");
  int32_t dims[2] = {n, (int32_t)E};
  dump_i32(f, "dims", dims, 2);
  dump_i32(f, "ei", ei, E); dump_i32(f, "ej", ej, E); dump_f64(f, "R_rel", R, 9 * E); dump_f64(f, "weight", w, E); dump_f64(f, "theta", theta, 3ll * n);
  fclose(f);
  memset(st, 0, sizeof(*st)); st->usable = 1;
  return B200SFM_OK;
}

/* ---- the rest of the ABI (stubs so that the Python host classes can be exercised without a GPU) ---- */
int b200sfm_create_dist(int device, int rank, int world, const void* id, b200sfm_ctx** o) { (void)device; (void)rank; (void)world; (void)id; *o = &g_ctx; return B200SFM_OK; }
int b200sfm_nccl_unique_id(void* id) { memset(id, 0, B200SFM_NCCL_ID_BYTES); return B200SFM_OK; }
int b200sfm_rank(const b200sfm_ctx* c) { (void)c; return 0; }
int b200sfm_world_size(const b200sfm_ctx* c) { (void)c; return 1; }
void* b200sfm_cuda_stream(const b200sfm_ctx* c) { (void)c; return NULL; }
int64_t b200sfm_kernel_launches(const b200sfm_ctx* c) { (void)c; return 0; }
int b200sfm_ba_problem_create(b200sfm_ctx* ctx, int32_t C, int32_t P, int64_t N, int32_t K, const int64_t* ptb,
                              const int32_t* obs_cam, const double* obs_xy, const int32_t* cam_intr, const int32_t* intr_model,
                              const uint8_t* mask, int32_t minv, b200sfm_ba_problem** o) {
  (void)obs_cam; (void)obs_xy; (void)cam_intr; (void)intr_model; (void)mask;
  FILE* f = mock_dump_open();
  fprintf(f, "call ba_problem_create\n");
  int32_t dims[5] = {C, P, (int32_t)N, K, minv};
  dump_i32(f, "dims", dims, 5);
  fclose(f);
  remember_ba(P, N, ptb);
  static struct b200sfm_ba_problem p; p.ctx = ctx; *o = &p;
  return B200SFM_OK;
}
int b200sfm_ba_problem_save_state(b200sfm_ba_problem* p) { (void)p; return B200SFM_OK; }
int b200sfm_ba_problem_restore_state(b200sfm_ba_problem* p) { (void)p; return B200SFM_OK; }
int b200sfm_ba_problem_cost(b200sfm_ba_problem* p, const b200sfm_ba_opts* o, double* c) { (void)p; (void)o; *c = 0.0; return B200SFM_OK; }
int b200sfm_ba_problem_filter_reprojection(b200sfm_ba_problem* p, double thr, uint8_t* keep, int64_t* n) {
  (void)p; const long long c = stub_filter("filter_reprojection", thr, keep); if (n) *n = c; return B200SFM_OK;
}
int b200sfm_ba_problem_filter_reprojection_normalized(b200sfm_ba_problem* p, const double* b, double thr, uint8_t* keep, int64_t* n) {
  (void)p; (void)b; const long long c = stub_filter("filter_reprojection_normalized", thr, keep); if (n) *n = c; return B200SFM_OK;
}
int b200sfm_ba_problem_filter_angle(b200sfm_ba_problem* p, const double* b, const uint8_t* cal, double thr, uint8_t* keep, int64_t* n) {
  (void)p; (void)b; (void)cal; const long long c = stub_filter("filter_angle", thr, keep); if (n) *n = c; return B200SFM_OK;
}
int b200sfm_ba_problem_filter_triangulation_angle(b200sfm_ba_problem* p, double thr, uint8_t* keep_track, int64_t* n) {
  (void)p;
  FILE* f = mock_dump_open();
  fprintf(f, "call filter_triangulation_angle\nthreshold 1 %.17g\n", thr);
  fclose(f);
  for (long long i = 0; i < g_ba_p; ++i) keep_track[i] = 1;
  if (n) *n = 0;
  return B200SFM_OK;
}
int b200sfm_gp_problem_save_state(b200sfm_gp_problem* p) { (void)p; return B200SFM_OK; }
int b200sfm_gp_problem_restore_state(b200sfm_gp_problem* p) { (void)p; return B200SFM_OK; }
int b200sfm_ra_solve_rig(b200sfm_ctx* ctx, const b200sfm_ra_opts* o, int32_t nf, int32_t nc, int64_t ne, const int32_t* ei,
                         const int32_t* ej, const int32_t* eci, const int32_t* ecj, const double* R, const double* w,
                         const int32_t* cfb, const int32_t* cf, int32_t fixed, double* theta, b200sfm_ra_stats* st) {
  (void)ctx; (void)o;
  FILE* f = mock_dump_open();
  fprintf(f, "call ra_solve_rig\n");
  int32_t dims[4] = {nf, nc, (int32_t)ne, fixed};
  dump_i32(f, "dims", dims, 4);
  dump_i32(f, "ei", ei, ne); dump_i32(f, "ej", ej, ne); dump_i32(f, "eci", eci, ne); dump_i32(f, "ecj", ecj, ne);
  dump_f64(f, "R_rel", R, 9 * ne); dump_f64(f, "w", w, ne);
  dump_i32(f, "cam_frames_begin", cfb, nc + 1); dump_i32(f, "cam_frames", cf, cfb ? cfb[nc] : 0);
  dump_f64(f, "theta", theta, 3ll * (nf + nc));
  fclose(f);
  /* a recognisable result for the camera nodes: rotation 0.3 rad about z */
  for (int c = 0; c < nc; ++c) { theta[3 * (nf + c)] = 0; theta[3 * (nf + c) + 1] = 0; theta[3 * (nf + c) + 2] = 0.3; }
  if (st) { memset(st, 0, sizeof(*st)); st->usable = 1; }
  return B200SFM_OK;
}
int b200sfm_ra_solve_gravity(b200sfm_ctx* ctx, const b200sfm_ra_opts* o, int32_t n, int64_t E, const int32_t* ei, const int32_t* ej,
                             const double* R, const double* w, const uint8_t* hg, int32_t fixed, double* theta, b200sfm_ra_stats* st) {
  (void)ctx; (void)o; (void)w;
  FILE* f = mock_dump_open();
  fprintf(f, "call ra_solve_gravity\n");
  int32_t dims[3] = {n, (int32_t)E, fixed};
  dump_i32(f, "dims", dims, 3);
  dump_i32(f, "ei", ei, E); dump_i32(f, "ej", ej, E); dump_f64(f, "R_rel", R, 9 * E); dump_u8(f, "has_gravity", hg, n); dump_f64(f, "theta", theta, 3ll * n);
  fclose(f);
  memset(st, 0, sizeof(*st)); st->usable = 1;
  return B200SFM_OK;
}

/* track establishment: not used by the host-logic tests; present so that the library exports the whole ABI */
int b200sfm_tracks_establish(b200sfm_ctx* ctx, int64_t m, const uint64_t* g1, const uint64_t* g2, const double* xy1, const double* xy2,
                             double thr, b200sfm_tracks** out, int64_t* nt, int64_t* no, int64_t* nd) {
  (void)ctx; (void)m; (void)g1; (void)g2; (void)xy1; (void)xy2; (void)thr;
  dump_call("tracks_establish");
  if (out) *out = NULL;
  if (nt) *nt = 0;
  if (no) *no = 0;
  if (nd) *nd = 0;
  return B200SFM_OK;
}
int b200sfm_tracks_get(b200sfm_tracks* t, uint64_t* ids, int64_t* begin, uint32_t* im, uint32_t* ft) {
  (void)t; (void)ids; (void)im; (void)ft;
  if (begin) begin[0] = 0;
  return B200SFM_OK;
}
void b200sfm_tracks_free(b200sfm_tracks* t) { (void)t; }
