// gp_kernels.cuh -- BATA global positioning kernels (sm_90a).
//
// Replaces the arithmetic Ceres performs for glomap::GlobalPositioner
// (reference: glomap/estimators/global_positioning.cc:83,212-375,432-489 and the
// functor cost_function.h:15-41):  r = t_obs - s (X - c), Huber (optionally
// ScaledLoss 0.5), one scale per observation with lower bound 1e-5, the first
// scale constant.  Where the reference lets Ceres' Schur eliminator remove the
// scales and CHOLMOD factor the rest, here both the scale (1x1) and the point
// (3x3) are eliminated in closed form per observation / per point and the
// reduced camera system (3x3 blocks) is solved by PCG:
//   with d = X - c, w = a rho'(|r|^2), h = w d.d + Ds:
//     M_o = w s^2 (I - w d d^T / h)        (symmetric 3x3; couples dX - dc)
//     b_o = w s   (I - w d d^T / h) r
//   V_p = sum M_o, g_X = -sum b_o, U_c = sum M_o, g_c = +sum b_o, W_o = -M_o.
// Layout: M[N][6] AoS (48-B rows, tile = one contiguous TMA bulk copy),
// bw[N][4] = (b_o, w s^2), per point Vinv[P][6] gX[P][3] Dp[P], per camera
// U[C][6] gc[C][3] Sd[C][6] Minv[C][6].
#pragma once
#include "ba_kernels.cuh"
#include "common.cuh"

namespace b200 {

constexpr int kMDoubles = 6;
// per-block record summed by the linearisation: U (6) | gc (3) | sum w s^2 (1) | Schur-Jacobi term (6) | raw gradient (3)
constexpr int kOutW = 19;
constexpr int kMBytes = 48;
constexpr double kScaleLowerBound = 1e-5;   // global_positioning.cc:373

struct GPView {
  int C, P;
  long long N;
  int n_tiles, n_segs, min_views;
  long long const_obs;            // observation whose scale is held constant (-1: none)
  int scales_var;                 // optimize_scales
  const int* obs_cam;
  const int* obs_pt;
  const double* obs_dir;          // [N][3] world-rotated unit bearings
  const double* obs_off;          // [N][3] or nullptr: known-rig offset R_cw^T t_cam_from_rig (RigBATA, rig scale = 1)
  const unsigned char* obs_cal;   // [N] or nullptr: prior-focal flag of the observing CAMERA (overrides the per-frame flag)
  // unknown cam_from_rig (RigUnknownBATAPairwiseDirectionError, cost_function.h:90-136, global_positioning.cc:347-364):
  //   r = t_obs - s (X - c_frame - R_rw^T u_s),  u_s = the camera centre of sensor s in the rig frame, an unknown shared by
  //   all images of the sensor.  The S_u unknown sensors are pseudo-camera blocks C .. C + S_u - 1 of the reduced system;
  //   the current -R_rw^T u_s is folded into obs_off before every evaluation (gp_dyn_offsets).
  int n_us;                       // S_u (0: none)
  const int* obs_us;              // [N] unknown-sensor index of the observing image, -1: none
  const double* frame_rot;        // [C][9] rig_from_world rotations (row-major), constants of global positioning
  const unsigned* pt_begin;
  const int* tile_pt_begin;
  const int* camord_obs;
  const int* pt_c;
  const int* seg_cam;
  const int* seg_begin;
  const int* seg_end;
  double* M;                      // [N][6]
  double* bw;                     // [N][4]
  double* jscale_s;               // [N]
  double* Vinv;                   // [P][6]
  double* gX;                     // [P][3]
  double* Dp;                     // [P]
  double* jscale_p;               // [P]
  double* graw;                   // [N][3] raw camera-side gradient w s r, before the scale is eliminated
};

__device__ __forceinline__ double lm_damp(double diag, double js, double radius) {
  const double js2 = js * js;
  return fmin(fmax(diag * js2, 1e-6), 1e32) / (radius * js2);
}

// everything one observation contributes at the current state
struct GPObs {
  double M[6], b[3], ws2, rho0;
  // for the back-substitution: w, h (0 if scale constant), d, r.d
  double w, h, d[3], r[3], dr;
};

__device__ __forceinline__ void gp_obs(const double t[3], double s, const double c4[4], const double X[3],
                                       double huber_a, bool svar, double js_in, bool set_js, double radius,
                                       double& js_out, GPObs& o) {
  const double a = c4[3];   // loss scale: 1 (calibrated) or 0.5 (ScaledLoss, global_positioning.cc:242-247)
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    o.d[k] = X[k] - c4[k];
    o.r[k] = t[k] - s * o.d[k];
  }
  const double sq = o.r[0] * o.r[0] + o.r[1] * o.r[1] + o.r[2] * o.r[2];
  double rho0, rho1;
  huber(sq, huber_a, rho0, rho1);
  o.rho0 = a * rho0;
  const double w = a * rho1;
  o.w = w;
  const double dd = o.d[0] * o.d[0] + o.d[1] * o.d[1] + o.d[2] * o.d[2];
  o.dr = o.d[0] * o.r[0] + o.d[1] * o.r[1] + o.d[2] * o.r[2];
  o.ws2 = w * s * s;
  double k = 0.0;   // w / h
  o.h = 0.0;
  js_out = js_in;
  if (svar) {
    const double diag = w * dd;
    if (set_js) js_out = 1.0 / (1.0 + sqrt(diag));
    const double Ds = lm_damp(diag, js_out, radius);
    o.h = diag + Ds;
    k = w / o.h;
  }
  // M = w s^2 (I - k d d^T), b = w s (r - k d (d.r))
  const double ws2 = o.ws2, ws = w * s;
  o.M[0] = ws2 * (1.0 - k * o.d[0] * o.d[0]);
  o.M[1] = -ws2 * k * o.d[0] * o.d[1];
  o.M[2] = -ws2 * k * o.d[0] * o.d[2];
  o.M[3] = ws2 * (1.0 - k * o.d[1] * o.d[1]);
  o.M[4] = -ws2 * k * o.d[1] * o.d[2];
  o.M[5] = ws2 * (1.0 - k * o.d[2] * o.d[2]);
#pragma unroll
  for (int i = 0; i < 3; ++i) o.b[i] = ws * (o.r[i] - k * o.d[i] * o.dr);
}

// obs_off[o] = static known-rig offset (or 0) - R_rw^T u_s  for the observations of unknown sensors
__global__ void gp_dyn_offsets(long long N, const int* __restrict__ obs_cam, const int* __restrict__ obs_us,
                               const double* __restrict__ frame_rot, const double* __restrict__ ucen,
                               const double* __restrict__ off_static, double* __restrict__ off) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= N) return;
  double f0 = 0, f1 = 0, f2 = 0;
  if (off_static) { f0 = off_static[3 * o]; f1 = off_static[3 * o + 1]; f2 = off_static[3 * o + 2]; }
  const int su = obs_us[o];
  if (su >= 0) {
    const double* R = frame_rot + 9 * (size_t)obs_cam[o];
    const double u0 = ucen[3 * su], u1 = ucen[3 * su + 1], u2 = ucen[3 * su + 2];
    f0 -= R[0] * u0 + R[3] * u1 + R[6] * u2;   // R^T u
    f1 -= R[1] * u0 + R[4] * u1 + R[7] * u2;
    f2 -= R[2] * u0 + R[5] * u1 + R[8] * u2;
  }
  off[3 * o] = f0; off[3 * o + 1] = f1; off[3 * o + 2] = f2;
}

// Blocks of the unknown sensors (dr/du_s = s R_rw^T = (dr/dc) R_rw^T):
//   out[C + su][0..5] += R M_o R^T, [6..8] += R b_o, [9] += w s^2, [16..18] += R g_raw  (one thread per observation,
//   CTA-level sums)
__global__ void __launch_bounds__(256) gp_linearize_sensors(GPView v, double* __restrict__ out16) {
  __shared__ double scratch[32];
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int su = -1;
  double val[13] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (o < v.N) {
    su = v.obs_us[o];
    const int pt = v.obs_pt[o];
    if ((int)(v.pt_begin[pt + 1] - v.pt_begin[pt]) < v.min_views) su = -1;
    if (su >= 0) {
      const double* R = v.frame_rot + 9 * (size_t)v.obs_cam[o];
      const double* m = v.M + kMDoubles * (size_t)o;
      const double M[3][3] = {{m[0], m[1], m[2]}, {m[1], m[3], m[4]}, {m[2], m[4], m[5]}};
      double T[3][3];   // R M
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) T[r][c] = R[3 * r] * M[0][c] + R[3 * r + 1] * M[1][c] + R[3 * r + 2] * M[2][c];
      int idx = 0;
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = r; c < 3; ++c) val[idx++] = T[r][0] * R[3 * c] + T[r][1] * R[3 * c + 1] + T[r][2] * R[3 * c + 2];
      const double4 bw = *reinterpret_cast<const double4*>(v.bw + 4 * (size_t)o);
#pragma unroll
      for (int r = 0; r < 3; ++r) val[6 + r] = R[3 * r] * bw.x + R[3 * r + 1] * bw.y + R[3 * r + 2] * bw.z;
      val[9] = bw.w;
      const double* g = v.graw + 3 * (size_t)o;
#pragma unroll
      for (int r = 0; r < 3; ++r) val[10 + r] = R[3 * r] * g[0] + R[3 * r + 1] * g[1] + R[3 * r + 2] * g[2];
    }
  }
  for (int s2 = 0; s2 < v.n_us; ++s2) {
#pragma unroll
    for (int k = 0; k < 13; ++k) {
      const double t = block_sum(su == s2 ? val[k] : 0.0, scratch);
      if (threadIdx.x == 0 && t != 0.0) atomicAdd(&out16[(size_t)(v.C + s2) * kOutW + (k < 10 ? k : k + 6)], t);
    }
  }
}

// centre records [C][4] = (c, loss scale)
__global__ void gp_build_records(int C, const double* __restrict__ centers, const unsigned char* __restrict__ calibrated,
                                 double* __restrict__ cen4) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  cen4[4 * c] = centers[3 * c];
  cen4[4 * c + 1] = centers[3 * c + 1];
  cen4[4 * c + 2] = centers[3 * c + 2];
  cen4[4 * c + 3] = (calibrated == nullptr || calibrated[c]) ? 1.0 : 0.5;
}

// ---------------------------------------------------------------------------
// G1: per-observation linearisation with the scale eliminated, per-point
// blocks (damped, inverted).  scal[0] += cost, scal[1] = max of the raw gradient over the variable points and the
// projected raw gradient over the variable scales (the camera blocks add theirs in gp_finalize_cams)
// ---------------------------------------------------------------------------
struct G1Smem {
  alignas(128) double Mt[kTile * kMDoubles];
  double red[13][kTile + 1];
  double acc[13][kTilePts + 1];
  unsigned pb[kTilePts + 1];
  double X[3][kTilePts + 1];
  double scratch[32];
};

__global__ void __launch_bounds__(kTile) gp_linearize_points(GPView v, const double* __restrict__ cen4,
                                                             const double* __restrict__ points,
                                                             const double* __restrict__ scales, double huber_a,
                                                             double radius, int set_js, int points_var,
                                                             double* __restrict__ scal) {
  extern __shared__ __align__(128) unsigned char smem_raw[];   // dynamic shared memory starts 128-B aligned (no static __shared__ in these kernels)
  G1Smem& sm = *reinterpret_cast<G1Smem*>(smem_raw);
  const int tile = blockIdx.x;
  const int p0 = v.tile_pt_begin[tile], p1 = v.tile_pt_begin[tile + 1];
  const unsigned o0 = v.pt_begin[p0], o1 = v.pt_begin[p1];
  const int n = (int)(o1 - o0);
  const int tid = threadIdx.x;
  const int npts = p1 - p0;
  if (tid < npts) {
    sm.pb[tid] = v.pt_begin[p0 + tid];
    if (tid == npts - 1) sm.pb[npts] = o1;
#pragma unroll
    for (int k = 0; k < 3; ++k) sm.X[k][tid] = points[3 * (size_t)(p0 + tid) + k];
#pragma unroll
    for (int k = 0; k < 13; ++k) sm.acc[k][tid] = 0.0;
  }
  __syncthreads();
  double cost = 0.0, gmax = 0.0;
  for (int c0 = 0; c0 < n; c0 += kTile) {
    const int nc = min(kTile, n - c0);
    GPObs o;
    bool use = false;
    if (tid < nc) {
      const size_t oi = (size_t)o0 + c0 + tid;
      const int cam = v.obs_cam[oi];
      const int pl = v.obs_pt[oi] - p0;
      use = (int)(sm.pb[pl + 1] - sm.pb[pl]) >= v.min_views;
      if (use) {
        const double t[3] = {v.obs_dir[3 * oi], v.obs_dir[3 * oi + 1], v.obs_dir[3 * oi + 2]};
        const double s = scales[oi];
        const double2 ca = *reinterpret_cast<const double2*>(cen4 + 4 * (size_t)cam);
        const double2 cb = *reinterpret_cast<const double2*>(cen4 + 4 * (size_t)cam + 2);
        const double c4[4] = {ca.x, ca.y, cb.x, v.obs_cal ? (v.obs_cal[oi] ? 1.0 : 0.5) : cb.y};
        double X[3] = {sm.X[0][pl], sm.X[1][pl], sm.X[2][pl]};
        if (v.obs_off) {   // d = X - c_frame + t_rig: fold the constant offset into the point
          X[0] += v.obs_off[3 * oi]; X[1] += v.obs_off[3 * oi + 1]; X[2] += v.obs_off[3 * oi + 2];
        }
        const bool svar = v.scales_var && (long long)oi != v.const_obs;
        double js = set_js ? 0.0 : v.jscale_s[oi];
        gp_obs(t, s, c4, X, huber_a, svar, js, set_js != 0, radius, js, o);
        if (set_js) v.jscale_s[oi] = js;
        cost += 0.5 * o.rho0;
        double4* bwp = reinterpret_cast<double4*>(v.bw + 4 * oi);
        *bwp = make_double4(o.b[0], o.b[1], o.b[2], o.ws2);
        // raw gradient (Ceres' g = J^T r of the unreduced program): w s r for the centre, -w s r for the point and
        // -w d.r for the scale, whose bound the norm projects on: |Project(s - g_s) - s|
        const double ws = o.w * s;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          o.r[k] *= ws;
          v.graw[3 * oi + k] = o.r[k];
        }
        if (svar) gmax = fmax(gmax, fabs(fmax(s + o.w * o.dr, kScaleLowerBound) - s));
      }
    }
    if (!use) {
#pragma unroll
      for (int k = 0; k < 6; ++k) o.M[k] = 0.0;
      o.b[0] = o.b[1] = o.b[2] = 0.0;
      o.r[0] = o.r[1] = o.r[2] = 0.0;
      o.ws2 = 0.0;
      if (tid < nc) {
        const size_t oi = (size_t)o0 + c0 + tid;
        *reinterpret_cast<double4*>(v.bw + 4 * oi) = make_double4(0, 0, 0, 0);
        v.graw[3 * oi] = v.graw[3 * oi + 1] = v.graw[3 * oi + 2] = 0.0;
      }
    }
    double* mrow = sm.Mt + tid * kMDoubles;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      mrow[k] = o.M[k];
      sm.red[k][tid] = o.M[k];
    }
    sm.red[6][tid] = -o.b[0];
    sm.red[7][tid] = -o.b[1];
    sm.red[8][tid] = -o.b[2];
    sm.red[9][tid] = o.ws2;
    sm.red[10][tid] = -o.r[0];
    sm.red[11][tid] = -o.r[1];
    sm.red[12][tid] = -o.r[2];
    fence_proxy_async_smem();
    __syncthreads();
    if (tid == 0) {
      tma_store_1d(v.M + ((size_t)o0 + c0) * kMDoubles, sm.Mt, (uint32_t)nc * kMBytes);
      tma_store_commit();
    }
    for (int item = tid; item < npts * 13; item += kTile) {
      const int j = item / 13, k = item - 13 * j;
      const int lo = max((int)sm.pb[j] - (int)(o0 + c0), 0), hi = min((int)sm.pb[j + 1] - (int)(o0 + c0), nc);
      double a = 0.0;
      for (int i = lo; i < hi; ++i) a += sm.red[k][i];
      sm.acc[k][j] += a;
    }
    if (tid == 0) tma_store_wait_read();
    __syncthreads();
  }
  if (tid < npts) {
    const size_t p = (size_t)(p0 + tid);
    const bool pvalid = (int)(sm.pb[tid + 1] - sm.pb[tid]) >= v.min_views;
    double vi[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0}, Dp = 0.0;
    if (pvalid && points_var) {
      double V6[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) V6[k] = sm.acc[k][tid];
      const double diag = sm.acc[9][tid];
      double js = set_js ? 1.0 / (1.0 + sqrt(diag)) : v.jscale_p[p];
      if (set_js) v.jscale_p[p] = js;
      Dp = lm_damp(diag, js, radius);
      V6[0] += Dp;
      V6[3] += Dp;
      V6[5] += Dp;
      sym3_inverse(V6, vi);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        g[k] = sm.acc[6 + k][tid];
        gmax = fmax(gmax, fabs(sm.acc[10 + k][tid]));
      }
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) v.Vinv[6 * p + k] = vi[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) v.gX[3 * p + k] = g[k];
    v.Dp[p] = Dp;
  }
  cost = block_sum(cost, sm.scratch);
  if (tid == 0 && cost != 0.0) atomicAdd(&scal[0], cost);
  gmax = block_max(gmax, sm.scratch);
  if (tid == 0 && gmax > 0.0) atomic_max_nonneg(&scal[1], gmax);
}

// ---------------------------------------------------------------------------
// G2: camera blocks (camera order, one warp per segment):
//   out[cam][0..5] += U = sum M_o, [6..8] += gc = sum b_o, [9] += sum w s^2,
//   [10..15] += Sd = sum M_o Vinv_p M_o, [16..18] += the raw gradient sum w s r
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) gp_linearize_cams(GPView v, int with_schur, double* __restrict__ out16) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= v.n_segs) return;
  const int cam = v.seg_cam[warp];
  const int b = v.seg_begin[warp], e = v.seg_end[warp];
  double acc[kOutW];
#pragma unroll
  for (int k = 0; k < kOutW; ++k) acc[k] = 0.0;
  for (int i = b + lane; i < e; i += 32) {
    const size_t o = (size_t)v.camord_obs[i];
    const double2* mp = reinterpret_cast<const double2*>(v.M + o * kMDoubles);
    const double2 m0 = mp[0], m1 = mp[1], m2 = mp[2];
    const double M[6] = {m0.x, m0.y, m1.x, m1.y, m2.x, m2.y};
    const double4 bw = *reinterpret_cast<const double4*>(v.bw + 4 * o);
#pragma unroll
    for (int k = 0; k < 6; ++k) acc[k] += M[k];
    acc[6] += bw.x;
    acc[7] += bw.y;
    acc[8] += bw.z;
    acc[9] += bw.w;
    acc[16] += v.graw[3 * o];
    acc[17] += v.graw[3 * o + 1];
    acc[18] += v.graw[3 * o + 2];
    if (with_schur) {
      const int pt = v.pt_c[i];
      const double2* vp = reinterpret_cast<const double2*>(v.Vinv + (size_t)pt * 6);
      const double2 v0 = vp[0], v1 = vp[1], v2 = vp[2];
      const double vi[6] = {v0.x, v0.y, v1.x, v1.y, v2.x, v2.y};
      // T = M Vinv (3x3, rows), S = T M (symmetric)
      const double Mr[3][3] = {{M[0], M[1], M[2]}, {M[1], M[3], M[4]}, {M[2], M[4], M[5]}};
      double T[3][3];
#pragma unroll
      for (int r = 0; r < 3; ++r) sym3_mul(vi, Mr[r], T[r]);   // (Vinv M_r) == row r of M Vinv (both symmetric)
      int idx = 10;
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = r; c < 3; ++c) acc[idx++] += T[r][0] * Mr[c][0] + T[r][1] * Mr[c][1] + T[r][2] * Mr[c][2];
    }
  }
#pragma unroll
  for (int k = 0; k < kOutW; ++k) {
    const double s = warp_sum(acc[k]);
    if (lane == k && s != 0.0) atomicAdd(&out16[(size_t)cam * kOutW + k], s);
  }
}

// Unpack out16 -> U, gc, Dc, Minv; constant / unobserved cameras become identity.
__global__ void gp_finalize_cams(int C, const double* __restrict__ out16, const unsigned char* __restrict__ cam_const,
                                 double* __restrict__ jscale_c, int set_js, double radius, int with_schur,
                                 double* __restrict__ U, double* __restrict__ gc, double* __restrict__ Dc,
                                 double* __restrict__ Minv, double* __restrict__ scal,
                                 const double* __restrict__ gslots, int nslots) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  double gmax = 0.0;
  if (blockIdx.x == 0 && threadIdx.x < nslots) gmax = gslots[threadIdx.x];   // per-rank max|g_X| slots (sum all-reduced)
  if (c < C) {
    const double* o = out16 + (size_t)c * kOutW;
    const double diag = o[9];
    const bool fixed = (cam_const && cam_const[c]) || !(diag > 0.0);
    double u[6], g[3], D = 0.0;
    if (fixed) {
      u[0] = u[3] = u[5] = 1.0;
      u[1] = u[2] = u[4] = 0.0;
      g[0] = g[1] = g[2] = 0.0;
      if (set_js) jscale_c[c] = -1.0;
    } else {
#pragma unroll
      for (int k = 0; k < 6; ++k) u[k] = o[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        g[k] = o[6 + k];
        gmax = fmax(gmax, fabs(o[16 + k]));
      }
      double js = set_js ? 1.0 / (1.0 + sqrt(diag)) : jscale_c[c];
      if (set_js) jscale_c[c] = js;
      D = lm_damp(diag, js, radius);
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) U[(size_t)c * 6 + k] = u[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      gc[(size_t)c * 3 + k] = g[k];
      Dc[(size_t)c * 3 + k] = D;
    }
    double m[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) m[k] = u[k] - ((with_schur && !fixed) ? o[10 + k] : 0.0);
    m[0] += D;
    m[3] += D;
    m[5] += D;
    double inv[6];
    spd_inverse_packed<3>(m, inv);
#pragma unroll
    for (int k = 0; k < 6; ++k) Minv[(size_t)c * 6 + k] = inv[k];
  }
  gmax = warp_max(gmax);
  if ((threadIdx.x & 31) == 0 && gmax > 0.0) atomic_max_nonneg(&scal[1], gmax);
}

// ---------------------------------------------------------------------------
// G3: implicit Schur pass (W_o = -M_o).
//   MODE 0: y_cam -= W_o Vinv sum W^T x            (mat-vec, x = xc[C][3])
//   MODE 1: y_cam -= W_o Vinv gX                   (rhs)
//   MODE 2: back-substitution: dX = -Vinv (gX + W^T dc), ds per observation;
//           writes dX[P][3], ds[N]; bscal[0] += g.delta (points+scales part),
//           bscal[1] += delta^T D delta (points + scales)
// ---------------------------------------------------------------------------
// the centre displacement an observation sees: x_c, plus R_rw^T x_u when its sensor's cam_from_rig centre is an unknown
__device__ __forceinline__ void gp_x_eff(const GPView& v, const double* __restrict__ x, size_t oi, double xe[3]) {
  const int cam = v.obs_cam[oi];
  xe[0] = x[3 * (size_t)cam];
  xe[1] = x[3 * (size_t)cam + 1];
  xe[2] = x[3 * (size_t)cam + 2];
  if (v.n_us > 0) {
    const int su = v.obs_us[oi];
    if (su >= 0) {
      const double* R = v.frame_rot + 9 * (size_t)cam;
      const double* xu = x + 3 * (size_t)(v.C + su);
      xe[0] += R[0] * xu[0] + R[3] * xu[1] + R[6] * xu[2];
      xe[1] += R[1] * xu[0] + R[4] * xu[1] + R[7] * xu[2];
      xe[2] += R[2] * xu[0] + R[5] * xu[1] + R[8] * xu[2];
    }
  }
}

struct G3Smem {
  alignas(128) double Mt[kTile * kMDoubles];
  double t[3][kTile + 1];
  double z[3][kTilePts + 1];
  unsigned pb[kTilePts + 1];
  double scratch[32];
  alignas(8) uint64_t mbar;
};

template <int MODE, bool SPEC = false>   // SPEC: launched ahead of the PCG read-back, tests the stopping flag
__global__ void __launch_bounds__(kTile) gp_schur_pass(GPView v, const double* __restrict__ x, double* __restrict__ y,
                                                       const double* __restrict__ cen4,
                                                       const double* __restrict__ points,
                                                       const double* __restrict__ scales, double huber_a, double radius,
                                                       double* __restrict__ dX, double* __restrict__ ds,
                                                       double* __restrict__ bscal,
                                                       const PcgCtl* __restrict__ ctl = nullptr) {
  extern __shared__ __align__(128) unsigned char smem_raw[];   // dynamic shared memory starts 128-B aligned (no static __shared__ in these kernels)
  // the PCG stopping rule may have fired (queued-ahead iterations are no-ops).  The flag is LOADED here but only
  // tested after the first TMA wait: a dependent global load in front of the tile pipeline would make this latency-bound
  // kernel wait a full memory round trip before its first bulk copy, and a CTA must not exit with a bulk copy in flight.
  const int pcg_done = (SPEC && ctl) ? ctl->done : 0;
  G3Smem& sm = *reinterpret_cast<G3Smem*>(smem_raw);
  const int tile = blockIdx.x;
  const int p0 = v.tile_pt_begin[tile], p1 = v.tile_pt_begin[tile + 1];
  const unsigned o0 = v.pt_begin[p0], o1 = v.pt_begin[p1];
  const int n = (int)(o1 - o0);
  const int tid = threadIdx.x;
  const int npts = p1 - p0;
  const int nchunks = (n + kTile - 1) / kTile;
  if (tid == 0) {
    mbar_init(&sm.mbar, 1);
    fence_mbar_init();
  }
  if (tid < npts) {
    sm.pb[tid] = v.pt_begin[p0 + tid];
    if (tid == npts - 1) sm.pb[npts] = o1;
    sm.z[0][tid] = sm.z[1][tid] = sm.z[2][tid] = 0.0;
  }
  __syncthreads();
  uint32_t phase = 0;
  if (MODE != 1) {
    for (int ch = 0; ch < nchunks; ++ch) {
      const int c0 = ch * kTile;
      const int nc = min(kTile, n - c0);
      if (tid == 0) {
        mbar_arrive_expect_tx(&sm.mbar, (uint32_t)nc * kMBytes);
        tma_load_1d(sm.Mt, v.M + ((size_t)o0 + c0) * kMDoubles, (uint32_t)nc * kMBytes, &sm.mbar);
      }
      double xc[3] = {0, 0, 0};
      const bool active = tid < nc;
      if (active) gp_x_eff(v, x, (size_t)o0 + c0 + tid, xc);
      mbar_wait(&sm.mbar, phase);
      phase ^= 1;
      if (SPEC && pcg_done) return;   // uniform; nothing has been written and no copy is in flight
      double t0 = 0, t1 = 0, t2 = 0;
      if (active) {
        const double2* mr = reinterpret_cast<const double2*>(sm.Mt + tid * kMDoubles);
        const double2 m0 = mr[0], m1 = mr[1], m2 = mr[2];
        // W^T x = -M x
        t0 = -(m0.x * xc[0] + m0.y * xc[1] + m1.x * xc[2]);
        t1 = -(m0.y * xc[0] + m1.y * xc[1] + m2.x * xc[2]);
        t2 = -(m1.x * xc[0] + m2.x * xc[1] + m2.y * xc[2]);
      }
      sm.t[0][tid] = t0;
      sm.t[1][tid] = t1;
      sm.t[2][tid] = t2;
      __syncthreads();
      for (int item = tid; item < npts * 3; item += kTile) {
        const int j = item / 3, k = item - 3 * j;
        const int lo = max((int)sm.pb[j] - (int)(o0 + c0), 0), hi = min((int)sm.pb[j + 1] - (int)(o0 + c0), nc);
        double a = 0.0;
        for (int i = lo; i < hi; ++i) a += sm.t[k][i];
        sm.z[k][j] += a;
      }
      __syncthreads();
    }
  }
  double b0 = 0, b1 = 0;
  if (tid < npts) {
    const size_t p = (size_t)(p0 + tid);
    const bool pvalid = (int)(sm.pb[tid + 1] - sm.pb[tid]) >= v.min_views;
    double z[3] = {0, 0, 0};
    if (pvalid) {
      double s[3] = {sm.z[0][tid], sm.z[1][tid], sm.z[2][tid]};
      double g[3] = {0, 0, 0};
      if (MODE != 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          g[k] = v.gX[3 * p + k];
          s[k] += g[k];
        }
      }
      double vi[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) vi[k] = v.Vinv[6 * p + k];
      sym3_mul(vi, s, z);
      if (MODE == 2) {
        const double Dp = v.Dp[p];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double d = -z[k];
          dX[3 * p + k] = d;
          b1 += Dp * d * d;
        }
      }
    } else if (MODE == 2) {
      dX[3 * p] = dX[3 * p + 1] = dX[3 * p + 2] = 0.0;
    }
    // MODE 2 keeps dX (= -z) in smem for the per-observation scale steps
    const double sgn = (MODE == 2) ? -1.0 : 1.0;
    sm.z[0][tid] = sgn * z[0];
    sm.z[1][tid] = sgn * z[1];
    sm.z[2][tid] = sgn * z[2];
  }
  __syncthreads();
  if (MODE == 2) {
    // per observation: q = dX - dc;  ds = (w d.r - w s d.q) / h;  raw-gradient . delta
    for (int c0 = 0; c0 < n; c0 += kTile) {
      const int nc = min(kTile, n - c0);
      if (tid < nc) {
        const size_t oi = (size_t)o0 + c0 + tid;
        const int pl = v.obs_pt[oi] - p0;
        double dsv = 0.0;
        if ((int)(sm.pb[pl + 1] - sm.pb[pl]) >= v.min_views) {
          const int cam = v.obs_cam[oi];
          const double t[3] = {v.obs_dir[3 * oi], v.obs_dir[3 * oi + 1], v.obs_dir[3 * oi + 2]};
          const double s = scales[oi];
          const double2 ca = *reinterpret_cast<const double2*>(cen4 + 4 * (size_t)cam);
          const double2 cb = *reinterpret_cast<const double2*>(cen4 + 4 * (size_t)cam + 2);
          const double c4[4] = {ca.x, ca.y, cb.x, v.obs_cal ? (v.obs_cal[oi] ? 1.0 : 0.5) : cb.y};
          const size_t p = (size_t)(p0 + pl);
          double X[3] = {points[3 * p], points[3 * p + 1], points[3 * p + 2]};
          if (v.obs_off) {
            X[0] += v.obs_off[3 * oi]; X[1] += v.obs_off[3 * oi + 1]; X[2] += v.obs_off[3 * oi + 2];
          }
          const bool svar = v.scales_var && (long long)oi != v.const_obs;
          GPObs o;
          double js = v.jscale_s[oi];
          gp_obs(t, s, c4, X, huber_a, svar, js, false, radius, js, o);
          double xe[3];
          gp_x_eff(v, x, oi, xe);
          const double q[3] = {sm.z[0][pl] - xe[0], sm.z[1][pl] - xe[1], sm.z[2][pl] - xe[2]};
          const double dq = o.d[0] * q[0] + o.d[1] * q[1] + o.d[2] * q[2];
          const double rq = o.r[0] * q[0] + o.r[1] * q[1] + o.r[2] * q[2];
          if (svar) {
            dsv = (o.w * o.dr - o.w * s * dq) / o.h;
            const double Ds = o.h - o.w * (o.d[0] * o.d[0] + o.d[1] * o.d[1] + o.d[2] * o.d[2]);
            b1 += Ds * dsv * dsv;
          }
          // g.delta over (c, X, s) of this observation: w (-s r.q - (d.r) ds)
          b0 += o.w * (-s * rq - o.dr * dsv);
        }
        ds[oi] = dsv;
      }
    }
    b0 = block_sum(b0, sm.scratch);
    b1 = block_sum(b1, sm.scratch);
    if (tid == 0) {
      atomicAdd(&bscal[0], b0);
      atomicAdd(&bscal[1], b1);
    }
    return;
  }
  // phase B: y_cam -= W_o z_p = + M_o z_p
  for (int ch = 0; ch < nchunks; ++ch) {
    const int c0 = ch * kTile;
    const int nc = min(kTile, n - c0);
    const bool reload = (MODE == 1) || (nchunks > 1);
    if (reload) {
      __syncthreads();
      if (tid == 0) {
        mbar_arrive_expect_tx(&sm.mbar, (uint32_t)nc * kMBytes);
        tma_load_1d(sm.Mt, v.M + ((size_t)o0 + c0) * kMDoubles, (uint32_t)nc * kMBytes, &sm.mbar);
      }
      mbar_wait(&sm.mbar, phase);
      phase ^= 1;
    }
    if (tid < nc) {
      const size_t oi = (size_t)o0 + c0 + tid;
      const int cam = v.obs_cam[oi];
      const int pl = v.obs_pt[oi] - p0;
      double z0 = sm.z[0][pl], z1 = sm.z[1][pl], z2 = sm.z[2][pl];
      const bool pvalid2 = (int)(sm.pb[pl + 1] - sm.pb[pl]) >= v.min_views;
      if (v.n_us > 0 && MODE == 0 && pvalid2) {
        // unknown sensors: the direct term is applied here too (y = M (x_eff + z): pcg_apply_diag then adds D x only),
        // because x_eff = x_c + R^T x_u differs per observation
        double xe[3];
        gp_x_eff(v, x, oi, xe);
        z0 += xe[0]; z1 += xe[1]; z2 += xe[2];
      }
      if (z0 != 0.0 || z1 != 0.0 || z2 != 0.0) {
        const double2* mr = reinterpret_cast<const double2*>(sm.Mt + tid * kMDoubles);
        const double2 m0 = mr[0], m1 = mr[1], m2 = mr[2];
        double* yc = y + 3 * (size_t)cam;
        const double a0 = m0.x * z0 + m0.y * z1 + m1.x * z2;
        const double a1 = m0.y * z0 + m1.y * z1 + m2.x * z2;
        const double a2 = m1.x * z0 + m2.x * z1 + m2.y * z2;
        atomicAdd(&yc[0], a0);
        atomicAdd(&yc[1], a1);
        atomicAdd(&yc[2], a2);
        const int su = v.n_us > 0 ? v.obs_us[oi] : -1;
        if (su >= 0) {   // y_u += R (M z)
          const double* R = v.frame_rot + 9 * (size_t)cam;
          double* yu = y + 3 * (size_t)(v.C + su);
          atomicAdd(&yu[0], R[0] * a0 + R[1] * a1 + R[2] * a2);
          atomicAdd(&yu[1], R[3] * a0 + R[4] * a1 + R[5] * a2);
          atomicAdd(&yu[2], R[6] * a0 + R[7] * a1 + R[8] * a2);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------
// candidate = Project(x + alpha delta)  (Ceres ParameterBlock::Plus projects on
// the bounds); norms for the parameter tolerance.
//   nscal[0] += |x_new - x|^2, nscal[1] += |x|^2  over variable blocks (Ceres' reduced program: constant points and
//   scales, and centres with jscale_c < 0, are not in it)
// ---------------------------------------------------------------------------
__global__ void gp_apply_step(GPView v, double alpha, const double* __restrict__ centers,
                              const double* __restrict__ points, const double* __restrict__ scales,
                              const double* __restrict__ dc, const double* __restrict__ dX,
                              const double* __restrict__ ds, const double* __restrict__ jscale_c, int count_cams,
                              int points_var, double* __restrict__ centers_new, double* __restrict__ points_new,
                              double* __restrict__ scales_new, double* __restrict__ nscal,
                              const double* __restrict__ ucen, double* __restrict__ ucen_new) {
  __shared__ double scratch[32];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double a0 = 0, a1 = 0;
  if (i < v.N) {
    const double s = scales[i];
    const int pt = v.obs_pt[i];
    const bool valid = (int)(v.pt_begin[pt + 1] - v.pt_begin[pt]) >= v.min_views;
    const bool svar = valid && v.scales_var && i != v.const_obs;
    const double sn = svar ? fmax(s + alpha * ds[i], kScaleLowerBound) : s;
    scales_new[i] = sn;
    if (svar) {
      a0 += (sn - s) * (sn - s);
      a1 += s * s;
    }
  }
  if (i < (long long)v.P * 3) {
    const double xo = points[i];
    const double d = alpha * dX[i];
    points_new[i] = xo + d;
    const int pt = (int)(i / 3);
    if (points_var && (int)(v.pt_begin[pt + 1] - v.pt_begin[pt]) >= v.min_views) {
      a0 += d * d;
      a1 += xo * xo;
    }
  }
  if (i < (long long)v.C * 3) {
    const bool var = jscale_c[i / 3] >= 0.0;
    const double co = centers[i];
    const double d = var ? alpha * dc[i] : 0.0;
    centers_new[i] = co + d;
    if (var && count_cams) {
      a0 += d * d;
      a1 += co * co;
    }
  }
  if (i < (long long)v.n_us * 3) {   // unknown cam_from_rig centres: blocks C .. C + S_u - 1
    const bool var = jscale_c[v.C + i / 3] >= 0.0;
    const double uo = ucen[i];
    const double d = var ? alpha * dc[(long long)v.C * 3 + i] : 0.0;
    ucen_new[i] = uo + d;
    if (var && count_cams) {
      a0 += d * d;
      a1 += uo * uo;
    }
  }
  a0 = block_sum(a0, scratch);
  a1 = block_sum(a1, scratch);
  if (threadIdx.x == 0) {
    if (a0 != 0.0) atomicAdd(&nscal[0], a0);
    if (a1 != 0.0) atomicAdd(&nscal[1], a1);
  }
}

// cost only: scal[0] += 1/2 sum a rho
__global__ void __launch_bounds__(256) gp_cost(GPView v, const double* __restrict__ cen4,
                                               const double* __restrict__ points, const double* __restrict__ scales,
                                               double huber_a, double* __restrict__ scal) {
  __shared__ double scratch[32];
  double cost = 0.0;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < v.N; o += (long long)gridDim.x * blockDim.x) {
    const int pt = v.obs_pt[o];
    if ((int)(v.pt_begin[pt + 1] - v.pt_begin[pt]) < v.min_views) continue;
    const int cam = v.obs_cam[o];
    const double s = scales[o];
    const double2 ca = *reinterpret_cast<const double2*>(cen4 + 4 * (size_t)cam);
    const double2 cb = *reinterpret_cast<const double2*>(cen4 + 4 * (size_t)cam + 2);
    double f0 = 0.0, f1 = 0.0, f2 = 0.0;
    if (v.obs_off) { f0 = v.obs_off[3 * o]; f1 = v.obs_off[3 * o + 1]; f2 = v.obs_off[3 * o + 2]; }
    const double r0 = v.obs_dir[3 * o] - s * (points[3 * (size_t)pt] + f0 - ca.x);
    const double r1 = v.obs_dir[3 * o + 1] - s * (points[3 * (size_t)pt + 1] + f1 - ca.y);
    const double r2 = v.obs_dir[3 * o + 2] - s * (points[3 * (size_t)pt + 2] + f2 - cb.x);
    double rho0, rho1;
    huber(r0 * r0 + r1 * r1 + r2 * r2, huber_a, rho0, rho1);
    cost += 0.5 * (v.obs_cal ? (v.obs_cal[o] ? 1.0 : 0.5) : cb.y) * rho0;
  }
  cost = block_sum(cost, scratch);
  if (threadIdx.x == 0 && cost != 0.0) atomicAdd(&scal[0], cost);
}

// camera part of the step scalars: cscal[0] += gc_raw.dc ... here the raw camera
// gradient is sum w s r = what G2 accumulates BEFORE scale elimination; with the
// scales eliminated exactly the identity g.delta = sum_o w(-s r.q - d.r ds) of
// gp_schur_pass<2> already contains the camera terms, so only the damping and
// the PCG residual terms remain:  cscal[0] += dc.resid, cscal[1] += sum Dc dc^2
__global__ void gp_cam_scalars(int C, const double* __restrict__ dc, const double* __restrict__ resid,
                               const double* __restrict__ Dc, const double* __restrict__ jscale_c,
                               double* __restrict__ cscal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double a0 = 0, a1 = 0;
  if (i < C * 3 && jscale_c[i / 3] >= 0.0) {
    const double d = dc[i];
    a0 = resid[i] * d;
    a1 = Dc[i] * d * d;
  }
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  if ((threadIdx.x & 31) == 0) {
    if (a0 != 0.0) atomicAdd(&cscal[0], a0);
    if (a1 != 0.0) atomicAdd(&cscal[1], a1);
  }
}

}  // namespace b200
