// gravity_kernels.cuh -- device side of GravityRefiner::RefineGravity (glomap/estimators/gravity_refinement.cc:9-181)
// in frame space (FP64, sm_90a).  The host passes, per valid pair whose two images have gravity, the frame-level relative
// rotation M = R_c2^T R_rel R_c1 (rig2_from_rig1), so no rig data reaches the device:
//   1. per pair: R = Ra2^T M Ra1, R_up = AngleToRotUp(RotUpToAngle(R)), mistake = CalcAngle(R, R_up) > max_gravity_error
//      (IdentifyErrorProneGravity, .cc:144-170)
//   2. frame incidence CSR: a stable radix sort of the incidences 2 pair + side by frame gives each frame its incidences
//      in ascending order; per-frame (mistakes, total) are segment differences of a prefix sum, so no atomics.  A frame is
//      error-prone when total >= min_num_neighbors and mistakes / total >= max_outlier_ratio (.cc:172-179)
//   3. one warp per error-prone frame: observed gravities (M^T g2 for the frame of image 1, M g1 for the frame of image 2,
//      .cc:81-95; one term for a pair inside the frame), AverageGravity (math/gravity.cc:37-91), a trust-region LM on the
//      tangent space of SphereManifold<3> with residual g - g_obs under ArctanLoss(1 - cos(max_gravity_error)), and the
//      consistency check (.cc:111-123).  Every reduction is a fixed-order warp butterfly, so a call is bit-reproducible.
// Every error-prone frame is refined against the gravities as they were on entry (Jacobi; the reference updates them in
// hash-set order).  The LM restates oracle/ceres_lm.py with the closed-form 2x2 system.
#pragma once
#include <cub/cub.cuh>
#include <math_constants.h>
#include <thrust/iterator/counting_iterator.h>

#include <cfloat>

#include "../../include/b200sfm_testing.h"
#include "context.cuh"
#include "ra_kernels.cuh"

namespace b200 {

struct GravityParams {
  double max_outlier_ratio, max_gravity_error;   // degrees
  int min_num_neighbors, max_num_iterations;
  double function_tolerance, gradient_tolerance, parameter_tolerance;
  int trace_cap = 0;   // LM iterations recorded per frame when grv_refine is given a trace (test probe only)
};

// The LM trace of one error-prone frame (grv_refine's optional output; stride GRV_TRACE_HEAD + 5 trace_cap doubles):
// the AverageGravity start x0 [3], the termination code, the number of recorded iterations, then per iteration
// (cost, radius, model cost change, candidate cost, code).  Termination: -1 too few terms, 0 gradient tolerance at x0,
// 1 max iterations, 2 min radius, 3 too many invalid steps, 4 parameter tolerance, 5 function tolerance, 6 gradient
// tolerance.  Iteration code: -1 invalid step (candidate cost NaN), 0 rejected, 1 accepted, 2 stopped by the parameter
// tolerance, 3 stopped by the function tolerance.
constexpr int GRV_TRACE_HEAD = 5;

// 0: every frame with a gravity prior has a finite R_align with a non-zero gravity column; sets bit 2 of *bad otherwise
__global__ void grv_frame_check(int F, const double* __restrict__ R_align, const unsigned char* __restrict__ has_g,
                                int* __restrict__ bad) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F || !has_g[f]) return;
  const double* R = R_align + 9LL * f;
  bool ok = true;
  for (int k = 0; k < 9; ++k) ok &= isfinite(R[k]);
  ok &= (R[1] != 0.0 || R[4] != 0.0 || R[7] != 0.0);
  if (!ok) atomicOr(bad, 2);
}

// 1. per pair: range check (bit 1 of *bad), finite M (bit 4), mistake flag, and the two incidences (key = frame, F for a pair that has a
// frame without gravity: it sorts last and belongs to no frame)
// CalcAngle(R, AngleToRotUp(RotUpToAngle(R))) in degrees (.cc:150-158); up = RotUpToAngle(R), the y component of the
// rotation vector.  CalcAngle(R1, R2) (math/rigid3d.cc:22-27) is acos(clamp((tr(R1^T R2) - 1) / 2)).
__device__ __forceinline__ double grv_pair_angle(const double R[9], double& up) {
  double aa[3];
  R_to_aa(R, aa);
  up = aa[1];
  const double w[3] = {0.0, aa[1], 0.0};
  double Rup[9];
  aa_to_R(w, Rup);
  double tr = 0.0;
  for (int k = 0; k < 9; ++k) tr += R[k] * Rup[k];
  double c = (tr - 1.0) / 2.0;
  c = fmin(fmax(c, -1.0), 1.0);
  return acos(c) * 180.0 / CUDART_PI;
}

// ang_out [E] (may be null): the pair's angle in degrees, written where the mistake flag is computed
__global__ void grv_pair(long long E, int F, const int* __restrict__ frame1, const int* __restrict__ frame2,
                         const double* __restrict__ M, const double* __restrict__ R_align, const unsigned char* __restrict__ has_g,
                         double max_err_deg, unsigned char* __restrict__ mistake, unsigned* __restrict__ keys,
                         int* __restrict__ vals, int* __restrict__ bad, double* __restrict__ ang_out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int f1 = frame1[e], f2 = frame2[e];
  vals[2 * e] = (int)(2 * e);
  vals[2 * e + 1] = (int)(2 * e + 1);
  mistake[e] = 0;
  if (f1 < 0 || f1 >= F || f2 < 0 || f2 >= F) {
    atomicOr(bad, 1);
    keys[2 * e] = keys[2 * e + 1] = (unsigned)F;
    return;
  }
  if (!has_g[f1] || !has_g[f2]) {
    keys[2 * e] = keys[2 * e + 1] = (unsigned)F;
    return;
  }
  keys[2 * e] = (unsigned)f1;
  keys[2 * e + 1] = (unsigned)f2;
  double Ra1[9], Ra2[9], Me[9], T[9], R[9];
  bool finite = true;
  for (int k = 0; k < 9; ++k) {
    Ra1[k] = R_align[9LL * f1 + k];
    Ra2[k] = R_align[9LL * f2 + k];
    Me[k] = M[9 * e + k];
    finite &= isfinite(Me[k]);
  }
  if (!finite) {   // the refinement marks skipped terms with NaN, so a non-finite M is refused (bit 4)
    atomicOr(bad, 4);
    return;
  }
  mat3_mul(Me, Ra1, T);     // M Ra1
  mat3_tmul(Ra2, T, R);     // Ra2^T M Ra1
  double up;
  const double ang = grv_pair_angle(R, up);
  if (ang_out) ang_out[e] = ang;
  mistake[e] = ang > max_err_deg ? 1 : 0;
}

// frame f's incidences are [offs[f], offs[f + 1]) of the sorted keys; offs[F] = incidences of pairs with gravity
__global__ void grv_offsets(int F, long long n, const unsigned* __restrict__ sorted_keys, int* __restrict__ offs) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > F) return;
  long long lo = 0, hi = n;   // first index with key >= f
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (sorted_keys[mid] < (unsigned)f) lo = mid + 1; else hi = mid;
  }
  offs[f] = (int)lo;
}

__global__ void grv_gather_mistake(long long n, const int* __restrict__ sorted_vals, const unsigned char* __restrict__ mistake,
                                   int* __restrict__ m_sorted) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) m_sorted[i] = mistake[sorted_vals[i] >> 1];
}

// 2. per-frame counts and the error-prone flag
__global__ void grv_flag(int F, const int* __restrict__ offs, const int* __restrict__ m_scan, int min_nb, double max_ratio,
                         unsigned char* __restrict__ flag) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int b = offs[f], e = offs[f + 1];
  const int total = e - b, mistakes = m_scan[e] - m_scan[b];
  flag[f] = (total >= min_nb && (double)mistakes / (double)total >= max_ratio) ? 1 : 0;
}

// ---- SphereManifold<3> (ceres/sphere_manifold.h, internal/sphere_manifold_functions.h; UPSTREAM-UNVERIFIED) --------
// Householder vector of x: (I - beta v v^T) x = |x| e_3
__device__ __forceinline__ void grv_householder(const double x[3], double v[3], double& beta) {
  const double sigma = x[0] * x[0] + x[1] * x[1];
  v[0] = x[0]; v[1] = x[1]; v[2] = 1.0;
  beta = 0.0;
  if (sigma <= DBL_EPSILON) {
    if (x[2] < 0.0) beta = 2.0;
    return;
  }
  const double mu = sqrt(x[2] * x[2] + sigma);
  const double vp = x[2] <= 0.0 ? x[2] - mu : -sigma / (x[2] + mu);
  beta = 2.0 * vp * vp / (sigma + vp * vp);
  v[0] /= vp;
  v[1] /= vp;
}
// x [+] d = |x| H (0.5 sin(|d|/2)/(|d|/2) d, cos(|d|/2))
__device__ __forceinline__ void grv_plus(const double x[3], double d0, double d1, double out[3]) {
  const double nd = sqrt(d0 * d0 + d1 * d1);
  if (nd == 0.0) {
    out[0] = x[0]; out[1] = x[1]; out[2] = x[2];
    return;
  }
  double v[3], beta;
  grv_householder(x, v, beta);
  const double nx = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  const double h = 0.5 * nd;
  const double sbd = sin(h) / h;
  const double y[3] = {0.5 * sbd * d0, 0.5 * sbd * d1, cos(h)};
  const double vy = beta * (v[0] * y[0] + v[1] * y[1] + v[2] * y[2]);
  for (int k = 0; k < 3; ++k) out[k] = nx * (y[k] - v[k] * vy);
}
// d(x [+] d)/dd at d = 0: 0.5 |x| (I - beta v v^T)[:, 0:2], row-major [3][2]
__device__ __forceinline__ void grv_plus_jacobian(const double x[3], double P[6]) {
  double v[3], beta;
  grv_householder(x, v, beta);
  const double nx = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 2; ++c) P[2 * r + c] = 0.5 * nx * ((r == c ? 1.0 : 0.0) - beta * v[r] * v[c]);
}

// one pass over the terms at x: cost = 1/2 sum a atan2(s, a), w = sum rho'(s), rs = sum rho'(s) (x - g_obs)
// (ArctanLoss, ceres/loss_function.cc; UPSTREAM-UNVERIFIED; its corrector is sqrt(rho') since rho'' <= 0)
__device__ __forceinline__ void grv_eval(const double* __restrict__ gobs, int b, int e, int lane, const double x[3], double a,
                                         double& cost, double& w, double rs[3]) {
  double c = 0.0, ww = 0.0, r0 = 0.0, r1 = 0.0, r2 = 0.0;
  const double inv_a2 = 1.0 / (a * a);
  for (int i = b + lane; i < e; i += 32) {
    const double g0 = gobs[3LL * i];
    if (isnan(g0)) continue;
    const double d0 = x[0] - g0, d1 = x[1] - gobs[3LL * i + 1], d2 = x[2] - gobs[3LL * i + 2];
    const double s = d0 * d0 + d1 * d1 + d2 * d2;
    c += a * atan2(s, a);
    const double rho1 = fmax(DBL_MIN, 1.0 / (1.0 + s * s * inv_a2));
    ww += rho1;
    r0 += rho1 * d0; r1 += rho1 * d1; r2 += rho1 * d2;
  }
  cost = 0.5 * warp_sum(c);
  w = warp_sum(ww);
  rs[0] = warp_sum(r0); rs[1] = warp_sum(r1); rs[2] = warp_sum(r2);
}

// max |x [+] (-g) - x| (Ceres' gradient max-norm under a manifold)
__device__ __forceinline__ double grv_gmax(const double x[3], const double g[2]) {
  double p[3];
  grv_plus(x, -g[0], -g[1], p);
  return fmax(fabs(p[0] - x[0]), fmax(fabs(p[1] - x[1]), fabs(p[2] - x[2])));
}

// principal eigenvector of the symmetric 3x3 A (row-major) by cyclic Jacobi, fixed sweeps
__device__ __forceinline__ void grv_principal(double A[9], double out[3]) {
  double V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int sweep = 0; sweep < 12; ++sweep) {
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      const double apq = A[3 * p + q];
      if (apq == 0.0) continue;
      const double theta = (A[3 * q + q] - A[3 * p + p]) / (2.0 * apq);
      const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      for (int k = 0; k < 3; ++k) {   // A <- J^T A J, J = rotation in (p, q)
        const double akp = A[3 * k + p], akq = A[3 * k + q];
        A[3 * k + p] = c * akp - s * akq;
        A[3 * k + q] = s * akp + c * akq;
      }
      for (int k = 0; k < 3; ++k) {
        const double apk = A[3 * p + k], aqk = A[3 * q + k];
        A[3 * p + k] = c * apk - s * aqk;
        A[3 * q + k] = s * apk + c * aqk;
      }
      for (int k = 0; k < 3; ++k) {
        const double vkp = V[3 * k + p], vkq = V[3 * k + q];
        V[3 * k + p] = c * vkp - s * vkq;
        V[3 * k + q] = s * vkp + c * vkq;
      }
    }
  }
  int m = 0;
  if (A[4] > A[0]) m = 1;
  if (A[8] > A[4 * m]) m = 2;
  for (int k = 0; k < 3; ++k) out[k] = V[3 * k + m];
}

// 3. one warp per error-prone frame.  status: 1 = fewer than min_num_neighbors terms, 2 = accepted, 3 = rejected.
// gobs [incidences][3] is scratch at the frame's incidence range (NaN x: the second incidence of a pair inside the frame).
// trace (null in production) receives each frame's LM trace (GRV_TRACE_HEAD); lane 0 writes it, no result depends on it.
__global__ void __launch_bounds__(128) grv_refine(int nep, const int* __restrict__ ep, const int* __restrict__ offs,
                                                  const int* __restrict__ sorted_vals, const int* __restrict__ frame1,
                                                  const int* __restrict__ frame2, const double* __restrict__ M,
                                                  const double* __restrict__ R_align, GravityParams prm,
                                                  double* __restrict__ gobs, double* __restrict__ g_out,
                                                  unsigned char* __restrict__ st_out, int* __restrict__ it_out,
                                                  double* __restrict__ trace) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= nep) return;
  double* tr = (trace && lane == 0) ? trace + (long long)w * (GRV_TRACE_HEAD + 5LL * prm.trace_cap) : nullptr;
  int nrec = 0;
  auto record = [&](double c0, double c1, double c2, double c3, int code) {
    if (tr && nrec < prm.trace_cap) {
      double* r = tr + GRV_TRACE_HEAD + 5LL * nrec;
      r[0] = c0; r[1] = c1; r[2] = c2; r[3] = c3; r[4] = code;
    }
    ++nrec;
  };
  auto finish_trace = [&](int term) {
    if (tr) { tr[3] = term; tr[4] = nrec < prm.trace_cap ? nrec : prm.trace_cap; }
  };
  const int f = ep[w], b = offs[f], e = offs[f + 1];
  // observed gravities, and AverageGravity's mean outer product
  int nloc = 0;
  double A0 = 0, A1 = 0, A2 = 0, A4 = 0, A5 = 0, A8 = 0;
  for (int i = b + lane; i < e; i += 32) {
    const int id = sorted_vals[i], pr = id >> 1, side = id & 1;
    const int f1 = frame1[pr], f2 = frame2[pr];
    double* go = gobs + 3LL * i;
    if (side == 1 && f1 == f2) {   // a pair inside the frame is one term (.cc:79-95)
      go[0] = go[1] = go[2] = CUDART_NAN;
      continue;
    }
    const double* Me = M + 9LL * pr;
    const double* Ro = R_align + 9LL * (side == 0 ? f2 : f1);
    const double o0 = Ro[1], o1 = Ro[4], o2 = Ro[7];
    double g[3];
    if (side == 0)
      for (int r = 0; r < 3; ++r) g[r] = Me[r] * o0 + Me[3 + r] * o1 + Me[6 + r] * o2;   // M^T g2
    else
      for (int r = 0; r < 3; ++r) g[r] = Me[3 * r] * o0 + Me[3 * r + 1] * o1 + Me[3 * r + 2] * o2;   // M g1
    go[0] = g[0]; go[1] = g[1]; go[2] = g[2];
    ++nloc;
    A0 += g[0] * g[0]; A1 += g[0] * g[1]; A2 += g[0] * g[2];
    A4 += g[1] * g[1]; A5 += g[1] * g[2]; A8 += g[2] * g[2];
  }
  const int n = (int)warp_sum((double)nloc);
  if (n < prm.min_num_neighbors) {
    if (lane == 0) { st_out[w] = 1; it_out[w] = 0; }
    finish_trace(-1);
    return;
  }
  const double inv_n = 1.0 / (double)n;
  double A[9];
  A[0] = warp_sum(A0) * inv_n; A[1] = warp_sum(A1) * inv_n; A[2] = warp_sum(A2) * inv_n;
  A[4] = warp_sum(A4) * inv_n; A[5] = warp_sum(A5) * inv_n; A[8] = warp_sum(A8) * inv_n;
  A[3] = A[1]; A[6] = A[2]; A[7] = A[5];
  double x[3];
  grv_principal(A, x);
  int negl = 0;
  for (int i = b + lane; i < e; i += 32) {
    const double g0 = gobs[3LL * i];
    if (isnan(g0)) continue;
    negl += (g0 * x[0] + gobs[3LL * i + 1] * x[1] + gobs[3LL * i + 2] * x[2]) < 0.0;
  }
  const int neg = (int)warp_sum((double)negl);
  const double* Rf = R_align + 9LL * f;
  if (neg > n / 2 || (2 * neg == n && x[0] * Rf[1] + x[1] * Rf[4] + x[2] * Rf[7] < 0.0)) {   // sign tie: toward the prior
    x[0] = -x[0]; x[1] = -x[1]; x[2] = -x[2];
  }
  if (tr) { tr[0] = x[0]; tr[1] = x[1]; tr[2] = x[2]; }

  // ---- LM (oracle/ceres_lm.py with Ceres' defaults; the Jacobian of every term is sqrt(rho') P, P = PlusJacobian)
  const double a = 1.0 - cos(prm.max_gravity_error * CUDART_PI / 180.0);
  double cost, wsum, rs[3], P[6];
  grv_eval(gobs, b, e, lane, x, a, cost, wsum, rs);
  grv_plus_jacobian(x, P);
  double PtP[3] = {P[0] * P[0] + P[2] * P[2] + P[4] * P[4], P[0] * P[1] + P[2] * P[3] + P[4] * P[5],
                   P[1] * P[1] + P[3] * P[3] + P[5] * P[5]};
  const double sc0 = 1.0 / (1.0 + sqrt(wsum * PtP[0])), sc1 = 1.0 / (1.0 + sqrt(wsum * PtP[2]));
  double g[2] = {P[0] * rs[0] + P[2] * rs[1] + P[4] * rs[2], P[1] * rs[0] + P[3] * rs[1] + P[5] * rs[2]};
  double radius = 1e4, decrease = 2.0;
  int invalid = 0, it = 0;
  double x_norm = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
  int term = 0;
  if (grv_gmax(x, g) > prm.gradient_tolerance) {
    term = 1;
    while (true) {
      if (it >= prm.max_num_iterations) { term = 1; break; }
      if (!(radius >= 1e-32)) { term = 2; break; }
      ++it;
      // scaled normal matrix S (wsum PtP) S, LM diagonal clamp(diag, 1e-6, 1e32) / radius
      const double H00 = wsum * PtP[0] * sc0 * sc0, H01 = wsum * PtP[1] * sc0 * sc1, H11 = wsum * PtP[2] * sc1 * sc1;
      const double D0 = fmin(fmax(H00, 1e-6), 1e32) / radius, D1 = fmin(fmax(H11, 1e-6), 1e32) / radius;
      const double a00 = H00 + D0, a11 = H11 + D1;
      const double q0 = -sc0 * g[0], q1 = -sc1 * g[1];
      const double det = a00 * a11 - H01 * H01;
      const double y0 = (a11 * q0 - H01 * q1) / det, y1 = (a00 * q1 - H01 * q0) / det;
      // -(J y)^T (r + J y / 2) = y^T q - 1/2 y^T H y
      const double mcc = (y0 * q0 + y1 * q1) - 0.5 * (y0 * (H00 * y0 + H01 * y1) + y1 * (H01 * y0 + H11 * y1));
      if (!isfinite(y0) || !isfinite(y1) || mcc <= 0.0) {
        record(cost, radius, mcc, CUDART_NAN, -1);
        if (++invalid >= 5) { term = 3; break; }
        radius /= decrease;
        decrease *= 2.0;
        continue;
      }
      invalid = 0;
      double xc[3];
      grv_plus(x, y0 * sc0, y1 * sc1, xc);
      double ccost, cw, crs[3];
      grv_eval(gobs, b, e, lane, xc, a, ccost, cw, crs);
      const double sn = sqrt((xc[0] - x[0]) * (xc[0] - x[0]) + (xc[1] - x[1]) * (xc[1] - x[1]) + (xc[2] - x[2]) * (xc[2] - x[2]));
      if (sn <= prm.parameter_tolerance * (x_norm + prm.parameter_tolerance)) {
        record(cost, radius, mcc, ccost, 2);
        term = 4;
        break;
      }
      const double change = cost - ccost;
      if (fabs(change) <= prm.function_tolerance * cost) {
        record(cost, radius, mcc, ccost, 3);
        term = 5;
        break;
      }
      const double rel = change / mcc;
      record(cost, radius, mcc, ccost, rel > 1e-3 ? 1 : 0);
      if (rel > 1e-3) {
        x[0] = xc[0]; x[1] = xc[1]; x[2] = xc[2];
        cost = ccost; wsum = cw; rs[0] = crs[0]; rs[1] = crs[1]; rs[2] = crs[2];
        grv_plus_jacobian(x, P);
        PtP[0] = P[0] * P[0] + P[2] * P[2] + P[4] * P[4];
        PtP[1] = P[0] * P[1] + P[2] * P[3] + P[4] * P[5];
        PtP[2] = P[1] * P[1] + P[3] * P[3] + P[5] * P[5];
        g[0] = P[0] * rs[0] + P[2] * rs[1] + P[4] * rs[2];
        g[1] = P[1] * rs[0] + P[3] * rs[1] + P[5] * rs[2];
        x_norm = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
        const double t = 2.0 * rel - 1.0;
        radius = fmin(1e16, radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
        decrease = 2.0;
        if (grv_gmax(x, g) <= prm.gradient_tolerance) { term = 6; break; }
      } else {
        radius /= decrease;
        decrease *= 2.0;
      }
    }
  }
  finish_trace(term);
  // consistency with the neighbours (.cc:111-123)
  int outl = 0;
  for (int i = b + lane; i < e; i += 32) {
    const double g0 = gobs[3LL * i];
    if (isnan(g0)) continue;
    const double d = g0 * x[0] + gobs[3LL * i + 1] * x[1] + gobs[3LL * i + 2] * x[2];
    outl += acos(fmax(fmin(d, 1.0), -1.0)) * 180.0 / CUDART_PI > prm.max_gravity_error * 2.0;
  }
  const int outliers = (int)warp_sum((double)outl);
  if (lane == 0) {
    st_out[w] = ((double)outliers / (double)n < prm.max_outlier_ratio) ? 2 : 3;
    it_out[w] = it;
    g_out[3LL * w] = x[0]; g_out[3LL * w + 1] = x[1]; g_out[3LL * w + 2] = x[2];
  }
}

// b200sfm_test_device_helpers: one thread per input row, through the production helpers (op table in
// include/b200sfm_testing.h)
constexpr int GRV_HELPER_IN[6] = {3, 5, 3, 9, 14, 9}, GRV_HELPER_OUT[6] = {4, 3, 6, 3, 4, 2};
__global__ void grv_test_helpers(int op, long long n, const double* __restrict__ in, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int wi = op == 0 ? 3 : op == 1 ? 5 : op == 2 ? 3 : op == 3 ? 9 : op == 4 ? 14 : 9;
  const int wo = op == 0 ? 4 : op == 1 ? 3 : op == 2 ? 6 : op == 3 ? 3 : op == 4 ? 4 : 2;
  double a[14], r[6];
  for (int k = 0; k < wi; ++k) a[k] = in[i * wi + k];
  switch (op) {
    case 0: grv_householder(a, r, r[3]); break;
    case 1: grv_plus(a, a[3], a[4], r); break;
    case 2: grv_plus_jacobian(a, r); break;
    case 3: grv_principal(a, r); break;
    case 4: quat_avg_eig(a, a + 10, r); break;
    default: r[1] = grv_pair_angle(a, r[0]); break;
  }
  for (int k = 0; k < wo; ++k) out[i * wo + k] = r[k];
}

struct GravityStats {
  int error_prone = 0, rectified = 0, too_few = 0;
  long long lm_iterations = 0;
  int max_lm_iterations = 0;
  double ms_h2d = 0, ms_error_test = 0, ms_csr = 0, ms_refine = 0;
};

// Device scratch and the steps of one call; the host reads back one flag word, the error-prone count and the results of
// the error-prone frames.
struct GravityRunner {
  b200sfm_ctx* ctx;
  cudaStream_t s;
  DevBuf<unsigned char> tmp;
  struct Event {   // destroyed with the runner, also when a later event of the constructor fails
    cudaEvent_t e = nullptr;
    Event() { B200_CUDA_OK(cudaEventCreate(&e)); }
    ~Event() { cudaEventDestroy(e); }
  };
  Event evs[5];
  cudaEvent_t ev[5] = {evs[0].e, evs[1].e, evs[2].e, evs[3].e, evs[4].e};

  explicit GravityRunner(b200sfm_ctx* c) : ctx(c), s(c->stream) {}
  void ensure_tmp(size_t need) {
    if (need > tmp.n) tmp.alloc(need);
  }
  template <class T>
  T read(const T* d) {
    T h{};
    B200_CUDA_OK(cudaMemcpyAsync(&h, d, sizeof(T), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return h;
  }
  float elapsed(int i) {
    float ms = 0;
    B200_CUDA_OK(cudaEventElapsedTime(&ms, ev[i], ev[i + 1]));
    return ms;
  }

  // Returns 0, or the *bad bits: 1 = a frame index out of range, 2 = a frame with gravity and a non-finite or zero
  // gravity, 4 = a non-finite M.  g_out [F][3] and status [F] are host arrays, written only when a frame is error-prone.
  // probe (null in production; b200sfm_test_gravity) receives every stage's outputs; prm.trace_cap sizes its LM trace.
  int run(const GravityParams& prm, int F, const double* h_R_align, const unsigned char* h_has_g, long long E,
          const int* h_frame1, const int* h_frame2, const double* h_M, double* h_g_out, unsigned char* h_status,
          GravityStats& st, b200sfm_test_gravity_out* probe = nullptr) {
    DevBuf<double> R_align, M;
    DevBuf<unsigned char> has_g, mistake, flag;
    DevBuf<int> frame1, frame2, bad;
    B200_CUDA_OK(cudaEventRecord(ev[0], s));
    R_align.alloc(9LL * F); has_g.alloc(F); frame1.alloc(E); frame2.alloc(E); M.alloc(9 * E); bad.alloc(1);
    R_align.upload(h_R_align, 9LL * F, s);
    has_g.upload(h_has_g, F, s);
    frame1.upload(h_frame1, E, s);
    frame2.upload(h_frame2, E, s);
    M.upload(h_M, 9 * E, s);
    bad.zero(s);
    B200_CUDA_OK(cudaEventRecord(ev[1], s));
    // 1. error test
    const long long n = 2 * E;
    DevBuf<unsigned> keys, skeys;
    DevBuf<int> vals, svals;
    mistake.alloc(E); keys.alloc(n); skeys.alloc(n); vals.alloc(n); svals.alloc(n);
    DevBuf<double> ang;
    if (probe) ang.alloc(E);
    B200_LAUNCH(ctx, grv_frame_check, cdiv(F, 256), 256, 0, F, R_align.p, has_g.p, bad.p);
    B200_LAUNCH(ctx, grv_pair, cdiv(E, 256), 256, 0, E, F, frame1.p, frame2.p, M.p, R_align.p, has_g.p, prm.max_gravity_error,
                mistake.p, keys.p, vals.p, bad.p, probe ? ang.p : nullptr);
    B200_CUDA_OK(cudaEventRecord(ev[2], s));
    const int b = read(bad.p);
    if (b) return b;
    if (probe) {
      if (probe->mistake) mistake.download(probe->mistake, E, s);
      if (probe->angle) ang.download(probe->angle, E, s);
    }
    // 2. incidence CSR, counts, error-prone list
    int end_bit = 1;
    while (end_bit < 32 && ((unsigned long long)F >> end_bit) != 0) ++end_bit;
    DevBuf<int> offs, m_sorted, m_scan, ep, nsel;
    offs.alloc((size_t)F + 1); m_sorted.alloc(n + 1); m_scan.alloc(n + 1); flag.alloc(F); ep.alloc(F); nsel.alloc(1);
    {
      size_t a = 0, c = 0, d = 0;
      thrust::counting_iterator<int> cnt(0);
      B200_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, a, keys.p, skeys.p, vals.p, svals.p, (int)n, 0, end_bit, s));
      B200_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, c, m_sorted.p, m_scan.p, (int)(n + 1), s));
      B200_CUDA_OK(cub::DeviceSelect::Flagged(nullptr, d, cnt, flag.p, ep.p, nsel.p, F, s));
      ensure_tmp(std::max(a, std::max(c, d)));
      size_t nb = tmp.n;
      B200_CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp.p, nb, keys.p, skeys.p, vals.p, svals.p, (int)n, 0, end_bit, s));
      B200_LAUNCH(ctx, grv_offsets, cdiv(F + 1, 256), 256, 0, F, n, skeys.p, offs.p);
      B200_CUDA_OK(cudaMemsetAsync(m_sorted.p + n, 0, sizeof(int), s));
      B200_LAUNCH(ctx, grv_gather_mistake, cdiv(n, 256), 256, 0, n, svals.p, mistake.p, m_sorted.p);
      nb = tmp.n;
      B200_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp.p, nb, m_sorted.p, m_scan.p, (int)(n + 1), s));
      B200_LAUNCH(ctx, grv_flag, cdiv(F, 256), 256, 0, F, offs.p, m_scan.p, prm.min_num_neighbors, prm.max_outlier_ratio, flag.p);
      nb = tmp.n;
      B200_CUDA_OK(cub::DeviceSelect::Flagged(tmp.p, nb, cnt, flag.p, ep.p, nsel.p, F, s));
    }
    B200_CUDA_OK(cudaEventRecord(ev[3], s));
    const int nep = read(nsel.p);
    st.error_prone = nep;
    if (probe) {
      probe->n_error_prone = nep;
      if (probe->offs) offs.download(probe->offs, (size_t)F + 1, s);
      if (probe->inc) svals.download(probe->inc, n, s);
      if (probe->error_prone) flag.download(probe->error_prone, F, s);
      if (probe->ep) ep.download(probe->ep, nep, s);
      if (probe->total || probe->mistakes) {
        std::vector<int> o(F + 1), sc(n + 1);
        offs.download(o.data(), (size_t)F + 1, s);
        m_scan.download(sc.data(), n + 1, s);
        B200_CUDA_OK(cudaStreamSynchronize(s));
        for (int f = 0; f < F; ++f) {
          if (probe->total) probe->total[f] = o[f + 1] - o[f];
          if (probe->mistakes) probe->mistakes[f] = sc[o[f + 1]] - sc[o[f]];
        }
      }
      B200_CUDA_OK(cudaStreamSynchronize(s));
    }
    if (nep == 0) {
      st.ms_h2d = elapsed(0);
      st.ms_error_test = elapsed(1);
      st.ms_csr = elapsed(2);
      return 0;
    }
    // 3. refinement (gobs spans every incidence; only the error-prone frames' ranges are written)
    DevBuf<double> gobs, g_out;
    DevBuf<unsigned char> st_out;
    DevBuf<int> it_out;
    gobs.alloc(3 * n); g_out.alloc(3LL * nep); st_out.alloc(nep); it_out.alloc(nep);
    DevBuf<double> trace;
    const long long tstride = GRV_TRACE_HEAD + 5LL * prm.trace_cap;
    if (probe) {
      trace.alloc(tstride * nep);
      B200_CUDA_OK(cudaMemsetAsync(gobs.p, 0xff, sizeof(double) * 3 * n, s));   // NaN where no frame writes
    }
    B200_LAUNCH(ctx, grv_refine, cdiv(32LL * nep, 128), 128, 0, nep, ep.p, offs.p, svals.p, frame1.p, frame2.p, M.p, R_align.p,
                prm, gobs.p, g_out.p, st_out.p, it_out.p, probe ? trace.p : nullptr);
    B200_CUDA_OK(cudaEventRecord(ev[4], s));
    std::vector<int> h_ep(nep), h_it(nep);
    std::vector<double> h_g(3LL * nep);
    std::vector<unsigned char> h_st(nep);
    ep.download(h_ep.data(), nep, s);
    it_out.download(h_it.data(), nep, s);
    g_out.download(h_g.data(), 3LL * nep, s);
    st_out.download(h_st.data(), nep, s);
    if (probe) {
      if (probe->gobs) gobs.download(probe->gobs, 3 * n, s);
      if (probe->x) g_out.download(probe->x, 3LL * nep, s);
      if (probe->status) st_out.download(probe->status, nep, s);
      if (probe->iterations) it_out.download(probe->iterations, nep, s);
      if (probe->trace) trace.download(probe->trace, tstride * nep, s);
    }
    B200_CUDA_OK(cudaStreamSynchronize(s));
    for (int f = 0; f < F; ++f) h_status[f] = 0;
    for (int k = 0; k < nep; ++k) {
      const int f = h_ep[k];
      h_status[f] = h_st[k];
      if (h_st[k] == 2) {
        for (int r = 0; r < 3; ++r) h_g_out[3LL * f + r] = h_g[3LL * k + r];
        ++st.rectified;
      }
      if (h_st[k] == 1) ++st.too_few;
      st.lm_iterations += h_it[k];
      st.max_lm_iterations = std::max(st.max_lm_iterations, h_it[k]);
    }
    st.ms_h2d = elapsed(0);
    st.ms_error_test = elapsed(1);
    st.ms_csr = elapsed(2);
    st.ms_refine = elapsed(3);
    return 0;
  }
};

}  // namespace b200
