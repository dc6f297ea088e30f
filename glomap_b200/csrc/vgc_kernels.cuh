// vgc_kernels.cuh -- device kernels of the view-graph calibrator: one focal length per camera refined from the
// fundamental matrices of the image pairs with Fetzer's focal-length residuals.  Reference path replaced:
// glomap/estimators/view_graph_calibration.cc:11-185 (ViewGraphCalibrator::Solve and its helpers) and the cost functions
// FetzerFocalLengthCost / FetzerFocalLengthSameCameraCost (glomap/estimators/cost_function.h:138-310); restated on the CPU
// in oracle/vgc_oracle.py.
//
// Per pair e (cameras i = cam1[e], j = cam2[e]) the setup keeps the eight constants d_01, d_12 (64 B) of the SVD of
// G = K1^T F K0.  The normal matrix J^T J of the K focal unknowns has one off-diagonal weight per pair with i != j; it
// stays implicit.  Camera rows are gathered over a CSR of pair incidences sorted by (camera, pair id).  A camera's row is
// split into segments of at most kVgcChunk incidences: one warp sums a segment, a second kernel sums the segments of a
// camera in their order.  No atomics touch a floating-point value, so every result is bit-reproducible, and a single
// camera shared by millions of pairs is spread over thousands of warps.
#pragma once
#include "common.cuh"
#include "context.cuh"
#include "pcg.cuh"

namespace b200 {

constexpr int kVgcChunk = 256;      // incidences per segment (8 per lane)
constexpr int kVgcThreads = 256;    // per-pair kernels: one partial per CTA of this size
constexpr double kVgcLowerBound = 1e-3;   // SetParameterLowerBound(focal, 0, 1e-3) (view_graph_calibration.cc:112)

struct VGCView {
  long long E;
  int K;
  const int* ci;              // [E] camera of image 1
  const int* cj;              // [E] camera of image 2
  const double* d;            // [E][8] d_01, d_12
  const unsigned char* var;   // [K] 1: variable focal (has a block and no prior)
};

// ---------------------------------------------------------------------------
// setup: G = K1^T F K0, one-sided Jacobi SVD, Fetzer constants
// ---------------------------------------------------------------------------
constexpr int kVgcSweeps = 8;   // fixed: a 3x3 one-sided Jacobi converges quadratically, 8 sweeps reach the rounding floor

__device__ __forceinline__ void fetzer_d(const double ai[3], const double bi[3], const double aj[3], const double bj[3], int u,
                                         int v, double* d) {
  d[0] = ai[u] * aj[v] - ai[v] * aj[u];
  d[1] = ai[u] * bj[v] - ai[v] * bj[u];
  d[2] = bi[u] * aj[v] - bi[v] * aj[u];
  d[3] = bi[u] * bj[v] - bi[v] * bj[u];
}

__global__ void __launch_bounds__(kVgcThreads) vgc_setup(long long E, const double* __restrict__ F,
                                                         const double* __restrict__ pp, const int* __restrict__ ci,
                                                         const int* __restrict__ cj, double* __restrict__ d_out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  double f[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) f[k] = F[9 * e + k];
  const double c0x = pp[2 * (size_t)ci[e]], c0y = pp[2 * (size_t)ci[e] + 1];
  const double c1x = pp[2 * (size_t)cj[e]], c1y = pp[2 * (size_t)cj[e] + 1];
  // F K0 (K0 = I with (c0x, c0y) in its last column), then K1^T (F K0)
  double a[3][3];   // a[r][c] = G(r, c), the columns are orthogonalised in place
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double m0 = f[3 * r], m1 = f[3 * r + 1];
    const double m2 = f[3 * r] * c0x + f[3 * r + 1] * c0y + f[3 * r + 2];
    a[r][0] = m0; a[r][1] = m1; a[r][2] = m2;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) a[2][c] = c1x * a[0][c] + c1y * a[1][c] + a[2][c];
  double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < kVgcSweeps; ++sweep) {
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
      double al = 0, be = 0, ga = 0;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        al += a[r][p] * a[r][p];
        be += a[r][q] * a[r][q];
        ga += a[r][p] * a[r][q];
      }
      if (ga == 0.0) continue;
      const double zeta = (be - al) / (2.0 * ga);
      const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const double x = a[r][p], y = a[r][q];
        a[r][p] = c * x - s * y;
        a[r][q] = s * x + c * y;
        const double vx = v[r][p], vy = v[r][q];
        v[r][p] = c * vx - s * vy;
        v[r][q] = s * vx + c * vy;
      }
    }
  }
  // singular values = column norms; the two largest (descending, as JacobiSVD orders them) with their U and V columns
  double sv[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) sv[c] = sqrt(a[0][c] * a[0][c] + a[1][c] * a[1][c] + a[2][c] * a[2][c]);
  int i0 = 0, i1 = 1, i2 = 2, tmp;
  if (sv[i1] > sv[i0]) { tmp = i0; i0 = i1; i1 = tmp; }
  if (sv[i2] > sv[i0]) { tmp = i0; i0 = i2; i2 = tmp; }
  if (sv[i2] > sv[i1]) { tmp = i1; i1 = i2; i2 = tmp; }
  const double s0 = sv[i0], s1 = sv[i1];
  double u0[3], u1[3], v0[3], v1[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    u0[r] = a[r][i0] / s0; u1[r] = a[r][i1] / s1;
    v0[r] = v[r][i0]; v1[r] = v[r][i1];
  }
  const double ai[3] = {s0 * s0 * (v0[0] * v0[0] + v0[1] * v0[1]), s0 * s1 * (v0[0] * v1[0] + v0[1] * v1[1]),
                        s1 * s1 * (v1[0] * v1[0] + v1[1] * v1[1])};
  const double aj[3] = {u1[0] * u1[0] + u1[1] * u1[1], -(u0[0] * u1[0] + u0[1] * u1[1]), u0[0] * u0[0] + u0[1] * u0[1]};
  const double bi[3] = {s0 * s0 * v0[2] * v0[2], s0 * s1 * v0[2] * v1[2], s1 * s1 * v1[2] * v1[2]};
  const double bj[3] = {u1[2] * u1[2], -(u0[2] * u1[2]), u0[2] * u0[2]};
  double dd[8];
  fetzer_d(ai, bi, aj, bj, 1, 0, dd);       // d_01
  fetzer_d(ai, bi, aj, bj, 2, 1, dd + 4);   // d_12
#pragma unroll
  for (int k = 0; k < 8; ++k) d_out[8 * e + k] = dd[k];
}

// ---------------------------------------------------------------------------
// residuals (cost_function.h:211-229) and their analytic derivatives
// ---------------------------------------------------------------------------
// r[2] at (fi, fj); dri[2] = dr/dfi, drj[2] = dr/dfj.  An exact zero denominator is replaced by 1e-6 without a derivative
// (a Jet constant in the reference).
__device__ __forceinline__ void vgc_residual(const double* __restrict__ d, double fi, double fj, double r[2], double dri[2],
                                             double drj[2]) {
  const double d0 = d[0], d1 = d[1], d2 = d[2], d3 = d[3], e0 = d[4], e1 = d[5], e2 = d[6], e3 = d[7];
  double di = fj * fj * d0 + d1;
  double dj = fi * fi * e0 + e2;
  const double nzi = di == 0.0 ? 0.0 : 1.0, nzj = dj == 0.0 ? 0.0 : 1.0;
  di = di == 0.0 ? 1e-6 : di;
  dj = dj == 0.0 ? 1e-6 : dj;
  const double K0 = -(fj * fj * d2 + d3) / di;
  const double K1 = -(fi * fi * e1 + e3) / dj;
  const double fi2 = fi * fi, fj2 = fj * fj;
  r[0] = (fi2 - K0) / fi2;
  r[1] = (fj2 - K1) / fj2;
  dri[0] = 2.0 * K0 / (fi2 * fi);
  drj[0] = 2.0 * fj * (d2 + K0 * d0 * nzi) / (di * fi2);
  drj[1] = 2.0 * K1 / (fj2 * fj);
  dri[1] = 2.0 * fi * (e1 + K1 * e0 * nzj) / (dj * fj2);
}

// CauchyLoss(a), b = a^2, c = 1 / b: rho = b log(1 + s c), rho' = max(DBL_MIN, 1 / (1 + s c))  (ceres loss_function.cc)
__device__ __forceinline__ void vgc_cauchy(double s, double b, double c, double& rho, double& rho1) {
  const double sum = 1.0 + s * c;
  const double inv = 1.0 / sum;
  rho = b * log(sum);
  rho1 = fmax(2.2250738585072014e-308, inv);
}

// corrected residual and Jacobian columns of pair e at focal x (rho'' < 0: both scaled by sqrt(rho'), corrector.cc).
// Columns of constant cameras are zero; a same-camera pair has its derivative (the sum of both partials) in Ji.
struct VgcPairLin {
  double r[2], Ji[2], Jj[2], rho;
  int i, j;
};
__device__ __forceinline__ VgcPairLin vgc_pair_lin(const VGCView& v, long long e, const double* __restrict__ x, double b,
                                                   double c) {
  VgcPairLin o;
  o.i = v.ci[e];
  o.j = v.cj[e];
  const double fi = x[o.i], fj = x[o.j];
  double dri[2], drj[2];
  vgc_residual(v.d + 8 * e, fi, fj, o.r, dri, drj);
  double rho1;
  vgc_cauchy(o.r[0] * o.r[0] + o.r[1] * o.r[1], b, c, o.rho, rho1);
  const double sq = sqrt(rho1);
  const bool same = o.i == o.j;
  const double vi = v.var[o.i] ? 1.0 : 0.0, vj = (v.var[o.j] && !same) ? 1.0 : 0.0;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    o.Ji[k] = vi * sq * (same ? dri[k] + drj[k] : dri[k]);
    o.Jj[k] = vj * sq * drj[k];
    o.r[k] *= sq;
  }
  return o;
}

// per pair: cost partial (per CTA), and the pair's contributions to the two cameras' J^T J diagonal and gradient
// (jd[e] = {A_i, A_j, g_i, g_j}, unscaled) and its off-diagonal weight c_e = J_i . J_j
__global__ void __launch_bounds__(kVgcThreads) vgc_linearize(VGCView v, const double* __restrict__ x, double b, double c,
                                                             double4* __restrict__ jd, double* __restrict__ off,
                                                             double* __restrict__ part_cost) {
  __shared__ double scratch[32];
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double cost = 0.0;
  if (e < v.E) {
    const VgcPairLin o = vgc_pair_lin(v, e, x, b, c);
    cost = 0.5 * o.rho;
    jd[e] = make_double4(o.Ji[0] * o.Ji[0] + o.Ji[1] * o.Ji[1], o.Jj[0] * o.Jj[0] + o.Jj[1] * o.Jj[1],
                         o.Ji[0] * o.r[0] + o.Ji[1] * o.r[1], o.Jj[0] * o.r[0] + o.Jj[1] * o.r[1]);
    off[e] = o.Ji[0] * o.Jj[0] + o.Ji[1] * o.Jj[1];
  }
  write_partial(cost, part_cost, scratch);
}

// per pair: robust cost partial at x (candidates and line-search trials)
__global__ void __launch_bounds__(kVgcThreads) vgc_cost(VGCView v, const double* __restrict__ x, double b, double c,
                                                        double* __restrict__ part_cost) {
  __shared__ double scratch[32];
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double cost = 0.0;
  if (e < v.E) {
    double r[2], dri[2], drj[2], rho, rho1;
    vgc_residual(v.d + 8 * e, x[v.ci[e]], x[v.cj[e]], r, dri, drj);
    vgc_cauchy(r[0] * r[0] + r[1] * r[1], b, c, rho, rho1);
    cost = 0.5 * rho;
  }
  write_partial(cost, part_cost, scratch);
}

// per pair: model cost change -(J dx) . (r + J dx / 2) of the step dx (unscaled), partial per CTA
__global__ void __launch_bounds__(kVgcThreads) vgc_model(VGCView v, const double* __restrict__ x, const double* __restrict__ dx,
                                                         double b, double c, double* __restrict__ part) {
  __shared__ double scratch[32];
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double m = 0.0;
  if (e < v.E) {
    const VgcPairLin o = vgc_pair_lin(v, e, x, b, c);
    const double di = dx[o.i], dj = o.i == o.j ? 0.0 : dx[o.j];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const double jd = o.Ji[k] * di + o.Jj[k] * dj;
      m -= jd * (o.r[k] + 0.5 * jd);
    }
  }
  write_partial(m, part, scratch);
}

// per pair: unlossed residuals at x and the validity test |r|^2 > thres^2 (view_graph_calibration.cc:150-185)
__global__ void __launch_bounds__(kVgcThreads) vgc_filter(VGCView v, const double* __restrict__ x, double thres2,
                                                          double* __restrict__ res, unsigned char* __restrict__ valid) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= v.E) return;
  double r[2], dri[2], drj[2];
  vgc_residual(v.d + 8 * e, x[v.ci[e]], x[v.cj[e]], r, dri, drj);
  res[2 * e] = r[0];
  res[2 * e + 1] = r[1];
  valid[e] = (r[0] * r[0] + r[1] * r[1] > thres2) ? 0 : 1;
}

// ---------------------------------------------------------------------------
// incidence CSR (built once per call)
// ---------------------------------------------------------------------------
// keys: camera of each incidence of a variable camera, K (sorts behind) otherwise; vals: e | side << 31
__global__ void vgc_inc_keys(VGCView v, int* __restrict__ cnt, int* __restrict__ keys, unsigned* __restrict__ vals) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= v.E) return;
  const int i = v.ci[e], j = v.cj[e];
  const bool vi = v.var[i], vj = v.var[j] && j != i;
  if (vi) atomicAdd(&cnt[i], 1);
  if (vj) atomicAdd(&cnt[j], 1);
  keys[2 * e] = vi ? i : v.K;
  keys[2 * e + 1] = vj ? j : v.K;
  vals[2 * e] = (unsigned)e;
  vals[2 * e + 1] = (unsigned)e | 0x80000000u;
}

// the other camera of each incidence, -1 when it carries no off-diagonal term (same camera or constant other camera)
__global__ void vgc_inc_other(int n_inc, VGCView v, const unsigned* __restrict__ val, int* __restrict__ other) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_inc) return;
  const unsigned w = val[s];
  const unsigned e = w & 0x7fffffffu;
  const int i = v.ci[e], j = v.cj[e];
  const int o = (w >> 31) ? i : j;
  other[s] = (i == j || !v.var[o]) ? -1 : o;
}

// segments: camera k owns segments [seg_off[k], seg_off[k + 1]), each of at most kVgcChunk incidences
__global__ void vgc_seg_counts(int K, const int* __restrict__ inc_begin, int* __restrict__ seg_count) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < K) seg_count[k] = (inc_begin[k + 1] - inc_begin[k] + kVgcChunk - 1) / kVgcChunk;
}
__global__ void vgc_fill_segs(int n_seg, int K, const int* __restrict__ seg_off, const int* __restrict__ inc_begin,
                              int* __restrict__ seg_begin, int* __restrict__ seg_end) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_seg) return;
  int lo = 0, hi = K;   // camera k with seg_off[k] <= s < seg_off[k + 1]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (seg_off[mid] <= s) lo = mid;
    else hi = mid;
  }
  const int b = inc_begin[lo] + (s - seg_off[lo]) * kVgcChunk;
  seg_begin[s] = b;
  seg_end[s] = min(b + kVgcChunk, inc_begin[lo + 1]);
}

// ---------------------------------------------------------------------------
// per-camera sums over the segments
// ---------------------------------------------------------------------------
// warp per segment: its incidences' diagonal and gradient contributions -> seg_part[s] = {A, g}
__global__ void __launch_bounds__(128) vgc_seg_sums(int n_seg, const int* __restrict__ seg_begin, const int* __restrict__ seg_end,
                                                    const unsigned* __restrict__ inc_val, const double4* __restrict__ jd,
                                                    double2* __restrict__ seg_part) {
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (s >= n_seg) return;
  double A = 0.0, g = 0.0;
  for (int t = seg_begin[s] + lane; t < seg_end[s]; t += 32) {
    const unsigned w = inc_val[t];
    const double4 q = jd[w & 0x7fffffffu];
    if (w >> 31) { A += q.y; g += q.w; }
    else { A += q.x; g += q.z; }
  }
  A = warp_sum(A);
  g = warp_sum(g);
  if (lane == 0) seg_part[s] = make_double2(A, g);
}

// warp per camera: A_k, g_k from its segments in order; then the scaled LM system of Ceres' Jacobi-scaled LM
// (oracle/ceres_lm.py): first call scale_k = 1 / (1 + sqrt(A_k)); A_s = scale^2 A, D = clamp(A_s, 1e-6, 1e32) / radius,
// Minv = 1 / (A_s + D), b = -scale g.  Constant cameras: an identity row with b = 0 (x_k stays 0).  part_gmax[blk]: the
// CTA's max over its cameras of |Project(x - g) - x| (the projected gradient norm of the bounds-constrained problem).
__global__ void __launch_bounds__(128) vgc_cam_system(int K, const int* __restrict__ seg_off, const double2* __restrict__ seg_part,
                                                      const unsigned char* __restrict__ var, const double* __restrict__ x,
                                                      int first, double radius, double* __restrict__ jscale,
                                                      double* __restrict__ A_s, double* __restrict__ D,
                                                      double* __restrict__ Minv, double* __restrict__ bvec,
                                                      double* __restrict__ g_out, double* __restrict__ part_gmax) {
  __shared__ double scratch[32];
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  double gm = 0.0;
  if (k < K) {
    double A = 0.0, g = 0.0;
    for (int s = seg_off[k] + lane; s < seg_off[k + 1]; s += 32) {
      const double2 p = seg_part[s];
      A += p.x;
      g += p.y;
    }
    A = warp_sum(A);
    g = warp_sum(g);
    if (lane == 0) {
      if (var[k]) {
        if (first) jscale[k] = 1.0 / (1.0 + sqrt(A));
        const double sc = jscale[k];
        const double as = sc * sc * A;
        const double dk = fmin(fmax(as, 1e-6), 1e32) / radius;
        A_s[k] = as;
        D[k] = dk;
        Minv[k] = 1.0 / (as + dk);
        bvec[k] = -sc * g;
        g_out[k] = g;
        gm = fabs(fmax(x[k] - g, kVgcLowerBound) - x[k]);
      } else {
        if (first) jscale[k] = 0.0;
        A_s[k] = 0.0; D[k] = 1.0; Minv[k] = 1.0; bvec[k] = 0.0; g_out[k] = 0.0;
      }
    }
  }
  gm = block_max(gm, scratch);
  if (threadIdx.x == 0) part_gmax[blockIdx.x] = gm;
}

// mat-vec, pass 1 (warp per segment): sum of c_e scale_o p_o over the segment's incidences
__global__ void __launch_bounds__(128) vgc_mv_seg(int n_seg, const int* __restrict__ seg_begin, const int* __restrict__ seg_end,
                                                  const unsigned* __restrict__ inc_val, const int* __restrict__ inc_other,
                                                  const double* __restrict__ off, const double* __restrict__ jscale,
                                                  const double* __restrict__ p, double* __restrict__ seg_part,
                                                  const PcgCtl* __restrict__ ctl) {
  if (ctl && ctl->done) return;
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (s >= n_seg) return;
  double y = 0.0;
  for (int t = seg_begin[s] + lane; t < seg_end[s]; t += 32) {
    const int o = ld_stream(inc_other + t);
    if (o >= 0) y += off[ld_stream(inc_val + t) & 0x7fffffffu] * (jscale[o] * p[o]);
  }
  y = warp_sum(y);
  if (lane == 0) seg_part[s] = y;
}

// mat-vec, pass 2 (warp per camera): yw_k = scale_k * sum of its segments (the off-diagonal part of the scaled J^T J p)
__global__ void __launch_bounds__(128) vgc_mv_cam(int K, const int* __restrict__ seg_off, const double* __restrict__ seg_part,
                                                  const double* __restrict__ jscale, double* __restrict__ yw,
                                                  const PcgCtl* __restrict__ ctl) {
  if (ctl && ctl->done) return;
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= K) return;
  double y = 0.0;
  for (int s = seg_off[k] + lane; s < seg_off[k + 1]; s += 32) y += seg_part[s];
  y = warp_sum(y);
  if (lane == 0) yw[k] = jscale[k] * y;
}

// ---------------------------------------------------------------------------
// step and candidates (per camera)
// ---------------------------------------------------------------------------
// dx = scale * y; partials: g . dx, max |dx|
__global__ void __launch_bounds__(kVgcThreads) vgc_step(int K, const double* __restrict__ y, const double* __restrict__ jscale,
                                                        const double* __restrict__ g, double* __restrict__ dx,
                                                        double* __restrict__ part_gd, double* __restrict__ part_max) {
  __shared__ double scratch[32];
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  double gd = 0.0, m = 0.0;
  if (k < K) {
    const double v = jscale[k] * y[k];
    dx[k] = v;
    gd = g[k] * v;
    m = fabs(v);
  }
  write_partial(gd, part_gd, scratch);
  m = block_max(m, scratch);
  if (threadIdx.x == 0) part_max[blockIdx.x] = m;
}

// x_new = Project(x + alpha dx) on the variable cameras (ParameterBlock::Plus with the lower bound); partials of
// |x_new - x|^2 and |x|^2 over the variable cameras
__global__ void __launch_bounds__(kVgcThreads) vgc_candidate(int K, double alpha, const unsigned char* __restrict__ var,
                                                             const double* __restrict__ x, const double* __restrict__ dx,
                                                             double* __restrict__ x_new, double* __restrict__ part_step,
                                                             double* __restrict__ part_x) {
  __shared__ double scratch[32];
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  double st = 0.0, xx = 0.0;
  if (k < K) {
    const double xv = x[k];
    double xn = xv;
    if (var[k]) {
      xn = fmax(xv + alpha * dx[k], kVgcLowerBound);
      st = (xn - xv) * (xn - xv);
      xx = xv * xv;
    }
    x_new[k] = xn;
  }
  write_partial(st, part_step, scratch);
  write_partial(xx, part_x, scratch);
}

// single CTA: out[0] = fixed-order sum (mode 0) or max (mode 1) of n partials
__global__ void __launch_bounds__(1024) vgc_reduce(const double* __restrict__ part, int n, int mode, double* __restrict__ out) {
  __shared__ double scratch[32];
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v = mode ? fmax(v, part[i]) : v + part[i];
  v = mode ? block_max(v, scratch) : block_sum(v, scratch);
  if (threadIdx.x == 0) *out = v;
}

}  // namespace b200
