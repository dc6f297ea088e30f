// ba_kernels_ext.cuh -- bundle adjustment with parameter blocks beyond the frame poses ("extended" path):
//   * camera intrinsics (the reference default optimize_intrinsics = true, bundle_adjustment.h:18; SubsetManifold
//     over the principal point, bundle_adjustment.cc:273-293) -- ONE BLOCK PER colmap::Camera, shared by any number
//     of images or owned by a single image (a database with one camera per image), no limit on their number;
//   * unknown cam_from_rig poses (optimize_rig_poses, bundle_adjustment.cc:162-180,296-308,
//     colmap::RigReprojErrorCostFunctor): one 6-dof block per non-reference sensor, shared by all its images.
//
// Layout of the reduced system.  Every extra block is appended to the frame blocks as a PSEUDO-CAMERA of 6 dofs
// (intrinsics blocks use their first m <= 5 slots, the rest are identity rows):
//     block index:  frame f -> f,   intrinsics block k -> C + k,   sensor s -> C + K + s         (CB = C + K + S)
// so the LM bookkeeping (Jacobi scaling, damping, block-Jacobi preconditioner, PCG, step scalars) is the code that
// already runs on [C][6] arrays, now over [CB][6].
//
// The mat-vec is MATRIX-FREE in the Jacobian: no per-observation block is stored for the extra parameters.  With
// J_o = [J_frame | J_intr | J_sensor] (2 x 6+m+6, corrector-scaled) and J_pt (2 x 3) recomputed per observation,
//     pass A (point order):   s_p = sum_o J_pt^T (J_o x_o),  z_p = Vinv s_p
//     pass B (camera order):  y_b += J_{o,b}^T (J_o x_o - J_pt z_p)      for the blocks b the observation touches
// gives y = (J^T J - W Vinv W^T) x = S x; the damping D x is added by pcg_apply_diag (A = nullptr).  The same pass B
// with x = 0 and z = Vinv g_p is the right-hand side.  Recomputing the projection chain in both passes costs
// arithmetic instead of bytes; the constant-intrinsics fast path (ba_kernels_v2/v3.cuh) is untouched.
#pragma once
#include "ba_kernels_v3.cuh"

namespace b200 {

struct ExtView {
  int C, K, S;                            // frames, intrinsics blocks, sensors (0 without rigs)
  const IntrVarRec* ivar;                 // [K] variable parameters of each intrinsics block (mb = 0: constant)
  const unsigned char* sensor_var;        // [S] 1: the sensor's cam_from_rig is an unknown; nullptr: none
};

// Everything one observation contributes, corrector-scaled (rows * sqrt(rho')); masked frame dofs are zero columns.
template <bool WK, bool WS>
struct ObsFull {
  double Jr[6], Jt[6], Jp[6], r[2], rho0;
  double Jk[WK ? 2 : 1][kMaxBlockDof];
  double Jsr[WS ? 6 : 1], Jst[WS ? 6 : 1];
  bool valid;
};

template <bool WK, bool WS>
__device__ __forceinline__ void obs_full(const double4& q4, const double4& t4, const double* __restrict__ ir,
                                         const IntrVarRec& iv, const double* __restrict__ sr, bool svar, double X0,
                                         double X1, double X2, double2 xy, double huber_a, ObsFull<WK, WS>& o) {
  const int mask = (int)(__double_as_longlong(t4.w) & 0xff);
  const double q[4] = {q4.x, q4.y, q4.z, q4.w};
  double R[9];
  quat_to_R(q, R);
  const double rx = R[0] * X0 + R[1] * X1 + R[2] * X2;
  const double ry = R[3] * X0 + R[4] * X1 + R[5] * X2;
  const double rz = R[6] * X0 + R[7] * X1 + R[8] * X2;
  double xc = rx + t4.x, yc = ry + t4.y, zc = rz + t4.z;
  if (sr) sensor_apply(sr, xc, yc, zc);
  o.valid = zc > kZEps;
#pragma unroll
  for (int k = 0; k < 6; ++k) o.Jr[k] = o.Jt[k] = o.Jp[k] = 0.0;
  o.r[0] = o.r[1] = 0.0;
  o.rho0 = 0.0;
  if (WK) {
#pragma unroll
    for (int j = 0; j < kMaxBlockDof; ++j) o.Jk[0][j] = o.Jk[WK ? 1 : 0][j] = 0.0;
  }
  if (WS) {
#pragma unroll
    for (int k = 0; k < 6; ++k) o.Jsr[WS ? k : 0] = o.Jst[WS ? k : 0] = 0.0;
  }
  if (!o.valid) return;
  double px, py, J[6];
  project_jac(ir, xc, yc, zc, px, py, J);
  const double u = xc / zc, v = yc / zc;
  const double e0 = px - xy.x, e1 = py - xy.y;
  double rho1;
  huber(e0 * e0 + e1 * e1, huber_a, o.rho0, rho1);
  const double w = sqrt(rho1);
  o.r[0] = w * e0;
  o.r[1] = w * e1;
#pragma unroll
  for (int k = 0; k < 6; ++k) J[k] *= w;
  if (WS) {
    if (svar) {   // left perturbation of cam_from_rig: dX_c = -2 [R_cr X_f]x d_rot + d_t,  R_cr X_f = X_c - t_cr
      const double a0 = xc - sr[9], a1 = yc - sr[10], a2 = zc - sr[11];
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const double j0 = J[3 * a], j1 = J[3 * a + 1], j2 = J[3 * a + 2];
        o.Jsr[WS ? 3 * a + 0 : 0] = -2.0 * (j1 * a2 - j2 * a1);
        o.Jsr[WS ? 3 * a + 1 : 0] = -2.0 * (j2 * a0 - j0 * a2);
        o.Jsr[WS ? 3 * a + 2 : 0] = -2.0 * (j0 * a1 - j1 * a0);
        o.Jst[WS ? 3 * a + 0 : 0] = j0;
        o.Jst[WS ? 3 * a + 1 : 0] = j1;
        o.Jst[WS ? 3 * a + 2 : 0] = j2;
      }
    }
  }
  if (WK) {
#pragma unroll
    for (int j = 0; j < kMaxBlockDof; ++j)
      if (j < iv.mb) intr_param_jac(ld_intr(ir), iv.pidx[j], u, v, w, o.Jk[0][j], o.Jk[WK ? 1 : 0][j]);
  }
  if (sr) {   // chain through the cam_from_rig rotation: J <- J R_cr
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const double j0 = J[3 * a], j1 = J[3 * a + 1], j2 = J[3 * a + 2];
      J[3 * a] = j0 * sr[0] + j1 * sr[3] + j2 * sr[6];
      J[3 * a + 1] = j0 * sr[1] + j1 * sr[4] + j2 * sr[7];
      J[3 * a + 2] = j0 * sr[2] + j1 * sr[5] + j2 * sr[8];
    }
  }
  const bool tvar = !(mask & 2), rvar = !(mask & 1);
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const double j0 = J[3 * a], j1 = J[3 * a + 1], j2 = J[3 * a + 2];
    if (tvar) { o.Jt[3 * a] = j0; o.Jt[3 * a + 1] = j1; o.Jt[3 * a + 2] = j2; }
    if (rvar) {
      o.Jr[3 * a + 0] = -2.0 * (j1 * rz - j2 * ry);
      o.Jr[3 * a + 1] = -2.0 * (j2 * rx - j0 * rz);
      o.Jr[3 * a + 2] = -2.0 * (j0 * ry - j1 * rx);
    }
#pragma unroll
    for (int b = 0; b < 3; ++b) o.Jp[3 * a + b] = j0 * R[b] + j1 * R[3 + b] + j2 * R[6 + b];
  }
}

// tau = J_o x_o (2-vector) from the blocks' x
template <bool WK, bool WS>
__device__ __forceinline__ void obs_apply(const ObsFull<WK, WS>& o, const double* xc, const double* xk, const double* xs,
                                          double& t0, double& t1) {
  t0 = o.Jr[0] * xc[0] + o.Jr[1] * xc[1] + o.Jr[2] * xc[2] + o.Jt[0] * xc[3] + o.Jt[1] * xc[4] + o.Jt[2] * xc[5];
  t1 = o.Jr[3] * xc[0] + o.Jr[4] * xc[1] + o.Jr[5] * xc[2] + o.Jt[3] * xc[3] + o.Jt[4] * xc[4] + o.Jt[5] * xc[5];
  if (WK) {
#pragma unroll
    for (int j = 0; j < kMaxBlockDof; ++j) {
      t0 += o.Jk[0][j] * xk[j];
      t1 += o.Jk[WK ? 1 : 0][j] * xk[j];
    }
  }
  if (WS) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      t0 += o.Jsr[WS ? k : 0] * xs[k] + o.Jst[WS ? k : 0] * xs[3 + k];
      t1 += o.Jsr[WS ? 3 + k : 0] * xs[k] + o.Jst[WS ? 3 + k : 0] * xs[3 + k];
    }
  }
}

// sensor records from the sensor pose state (rebuilt whenever a cam_from_rig is an unknown)
__global__ void bax_build_sensor_rec(int S, const double* __restrict__ sq, const double* __restrict__ st,
                                     const int* __restrict__ sensor_intr, double* __restrict__ rec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S) return;
  const double q[4] = {sq[4 * i], sq[4 * i + 1], sq[4 * i + 2], sq[4 * i + 3]};
  double R[9];
  quat_to_R(q, R);
  double* r = rec + (size_t)i * kSensorRec;
#pragma unroll
  for (int k = 0; k < 9; ++k) r[k] = R[k];
  r[9] = st[3 * i]; r[10] = st[3 * i + 1]; r[11] = st[3 * i + 2];
  r[12] = (double)sensor_intr[i];
}

// ---- linearisation of the block-diagonal and the gradient, camera order (one warp per segment) ---------------------
//   WHAT 0: frame block (U_cc, g_c);  1: intrinsics block of the segment;  2: sensor block of the segment
template <int WHAT>
__global__ void __launch_bounds__(128) bax_linearize_blocks(BAView v, ExtView ex, const double* __restrict__ cam_rec,
                                                           const double* __restrict__ intr_rec,
                                                           const double* __restrict__ points, double huber_a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= v.n_segs) return;
  const int cam = v.seg_cam[warp];
  const int b = v.seg_begin[warp], e = v.seg_end[warp];
  const double4 q4c = ld_rec32(cam_rec + (size_t)cam * kCamRec);
  const double4 t4c = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
  const int blk = v.seg_intr[warp];
  const double* irc = intr_rec + (size_t)blk * kIntrRec;
  const double* src = sensor_of_seg(v, warp);
  const int sidx = v.S > 0 ? v.seg_sensor[warp] : 0;
  const bool svar = v.S > 0 && ex.sensor_var && ex.sensor_var[sidx];
  IntrVarRec iv{};
  if (WHAT == 1) iv = ex.ivar[blk];
  int target = cam;
  if (WHAT == 1) {
    if (iv.mb == 0) return;
    target = ex.C + blk;
  }
  if (WHAT == 2) {
    if (!svar) return;
    target = ex.C + ex.K + sidx;
  }
  double U[21], g[6];
#pragma unroll
  for (int k = 0; k < 21; ++k) U[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) g[k] = 0.0;
  for (int i = b + lane; i < e; i += 32) {
    const int pt = v.pt_c[i];
    const double2 xy = v.xy_c[i];
    const double X0 = points[3 * (size_t)pt], X1 = points[3 * (size_t)pt + 1], X2 = points[3 * (size_t)pt + 2];
    ObsFull<WHAT == 1, WHAT == 2> o;
    obs_full<WHAT == 1, WHAT == 2>(q4c, t4c, irc, iv, src, svar, X0, X1, X2, xy, huber_a, o);
    double Jb[2][6];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        if (WHAT == 0) { Jb[a][k] = o.Jr[3 * a + k]; Jb[a][3 + k] = o.Jt[3 * a + k]; }
        if (WHAT == 2) { Jb[a][k] = o.Jsr[WHAT == 2 ? 3 * a + k : 0]; Jb[a][3 + k] = o.Jst[WHAT == 2 ? 3 * a + k : 0]; }
      }
    if (WHAT == 1) {
#pragma unroll
      for (int a = 0; a < 2; ++a) {
#pragma unroll
        for (int j = 0; j < kMaxBlockDof; ++j) Jb[a][j] = o.Jk[WHAT == 1 ? a : 0][j];
        Jb[a][5] = 0.0;
      }
    }
    int idx = 0;
#pragma unroll
    for (int i2 = 0; i2 < 6; ++i2) {
#pragma unroll
      for (int j = i2; j < 6; ++j) U[idx++] += Jb[0][i2] * Jb[0][j] + Jb[1][i2] * Jb[1][j];
      g[i2] += Jb[0][i2] * o.r[0] + Jb[1][i2] * o.r[1];
    }
  }
  double vals[27];
#pragma unroll
  for (int k = 0; k < 21; ++k) vals[k] = U[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) vals[21 + k] = g[k];
  const double s = warp_reduce_scatter(vals);   // total k in lane k
  if (lane < 27 && s != 0.0)
    atomicAdd(lane < 21 ? &v.U[(size_t)target * 21 + lane] : &v.gc[(size_t)target * 6 + (lane - 21)], s);
}

// ---- pass A (ELL, one thread per point): s_p = [g_p] + sum_o J_pt^T (J_o x_o), z_p = Vinv s_p ----------------------
template <int MODE, bool WK, bool WS>
__global__ void __launch_bounds__(kEllThreads) bax_pass_a(BAView v, EllView ell, ExtView ex, BAViewV2 v2,
                                                           const double* __restrict__ cam_rec,
                                                           const double* __restrict__ intr_rec,
                                                           const double* __restrict__ x, const double* __restrict__ points,
                                                           double* __restrict__ points_new, double huber_a, double radius,
                                                           double* __restrict__ bscal, const PcgCtl* __restrict__ ctl) {
  __shared__ double scratch[32];
  if (ctl && ctl->done) return;
  const int slot = blockIdx.x * kEllThreads + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int g = slot >> 5;
  double b0 = 0, b1 = 0, b2 = 0, b3 = 0;
  if (g < ell.n_groups) {
    const int pt = ell.pt[slot];
    const int mylen = ell.len[slot];
    const int r0 = ell.row0[g], nrow = ell.row0[g + 1] - r0;
    double X0 = 0, X1 = 0, X2 = 0;
    if (pt >= 0) {
      X0 = points[3 * (size_t)pt]; X1 = points[3 * (size_t)pt + 1]; X2 = points[3 * (size_t)pt + 2];
    }
    double s0 = 0, s1 = 0, s2 = 0;
    for (int j = 0; j < nrow; ++j) {
      if (j >= mylen) continue;
      const size_t idx = ((size_t)r0 + j) * 32 + lane;
      const int cam = ell.cam[idx];
      const double2 xy = ell.xy[idx];
      const double4 q4 = ld_rec32(cam_rec + (size_t)cam * kCamRec);
      const double4 t4 = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
      const int sidx = ell.sensor ? (int)ell.sensor[idx] : 0;
      const double* sr = ell.sensor ? v.sensor_rec + (size_t)sidx * kSensorRec : nullptr;
      const int blk = obs_intr_idx(t4, sr);
      const double* ir = intr_rec + (size_t)blk * kIntrRec;
      const bool svar = WS && ell.sensor && ex.sensor_var && ex.sensor_var[sidx];
      IntrVarRec iv{};
      if (WK) iv = ex.ivar[blk];
      ObsFull<WK, WS> o;
      obs_full<WK, WS>(q4, t4, ir, iv, sr, svar, X0, X1, X2, xy, huber_a, o);
      double xc[6], xk[kMaxBlockDof], xs[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) xc[k] = x[(size_t)cam * 6 + k];
#pragma unroll
      for (int k = 0; k < kMaxBlockDof; ++k) xk[k] = WK ? x[(size_t)(ex.C + blk) * 6 + k] : 0.0;
#pragma unroll
      for (int k = 0; k < 6; ++k) xs[k] = (WS && svar) ? x[(size_t)(ex.C + ex.K + sidx) * 6 + k] : 0.0;
      double t0, t1;
      obs_apply<WK, WS>(o, xc, xk, xs, t0, t1);
      s0 += o.Jp[0] * t0 + o.Jp[3] * t1;
      s1 += o.Jp[1] * t0 + o.Jp[4] * t1;
      s2 += o.Jp[2] * t0 + o.Jp[5] * t1;
    }
    if (pt >= 0) {
      const size_t p = (size_t)pt;
      double z[3] = {0.0, 0.0, 0.0};
      if (mylen > 0) {
        double s[3] = {s0, s1, s2};
        double gq[3] = {0, 0, 0};
        if (MODE != 0) {
          gq[0] = v.gp[3 * p]; gq[1] = v.gp[3 * p + 1]; gq[2] = v.gp[3 * p + 2];
          s[0] += gq[0]; s[1] += gq[1]; s[2] += gq[2];
        }
        const double2* vp = reinterpret_cast<const double2*>(v.Vinv + 6 * p);
        const double2 va = vp[0], vb = vp[1], vc = vp[2];
        const double vi[6] = {va.x, va.y, vb.x, vb.y, vc.x, vc.y};
        sym3_mul(vi, s, z);
        if (MODE == 2) {
          double v6[6], js[3], Dp[3];
#pragma unroll
          for (int k = 0; k < 6; ++k) v6[k] = v.V[6 * p + k];
#pragma unroll
          for (int k = 0; k < 3; ++k) js[k] = v.jscale_p[3 * p + k];
          point_damping(v6, js, radius, Dp);
          const double Xo[3] = {X0, X1, X2};
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const double dp = -z[k];
            points_new[3 * p + k] = Xo[k] + dp;
            b0 += gq[k] * dp;
            b1 += Dp[k] * dp * dp;
            b2 += dp * dp;
            b3 += Xo[k] * Xo[k];
          }
        }
      } else if (MODE == 2) {
        points_new[3 * p] = X0; points_new[3 * p + 1] = X1; points_new[3 * p + 2] = X2;
      }
      if (MODE == 0) *reinterpret_cast<double4*>(v2.z4 + 4 * p) = make_double4(z[0], z[1], z[2], 0.0);
    }
  }
  if (MODE == 2) {
    b0 = block_sum(b0, scratch);
    b1 = block_sum(b1, scratch);
    b2 = block_sum(b2, scratch);
    b3 = block_sum(b3, scratch);
    if (threadIdx.x == 0) {
      double* o = bscal + (size_t)blockIdx.x * 4;
      o[0] = b0; o[1] = b1; o[2] = b2; o[3] = b3;
    }
  }
}

// ---- pass B (camera order, one warp per segment):  y_b += J_b^T (J_o x_o - J_pt z_p) ---------------------------------
//   x == nullptr: right-hand-side mode (x = 0, z = Vinv g_p)  ->  y = -W Vinv g_p
template <bool WK, bool WS>
__global__ void __launch_bounds__(128) bax_pass_b(BAView v, ExtView ex, BAViewV2 v2, const double* __restrict__ cam_rec,
                                                 const double* __restrict__ intr_rec, const double* __restrict__ points,
                                                 const double* __restrict__ x, double huber_a, double* __restrict__ y,
                                                 const PcgCtl* __restrict__ ctl) {
  if (ctl && ctl->done) return;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= v.n_segs) return;
  const int cam = v.seg_cam[warp];
  const int b = v.seg_begin[warp], e = v.seg_end[warp];
  const double4 q4c = ld_rec32(cam_rec + (size_t)cam * kCamRec);
  const double4 t4c = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
  const int blk = v.seg_intr[warp];
  const double* irc = intr_rec + (size_t)blk * kIntrRec;
  const double* src = sensor_of_seg(v, warp);
  const int sidx = v.S > 0 ? v.seg_sensor[warp] : 0;
  const bool svar = WS && v.S > 0 && ex.sensor_var && ex.sensor_var[sidx];
  IntrVarRec iv{};
  if (WK) iv = ex.ivar[blk];
  double xc[6], xk[kMaxBlockDof], xs[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) xc[k] = x ? x[(size_t)cam * 6 + k] : 0.0;
#pragma unroll
  for (int k = 0; k < kMaxBlockDof; ++k) xk[k] = (WK && x) ? x[(size_t)(ex.C + blk) * 6 + k] : 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) xs[k] = (WS && svar && x) ? x[(size_t)(ex.C + ex.K + sidx) * 6 + k] : 0.0;
  double ac[6] = {0, 0, 0, 0, 0, 0}, ak[kMaxBlockDof] = {0, 0, 0, 0, 0}, as[6] = {0, 0, 0, 0, 0, 0};
  for (int i = b + lane; i < e; i += 32) {
    const int pt = v.pt_c[i];
    const double2 xy = v.xy_c[i];
    const double X0 = points[3 * (size_t)pt], X1 = points[3 * (size_t)pt + 1], X2 = points[3 * (size_t)pt + 2];
    const double4 z = *reinterpret_cast<const double4*>(v2.z4 + 4 * (size_t)pt);
    ObsFull<WK, WS> o;
    obs_full<WK, WS>(q4c, t4c, irc, iv, src, svar, X0, X1, X2, xy, huber_a, o);
    double t0, t1;
    obs_apply<WK, WS>(o, xc, xk, xs, t0, t1);
    t0 -= o.Jp[0] * z.x + o.Jp[1] * z.y + o.Jp[2] * z.z;
    t1 -= o.Jp[3] * z.x + o.Jp[4] * z.y + o.Jp[5] * z.z;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      ac[k] += o.Jr[k] * t0 + o.Jr[3 + k] * t1;
      ac[3 + k] += o.Jt[k] * t0 + o.Jt[3 + k] * t1;
    }
    if (WK) {
#pragma unroll
      for (int j = 0; j < kMaxBlockDof; ++j) ak[j] += o.Jk[0][j] * t0 + o.Jk[WK ? 1 : 0][j] * t1;
    }
    if (WS) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        as[k] += o.Jsr[WS ? k : 0] * t0 + o.Jsr[WS ? 3 + k : 0] * t1;
        as[3 + k] += o.Jst[WS ? k : 0] * t0 + o.Jst[WS ? 3 + k : 0] * t1;
      }
    }
  }
  // the frame, intrinsics and sensor sums in one reduce-scatter, one atomic per lane that holds a total
  constexpr int NKV = WK ? kMaxBlockDof : 0, KV = 6 + NKV + (WS ? 6 : 0), S = warp_rs_stride<KV>();
  double vals[KV];
#pragma unroll
  for (int k = 0; k < 6; ++k) vals[k] = ac[k];
#pragma unroll
  for (int j = 0; j < NKV; ++j) vals[6 + j] = ak[j];
#pragma unroll
  for (int k = 0; k < (WS ? 6 : 0); ++k) vals[6 + NKV + k] = as[k];
  const double s = warp_reduce_scatter(vals);
  const int k = lane / S;
  bool live = lane % S == 0 && k < KV && s != 0.0;
  double* dst = &y[(size_t)cam * 6 + k];
  if (k >= 6 && k < 6 + NKV) {
    live = live && k - 6 < iv.mb;
    dst = &y[(size_t)(ex.C + blk) * 6 + (k - 6)];
  } else if (k >= 6 + NKV) {
    live = live && svar;
    dst = &y[(size_t)(ex.C + ex.K + sidx) * 6 + (k - 6 - NKV)];
  }
  if (live) atomicAdd(dst, s);
}

// ---- trial step of the extra blocks -----------------------------------------------------------------------------------
//   intrinsics: params[pidx[j]] += d[j];  sensors: q <- exp(d_rot) (x) q (EigenQuaternionManifold), t += d_t
//   cscal as ba_update_cams: [0] g.d  [1] d.resid  [2] sum D d^2  [3] |x_new - x|^2  [4] |x|^2 over the blocks of the problem
__global__ void bax_update_extras(ExtView ex, const IntrVarRec* __restrict__ ivar, const int* __restrict__ intr_model,
                                  const double* __restrict__ intr, double* __restrict__ intr_new,
                                  const double* __restrict__ sq, const double* __restrict__ st, double* __restrict__ sq_new,
                                  double* __restrict__ st_new, const double* __restrict__ dc, const double* __restrict__ gc,
                                  const double* __restrict__ resid, const double* __restrict__ Dc,
                                  const double* __restrict__ jscale_c, const double* __restrict__ blk_used, int count_norms,
                                  double* __restrict__ cscal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double a0 = 0, a1 = 0, a2 = 0, a3 = 0, a4 = 0;
  if (i < ex.K) {
    const IntrVarRec iv = ivar[i];
    const size_t blk = (size_t)(ex.C + i);
    double p[12];
#pragma unroll
    for (int j = 0; j < 12; ++j) p[j] = intr[(size_t)i * 12 + j];
    for (int j = 0; j < iv.mb; ++j) {
      const size_t k = blk * 6 + j;
      if (!(jscale_c[k] >= 0.0)) continue;
      const double d = dc[k];
      a0 += gc[k] * d;
      a1 += resid[k] * d;
      a2 += Dc[k] * d * d;
      a3 += d * d;
      p[iv.pidx[j]] += d;
    }
    if (iv.mb > 0 && blk_used[blk] > 0.0) {   // x norm: every block of the problem, whatever its curvature
      const int npar = intr_model[i] == 0 ? 3 : (intr_model[i] == 3 ? 5 : 4);
      for (int j = 0; j < npar; ++j) a4 += intr[(size_t)i * 12 + j] * intr[(size_t)i * 12 + j];
    }
#pragma unroll
    for (int j = 0; j < 12; ++j) intr_new[(size_t)i * 12 + j] = p[j];
  } else if (i < ex.K + ex.S) {
    const int s = i - ex.K;
    const size_t blk = (size_t)(ex.C + ex.K + s);
    double d[6];
    bool rvar = false, tvar = false;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const size_t j = blk * 6 + k;
      const bool var = jscale_c[j] >= 0.0;
      d[k] = var ? dc[j] : 0.0;
      if (var) {
        a0 += gc[j] * d[k];
        a1 += resid[j] * d[k];
        a2 += Dc[j] * d[k] * d[k];
        if (k < 3) rvar = true; else tvar = true;
      }
    }
    // x norm: the sensor is a parameter block of the problem when it is an unknown and observed
    const bool in_problem = ex.sensor_var && ex.sensor_var[s] && blk_used[blk] > 0.0;
    const double q[4] = {sq[4 * s], sq[4 * s + 1], sq[4 * s + 2], sq[4 * s + 3]};
    double qn[4] = {q[0], q[1], q[2], q[3]};
    const double nrm = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (nrm > 0.0) {
      const double sn = sin(nrm) / nrm, cs = cos(nrm);
      const double ax = sn * d[0], ay = sn * d[1], az = sn * d[2], aw = cs;
      qn[0] = aw * q[0] + ax * q[3] + ay * q[2] - az * q[1];
      qn[1] = aw * q[1] - ax * q[2] + ay * q[3] + az * q[0];
      qn[2] = aw * q[2] + ax * q[1] - ay * q[0] + az * q[3];
      qn[3] = aw * q[3] - ax * q[0] - ay * q[1] - az * q[2];
      const double inv = 1.0 / sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
#pragma unroll
      for (int k = 0; k < 4; ++k) qn[k] *= inv;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      sq_new[4 * s + k] = qn[k];
      if (rvar) a3 += (qn[k] - q[k]) * (qn[k] - q[k]);
      if (in_problem) a4 += q[k] * q[k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double t = st[3 * s + k];
      st_new[3 * s + k] = t + d[3 + k];
      if (tvar) a3 += d[3 + k] * d[3 + k];
      if (in_problem) a4 += t * t;
    }
  }
  if (!count_norms) { a3 = 0; a4 = 0; }
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  a2 = warp_sum(a2);
  a3 = warp_sum(a3);
  a4 = warp_sum(a4);
  if ((threadIdx.x & 31) == 0) {
    if (a0 != 0.0) atomicAdd(&cscal[0], a0);
    if (a1 != 0.0) atomicAdd(&cscal[1], a1);
    if (a2 != 0.0) atomicAdd(&cscal[2], a2);
    if (a3 != 0.0) atomicAdd(&cscal[3], a3);
    if (a4 != 0.0) atomicAdd(&cscal[4], a4);
  }
}

}  // namespace b200
