// ba_kernels_v2.cuh -- "compact row" layout of the BA hot path (design v2).
//
// v1 stores the 6x3 block W_o = J_cam^T J_pt (144 B/observation) and scatters
// W_o z_p into y[cam] with 6 FP64 atomics per observation, which bounds that
// mat-vec by L2 operations.  v2 exploits
//     J_cam = J_pt G,   G = [ -2 [X]x R^T | R^T ]   (3 x 6;  X = the world point, R = R(q_cam))
// (left-perturbed rotation, translation), so that with the symmetric 3x3
//     A_o = J_pt^T J_pt        (what the observation adds to V_p)
// W_o = G^T A_o,  W_o^T x = A_o v  with  v = R^T x_t - 2 X x (R^T x_r),
// W_o z = [ 2 R (X x w) ; R w ],  w = A_o z.   A_o (48 B) is stored per observation in POINT order only
// (Ap[N][6], or the ELL rows of ba_kernels_v3.cuh), and the implicit-Schur mat-vec is two passes
//     pass A (point order):  s_p = sum_o A_o v_o,  z_p = Vinv s_p -> z4[P]      streams A_o, gathers R^T x (64 B)
//     pass B (camera order): y_c -= R-rotated sum_o [2 X x (A_o z_p) ; A_o z_p]  gathers X_p (pts4) and z_p (32 B each)
//                            one warp per <= 256-observation segment of ONE camera: register
//                            accumulation, shuffle reduction, 6 atomics per segment.
// In camera order the segment's camera, intrinsics and sensor records are warp-uniform and held in registers, so pass B
// (and the Schur-Jacobi diagonal) recompute each observation's residual with the linearisation's own arithmetic
// (obs_core_R) instead of streaming a stored camera-order row, and apply its Jacobian in the camera frame without
// forming A_o (see "Camera-frame form" below): about 80 FP64 instructions per pinhole observation in place of 72 B of
// HBM traffic, the cheaper side on an H100.  All arithmetic stays FP64.
// Algorithmic bytes per mat-vec: 52 N + 80 P (A) + 20 N + 64 P (B, point records gathered from L2: see the slices of
// BAProblem::create).
#pragma once
#include "ba_kernels.cuh"
#include "pcg.cuh"

namespace b200 {

struct BAViewV2 {
  const double* Ap;     // [N][6]   (aliases BAView::W)
  double* z4;           // [P][4]
  const double* pts4;   // [P][4]   {X_p, 0} of the current state (ba2_pad_points at every linearisation)
  // stored-row intrinsics path (NK > 0, see below): the frame x intrinsics cross blocks of every image, the
  // variable-parameter table and the number of frames (block C + k = intrinsics k)
  double* Ufk = nullptr;             // [C][6][NK]
  const IntrVarRec* ivar = nullptr;  // [K]
  int C = 0;
};

// ---------------------------------------------------------------------------
// Variable intrinsics WITHOUT recomputing the projection chain in the mat-vec ("stored-row" path, NK <= 2 variable
// parameters per camera: SIMPLE_PINHOLE f; SIMPLE_RADIAL f, k; PINHOLE fx, fy -- the reference default
// optimize_intrinsics = true, optimize_principal_point = false, bundle_adjustment.cc:273-293).
// Intrinsics block k is pseudo-camera block C + k of the reduced system (ba_kernels_ext.cuh).  With J_k = d e / d(params)
// (2 x NK) and B_o = rho' J_pt^T J_k (3 x NK, stored next to A_o in point order, 24 NK bytes; recomputed in camera order):
//     W^T x   per point:   s_p = sum_o ( A_o w_o + B_o x_k(o) )                    (pass A, x_k rides in the xq record)
//     W z     per image:   y_f -= G^T sum_o A_o z_p,   y_k -= sum_o B_o^T z_p       (pass B)
//     U x:    block diagonal U_ff, U_kk by pcg_apply_diag; the frame x intrinsics coupling is ONE 6 x NK block per image
//             (an image has one camera):  y_f += U_fk x_k,  y_k += U_fk^T x_f       (ba2k_cross, C threads)
// so the per-iteration cost over the constant-intrinsics path is 24 NK bytes per observation of streamed rows.
// ---------------------------------------------------------------------------
template <int NK>
__device__ __forceinline__ void obs_intr_jac(const ObsCore& o, const Intr& in, const IntrVarRec& iv,
                                             double Jk[2][NK > 0 ? NK : 1]) {
#pragma unroll
  for (int j = 0; j < NK; ++j) {
    double jx = 0.0, jy = 0.0;
    if (j < iv.mb) intr_param_jac(in, iv.pidx[j], o.uv[0], o.uv[1], 1.0, jx, jy);
    if (!o.valid) jx = jy = 0.0;
    Jk[0][j] = jx;
    Jk[1][j] = jy;
  }
}
template <int NK>
__device__ __forceinline__ void obs_intr_rows(const ObsCore& o, const Intr& in, const IntrVarRec& iv,
                                              const double Jp[6], double Jk[2][NK > 0 ? NK : 1],
                                              double B[NK > 0 ? 3 * NK : 1]) {
  obs_intr_jac<NK>(o, in, iv, Jk);
#pragma unroll
  for (int j = 0; j < NK; ++j)
#pragma unroll
    for (int c = 0; c < 3; ++c) B[3 * j + c] = o.rho1 * (Jp[c] * Jk[0][j] + Jp[3 + c] * Jk[1][j]);
}

// ---------------------------------------------------------------------------
// Camera-frame form of the camera-order kernels.  With Rs = R_cr R (R for a trivial frame, R_cr = cam_from_rig of a
// known rig), P = R_cr R X (the rotated point in the sensor-camera frame) and J_pi = iz M [I | -(u, v)^T] the
// projection Jacobian (ProjJac),
//     J_pt = J_pi Rs,   J_cam = J_pi [ -2 [P]x | I ] B,   B = blockdiag(R_cr, R_cr)
// so every per-segment sum is taken in the sensor-camera frame and conjugated by B once at the end of the segment
// (B = I for a trivial frame).  No world-frame J_pt or A_o is formed.  Only R is held in registers: the R_cr factor of
// a known rig is applied from its sensor record (a branch the trivial frames never take).
// ---------------------------------------------------------------------------
// the segment's warp-uniform records, in registers
struct SegRec {
  double R[9];
  double4 t4;
  Intr in;
  const double* sr;   // sensor record (known rig) or nullptr
};
__device__ __forceinline__ void seg_records(const BAView& v, int seg, int cam, const double* __restrict__ cam_rec,
                                            const double* __restrict__ intr_rec, SegRec& s) {
  const double4 q4 = ld_rec32(cam_rec + (size_t)cam * kCamRec);
  s.t4 = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
  s.in = ld_intr(intr_rec + (size_t)v.seg_intr[seg] * kIntrRec);
  s.sr = sensor_of_seg(v, seg);
  const double q[4] = {q4.x, q4.y, q4.z, q4.w};
  quat_to_R(q, s.R);
}
// x <- R_cr x  (nothing for a trivial frame)
__device__ __forceinline__ void to_sensor(const double* __restrict__ sr, double x[3]) {
  if (!sr) return;
  const double x0 = x[0], x1 = x[1], x2 = x[2];
#pragma unroll
  for (int k = 0; k < 3; ++k) x[k] = sr[3 * k] * x0 + sr[3 * k + 1] * x1 + sr[3 * k + 2] * x2;
}
// a = rho' J_pi r  and  w = J_pi^T a
__device__ __forceinline__ void cam_frame_jac(const ObsCore& o, const double r[3], double a[2], double w[3]) {
  const ProjJac& p = o.pj;
  const double t0 = r[0] - p.u * r[2], t1 = r[1] - p.v * r[2];
  const double c = o.rho1 * p.iz;
  a[0] = c * (p.m00 * t0 + p.m01 * t1);
  a[1] = c * (p.m10 * t0 + p.m11 * t1);
  const double s0 = p.iz * (p.m00 * a[0] + p.m10 * a[1]), s1 = p.iz * (p.m01 * a[0] + p.m11 * a[1]);
  w[0] = s0;
  w[1] = s1;
  w[2] = -(p.u * s0 + p.v * s1);
}

// xp[c] = { R^T x_r , R^T x_t, pad, pad }: 64-B rows, so pass A gathers a camera with three 128-bit
// loads out of a single line  (masked dofs of x are zero already: PCG keeps them at 0)
constexpr int kXqStride = 8;
__global__ void ba2_pack_x(int C, const double* __restrict__ x, const double* __restrict__ cam_rec,
                           double* __restrict__ xp) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double* r = cam_rec + (size_t)c * kCamRec;
  const double q[4] = {r[0], r[1], r[2], r[3]};
  double R[9];
  quat_to_R(q, R);
  const double* xc = x + (size_t)c * 6;
  double* o = xp + (size_t)c * kXqStride;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    o[k] = R[k] * xc[0] + R[3 + k] * xc[1] + R[6 + k] * xc[2];
    o[3 + k] = R[k] * xc[3] + R[3 + k] * xc[4] + R[6 + k] * xc[5];
  }
}

// Head of a PCG iteration fused with the packing of its search direction: p = z + beta p (pcg_direction) and
// xp[c] = {R^T p_r, R^T p_t} for pass A, one thread per camera -- one launch instead of two per iteration.
__global__ void __launch_bounds__(kPcgThreads) ba2_pcg_direction_pack(int nb, int nblk, int it, int min_it, double rel_tol,
                                                                      const double* __restrict__ z, double* __restrict__ p,
                                                                      double* __restrict__ yw,
                                                                      const double* __restrict__ dots_pp,
                                                                      const double* __restrict__ part_rz,
                                                                      const double* __restrict__ part_rr,
                                                                      double* __restrict__ dots_pub, PcgCtl* __restrict__ ctl,
                                                                      const double* __restrict__ cam_rec,
                                                                      double* __restrict__ xp, int n_pack) {
  __shared__ double sh3[3];
  double beta;
  if (!pcg_direction_head(nblk, it, min_it, rel_tol, dots_pp, part_rz, part_rr, nullptr, dots_pub, ctl, sh3, beta)) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nb) return;
  double pv[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const size_t i = (size_t)c * 6 + k;
    pv[k] = (it == 1) ? z[i] : z[i] + beta * p[i];
    p[i] = pv[k];
    yw[i] = 0.0;
  }
  if (c >= n_pack) return;   // pseudo-camera blocks (intrinsics) have no record: their x rides in the frames' rows
  const double* r = cam_rec + (size_t)c * kCamRec;
  const double q[4] = {r[0], r[1], r[2], r[3]};
  double R[9];
  quat_to_R(q, R);
  double* o = xp + (size_t)c * kXqStride;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    o[k] = R[k] * pv[0] + R[3 + k] * pv[1] + R[6 + k] * pv[2];
    o[3 + k] = R[k] * pv[3] + R[3 + k] * pv[4] + R[6 + k] * pv[5];
  }
}

// pts4[p] = {X_p, 0}: 32-B rows for the camera-order gathers (one sector per observation).  Written at every
// linearisation from points[cur]; a rejected step keeps points[cur], so it stays valid until the next one.
__global__ void ba2_pad_points(int P, const double* __restrict__ points, double* __restrict__ pts4) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const double x = points[3 * (size_t)p], y = points[3 * (size_t)p + 1], z = points[3 * (size_t)p + 2];
  st_rec32(pts4 + 4 * (size_t)p, x, y, z, 0.0);
}

// ---------------------------------------------------------------------------
// camera-order linearisation: U_c, g_c (and, NK > 0, U_kk, g_k, U_fk)
// ---------------------------------------------------------------------------
template <int NK>
__global__ void __launch_bounds__(128, NK > 0 ? 3 : B200_LC_MIN_CTAS) ba2_linearize_cams(BAView v, BAViewV2 v2, const double* __restrict__ cam_rec,
                                                         const double* __restrict__ intr_rec, double huber_a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= v.n_segs) return;
  const int cam = v.seg_cam[warp];
  const int b = v.seg_begin[warp], e = v.seg_end[warp];
  SegRec sg;
  seg_records(v, warp, cam, cam_rec, intr_rec, sg);
  double U[21], g[6];
#pragma unroll
  for (int k = 0; k < 21; ++k) U[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) g[k] = 0.0;
  const int cmask = (int)(__double_as_longlong(sg.t4.w) & 0xff);
  const bool tvar = !(cmask & 2), rvar = !(cmask & 1);
  // stored-row intrinsics path: U_kk / g_k of the segment's intrinsics block and the image's 6 x NK cross block
  constexpr int NKK = NK > 0 ? NK : 1;
  const int blk = v.seg_intr[warp];
  IntrVarRec iv{};
  if (NK > 0) iv = v2.ivar[blk];
  double Ukk[NKK * (NKK + 1) / 2], gk[NKK], Ufk[6][NKK];
#pragma unroll
  for (int k = 0; k < NKK * (NKK + 1) / 2; ++k) Ukk[k] = 0.0;
#pragma unroll
  for (int k = 0; k < NKK; ++k) {
    gk[k] = 0.0;
#pragma unroll
    for (int i2 = 0; i2 < 6; ++i2) Ufk[i2][k] = 0.0;
  }
  // index -> point gather -> ~400 instructions: the first use of the gathered point and the address computed from the
  // streamed index each wait a full memory latency.  Register pipeline: the index of iteration + 2 and the
  // point / pixel of iteration + 1 are in flight while iteration + 0 is computed.  The points come from the 32-B padded
  // copy pts4: ONE 32-B record (two 128-bit loads of one sector) instead of three 64-bit gathers.
  const double* __restrict__ pts4 = v2.pts4;
  int i = b + lane;
  int pt_nxt = 0;
  double2 xy = make_double2(0, 0);
  double4 Xc = make_double4(0, 0, 0, 0);
  if (i < e) {
    const int pt0 = ld_stream(v.pt_c + i);
    if (i + 32 < e) pt_nxt = ld_stream(v.pt_c + i + 32);
    xy = ld_stream(v.xy_c + i);
    Xc = ld_rec32(pts4 + 4 * (size_t)pt0);
  }
  for (; i < e; i += 32) {
    double4 Xn = Xc;
    double2 xyn = xy;
    int pt_nn = 0;
    if (i + 32 < e) {
      Xn = ld_rec32(pts4 + 4 * (size_t)pt_nxt);
      xyn = ld_stream(v.xy_c + i + 32);
    }
    if (i + 64 < e) pt_nn = ld_stream(v.pt_c + i + 64);
    const double X0 = Xc.x, X1 = Xc.y, X2 = Xc.z;
    ObsCore o;
    obs_core_R(sg.R, sg.t4, sg.in, sg.sr, X0, X1, X2, xy, huber_a, o);
    // camera blocks: J_t = J, J_r = J (-2 [R X]x)  (EigenQuaternionManifold: left perturbation of angle 2|d|), masked;
    // U += rho' Jc^T Jc, g += rho' Jc^T e
    double Jc[2][6];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const double j0 = o.J[3 * a], j1 = o.J[3 * a + 1], j2 = o.J[3 * a + 2];
      Jc[a][0] = rvar ? -2.0 * (j1 * o.RX[2] - j2 * o.RX[1]) : 0.0;
      Jc[a][1] = rvar ? -2.0 * (j2 * o.RX[0] - j0 * o.RX[2]) : 0.0;
      Jc[a][2] = rvar ? -2.0 * (j0 * o.RX[1] - j1 * o.RX[0]) : 0.0;
      Jc[a][3] = tvar ? j0 : 0.0;
      Jc[a][4] = tvar ? j1 : 0.0;
      Jc[a][5] = tvar ? j2 : 0.0;
    }
    const double e0 = o.rho1 * o.e[0], e1 = o.rho1 * o.e[1];
    int idx = 0;
#pragma unroll
    for (int i2 = 0; i2 < 6; ++i2) {
      const double s0 = o.rho1 * Jc[0][i2], s1 = o.rho1 * Jc[1][i2];
#pragma unroll
      for (int j = i2; j < 6; ++j) U[idx++] += s0 * Jc[0][j] + s1 * Jc[1][j];
      g[i2] += Jc[0][i2] * e0 + Jc[1][i2] * e1;
    }
    if (NK > 0) {
      double Jk[2][NKK];
      obs_intr_jac<NK>(o, sg.in, iv, Jk);
      int ik = 0;
#pragma unroll
      for (int a = 0; a < NK; ++a) {
        const double s0 = o.rho1 * Jk[0][a], s1 = o.rho1 * Jk[1][a];
#pragma unroll
        for (int c = a; c < NK; ++c) Ukk[ik++] += s0 * Jk[0][c] + s1 * Jk[1][c];
        gk[a] += Jk[0][a] * e0 + Jk[1][a] * e1;
#pragma unroll
        for (int i2 = 0; i2 < 6; ++i2) Ufk[i2][a] += Jc[0][i2] * s0 + Jc[1][i2] * s1;
      }
    }
    Xc = Xn; xy = xyn; pt_nxt = pt_nn;
  }
  // epilogue: reduce-scatter rounds of <= 32 sums, one atomic per lane that holds a total
  if (NK > 0) {   // U_kk (upper triangle), g_k, then U_fk row-major: 17 sums for NK = 2
    constexpr int nU = NKK * (NKK + 1) / 2, KV = nU + NKK + 6 * NKK, S = warp_rs_stride<KV>();
    double vals[KV];
#pragma unroll
    for (int k = 0; k < nU; ++k) vals[k] = Ukk[k];
#pragma unroll
    for (int a = 0; a < NKK; ++a) {
      vals[nU + a] = gk[a];
#pragma unroll
      for (int i2 = 0; i2 < 6; ++i2) vals[nU + NKK + i2 * NKK + a] = Ufk[i2][a];
    }
    const double s = warp_reduce_scatter(vals);
    const int k = lane / S;
    const size_t kb = (size_t)(v2.C + blk);
    double* dst = &v2.Ufk[(size_t)cam * 6 * NKK + (k - nU - NKK)];
    if (k < nU + NKK) dst = &v.gc[kb * 6 + (k - nU)];
    int ik = 0;
#pragma unroll
    for (int a = 0; a < NKK; ++a)
#pragma unroll
      for (int c = a; c < NKK; ++c, ++ik)
        if (k == ik) dst = &v.U[kb * 21 + sym_idx(6, a, c)];
    if (lane % S == 0 && k < KV && s != 0.0) atomicAdd(dst, s);
  }
  double vals[27];
#pragma unroll
  for (int k = 0; k < 21; ++k) vals[k] = U[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) vals[21 + k] = g[k];
  const double s = warp_reduce_scatter(vals);   // total k in lane k
  if (lane < 27 && s != 0.0) atomicAdd(lane < 21 ? &v.U[(size_t)cam * 21 + lane] : &v.gc[(size_t)cam * 6 + (lane - 21)], s);
}

// ---------------------------------------------------------------------------
// Schur-Jacobi diagonal in camera order, accumulated in the sensor-camera frame (per observation, W_o Vinv_p W_o^T):
//   Sd_c = B^T ( sum_o Gh^T N Gh ) B,   N = J_pi^T Q J_pi,   Q = rho'^2 L Vinv_p L^T,   L = J_pi Rs,
//   Gh = [ -2 [P]x | I ]
// with Q = (rho' iz^2)^2 K Q' K, Q' = L' Vinv L'^T, L' = [I | -(u, v)^T] Rs, K = M^T M.  Per observation the kernel
// gathers the point (pts4, 32 B) and Vinv_p (48 B).
// ---------------------------------------------------------------------------
// The 21 per-segment sums of ba2_schur_diag, in order RR (packed upper 3 x 3), RT (row-major 3 x 3), TT (packed upper
// 3 x 3), are the upper triangle of the symmetric 6 x 6 M = [RR RT; RT^T TT].  sd_entry: sum k -> its entry (r, c),
// r <= c (k < 21);  sd_value: entry (p, q) of M -> the sum that holds it.
__device__ __forceinline__ void sd_entry(int k, int& r, int& c) {
  if (k >= 6 && k < 15) {
    r = (k - 6) / 3;
    c = 3 + (k - 6) % 3;
  } else {
    const int o = k < 6 ? 0 : 3, t = k < 6 ? k : k - 15;   // packed 3 x 3: 00 01 02 11 12 22
    const int i = (t >= 3) + (t >= 5);
    r = o + i;
    c = o + t - (i == 0 ? 0 : i == 1 ? 2 : 3);
  }
}
__device__ __forceinline__ int sd_value(int p, int q) {
  const int i = min(p, q), j = max(p, q);
  if (j < 3) return sym_idx(3, i, j);
  if (i >= 3) return 15 + sym_idx(3, i - 3, j - 3);
  return 6 + 3 * i + (j - 3);
}
__global__ void __launch_bounds__(128, B200_SD_MIN_CTAS) ba2_schur_diag(BAView v, BAViewV2 v2, const double* __restrict__ cam_rec,
                                                                        const double* __restrict__ intr_rec, double huber_a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= v.n_segs) return;
  const int cam = v.seg_cam[warp];
  const int b = v.seg_begin[warp], e = v.seg_end[warp];
  SegRec sg;
  seg_records(v, warp, cam, cam_rec, intr_rec, sg);
  // accumulators: RR (sym 6), RT (full 9), TT (sym 6)
  double RR[6] = {0, 0, 0, 0, 0, 0}, RT[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, TT[6] = {0, 0, 0, 0, 0, 0};
  // register pipeline of ba2_linearize_cams: the index of iteration + 2 and the point / pixel / Vinv of iteration + 1
  // are in flight while iteration + 0 is computed
  int i = b + lane;
  int pt_nxt = 0;
  double2 xy = make_double2(0, 0), va = xy, vb = xy, vc = xy;
  double4 Xc = make_double4(0, 0, 0, 0);
  if (i < e) {
    const int pt0 = ld_stream(v.pt_c + i);
    if (i + 32 < e) pt_nxt = ld_stream(v.pt_c + i + 32);
    xy = ld_stream(v.xy_c + i);
    Xc = ld_rec32(v2.pts4 + 4 * (size_t)pt0);
    const double2* vp = reinterpret_cast<const double2*>(v.Vinv + (size_t)pt0 * 6);
    va = vp[0]; vb = vp[1]; vc = vp[2];
  }
  for (; i < e; i += 32) {
    double4 Xn = Xc;
    double2 xyn = xy, van = va, vbn = vb, vcn = vc;
    int pt_nn = 0;
    if (i + 32 < e) {
      Xn = ld_rec32(v2.pts4 + 4 * (size_t)pt_nxt);
      xyn = ld_stream(v.xy_c + i + 32);
      const double2* vp = reinterpret_cast<const double2*>(v.Vinv + (size_t)pt_nxt * 6);
      van = vp[0]; vbn = vp[1]; vcn = vp[2];
    }
    if (i + 64 < e) pt_nn = ld_stream(v.pt_c + i + 64);
    ObsCore o;
    obs_core_R(sg.R, sg.t4, sg.in, sg.sr, Xc.x, Xc.y, Xc.z, xy, huber_a, o);
    double X[3] = {o.RX[0], o.RX[1], o.RX[2]};
    to_sensor(sg.sr, X);
    const ProjJac& pj = o.pj;
    const double vi[6] = {va.x, va.y, vb.x, vb.y, vc.x, vc.y};
    // Q' = L' Vinv L'^T,  L' = E Rs = (E R_cr) R,  E = [I | -(u, v)^T]
    double e0[3] = {1.0, 0.0, -pj.u}, e1[3] = {0.0, 1.0, -pj.v};
    if (sg.sr) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        e0[c] = sg.sr[c] - pj.u * sg.sr[6 + c];
        e1[c] = sg.sr[3 + c] - pj.v * sg.sr[6 + c];
      }
    }
    double l0[3], l1[3], t0[3], t1[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      l0[c] = e0[0] * sg.R[c] + e0[1] * sg.R[3 + c] + e0[2] * sg.R[6 + c];
      l1[c] = e1[0] * sg.R[c] + e1[1] * sg.R[3 + c] + e1[2] * sg.R[6 + c];
    }
    sym3_mul(vi, l0, t0);
    sym3_mul(vi, l1, t1);
    const double q00 = l0[0] * t0[0] + l0[1] * t0[1] + l0[2] * t0[2];
    const double q01 = l0[0] * t1[0] + l0[1] * t1[1] + l0[2] * t1[2];
    const double q11 = l1[0] * t1[0] + l1[1] * t1[1] + l1[2] * t1[2];
    // H = (rho' iz^2)^2 K Q' K  (J_pi^T Q J_pi = [I | -(u, v)^T]^T H [I | -(u, v)^T])
    const double k00 = pj.m00 * pj.m00 + pj.m10 * pj.m10, k01 = pj.m00 * pj.m01 + pj.m10 * pj.m11,
                 k11 = pj.m01 * pj.m01 + pj.m11 * pj.m11;
    const double a00 = k00 * q00 + k01 * q01, a01 = k00 * q01 + k01 * q11;
    const double a10 = k01 * q00 + k11 * q01, a11 = k01 * q01 + k11 * q11;
    const double sc = o.rho1 * pj.iz * pj.iz, c2 = sc * sc;
    const double h00 = c2 * (a00 * k00 + a01 * k01), h01 = c2 * (a00 * k01 + a01 * k11), h11 = c2 * (a10 * k01 + a11 * k11);
    double N[3][3];
    N[0][0] = h00; N[0][1] = N[1][0] = h01; N[1][1] = h11;
    N[0][2] = N[2][0] = -(h00 * pj.u + h01 * pj.v);
    N[1][2] = N[2][1] = -(h01 * pj.u + h11 * pj.v);
    N[2][2] = -(N[0][2] * pj.u + N[1][2] * pj.v);
    // P = 2 [X]x N  (rows: 2 X x N_col);  rr = -2 P [X]x;  rt = P;  tt = N   (X: the camera-frame point)
    double P[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double n0 = N[0][c], n1 = N[1][c], n2 = N[2][c];
      P[0][c] = 2.0 * (X[1] * n2 - X[2] * n1);
      P[1][c] = 2.0 * (X[2] * n0 - X[0] * n2);
      P[2][c] = 2.0 * (X[0] * n1 - X[1] * n0);
    }
    // (P [X]x)[r][c] = sum_k P[r][k] K[k][c],  K = [X]x = [[0,-X2,X1],[X2,0,-X0],[-X1,X0,0]]
    double PK[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      PK[r][0] = P[r][1] * X[2] - P[r][2] * X[1];
      PK[r][1] = -P[r][0] * X[2] + P[r][2] * X[0];
      PK[r][2] = P[r][0] * X[1] - P[r][1] * X[0];
    }
    RR[0] += -2.0 * PK[0][0]; RR[1] += -2.0 * PK[0][1]; RR[2] += -2.0 * PK[0][2];
    RR[3] += -2.0 * PK[1][1]; RR[4] += -2.0 * PK[1][2]; RR[5] += -2.0 * PK[2][2];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) RT[3 * r + c] += P[r][c];
    TT[0] += N[0][0]; TT[1] += N[0][1]; TT[2] += N[0][2]; TT[3] += N[1][1]; TT[4] += N[1][2]; TT[5] += N[2][2];
    Xc = Xn; xy = xyn; va = van; vb = vbn; vc = vcn; pt_nxt = pt_nn;
  }
  // epilogue: the 21 sums of M (the 6 x 6 block in the sensor-camera frame) reduce-scattered, total k in lane k, and
  // lane k stores entry (r, c) of S = B^T M B with one atomic
  double vals[21];
#pragma unroll
  for (int k = 0; k < 6; ++k) vals[k] = RR[k];
#pragma unroll
  for (int k = 0; k < 9; ++k) vals[6 + k] = RT[k];
#pragma unroll
  for (int k = 0; k < 6; ++k) vals[15 + k] = TT[k];
  double s = warp_reduce_scatter(vals);
  int r, c;
  sd_entry(lane, r, c);
  if (sg.sr) {
    // known rig: S = Rb M Rb^T, Rb = blockdiag(R, R), R = R_cr^T.  Lane k forms S[r][c] from the 3 x 3 block of M
    // it needs, read from a per-warp stage.  (A trivial frame has B = I and stores M as it is.)
    __shared__ double stage[4][21];
    double* st = stage[threadIdx.x >> 5];
    if (lane < 21) st[lane] = s;
    __syncwarp();
    if (lane < 21) {
      const int rb = r - r % 3, cb = c - c % 3;
      const double* sr = sg.sr;
      double t[3];   // t_j = sum_a R[r % 3][a] M[rb + a][cb + j],  R[i][a] = sr[3a + i]
#pragma unroll
      for (int j = 0; j < 3; ++j)
        t[j] = sr[r % 3] * st[sd_value(rb, cb + j)] + sr[3 + r % 3] * st[sd_value(rb + 1, cb + j)] +
               sr[6 + r % 3] * st[sd_value(rb + 2, cb + j)];
      s = t[0] * sr[c % 3] + t[1] * sr[3 + c % 3] + t[2] * sr[6 + c % 3];
    }
  }
  const int mask = (int)(__double_as_longlong(sg.t4.w) & 0xff);
  const bool rfix = (r < 3) ? (mask & 1) : (mask & 2), cfix = (c < 3) ? (mask & 1) : (mask & 2);
  if (lane < 21 && !rfix && !cfix && s != 0.0) atomicAdd(&v.Sd[(size_t)cam * 21 + sym_idx(6, r, c)], s);
}

// ---------------------------------------------------------------------------
// pass A (point order):  s_p = [g_p] + sum_o A_o v_o,  v_o = x'_t - 2 X_p x x'_r ;  z_p = Vinv s_p
//   MODE 0: z -> z4[P][4]                      (mat-vec)
//   MODE 2: back-substitution epilogue (points_new, step scalars), as ba_schur_pass<2>
// ---------------------------------------------------------------------------
struct K3v2Smem {
  alignas(128) double At[kTile * kJpDoubles];
  double t[3][kTile + 1];
  double z[3][kTilePts + 1];
  double X[3][kTilePts + 1];
  unsigned pb[kTilePts + 1];
  double scratch[32];
  alignas(8) uint64_t mbar;
};

template <int MODE>
__global__ void __launch_bounds__(kTile, MODE == 0 ? B200_PA_MIN_CTAS : B200_K3_MIN_CTAS) ba2_pass_a(BAView v, BAViewV2 v2, const double* __restrict__ xp,
                                                                     const double* __restrict__ points,
                                                                     double* __restrict__ points_new, double radius,
                                                                     double* __restrict__ bscal,
                                                                     const PcgCtl* __restrict__ ctl) {
  extern __shared__ __align__(128) unsigned char smem_raw[];   // dynamic shared memory starts 128-B aligned (no static __shared__ in these kernels)
  if (ctl && ctl->done) return;   // the PCG stopping rule has fired: the queued iterations are no-ops
  K3v2Smem& sm = *reinterpret_cast<K3v2Smem*>(smem_raw);
  const int tile = blockIdx.x;
  const int tid = threadIdx.x;
  const int4 td = v.tile_desc[tile];
  const int p0 = td.x, npts = td.y, n = td.w;
  const unsigned o0 = (unsigned)td.z, o1 = o0 + (unsigned)n;
  const int nchunks = (n + kTile - 1) / kTile;
  constexpr uint32_t kRowBytes = kJpDoubles * 8;
  if (tid == 0) {
    mbar_init(&sm.mbar, 1);
    fence_mbar_init();
    if (n > 0) {
      const int nc0 = min(kTile, n);
      mbar_arrive_expect_tx(&sm.mbar, (uint32_t)nc0 * kRowBytes);
      tma_load_1d_stream(sm.At, v2.Ap + (size_t)o0 * kJpDoubles, (uint32_t)nc0 * kRowBytes, &sm.mbar);
    }
  }
  // prefetch the first chunk: camera index -> R^T x record, local point index
  double xr0 = 0, xr1 = 0, xr2 = 0, xt0 = 0;
  double2 xt12 = make_double2(0, 0);
  int pl_pf = 0;
  if (tid < n) {
    const int cam = ld_stream(v.obs_cam + o0 + tid);
    pl_pf = ld_stream(v.obs_pt + o0 + tid) - p0;
    ld_nc_256(xp + (size_t)cam * kXqStride, xr0, xr1, xr2, xt0);
    xt12 = __ldg(reinterpret_cast<const double2*>(xp + (size_t)cam * kXqStride + 4));
  }
  if (tid < npts) {
    sm.pb[tid] = v.pt_begin[p0 + tid];
    if (tid == npts - 1) sm.pb[npts] = o1;
#pragma unroll
    for (int k = 0; k < 3; ++k) sm.X[k][tid] = points[3 * (size_t)(p0 + tid) + k];
    sm.z[0][tid] = sm.z[1][tid] = sm.z[2][tid] = 0.0;
  }
  __syncthreads();
  uint32_t phase = 0;
  for (int ch = 0; ch < nchunks; ++ch) {
    const int c0 = ch * kTile;
    const int nc = min(kTile, n - c0);
    if (tid == 0 && ch > 0) {
      mbar_arrive_expect_tx(&sm.mbar, (uint32_t)nc * kRowBytes);
      tma_load_1d_stream(sm.At, v2.Ap + (size_t)(o0 + c0) * kJpDoubles, (uint32_t)nc * kRowBytes, &sm.mbar);
    }
    const bool active = tid < nc;
    if (active && ch > 0) {
      const int cam = ld_stream(v.obs_cam + o0 + c0 + tid);
      pl_pf = ld_stream(v.obs_pt + o0 + c0 + tid) - p0;
      ld_nc_256(xp + (size_t)cam * kXqStride, xr0, xr1, xr2, xt0);
      xt12 = __ldg(reinterpret_cast<const double2*>(xp + (size_t)cam * kXqStride + 4));
    }
    mbar_wait(&sm.mbar, phase);
    phase ^= 1;
    double t0 = 0, t1 = 0, t2 = 0;
    if (active) {
      const double2* ar = reinterpret_cast<const double2*>(sm.At + tid * kJpDoubles);
      const double2 a0 = ar[0], a1 = ar[1], a2 = ar[2];
      const double X[3] = {sm.X[0][pl_pf], sm.X[1][pl_pf], sm.X[2][pl_pf]};
      const double xr[3] = {xr0, xr1, xr2}, xt[3] = {xt0, xt12.x, xt12.y};
      const double vv[3] = {xt[0] - 2.0 * (X[1] * xr[2] - X[2] * xr[1]), xt[1] - 2.0 * (X[2] * xr[0] - X[0] * xr[2]),
                            xt[2] - 2.0 * (X[0] * xr[1] - X[1] * xr[0])};
      t0 = a0.x * vv[0] + a0.y * vv[1] + a1.x * vv[2];
      t1 = a0.y * vv[0] + a1.y * vv[1] + a2.x * vv[2];
      t2 = a1.x * vv[0] + a2.x * vv[1] + a2.y * vv[2];
    }
    // per-point sums through shared memory: thread -> (point j, component k).  (A warp-shuffle segmented
    // reduction was measured slower: SHFL shares the LSU data pipe that bounds this kernel.)
    sm.t[0][tid] = t0;
    sm.t[1][tid] = t1;
    sm.t[2][tid] = t2;
    __syncthreads();
    for (int item = tid; item < npts * 3; item += kTile) {
      const int j = item / 3, k = item - 3 * j;
      const int lo = max((int)sm.pb[j] - (int)(o0 + c0), 0), hi = min((int)sm.pb[j + 1] - (int)(o0 + c0), nc);
      double acc = 0.0;
      for (int i = lo; i < hi; ++i) acc += sm.t[k][i];
      sm.z[k][j] += acc;
    }
    __syncthreads();
  }
  double b0 = 0, b1 = 0, b2 = 0, b3 = 0;
  if (tid < npts) {
    const size_t p = (size_t)(p0 + tid);
    const bool pvalid = (int)(sm.pb[tid + 1] - sm.pb[tid]) >= v.min_views;
    double z[3] = {0.0, 0.0, 0.0};
    if (pvalid) {
      double s[3] = {sm.z[0][tid], sm.z[1][tid], sm.z[2][tid]};
      double g[3] = {0, 0, 0};
      if (MODE != 0) {
        g[0] = v.gp[3 * p]; g[1] = v.gp[3 * p + 1]; g[2] = v.gp[3 * p + 2];
        s[0] += g[0]; s[1] += g[1]; s[2] += g[2];
      }
      // 48-B rows are 16-B aligned: three 128-bit loads (8-B streaming loads would re-fetch the sector six times)
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
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double dp = -z[k];
          const double xo = sm.X[k][tid];
          points_new[3 * p + k] = xo + dp;
          b0 += g[k] * dp;
          b1 += Dp[k] * dp * dp;
          b2 += dp * dp;
          b3 += xo * xo;
        }
      }
    } else if (MODE == 2) {
#pragma unroll
      for (int k = 0; k < 3; ++k) points_new[3 * p + k] = sm.X[k][tid];
    }
    if (MODE == 0) st_keep4(v2.z4 + 4 * p, make_double4(z[0], z[1], z[2], 0.0), l2_policy_evict_last());
  }
  if (MODE == 2) {
    // step scalars: one partial row per tile (bscal = part[n_tiles][4]), column-summed by ba_colsum afterwards --
    // deterministic, and no 4 x n_tiles same-address atomics
    b0 = warp_sum(b0);
    b1 = warp_sum(b1);
    b2 = warp_sum(b2);
    b3 = warp_sum(b3);
    if ((tid & 31) == 0) {
      sm.scratch[(tid >> 5)] = b0;
      sm.scratch[4 + (tid >> 5)] = b1;
      sm.scratch[8 + (tid >> 5)] = b2;
      sm.scratch[12 + (tid >> 5)] = b3;
    }
    __syncthreads();
    if (tid < 4) {
      double a = 0.0;
#pragma unroll
      for (int w = 0; w < kTile / 32; ++w) a += sm.scratch[4 * tid + w];
      bscal[(size_t)tile * 4 + tid] = a;
    }
  }
}

// Column sums of the per-tile step scalars part[rows][4], stage 1: 4 partial sums per CTA (grid-stride over the
// rows, one 32-B load per row); stage 2 is ba_colsum over the gridDim.x partial rows.  Deterministic.
__global__ void __launch_bounds__(256) ba2_sum4_stage1(int rows, const double* __restrict__ part, double* __restrict__ out) {
  __shared__ double scratch[32];
  double a0 = 0, a1 = 0, a2 = 0, a3 = 0;
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    const double2* row = reinterpret_cast<const double2*>(part + 4 * r);
    const double2 u = row[0], w = row[1];
    a0 += u.x; a1 += u.y; a2 += w.x; a3 += w.y;
  }
  a0 = block_sum(a0, scratch);
  a1 = block_sum(a1, scratch);
  a2 = block_sum(a2, scratch);
  a3 = block_sum(a3, scratch);
  if (threadIdx.x == 0) {
    double* o = out + 4 * (size_t)blockIdx.x;
    o[0] = a0; o[1] = a1; o[2] = a2; o[3] = a3;
  }
}

// z4[p] = Vinv_p g_p   (right-hand side: no observation pass needed)
__global__ void ba2_point_rhs_z(BAView v, BAViewV2 v2) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= v.P) return;
  double vi[6], g[3], z[3];
#pragma unroll
  for (int k = 0; k < 6; ++k) vi[k] = v.Vinv[6 * (size_t)p + k];
#pragma unroll
  for (int k = 0; k < 3; ++k) g[k] = v.gp[3 * (size_t)p + k];
  sym3_mul(vi, g, z);
  const bool pvalid = (int)(v.pt_begin[p + 1] - v.pt_begin[p]) >= v.min_views;
  *reinterpret_cast<double4*>(v2.z4 + 4 * (size_t)p) = pvalid ? make_double4(z[0], z[1], z[2], 0.0) : make_double4(0, 0, 0, 0);
}

// ---------------------------------------------------------------------------
// pass B (camera order): y_c -= B^T [ 2 sum P x v ; sum v ],  v = J_pi^T a,  a = rho' J_pi Rs z_p
//                        (= [ 2 R sum (X x w) ; R sum w ] with w = A_o z_p;  NK > 0: y_k -= sum J_k^T a = sum B_o^T z_p)
// Per observation the kernel recomputes the residual (obs_core_R), streams the index and the pixel (20 B) and gathers
// two 32-B point records, X_p (pts4) and z_p (z4).
// ---------------------------------------------------------------------------
template <int NK>
__global__ void __launch_bounds__(128, B200_PB_MIN_CTAS) ba2_pass_b(BAView v, BAViewV2 v2, const double* __restrict__ cam_rec,
                                                 const double* __restrict__ intr_rec, double huber_a,
                                                 double* __restrict__ y, const PcgCtl* __restrict__ ctl, int seg_lo,
                                                 int seg_hi) {
  if (ctl && ctl->done) return;
  const int warp = seg_lo + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5);   // segments [seg_lo, seg_hi)
  const int lane = threadIdx.x & 31;
  if (warp >= seg_hi) return;
  const int cam = v.seg_cam[warp];
  const int b = v.seg_begin[warp], e = v.seg_end[warp];
  const int blk = v.seg_intr[warp];
  SegRec sg;
  seg_records(v, warp, cam, cam_rec, intr_rec, sg);
  constexpr int NKK = NK > 0 ? NK : 1;
  IntrVarRec iv{};
  if (NK > 0) iv = v2.ivar[blk];
  double acc[6] = {0, 0, 0, 0, 0, 0};   // sensor-camera frame: sum P x w, sum w
  double accK[NKK];
#pragma unroll
  for (int k = 0; k < NKK; ++k) accK[k] = 0.0;
  const uint64_t keep = l2_policy_evict_last();
  // register pipeline of ba2_linearize_cams: the index of iteration + 2 and the point, z and pixel of iteration + 1 are
  // in flight while iteration + 0 is computed
  int i = b + lane;
  int pt_nxt = 0;
  double4 X = make_double4(0, 0, 0, 0), z = X;
  double2 xy = make_double2(0, 0);
  if (i < e) {
    const int pt0 = ld_stream(v.pt_c + i);
    if (i + 32 < e) pt_nxt = ld_stream(v.pt_c + i + 32);
    X = ld_rec32(v2.pts4 + 4 * (size_t)pt0);
    z = ld_keep4(v2.z4 + 4 * (size_t)pt0, keep);
    xy = ld_stream(v.xy_c + i);
  }
  for (; i < e; i += 32) {
    double4 Xn = X, zn = z;
    double2 xyn = xy;
    int pt_nn = 0;
    if (i + 32 < e) {
      Xn = ld_rec32(v2.pts4 + 4 * (size_t)pt_nxt);
      zn = ld_keep4(v2.z4 + 4 * (size_t)pt_nxt, keep);
      xyn = ld_stream(v.xy_c + i + 32);
    }
    if (i + 64 < e) pt_nn = ld_stream(v.pt_c + i + 64);
    ObsCore o;
    obs_core_R(sg.R, sg.t4, sg.in, sg.sr, X.x, X.y, X.z, xy, huber_a, o);
    double P[3] = {o.RX[0], o.RX[1], o.RX[2]};
    to_sensor(sg.sr, P);
    // R w = J^T rho' J (R z) and R (X x w) = (R X) x (R w): w = A_o z_p is never formed in the world frame
    double r[3] = {sg.R[0] * z.x + sg.R[1] * z.y + sg.R[2] * z.z,
                   sg.R[3] * z.x + sg.R[4] * z.y + sg.R[5] * z.z,
                   sg.R[6] * z.x + sg.R[7] * z.y + sg.R[8] * z.z};
    to_sensor(sg.sr, r);
    double a[2], w[3];
    cam_frame_jac(o, r, a, w);
    acc[0] += P[1] * w[2] - P[2] * w[1];
    acc[1] += P[2] * w[0] - P[0] * w[2];
    acc[2] += P[0] * w[1] - P[1] * w[0];
    acc[3] += w[0];
    acc[4] += w[1];
    acc[5] += w[2];
    if (NK > 0) {   // B_o^T z_p = J_k^T a
      double Jk[2][NKK];
      obs_intr_jac<NK>(o, sg.in, iv, Jk);
#pragma unroll
      for (int k = 0; k < NK; ++k) accK[k] += Jk[0][k] * a[0] + Jk[1][k] * a[1];
    }
    X = Xn; z = zn; xy = xyn; pt_nxt = pt_nn;
  }
  // epilogue: one reduce-scatter of the 6 + NK sums, then one atomic per lane that holds a total
  constexpr int KV = 6 + NK, S = warp_rs_stride<KV>();
  double vals[KV];
#pragma unroll
  for (int k = 0; k < 6; ++k) vals[k] = acc[k];
#pragma unroll
  for (int k = 0; k < NK; ++k) vals[6 + k] = accK[k];
  double s = warp_reduce_scatter(vals);
  const int k = lane / S;
  if (sg.sr) {   // B^T of a known rig: dof k mixes the three totals of its half, read from a per-warp stage
    __shared__ double stage[4][6];
    double* st = stage[threadIdx.x >> 5];
    if (lane % S == 0 && k < 6) st[k] = s;
    __syncwarp();
    if (k < 6) {
      const int c = k % 3, h = k - c;
      s = sg.sr[c] * st[h] + sg.sr[3 + c] * st[h + 1] + sg.sr[6 + c] * st[h + 2];
    }
  }
  const int mask = (int)(__double_as_longlong(sg.t4.w) & 0xff);
  const bool fixed = k < 3 ? (mask & 1) : k < 6 ? (mask & 2) : false;
  if (lane % S == 0 && k < KV && !fixed && s != 0.0) {
    double* dst = k < 6 ? &y[(size_t)cam * 6 + k] : &y[(size_t)(v2.C + blk) * 6 + (k - 6)];
    atomicAdd(dst, k < 3 ? -(2.0 * s) : -s);
  }
}

// x_k of every image's intrinsics block into the two spare doubles of its xq row (pass A gathers ONE 64-B record)
__global__ void ba2k_pack_xk(int C, const double* __restrict__ cam_rec, const double* __restrict__ x, double* __restrict__ xp,
                             const PcgCtl* __restrict__ ctl) {
  if (ctl && ctl->done) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int blk = (int)(__double_as_longlong(cam_rec[(size_t)c * kCamRec + 7]) >> 8);
  xp[(size_t)c * kXqStride + 6] = x[(size_t)(C + blk) * 6];
  xp[(size_t)c * kXqStride + 7] = x[(size_t)(C + blk) * 6 + 1];
}

// frame x intrinsics coupling of U x:  y_f += U_fk x_k,  y_k += U_fk^T x_f   (one thread per image; the y_k sums of a
// CTA are combined in shared memory when the blocks fit, so a single shared camera costs one atomic per CTA and dof)
template <int NK>
__global__ void __launch_bounds__(256) ba2k_cross(int C, int K, const double* __restrict__ cam_rec, const double* __restrict__ Ufk,
                                                  const double* __restrict__ x, double* __restrict__ y,
                                                  const PcgCtl* __restrict__ ctl) {
  constexpr int kBins = 256;
  __shared__ double bins[kBins * NK];
  if (ctl && ctl->done) return;
  const bool use_bins = K <= kBins;
  if (use_bins) {
    for (int i = threadIdx.x; i < K * NK; i += blockDim.x) bins[i] = 0.0;
    __syncthreads();
  }
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    const int blk = (int)(__double_as_longlong(cam_rec[(size_t)c * kCamRec + 7]) >> 8);
    double xf[6], xk[NK], tk[NK];
#pragma unroll
    for (int i = 0; i < 6; ++i) xf[i] = x[(size_t)c * 6 + i];
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      xk[k] = x[(size_t)(C + blk) * 6 + k];
      tk[k] = 0.0;
    }
    const double* u = Ufk + (size_t)c * 6 * NK;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      double yf = 0.0;
#pragma unroll
      for (int k = 0; k < NK; ++k) {
        const double uik = u[i * NK + k];
        yf += uik * xk[k];
        tk[k] += uik * xf[i];
      }
      // plain read-modify-write: this thread owns y_f of its image, and pass B, which adds to y_f with atomics, is
      // launched after this kernel on the same stream
      if (yf != 0.0) y[(size_t)c * 6 + i] += yf;
    }
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      if (tk[k] == 0.0) continue;
      if (use_bins) atomicAdd(&bins[blk * NK + k], tk[k]);
      else atomicAdd(&y[(size_t)(C + blk) * 6 + k], tk[k]);
    }
  }
  if (use_bins) {
    __syncthreads();
    for (int i = threadIdx.x; i < K * NK; i += blockDim.x)
      if (bins[i] != 0.0) atomicAdd(&y[(size_t)(C + i / NK) * 6 + (i % NK)], bins[i]);
  }
}

}  // namespace b200
