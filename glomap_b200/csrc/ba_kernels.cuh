// ba_kernels.cuh -- bundle-adjustment kernels (sm_90a).
//
// Replaces the arithmetic Ceres performs for glomap::BundleAdjuster
// (reference: glomap/estimators/bundle_adjustment.cc:99,115-190,244-317):
// per-observation reprojection residual + analytic 2x(6+3) Jacobian, Huber
// corrector, per-point 3x3 Schur marginalisation, implicit-Schur mat-vec.
//
// Data layout in HBM (FP64, DESIGN.md "BA layout"):
//   observations in POINT order (CSR by point): obs_cam[N], obs_pt[N], obs_xy[N]
//   W[N][18]   (design v1) 6x3 block J_cam^T J_pt of every observation, AoS (144-B rows) so
//              that a tile of kTile = 128 consecutive observations is one contiguous
//              18,432-B chunk moved by a single TMA bulk copy; design v2 (ba_kernels_v2.cuh,
//              the default with constant intrinsics) stores 48-B A_o rows in the same buffer
//   V[P][6], Vinv[P][6], gp[P][3]         per point (packed symmetric)
//   U[C][21], gc[C][6], Sd[C][21], Minv[C][21]   per camera (packed symmetric)
//   camera-order copies pt_c[Nv], xy_c[Nv], camord_obs[Nv] + segments (about kSeg = 256, fewer than 1.5 kSeg,
//   observations of ONE camera -- or of one (frame, sensor) with known rigs -- handled by one warp)
// Point-order kernels run one CTA (kTile = 128 threads) per tile of whole points with
// <= 128 observations (longer tracks: several chunks); one thread per observation, per-point
// reductions through shared memory.
#pragma once
#include "common.cuh"
#include "pcg.cuh"

namespace b200 {

constexpr int kCamRec = 8;    // q(4) t(3) packed{mask, intr idx}
constexpr int kIntrRec = 8;   // fx fy cx cy k1 k2 model pad
constexpr double kZEps = 1e-12;
constexpr int kSeg = 256;     // observations per camera-order segment (one warp), nominal: see seg_split
// Number of camera-order segments of a bucket of n observations: n / kSeg rounded to the nearest (at least one), of
// equal length (so all are shorter than 1.5 kSeg).  Every segment costs its warp the camera records, a shuffle
// reduction and the atomics, and cutting at every kSeg would leave a warp only the few observations past a multiple of
// kSeg (at config 4, where a (slice, camera) bucket holds 250 +- 16, a quarter of the segments would be such tails).
__host__ __device__ constexpr int seg_split(int n) { return n <= 0 ? 0 : (n < kSeg + kSeg / 2 ? 1 : (n + kSeg / 2) / kSeg); }
constexpr int kIntrSmem = 16; // intrinsics blocks cached in shared memory by the point-order kernels
constexpr int kJpDoubles = 6;  // v2 point-order row: A_o = J_pt^T J_pt (packed symmetric 3x3) -> 48 B
constexpr int kSensorRec = 16; // known rigs: R_cam_from_rig (9, row-major), t_cam_from_rig (3), intrinsics idx, pad

struct BAView {
  int C, P, K;
  long long N;
  int n_tiles;
  int n_segs;
  int min_views;
  // structure
  const int* obs_cam;
  const int* obs_pt;
  const double2* obs_xy;
  const unsigned* pt_begin;     // [P+1]
  const int* tile_pt_begin;     // [n_tiles+1]
  const int4* tile_desc;        // [n_tiles] {first point, #points, first observation, #observations}
  const int* camord_obs;        // [Nv] observation ids sorted by camera
  const int* pt_c;              // [Nv]
  const double2* xy_c;          // [Nv]
  const int* seg_cam;           // [n_segs]
  const int* seg_begin;         // [n_segs+1] (only within one camera: seg_end = seg_begin2[s])
  const int* seg_end;
  // known (constant) rigs -- bundle_adjustment.cc:147-161.  S == 0: every frame is trivial, obs_cam is the
  // image and the intrinsics index rides in the camera record.  S > 0: obs_cam is the FRAME (rig_from_world),
  // obs_sensor picks the constant cam_from_rig + intrinsics of the observing image; camera-order segments
  // are homogeneous in (frame, sensor).
  int S;
  const unsigned short* obs_sensor;   // [N]
  const int* seg_sensor;              // [n_segs]
  const int* seg_intr;                // [n_segs] intrinsics block of the segment (always filled)
  const double* sensor_rec;           // [S][kSensorRec]
  // linear system
  double* W;
  double* V;
  double* Vinv;
  double* gp;
  double* U;
  double* gc;
  double* Sd;
  double* Minv;
  double* jscale_c;
  double* jscale_p;
  double* Dc;
};

// Huber (Ceres HuberLoss): returns rho'(s) and rho(s)
__device__ __forceinline__ void huber(double s, double a, double& rho0, double& rho1) {
  const double b = a * a;
  if (s > b) {
    const double r = sqrt(s);
    rho0 = 2.0 * a * r - b;
    rho1 = fmax(2.2250738585072014e-308, a / r);
  } else {
    rho0 = s;
    rho1 = 1.0;
  }
}

// Values of an intrinsics record (fx fy cx cy k1 k2 model).  The camera-order kernels load it once per segment.
struct Intr {
  double fx, fy, cx, cy, k1, k2;
  int model;
};
__device__ __forceinline__ Intr ld_intr(const double* __restrict__ ir) {
  return Intr{ir[0], ir[1], ir[2], ir[3], ir[4], ir[5], (int)ir[6]};
}

// Projection Jacobian in factored form:  d(px,py)/d(Xc) = iz M [I | -(u, v)^T],  M = d(pixel)/d(u, v)  (2x2;
// diag(fx, fy) for the pinhole models).
struct ProjJac {
  double iz, u, v, m00, m01, m10, m11;
};

// Pixel projection.  Records with k1 == k2 == 0 (SIMPLE_PINHOLE, PINHOLE) take the pinhole form; the others the
// generic radial form (simple models have fx = fy).  project_only computes the pixel with the same instructions.
__device__ __forceinline__ void project_jac(const Intr& in, double x, double y, double z, double& px, double& py,
                                            ProjJac& pj) {
  const double iz = 1.0 / z;
  const double u = x * iz, v = y * iz;
  pj.iz = iz;
  pj.u = u;
  pj.v = v;
  if (in.k1 == 0.0 && in.k2 == 0.0) {
    px = in.fx * u + in.cx;
    py = in.fy * v + in.cy;
    pj.m00 = in.fx; pj.m01 = 0.0; pj.m10 = 0.0; pj.m11 = in.fy;
  } else {
    const double r2 = u * u + v * v;
    const double d = 1.0 + r2 * (in.k1 + in.k2 * r2);
    const double dd = in.k1 + 2.0 * in.k2 * r2;
    px = in.fx * u * d + in.cx;
    py = in.fy * v * d + in.cy;
    const double a00 = d + 2.0 * u * u * dd, a01 = 2.0 * u * v * dd, a11 = d + 2.0 * v * v * dd;
    pj.m00 = in.fx * a00; pj.m01 = in.fx * a01; pj.m10 = in.fy * a01; pj.m11 = in.fy * a11;
  }
}
__device__ __forceinline__ void project_only(const Intr& in, double x, double y, double z, double& px, double& py) {
  const double iz = 1.0 / z;
  const double u = x * iz, v = y * iz;
  if (in.k1 == 0.0 && in.k2 == 0.0) {
    px = in.fx * u + in.cx;
    py = in.fy * v + in.cy;
  } else {
    const double r2 = u * u + v * v;
    const double d = 1.0 + r2 * (in.k1 + in.k2 * r2);
    px = in.fx * u * d + in.cx;
    py = in.fy * v * d + in.cy;
  }
}
// J = d(px,py)/d(Xc) row-major 2x3 from the factored form
__device__ __forceinline__ void proj_jac_rows(const ProjJac& pj, double J[6]) {
  J[0] = pj.m00 * pj.iz;
  J[1] = pj.m01 * pj.iz;
  J[2] = -(J[0] * pj.u + J[1] * pj.v);
  J[3] = pj.m10 * pj.iz;
  J[4] = pj.m11 * pj.iz;
  J[5] = -(J[3] * pj.u + J[4] * pj.v);
}
__device__ __forceinline__ void project_jac(const double* __restrict__ ir, double x, double y, double z, double& px,
                                            double& py, double J[6]) {
  ProjJac pj;
  project_jac(ld_intr(ir), x, y, z, px, py, pj);
  proj_jac_rows(pj, J);
}
__device__ __forceinline__ void project_only(const double* __restrict__ ir, double x, double y, double z, double& px,
                                             double& py) {
  project_only(ld_intr(ir), x, y, z, px, py);
}

// Everything one observation contributes.  Jc = [Jrot(2x3) | Jtrn(2x3)] and
// Jp (2x3), already scaled by sqrt(rho') and masked; r scaled by sqrt(rho').
struct ObsLin {
  double Jr[6], Jt[6], Jp[6], r[2], rho0;
  double u, v, w;   // normalised image coordinates and sqrt(rho') (for the intrinsics Jacobian)
  bool valid;
};

__device__ __forceinline__ int cam_rec_intr(const double4& t4) { return (int)(__double_as_longlong(t4.w) >> 8); }

// camera-frame point of a known-rig image: X_c = R_cr X_f + t_cr
__device__ __forceinline__ void sensor_apply(const double* __restrict__ sr, double& x, double& y, double& z) {
  const double a = sr[0] * x + sr[1] * y + sr[2] * z + sr[9];
  const double b = sr[3] * x + sr[4] * y + sr[5] * z + sr[10];
  const double c = sr[6] * x + sr[7] * y + sr[8] * z + sr[11];
  x = a; y = b; z = c;
}
__device__ __forceinline__ int obs_intr_idx(const double4& t4, const double* __restrict__ sr) {
  return sr ? (int)sr[12] : cam_rec_intr(t4);
}
__device__ __forceinline__ const double* sensor_of_obs(const BAView& v, long long o) {
  return v.S > 0 ? v.sensor_rec + (size_t)v.obs_sensor[o] * kSensorRec : nullptr;
}
__device__ __forceinline__ const double* sensor_of_seg(const BAView& v, int seg) {
  return v.S > 0 ? v.sensor_rec + (size_t)v.seg_sensor[seg] * kSensorRec : nullptr;
}

// q4/t4 = the camera (frame) record (already loaded), ir = the intrinsics record of the observing image,
// sr = its sensor record (nullptr: trivial frame, cam_from_rig = identity)
__device__ __forceinline__ void linearize_obs(const double4& q4, const double4& t4, const double* __restrict__ ir,
                                              const double* __restrict__ sr,
                                              double X0, double X1, double X2, double2 xy, double huber_a, ObsLin& o) {
  const long long packed = __double_as_longlong(t4.w);
  const int mask = (int)(packed & 0xff);
  const double q[4] = {q4.x, q4.y, q4.z, q4.w};
  double R[9];
  quat_to_R(q, R);
  const double rx = R[0] * X0 + R[1] * X1 + R[2] * X2;
  const double ry = R[3] * X0 + R[4] * X1 + R[5] * X2;
  const double rz = R[6] * X0 + R[7] * X1 + R[8] * X2;
  double xc = rx + t4.x, yc = ry + t4.y, zc = rz + t4.z;
  if (sr) sensor_apply(sr, xc, yc, zc);
  o.valid = zc > kZEps;
  if (!o.valid) {
#pragma unroll
    for (int k = 0; k < 6; ++k) o.Jr[k] = o.Jt[k] = o.Jp[k] = 0.0;
    o.r[0] = o.r[1] = 0.0;
    o.rho0 = 0.0;
    o.u = o.v = o.w = 0.0;
    return;
  }
  double px, py, J[6];
  project_jac(ir, xc, yc, zc, px, py, J);
  if (sr) {   // chain through the constant cam_from_rig rotation: J <- J R_cr
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const double j0 = J[3 * a], j1 = J[3 * a + 1], j2 = J[3 * a + 2];
      J[3 * a] = j0 * sr[0] + j1 * sr[3] + j2 * sr[6];
      J[3 * a + 1] = j0 * sr[1] + j1 * sr[4] + j2 * sr[7];
      J[3 * a + 2] = j0 * sr[2] + j1 * sr[5] + j2 * sr[8];
    }
  }
  o.u = xc / zc;
  o.v = yc / zc;
  const double r0 = px - xy.x, r1 = py - xy.y;
  double rho1;
  huber(r0 * r0 + r1 * r1, huber_a, o.rho0, rho1);
  const double w = sqrt(rho1);
  o.w = w;
  o.r[0] = w * r0;
  o.r[1] = w * r1;
#pragma unroll
  for (int k = 0; k < 6; ++k) J[k] *= w;
  // translation block
  const bool tvar = !(mask & 2), rvar = !(mask & 1);
#pragma unroll
  for (int k = 0; k < 6; ++k) o.Jt[k] = tvar ? J[k] : 0.0;
  // rotation block: J * (-2 [RX]x)   (EigenQuaternionManifold: left perturbation of angle 2|d|)
  // [v]x = [0 -vz vy; vz 0 -vx; -vy vx 0];  J*(-2[v]x) columns:
  //   col0 = -2*( J1*vz - J2*vy ), col1 = -2*( -J0*vz + J2*vx ), col2 = -2*( J0*vy - J1*vx )
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const double j0 = J[3 * a], j1 = J[3 * a + 1], j2 = J[3 * a + 2];
    o.Jr[3 * a + 0] = rvar ? -2.0 * (j1 * rz - j2 * ry) : 0.0;
    o.Jr[3 * a + 1] = rvar ? -2.0 * (j2 * rx - j0 * rz) : 0.0;
    o.Jr[3 * a + 2] = rvar ? -2.0 * (j0 * ry - j1 * rx) : 0.0;
  }
  // point block: J * R
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) o.Jp[3 * a + b] = J[3 * a] * R[b] + J[3 * a + 1] * R[3 + b] + J[3 * a + 2] * R[6 + b];
}

// Lean per-observation core of design v2 (both traversal orders): everything downstream is rho' * (unscaled
// Jacobian products), so sqrt(rho') is never formed -- one reciprocal and, for outliers only, one rsqrt:
//   J   = d(pixel)/d(X_frame)  2x3, unscaled (chained through the constant cam_from_rig of a known rig)
//   e   = pixel residual, rho0 = rho(|e|^2), rho1 = rho'(|e|^2)  (Huber; corrector with rho'' <= 0 => rows * sqrt(rho'))
//   RX  = R X (the rotated point, for the rotation block), R = R(q)
// valid == false (point behind the camera): the observation contributes nothing (ObsLin convention).
//   pj  = the factored projection Jacobian (camera-order kernels work with it in the camera frame; J is then dead code)
struct ObsCore {
  double J[6], e[2], rho0, rho1, RX[3], R[9];
  double uv[2];   // normalised image coordinates (only read by the intrinsics rows: dead code elsewhere)
  ProjJac pj;
  bool valid;
};
// R = R(q) of the camera (frame) record, computed by the caller (once per segment in camera order)
__device__ __forceinline__ void obs_core_R(const double R[9], const double4& t4, const Intr& in,
                                           const double* __restrict__ sr, double X0, double X1, double X2, double2 xy,
                                           double huber_a, ObsCore& o) {
#pragma unroll
  for (int k = 0; k < 9; ++k) o.R[k] = R[k];
  o.RX[0] = o.R[0] * X0 + o.R[1] * X1 + o.R[2] * X2;
  o.RX[1] = o.R[3] * X0 + o.R[4] * X1 + o.R[5] * X2;
  o.RX[2] = o.R[6] * X0 + o.R[7] * X1 + o.R[8] * X2;
  double xc = o.RX[0] + t4.x, yc = o.RX[1] + t4.y, zc = o.RX[2] + t4.z;
  if (sr) sensor_apply(sr, xc, yc, zc);
  o.valid = zc > kZEps;
  if (!o.valid) {
#pragma unroll
    for (int k = 0; k < 6; ++k) o.J[k] = 0.0;
    o.e[0] = o.e[1] = 0.0;
    o.rho0 = 0.0;
    o.rho1 = 0.0;
    o.uv[0] = o.uv[1] = 0.0;
    o.pj = ProjJac{0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    return;
  }
  double px, py;
  project_jac(in, xc, yc, zc, px, py, o.pj);
  proj_jac_rows(o.pj, o.J);
  o.uv[0] = xc / zc;
  o.uv[1] = yc / zc;
  if (sr) {   // chain through the constant cam_from_rig rotation: J <- J R_cr
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const double j0 = o.J[3 * a], j1 = o.J[3 * a + 1], j2 = o.J[3 * a + 2];
      o.J[3 * a] = j0 * sr[0] + j1 * sr[3] + j2 * sr[6];
      o.J[3 * a + 1] = j0 * sr[1] + j1 * sr[4] + j2 * sr[7];
      o.J[3 * a + 2] = j0 * sr[2] + j1 * sr[5] + j2 * sr[8];
    }
  }
  o.e[0] = px - xy.x;
  o.e[1] = py - xy.y;
  const double s = o.e[0] * o.e[0] + o.e[1] * o.e[1];
  const double b = huber_a * huber_a;
  if (s > b) {   // Ceres HuberLoss: rho = 2 a sqrt(s) - a^2, rho' = a / sqrt(s)
    const double t = rsqrt(s);
    o.rho1 = fmax(2.2250738585072014e-308, huber_a * t);
    o.rho0 = 2.0 * huber_a * (s * t) - b;
  } else {
    o.rho0 = s;
    o.rho1 = 1.0;
  }
}
__device__ __forceinline__ void obs_core(const double4& q4, const double4& t4, const double* __restrict__ ir,
                                         const double* __restrict__ sr, double X0, double X1, double X2, double2 xy,
                                         double huber_a, ObsCore& o) {
  const double q[4] = {q4.x, q4.y, q4.z, q4.w};
  double R[9];
  quat_to_R(q, R);
  obs_core_R(R, t4, ld_intr(ir), sr, X0, X1, X2, xy, huber_a, o);
}
// point block J_pt = J R (2x3, unscaled) -> A = rho' J_pt^T J_pt (packed symmetric), b = rho' J_pt^T e
__device__ __forceinline__ void obs_point_blocks(const ObsCore& o, double Jp[6], double A[6], double b[3]) {
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) Jp[3 * a + c] = o.J[3 * a] * o.R[c] + o.J[3 * a + 1] * o.R[3 + c] + o.J[3 * a + 2] * o.R[6 + c];
  const double s0 = o.rho1 * Jp[0], s1 = o.rho1 * Jp[1], s2 = o.rho1 * Jp[2];
  const double s3 = o.rho1 * Jp[3], s4 = o.rho1 * Jp[4], s5 = o.rho1 * Jp[5];
  A[0] = s0 * Jp[0] + s3 * Jp[3];
  A[1] = s0 * Jp[1] + s3 * Jp[4];
  A[2] = s0 * Jp[2] + s3 * Jp[5];
  A[3] = s1 * Jp[1] + s4 * Jp[4];
  A[4] = s1 * Jp[2] + s4 * Jp[5];
  A[5] = s2 * Jp[2] + s5 * Jp[5];
  b[0] = s0 * o.e[0] + s3 * o.e[1];
  b[1] = s1 * o.e[0] + s4 * o.e[1];
  b[2] = s2 * o.e[0] + s5 * o.e[1];
}

// ---------------------------------------------------------------------------
// camera / intrinsics records
// ---------------------------------------------------------------------------
__global__ void ba_build_records(int C, int K, const double* __restrict__ quat, const double* __restrict__ trans,
                                 const int* __restrict__ cam_intr, const unsigned char* __restrict__ cam_mask,
                                 const double* __restrict__ intr, const int* __restrict__ intr_model,
                                 double* __restrict__ cam_rec, double* __restrict__ intr_rec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < C) {
    double* r = cam_rec + (size_t)i * kCamRec;
    r[0] = quat[4 * i];
    r[1] = quat[4 * i + 1];
    r[2] = quat[4 * i + 2];
    r[3] = quat[4 * i + 3];
    r[4] = trans[3 * i];
    r[5] = trans[3 * i + 1];
    r[6] = trans[3 * i + 2];
    const long long packed = ((long long)cam_intr[i] << 8) | (long long)cam_mask[i];
    r[7] = __longlong_as_double(packed);
  }
  if (i < K) {
    const double* p = intr + (size_t)i * 12;
    double* r = intr_rec + (size_t)i * kIntrRec;
    const int m = intr_model[i];
    double fx, fy, cx, cy, k1 = 0, k2 = 0;
    if (m == 0) { fx = fy = p[0]; cx = p[1]; cy = p[2]; }
    else if (m == 1) { fx = p[0]; fy = p[1]; cx = p[2]; cy = p[3]; }
    else if (m == 2) { fx = fy = p[0]; cx = p[1]; cy = p[2]; k1 = p[3]; }
    else { fx = fy = p[0]; cx = p[1]; cy = p[2]; k1 = p[3]; k2 = p[4]; }
    r[0] = fx; r[1] = fy; r[2] = cx; r[3] = cy; r[4] = k1; r[5] = k2; r[6] = (double)m; r[7] = 0;
  }
}

// ---------------------------------------------------------------------------
// K1: Jacobian + point Schur blocks, point order.  scal[0] += cost,
// scal[1] = max |g_p|
// ---------------------------------------------------------------------------
struct K1Smem {
  alignas(128) double Wt[kTile * kWDoubles];
  double red[9][kTile + 1];  // +1: rows land in different banks for the (point, component) reduction
  double acc[9][kTilePts + 1];   // per-point sums (V packed 6 + g 3)
  unsigned pb[kTilePts + 1]; // observation range of each point of the tile
  double X[3][kTilePts + 1]; // the tile's points
  double intr[kIntrSmem][kIntrRec];   // intrinsics table (first kIntrSmem blocks)
  double scratch[32];
};

// V2 = false: writes W[N][18] (6x3 blocks).  V2 = true: writes the compact rows Ap[N][6] = J_pt^T J_pt
// of the world-frame layout (ba_kernels_v2.cuh) into v.W instead.
template <bool V2>
__global__ void __launch_bounds__(kTile, B200_K1_MIN_CTAS) ba_linearize_points(BAView v, const double* __restrict__ cam_rec,
                                                             const double* __restrict__ intr_rec,
                                                             const double* __restrict__ points, double huber_a,
                                                             int points_var, double* __restrict__ scal) {
  extern __shared__ __align__(128) unsigned char smem_raw[];   // dynamic shared memory starts 128-B aligned (no static __shared__ in these kernels)
  K1Smem& sm = *reinterpret_cast<K1Smem*>(smem_raw);
  const int tile = blockIdx.x;
  const int tid = threadIdx.x;
  // one 16-B descriptor per tile: the dependent-load chain is descriptor -> {observations, points} -> camera record
  const int4 td = v.tile_desc[tile];
  const int p0 = td.x, npts = td.y, n = td.w;
  const unsigned o0 = (unsigned)td.z;
  // prefetch the first chunk's observation + its camera record before the shared-memory fill / barrier
  int cam_pf = 0, pt_pf = 0;
  double2 xy_pf = make_double2(0.0, 0.0);
  double4 q4_pf = make_double4(0, 0, 0, 1), t4_pf = make_double4(0, 0, 0, 0);
  const double* sr_pf = nullptr;
  if (tid < n) {
    cam_pf = v.obs_cam[o0 + tid];
    xy_pf = v.obs_xy[o0 + tid];
    pt_pf = v.obs_pt[o0 + tid];
    q4_pf = *reinterpret_cast<const double4*>(cam_rec + (size_t)cam_pf * kCamRec);
    t4_pf = *reinterpret_cast<const double4*>(cam_rec + (size_t)cam_pf * kCamRec + 4);
    sr_pf = sensor_of_obs(v, o0 + tid);
  }
  for (int i = tid; i < min(v.K, kIntrSmem) * kIntrRec; i += kTile) (&sm.intr[0][0])[i] = intr_rec[i];
  // per-point accumulators live in shared memory (thread j <-> point p0 + j)
  unsigned pb = 0, pe = 0;
  bool pvalid = false;
  if (tid < npts) {
    pb = v.pt_begin[p0 + tid];
    pe = v.pt_begin[p0 + tid + 1];
    pvalid = (int)(pe - pb) >= v.min_views;
    sm.pb[tid] = pb;
    if (tid == npts - 1) sm.pb[npts] = pe;
#pragma unroll
    for (int k = 0; k < 3; ++k) sm.X[k][tid] = points[3 * (size_t)(p0 + tid) + k];
#pragma unroll
    for (int k = 0; k < 9; ++k) sm.acc[k][tid] = 0.0;
  }
  __syncthreads();
  double cost = 0.0;
  for (int c0 = 0; c0 < n; c0 += kTile) {
    const int nc = min(kTile, n - c0);
    const bool active = tid < nc;
    ObsLin o;
    bool use = false;
    if (active) {
      if (c0 > 0) {   // multi-chunk tiles (one track longer than the tile) reload per chunk
        const unsigned oi = o0 + c0 + tid;
        cam_pf = v.obs_cam[oi];
        xy_pf = v.obs_xy[oi];
        pt_pf = v.obs_pt[oi];
        q4_pf = *reinterpret_cast<const double4*>(cam_rec + (size_t)cam_pf * kCamRec);
        t4_pf = *reinterpret_cast<const double4*>(cam_rec + (size_t)cam_pf * kCamRec + 4);
        sr_pf = sensor_of_obs(v, oi);
      }
      const int pl = pt_pf - p0;     // point index within the tile: X and validity come from smem
      use = (int)(sm.pb[pl + 1] - sm.pb[pl]) >= v.min_views;
      if (use) {
        const double X0 = sm.X[0][pl], X1 = sm.X[1][pl], X2 = sm.X[2][pl];
        const int intr = obs_intr_idx(t4_pf, sr_pf);
        const double* ir = intr < kIntrSmem ? sm.intr[intr] : intr_rec + (size_t)intr * kIntrRec;
        linearize_obs(q4_pf, t4_pf, ir, sr_pf, X0, X1, X2, xy_pf, huber_a, o);
        cost += 0.5 * o.rho0;
      }
    }
    if (!use) {
#pragma unroll
      for (int k = 0; k < 6; ++k) o.Jr[k] = o.Jt[k] = o.Jp[k] = 0.0;
      o.r[0] = o.r[1] = 0.0;
    }
    if (points_var) {
      if (V2) {
        // compact row A_o = J_pt^T J_pt (packed symmetric 3x3, 48 B: every tile is a legal TMA bulk copy)
        double* arow = sm.Wt + tid * kJpDoubles;
        arow[0] = o.Jp[0] * o.Jp[0] + o.Jp[3] * o.Jp[3];
        arow[1] = o.Jp[0] * o.Jp[1] + o.Jp[3] * o.Jp[4];
        arow[2] = o.Jp[0] * o.Jp[2] + o.Jp[3] * o.Jp[5];
        arow[3] = o.Jp[1] * o.Jp[1] + o.Jp[4] * o.Jp[4];
        arow[4] = o.Jp[1] * o.Jp[2] + o.Jp[4] * o.Jp[5];
        arow[5] = o.Jp[2] * o.Jp[2] + o.Jp[5] * o.Jp[5];
      } else {
        // W = [Jr^T; Jt^T] Jp  (6x3), rows of 3 -> smem tile (stride 144 B: conflict-free STS.128)
        double* wrow = sm.Wt + tid * kWDoubles;
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int b = 0; b < 3; ++b) {
            wrow[3 * a + b] = o.Jr[a] * o.Jp[b] + o.Jr[3 + a] * o.Jp[3 + b];
            wrow[9 + 3 * a + b] = o.Jt[a] * o.Jp[b] + o.Jt[3 + a] * o.Jp[3 + b];
          }
      }
      // V_o (packed sym) and g_o
      sm.red[0][tid] = o.Jp[0] * o.Jp[0] + o.Jp[3] * o.Jp[3];
      sm.red[1][tid] = o.Jp[0] * o.Jp[1] + o.Jp[3] * o.Jp[4];
      sm.red[2][tid] = o.Jp[0] * o.Jp[2] + o.Jp[3] * o.Jp[5];
      sm.red[3][tid] = o.Jp[1] * o.Jp[1] + o.Jp[4] * o.Jp[4];
      sm.red[4][tid] = o.Jp[1] * o.Jp[2] + o.Jp[4] * o.Jp[5];
      sm.red[5][tid] = o.Jp[2] * o.Jp[2] + o.Jp[5] * o.Jp[5];
      sm.red[6][tid] = o.Jp[0] * o.r[0] + o.Jp[3] * o.r[1];
      sm.red[7][tid] = o.Jp[1] * o.r[0] + o.Jp[4] * o.r[1];
      sm.red[8][tid] = o.Jp[2] * o.r[0] + o.Jp[5] * o.r[1];
      fence_proxy_async_smem();
      __syncthreads();
      if (tid == 0) {
        if (V2) tma_store_1d(v.W + (size_t)(o0 + c0) * kJpDoubles, sm.Wt, (uint32_t)nc * kJpDoubles * 8);
        else tma_store_1d(v.W + (size_t)(o0 + c0) * kWDoubles, sm.Wt, (uint32_t)nc * kWBytes);
        tma_store_commit();
      }
      // per-point sums: thread -> (point j, component k), 9 threads per point
      for (int item = tid; item < npts * 9; item += kTile) {
        const int j = item / 9, k = item - 9 * j;
        const int lo = max((int)sm.pb[j] - (int)(o0 + c0), 0), hi = min((int)sm.pb[j + 1] - (int)(o0 + c0), nc);
        double a = 0.0;
        for (int i = lo; i < hi; ++i) a += sm.red[k][i];
        sm.acc[k][j] += a;
      }
      if (tid == 0) tma_store_wait_read();
      __syncthreads();
    }
  }
  double gmax = 0.0;
  if (points_var && tid < npts) {
    const size_t p = (size_t)(p0 + tid);
    if (pvalid) {
#pragma unroll
      for (int k = 0; k < 6; ++k) v.V[6 * p + k] = sm.acc[k][tid];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double gk = sm.acc[6 + k][tid];
        v.gp[3 * p + k] = gk;
        gmax = fmax(gmax, fabs(gk));
      }
    } else {
#pragma unroll
      for (int k = 0; k < 6; ++k) v.V[6 * p + k] = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) v.gp[3 * p + k] = 0.0;
    }
  }
  cost = block_sum(cost, sm.scratch);
  if (tid == 0 && cost != 0.0) atomicAdd(&scal[0], cost);
  gmax = block_max(gmax, sm.scratch);
  if (tid == 0 && gmax > 0.0) atomic_max_nonneg(&scal[1], gmax);
}

// ---------------------------------------------------------------------------
// K2a: camera blocks U = sum Jc^T Jc (packed 21), gc = sum Jc^T r, camera order.
// One warp per segment (one camera's observations, see seg_split).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) ba_linearize_cams(BAView v, const double* __restrict__ cam_rec,
                                                        const double* __restrict__ intr_rec,
                                                        const double* __restrict__ points, double huber_a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= v.n_segs) return;
  const int cam = v.seg_cam[warp];
  const int b = v.seg_begin[warp], e = v.seg_end[warp];
  const double4 q4c = *reinterpret_cast<const double4*>(cam_rec + (size_t)cam * kCamRec);
  const double4 t4c = *reinterpret_cast<const double4*>(cam_rec + (size_t)cam * kCamRec + 4);
  const double* irc = intr_rec + (size_t)v.seg_intr[warp] * kIntrRec;
  const double* src = sensor_of_seg(v, warp);
  double U[21], g[6];
#pragma unroll
  for (int k = 0; k < 21; ++k) U[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) g[k] = 0.0;
  for (int i = b + lane; i < e; i += 32) {
    const int pt = v.pt_c[i];
    const double2 xy = v.xy_c[i];
    const double X0 = points[3 * (size_t)pt], X1 = points[3 * (size_t)pt + 1], X2 = points[3 * (size_t)pt + 2];
    ObsLin o;
    linearize_obs(q4c, t4c, irc, src, X0, X1, X2, xy, huber_a, o);
    double Jc[2][6];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        Jc[a][k] = o.Jr[3 * a + k];
        Jc[a][3 + k] = o.Jt[3 * a + k];
      }
    int idx = 0;
#pragma unroll
    for (int i2 = 0; i2 < 6; ++i2) {
#pragma unroll
      for (int j = i2; j < 6; ++j) U[idx++] += Jc[0][i2] * Jc[0][j] + Jc[1][i2] * Jc[1][j];
      g[i2] += Jc[0][i2] * o.r[0] + Jc[1][i2] * o.r[1];
    }
  }
#pragma unroll
  for (int k = 0; k < 21; ++k) {
    const double s = warp_sum(U[k]);
    if (lane == k && s != 0.0) atomicAdd(&v.U[(size_t)cam * 21 + k], s);
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const double s = warp_sum(g[k]);
    if (lane == 21 + k && s != 0.0) atomicAdd(&v.gc[(size_t)cam * 6 + k], s);
  }
}

// After the (all-)reduction of U/gc: masked or unobserved dofs become identity
// rows, Jacobi scaling is fixed at the first linearisation, max|gc| -> scal[1].
__global__ void ba_finalize_cams(int C, double* __restrict__ U, double* __restrict__ gc,
                                 const unsigned char* __restrict__ cam_mask, double* __restrict__ jscale_c,
                                 int set_jscale, double* __restrict__ scal, const double* __restrict__ gslots, int nslots) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  double gmax = 0.0;
  // per-rank max|g_p| travelled through the sum all-reduce in one slot per rank: fold them into scal[1]
  if (blockIdx.x == 0 && threadIdx.x < nslots) gmax = gslots[threadIdx.x];
  if (c < C) {
    const int mask = cam_mask[c];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      const int di = sym_idx(6, i, i);
      const bool fixed = (i < 3) ? (mask & 1) : (mask & 2);
      double d = U[(size_t)c * 21 + di];
      if (fixed || !(d > 0.0)) {
        // decouple this dof completely
        for (int j = 0; j < 6; ++j) U[(size_t)c * 21 + (i <= j ? sym_idx(6, i, j) : sym_idx(6, j, i))] = 0.0;
        U[(size_t)c * 21 + di] = 1.0;
        gc[(size_t)c * 6 + i] = 0.0;
        if (set_jscale) jscale_c[(size_t)c * 6 + i] = -1.0;   // marks "not a variable"
      } else {
        if (set_jscale) jscale_c[(size_t)c * 6 + i] = 1.0 / (1.0 + sqrt(d));
        gmax = fmax(gmax, fabs(gc[(size_t)c * 6 + i]));
      }
    }
  }
  gmax = warp_max(gmax);
  if ((threadIdx.x & 31) == 0 && gmax > 0.0) atomic_max_nonneg(&scal[1], gmax);
}

// LM damping of the camera blocks: Dc = clamp(U_ii js^2, 1e-6, 1e32) / (radius js^2)
// (levenberg_marquardt_strategy.cc, in the Jacobi-scaled space)
__global__ void ba_damp_cams(int C, const double* __restrict__ U, const double* __restrict__ jscale_c, double radius,
                             double* __restrict__ Dc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * 6) return;
  const int c = i / 6, k = i % 6;
  const double js = jscale_c[i];
  if (js < 0.0) {
    Dc[i] = 0.0;
    return;
  }
  const double d = U[(size_t)c * 21 + sym_idx(6, k, k)];
  const double js2 = js * js;
  Dc[i] = fmin(fmax(d * js2, 1e-6), 1e32) / (radius * js2);
}

// Point blocks: Jacobi scale (first linearisation) and Vinv = (V + Dp)^-1
__device__ __forceinline__ void point_damping(const double* V6, const double* js, double radius, double Dp[3]) {
  const double d[3] = {V6[0], V6[3], V6[5]};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double js2 = js[k] * js[k];
    Dp[k] = fmin(fmax(d[k] * js2, 1e-6), 1e32) / (radius * js2);
  }
}
__global__ void ba_damp_points(int P, const double* __restrict__ V, double* __restrict__ jscale_p, int set_jscale,
                               double radius, double* __restrict__ Vinv) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  double v6[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) v6[k] = V[6 * (size_t)p + k];
  double js[3];
  if (set_jscale) {
    js[0] = 1.0 / (1.0 + sqrt(v6[0]));
    js[1] = 1.0 / (1.0 + sqrt(v6[3]));
    js[2] = 1.0 / (1.0 + sqrt(v6[5]));
#pragma unroll
    for (int k = 0; k < 3; ++k) jscale_p[3 * (size_t)p + k] = js[k];
  } else {
#pragma unroll
    for (int k = 0; k < 3; ++k) js[k] = jscale_p[3 * (size_t)p + k];
  }
  double Dp[3];
  point_damping(v6, js, radius, Dp);
  v6[0] += Dp[0];
  v6[3] += Dp[1];
  v6[5] += Dp[2];
  double inv[6];
  sym3_inverse(v6, inv);
#pragma unroll
  for (int k = 0; k < 6; ++k) Vinv[6 * (size_t)p + k] = inv[k];
}

// ---------------------------------------------------------------------------
// K2b: Schur-Jacobi diagonal  Sd_c = sum_{o in c} W_o Vinv_p W_o^T, camera order
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) ba_schur_diag(BAView v) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= v.n_segs) return;
  const int cam = v.seg_cam[warp];
  const int b = v.seg_begin[warp], e = v.seg_end[warp];
  double S[21];
#pragma unroll
  for (int k = 0; k < 21; ++k) S[k] = 0.0;
  for (int i = b + lane; i < e; i += 32) {
    const int o = v.camord_obs[i];
    const int pt = v.pt_c[i];
    double w[18], vi[6];
    const double2* wp = reinterpret_cast<const double2*>(v.W + (size_t)o * kWDoubles);
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const double2 t = wp[k];
      w[2 * k] = t.x;
      w[2 * k + 1] = t.y;
    }
    const double2* vp = reinterpret_cast<const double2*>(v.Vinv + (size_t)pt * 6);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double2 t = vp[k];
      vi[2 * k] = t.x;
      vi[2 * k + 1] = t.y;
    }
    double T[6][3];
#pragma unroll
    for (int r = 0; r < 6; ++r) sym3_mul(vi, &w[3 * r], T[r]);
    int idx = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
      for (int c = r; c < 6; ++c)
        S[idx++] += T[r][0] * w[3 * c] + T[r][1] * w[3 * c + 1] + T[r][2] * w[3 * c + 2];
  }
#pragma unroll
  for (int k = 0; k < 21; ++k) {
    const double s = warp_sum(S[k]);
    if (lane == k && s != 0.0) atomicAdd(&v.Sd[(size_t)cam * 21 + k], s);
  }
}

// Preconditioner blocks Minv = (U + Dc - Sd)^-1 (Sd == nullptr: block-Jacobi on U + Dc)
__global__ void ba_build_precond(int C, const double* __restrict__ U, const double* __restrict__ Dc,
                                 const double* __restrict__ Sd, double* __restrict__ Minv) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double m[21];
#pragma unroll
  for (int k = 0; k < 21; ++k) m[k] = U[(size_t)c * 21 + k] - (Sd ? Sd[(size_t)c * 21 + k] : 0.0);
#pragma unroll
  for (int i = 0; i < 6; ++i) m[sym_idx(6, i, i)] += Dc[(size_t)c * 6 + i];
  double inv[21];
  spd_inverse_packed<6>(m, inv);
#pragma unroll
  for (int k = 0; k < 21; ++k) Minv[(size_t)c * 21 + k] = inv[k];
}

// ---------------------------------------------------------------------------
// K3: implicit Schur pass over one tile of points.
//   s_p = [g_p] + sum_o W_o^T x_cam(o);  z_p = Vinv_p s_p
//   MODE 0 (mat-vec):  y_cam -= W_o z_p
//   MODE 1 (rhs):      s_p = g_p only (no x); y_cam -= W_o z_p
//   MODE 2 (back-substitution): s_p = g_p + W^T dc; dp = -z_p; points_new = points + dp;
//          bscal[0] += g_p.dp, bscal[1] += sum Dp dp^2, bscal[2] += |dp|^2, bscal[3] += |points|^2
// ---------------------------------------------------------------------------
struct K3Smem {
  alignas(128) double Wt[kTile * kWDoubles];
  double t[3][kTile + 1];
  double z[3][kTilePts + 1];     // s_p while accumulating, then z_p
  unsigned pb[kTilePts + 1];
  double scratch[32];
  alignas(8) uint64_t mbar;
};

template <int MODE>
__global__ void __launch_bounds__(kTile, B200_K3_MIN_CTAS) ba_schur_pass(BAView v, const double* __restrict__ x, double* __restrict__ y,
                                                          const double* __restrict__ points,
                                                          double* __restrict__ points_new, double radius,
                                                          double* __restrict__ bscal, const double* __restrict__ spk = nullptr,
                                                          const double* __restrict__ dk = nullptr, int m_intr = 0,
                                                          const PcgCtl* __restrict__ ctl = nullptr) {
  extern __shared__ __align__(128) unsigned char smem_raw[];   // dynamic shared memory starts 128-B aligned (no static __shared__ in these kernels)
  if (ctl && ctl->done) return;   // the PCG stopping rule has fired: the queued iterations are no-ops
  K3Smem& sm = *reinterpret_cast<K3Smem*>(smem_raw);
  const int tile = blockIdx.x;
  const int tid = threadIdx.x;
  const int4 td = v.tile_desc[tile];
  const int p0 = td.x, npts = td.y, n = td.w;
  const unsigned o0 = (unsigned)td.z, o1 = o0 + (unsigned)n;
  const int nchunks = (n + kTile - 1) / kTile;
  if (tid == 0) {
    mbar_init(&sm.mbar, 1);
    fence_mbar_init();
    if (MODE != 1 && n > 0) {   // first W tile is requested before anything else
      const int nc0 = min(kTile, n);
      mbar_arrive_expect_tx(&sm.mbar, (uint32_t)nc0 * kWBytes);
      tma_load_1d(sm.Wt, v.W + (size_t)o0 * kWDoubles, (uint32_t)nc0 * kWBytes, &sm.mbar);
    }
  }
  // prefetch the first chunk's camera index + x block before the barrier
  int cam_pf = 0, pt_pf = 0;
  double2 xa_pf = make_double2(0, 0), xb_pf = xa_pf, xc_pf = xa_pf;
  if (MODE != 1 && tid < n) {
    cam_pf = v.obs_cam[o0 + tid];
    if (MODE == 0) pt_pf = v.obs_pt[o0 + tid];
    const double2* xp = reinterpret_cast<const double2*>(x + (size_t)cam_pf * 6);
    xa_pf = xp[0];
    xb_pf = xp[1];
    xc_pf = xp[2];
  }
  if (tid < npts) {
    sm.pb[tid] = v.pt_begin[p0 + tid];
    if (tid == npts - 1) sm.pb[npts] = o1;
    sm.z[0][tid] = sm.z[1][tid] = sm.z[2][tid] = 0.0;
  }
  __syncthreads();
  uint32_t phase = 0;
  // ---- phase A: s_p = sum_o W_o^T x_cam(o) (accumulated in sm.z) --------------------
  if (MODE != 1) {
    for (int ch = 0; ch < nchunks; ++ch) {
      const int c0 = ch * kTile;
      const int nc = min(kTile, n - c0);
      if (tid == 0 && ch > 0) {
        mbar_arrive_expect_tx(&sm.mbar, (uint32_t)nc * kWBytes);
        tma_load_1d(sm.Wt, v.W + (size_t)(o0 + c0) * kWDoubles, (uint32_t)nc * kWBytes, &sm.mbar);
      }
      double xc[6] = {0, 0, 0, 0, 0, 0};
      const bool active = tid < nc;
      if (active) {
        if (ch > 0) {
          cam_pf = v.obs_cam[o0 + c0 + tid];
          const double2* xp = reinterpret_cast<const double2*>(x + (size_t)cam_pf * 6);
          xa_pf = xp[0];
          xb_pf = xp[1];
          xc_pf = xp[2];
        }
        xc[0] = xa_pf.x; xc[1] = xa_pf.y; xc[2] = xb_pf.x; xc[3] = xb_pf.y; xc[4] = xc_pf.x; xc[5] = xc_pf.y;
      }
      mbar_wait(&sm.mbar, phase);
      phase ^= 1;
      double t0 = 0, t1 = 0, t2 = 0;
      if (active) {
        const double2* wr = reinterpret_cast<const double2*>(sm.Wt + tid * kWDoubles);
#pragma unroll
        for (int r = 0; r < 6; r += 2) {
          const double2 q0 = wr[(3 * r) / 2], q1 = wr[(3 * r) / 2 + 1], q2 = wr[(3 * r) / 2 + 2];
          // rows r (q0.x q0.y q1.x) and r+1 (q1.y q2.x q2.y)
          t0 += q0.x * xc[r] + q1.y * xc[r + 1];
          t1 += q0.y * xc[r] + q2.x * xc[r + 1];
          t2 += q1.x * xc[r] + q2.y * xc[r + 1];
        }
      }
      sm.t[0][tid] = t0;
      sm.t[1][tid] = t1;
      sm.t[2][tid] = t2;
      __syncthreads();
      // per-point partial sums: thread -> (point j, component k)
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
  // ---- z_p = Vinv_p s_p -----------------------------------------------------------
  double b0 = 0, b1 = 0, b2 = 0, b3 = 0;
  if (tid < npts) {
    const size_t p = (size_t)(p0 + tid);
    const bool pvalid = (int)(sm.pb[tid + 1] - sm.pb[tid]) >= v.min_views;
    double z[3] = {0.0, 0.0, 0.0};
    if (pvalid) {
      double s[3] = {sm.z[0][tid], sm.z[1][tid], sm.z[2][tid]};
      double g[3] = {0, 0, 0};
      if (MODE != 0) {
        g[0] = v.gp[3 * p];
        g[1] = v.gp[3 * p + 1];
        g[2] = v.gp[3 * p + 2];
        s[0] += g[0];
        s[1] += g[1];
        s[2] += g[2];
      }
      if (MODE == 2 && m_intr > 0) {   // + W_k^T dk  (shared-intrinsics border)
        for (int j = 0; j < m_intr; ++j) {
          const double dkj = dk[j];
          s[0] += spk[p * 3 * m_intr + 3 * j] * dkj;
          s[1] += spk[p * 3 * m_intr + 3 * j + 1] * dkj;
          s[2] += spk[p * 3 * m_intr + 3 * j + 2] * dkj;
        }
      }
      double vi[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) vi[k] = v.Vinv[6 * p + k];
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
          const double xo = points[3 * p + k];
          points_new[3 * p + k] = xo + dp;
          b0 += g[k] * dp;
          b1 += Dp[k] * dp * dp;
          b2 += dp * dp;
          b3 += xo * xo;
        }
      }
    } else if (MODE == 2) {
#pragma unroll
      for (int k = 0; k < 3; ++k) points_new[3 * p + k] = points[3 * p + k];
    }
    if (MODE != 2) {
      sm.z[0][tid] = z[0];
      sm.z[1][tid] = z[1];
      sm.z[2][tid] = z[2];
    }
  }
  if (MODE == 2) {
    b0 = block_sum(b0, sm.scratch);
    b1 = block_sum(b1, sm.scratch);
    b2 = block_sum(b2, sm.scratch);
    b3 = block_sum(b3, sm.scratch);
    if (tid == 0) {
      atomicAdd(&bscal[0], b0);
      atomicAdd(&bscal[1], b1);
      atomicAdd(&bscal[2], b2);
      atomicAdd(&bscal[3], b3);
    }
    return;
  }
  __syncthreads();
  // ---- phase B: y_cam -= W_o z_p (W re-read from the shared-memory tile) --------------
  for (int ch = 0; ch < nchunks; ++ch) {
    const int c0 = ch * kTile;
    const int nc = min(kTile, n - c0);
    const bool reload = (MODE == 1) || (nchunks > 1);
    if (reload) {
      __syncthreads();
      if (tid == 0) {
        mbar_arrive_expect_tx(&sm.mbar, (uint32_t)nc * kWBytes);
        tma_load_1d(sm.Wt, v.W + (size_t)(o0 + c0) * kWDoubles, (uint32_t)nc * kWBytes, &sm.mbar);
      }
      mbar_wait(&sm.mbar, phase);
      phase ^= 1;
    }
    if (tid < nc) {
      const unsigned oi = o0 + c0 + tid;
      const int cam = reload ? v.obs_cam[oi] : cam_pf;
      const int pl = (reload ? v.obs_pt[oi] : pt_pf) - p0;
      const double z0 = sm.z[0][pl], z1 = sm.z[1][pl], z2 = sm.z[2][pl];
      if (z0 != 0.0 || z1 != 0.0 || z2 != 0.0) {
        const double2* wr = reinterpret_cast<const double2*>(sm.Wt + tid * kWDoubles);
        double* yc = y + (size_t)cam * 6;
#pragma unroll
        for (int r = 0; r < 6; r += 2) {
          const double2 q0 = wr[(3 * r) / 2], q1 = wr[(3 * r) / 2 + 1], q2 = wr[(3 * r) / 2 + 2];
          atomicAdd(&yc[r], -(q0.x * z0 + q0.y * z1 + q1.x * z2));
          atomicAdd(&yc[r + 1], -(q1.y * z0 + q2.x * z1 + q2.y * z2));
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------
// cost-only evaluation (trial step): scal[0] += 1/2 sum rho
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ba_cost(BAView v, const double* __restrict__ cam_rec,
                                               const double* __restrict__ intr_rec, const double* __restrict__ points,
                                               double huber_a, double* __restrict__ scal) {
  __shared__ double scratch[32];
  double cost = 0.0;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < v.N; o += (long long)gridDim.x * blockDim.x) {
    const int pt = v.obs_pt[o];
    if ((int)(v.pt_begin[pt + 1] - v.pt_begin[pt]) < v.min_views) continue;
    const int cam = v.obs_cam[o];
    const double2 xy = v.obs_xy[o];
    const double4 q4 = *reinterpret_cast<const double4*>(cam_rec + (size_t)cam * kCamRec);
    const double4 t4 = *reinterpret_cast<const double4*>(cam_rec + (size_t)cam * kCamRec + 4);
    const double* sr = sensor_of_obs(v, o);
    const int intr = obs_intr_idx(t4, sr);
    const double q[4] = {q4.x, q4.y, q4.z, q4.w};
    double R[9];
    quat_to_R(q, R);
    const double X0 = points[3 * (size_t)pt], X1 = points[3 * (size_t)pt + 1], X2 = points[3 * (size_t)pt + 2];
    double xc = R[0] * X0 + R[1] * X1 + R[2] * X2 + t4.x;
    double yc = R[3] * X0 + R[4] * X1 + R[5] * X2 + t4.y;
    double zc = R[6] * X0 + R[7] * X1 + R[8] * X2 + t4.z;
    if (sr) sensor_apply(sr, xc, yc, zc);
    if (zc > kZEps) {
      double px, py;
      project_only(intr_rec + (size_t)intr * kIntrRec, xc, yc, zc, px, py);
      const double r0 = px - xy.x, r1 = py - xy.y;
      double rho0, rho1;
      huber(r0 * r0 + r1 * r1, huber_a, rho0, rho1);
      cost += 0.5 * rho0;
    }
  }
  cost = block_sum(cost, scratch);
  if (threadIdx.x == 0 && cost != 0.0) atomicAdd(&scal[0], cost);
}

// ---------------------------------------------------------------------------
// camera update: q_new = exp(d_rot) (x) q (EigenQuaternionManifold), t_new = t + d_t
//   cscal[0] += gc.dc, cscal[1] += dc.rho (PCG residual), cscal[2] += sum Dc dc^2,
//   cscal[3] += |x_new - x|^2 (ambient), cscal[4] += |x|^2 (ambient, over the parameter blocks of the problem: observed
//   by a kept observation and not held constant, whatever their curvature -- Ceres' x_norm over the reduced program)
// ---------------------------------------------------------------------------
__global__ void ba_update_cams(int C, const double* __restrict__ quat, const double* __restrict__ trans,
                               const double* __restrict__ dc, const double* __restrict__ gc,
                               const double* __restrict__ resid, const double* __restrict__ Dc,
                               const double* __restrict__ jscale_c, const double* __restrict__ blk_used,
                               const unsigned char* __restrict__ cam_mask, double* __restrict__ quat_new,
                               double* __restrict__ trans_new, double* __restrict__ cscal) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  double a0 = 0, a1 = 0, a2 = 0, a3 = 0, a4 = 0;
  if (c < C) {
    double d[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const size_t i = (size_t)c * 6 + k;
      const bool var = jscale_c[i] >= 0.0;
      d[k] = var ? dc[i] : 0.0;
      a0 += gc[i] * d[k];
      a1 += resid[i] * d[k];
      a2 += Dc[i] * d[k] * d[k];
    }
    const double q[4] = {quat[4 * c], quat[4 * c + 1], quat[4 * c + 2], quat[4 * c + 3]};
    const bool used = blk_used[c] > 0.0;
    const bool rvar = used && !(cam_mask[c] & 1), tvar = used && !(cam_mask[c] & 2);
    const double nrm = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    double qn[4] = {q[0], q[1], q[2], q[3]};
    if (nrm > 0.0) {
      const double sn = sin(nrm) / nrm, cs = cos(nrm);
      const double ax = sn * d[0], ay = sn * d[1], az = sn * d[2], aw = cs;
      // Hamilton product (a (x) q), xyzw
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
      quat_new[4 * c + k] = qn[k];
      if (rvar) {
        a3 += (qn[k] - q[k]) * (qn[k] - q[k]);
        a4 += q[k] * q[k];
      }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double t = trans[3 * c + k];
      trans_new[3 * c + k] = t + d[3 + k];
      if (tvar) {
        a3 += d[3 + k] * d[3 + k];
        a4 += t * t;
      }
    }
  }
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  a2 = warp_sum(a2);
  a3 = warp_sum(a3);
  a4 = warp_sum(a4);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&cscal[0], a0);
    atomicAdd(&cscal[1], a1);
    atomicAdd(&cscal[2], a2);
    atomicAdd(&cscal[3], a3);
    atomicAdd(&cscal[4], a4);
  }
}


// ===========================================================================
// Intrinsics (optimize_intrinsics, bundle_adjustment.cc:273-293): the variable-parameter table of an intrinsics block and
// the Jacobian of the projection with respect to one parameter.  The blocks themselves are pseudo-camera blocks of the
// reduced system (ba_kernels_ext.cuh; stored-row fast path in ba_kernels_v2.cuh) -- round 1's dense border is gone.
// ===========================================================================
constexpr int kMaxBlockDof = 5;

struct IntrVarRec {   // per intrinsics block
  int col0;           // reserved (0)
  int mb;             // number of variable parameters
  int pidx[kMaxBlockDof];
  int pad;
};

// d(px,py)/d(param pidx), scaled by w = sqrt(rho')
__device__ __forceinline__ void intr_param_jac(const Intr& in, int pidx, double u, double v, double w,
                                               double& jx, double& jy) {
  const double r2 = u * u + v * v;
  const double d = 1.0 + r2 * (in.k1 + in.k2 * r2);
  jx = 0.0;
  jy = 0.0;
  if (in.model == 1) {                    // PINHOLE fx fy cx cy
    if (pidx == 0) jx = u;
    else if (pidx == 1) jy = v;
    else if (pidx == 2) jx = 1.0;
    else jy = 1.0;
  } else {                                // f cx cy [k1 [k2]]
    if (pidx == 0) { jx = u * d; jy = v * d; }
    else if (pidx == 1) jx = 1.0;
    else if (pidx == 2) jy = 1.0;
    else if (pidx == 3) { jx = in.fx * u * r2; jy = in.fy * v * r2; }
    else { jx = in.fx * u * r2 * r2; jy = in.fy * v * r2 * r2; }
  }
  jx *= w;
  jy *= w;
}

// column sums of a [rows][ncol] partial buffer (one CTA per column, deterministic)
__global__ void __launch_bounds__(256) ba_colsum(int rows, int ncol, const double* __restrict__ part,
                                                 double* __restrict__ out) {
  __shared__ double scratch[32];
  const int c = blockIdx.x;
  double a = 0.0;
  for (int r = threadIdx.x; r < rows; r += blockDim.x) a += part[(size_t)r * ncol + c];
  a = block_sum(a, scratch);
  if (threadIdx.x == 0) out[c] = a;
}

}  // namespace b200
