// ba_kernels_v3.cuh -- point side of design v2 in the "ELL-32" layout: ONE THREAD PER POINT.
//
// The tile kernels (ba_linearize_points<true>, ba2_pass_a) give one thread to every observation and then have to
// reduce over the observations of a point: rows staged through shared memory, a (point, component) re-read loop,
// two CTA barriers per tile, which leaves pass A bound by the LSU wavefront pipe (shared-memory wavefronts outnumber
// the global ones) well below the DRAM bandwidth, and the linearisation latency-bound.  Here the point-order data is transposed instead so that the
// reduction is a register accumulation:
//   * points are grouped by 32 (one warp).  Inside windows of 1024 consecutive points the points are stably sorted by
//     track length (descending), so the 32 tracks of a group have (nearly) the same length and neighbouring groups
//     still touch neighbouring per-point records; with uniform track lengths the permutation is the identity.
//   * group g owns rows ell_row0[g] .. ell_row0[g+1]-1; the j-th observation of the point in lane l sits in row
//     ell_row0[g] + j at lane l.  Per-observation arrays are [row][32] (ell_cam, ell_xy, ell_sensor) and the A_o rows
//     [row][6][32], so every warp access is a full 128-B / 256-B line -- no shared memory, no barrier, no atomics.
//   * tracks shorter than min_num_view_per_track (bundle_adjustment.cc:122) get no rows at all.
// Per-point records (X, V, g_p, Vinv, z) stay indexed by the caller's point id (ell_pt[slot]); the camera-order
// kernels of ba_kernels_v2.cuh (pass B, Schur-Jacobi, camera-order linearisation) are unchanged.
// Algorithmic bytes: linearise 20 N (xy, camera index) + 48 N (A_o) + 100 P; pass A 52 N + 4 N (index) + 108 P.
#pragma once
#include "ba_kernels_v2.cuh"

namespace b200 {

constexpr int kEllWindow = 1024;   // points per sorting window (32 groups)
constexpr int kEllThreads = 128;   // 4 groups per CTA

struct EllView {
  int n_groups;
  const int* row0;            // [n_groups + 1]
  const int* pt;              // [n_groups * 32] caller's point id of the slot, -1 = padding
  const int* len;             // [n_groups * 32] rows of the slot (0: padding or a track below min_num_view_per_track)
  const int* cam;             // [rows * 32]
  const double2* xy;          // [rows * 32]
  const unsigned short* sensor;   // [rows * 32] (known rigs) or nullptr
  double* A;                  // [rows][6][32]
  double* B = nullptr;        // [rows][3 * NK][32]  stored-row intrinsics path (ba_kernels_v2.cuh), else nullptr
};

// ---- structure build -------------------------------------------------------------------------------------------
// Stable sort of one window of points by descending effective track length; CTA = kEllWindow threads.
// Block-wide radix sort on the key (0xffff - min(len, 0xffff)) with the point's offset in the window as the value.
template <class Sort>
__global__ void __launch_bounds__(kEllWindow) ell_sort_window(int P, int min_views, const unsigned* __restrict__ pt_begin,
                                                              int* __restrict__ ell_pt, int* __restrict__ ell_len,
                                                              int* __restrict__ ell_slot, int* __restrict__ group_rows) {
  __shared__ typename Sort::TempStorage tmp;
  const int t = threadIdx.x;
  const int p = blockIdx.x * kEllWindow + t;
  int len = -1;
  if (p < P) {
    len = (int)(pt_begin[p + 1] - pt_begin[p]);
    if (len < min_views) len = 0;
  }
  unsigned key[1] = {p < P ? (unsigned)(0xffffff - min(len, 0xffffff)) : 0xffffffffu};   // padding sorts last
  int val[1] = {t};
  Sort(tmp).Sort(key, val, 0, 25);   // blocked arrangement: thread t holds rank t
  const int src = blockIdx.x * kEllWindow + val[0];
  const int slot = blockIdx.x * kEllWindow + t;
  const bool real = key[0] != 0xffffffffu;
  const int l = real ? (int)(0xffffff - key[0]) : 0;
  ell_pt[slot] = real ? src : -1;
  ell_len[slot] = l;
  if (real) ell_slot[src] = slot;
  if ((t & 31) == 0) group_rows[slot >> 5] = l;   // sorted descending: lane 0 holds the group's longest track
}

// scatter the caller's (point-order CSR) observations into the ELL rows
__global__ void ell_scatter_obs(long long N, int min_views, const int* __restrict__ obs_pt, const unsigned* __restrict__ pt_begin,
                                const int* __restrict__ obs_cam, const double2* __restrict__ obs_xy,
                                const unsigned short* __restrict__ obs_sensor, const int* __restrict__ ell_slot,
                                const int* __restrict__ row0, int* __restrict__ ell_cam, double2* __restrict__ ell_xy,
                                unsigned short* __restrict__ ell_sensor) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= N) return;
  const int p = obs_pt[o];
  const unsigned b = pt_begin[p];
  if ((int)(pt_begin[p + 1] - b) < min_views) return;
  const int slot = ell_slot[p];
  const size_t dst = ((size_t)row0[slot >> 5] + (size_t)(o - b)) * 32 + (slot & 31);
  ell_cam[dst] = obs_cam[o];
  ell_xy[dst] = obs_xy[o];
  if (obs_sensor) ell_sensor[dst] = obs_sensor[o];
}

// ---- linearisation, point side -----------------------------------------------------------------------------------
// residual, Jacobian wrt the point, Huber; A_o rows -> ell.A; V_p, g_p per point; per-WARP partial cost / max|g_p|
// (no CTA barrier: the warps of a CTA own groups of different length and would wait for the longest one).
// The per-observation chain  camera index -> camera record -> ~260 instructions  is latency-bound at 16-20 resident
// warps (two dependent memory latencies per observation); the index / pixel rows of iteration
// j + 2 and the camera record of iteration j + 1 are therefore prefetched into L1 while observation j is computed.
template <int NK>
__global__ void __launch_bounds__(kEllThreads, NK > 0 ? 3 : B200_E1_MIN_CTAS) ba3_linearize_points(BAView v, EllView ell,
                                                                               const double* __restrict__ cam_rec,
                                                                               const double* __restrict__ intr_rec,
                                                                               const double* __restrict__ points,
                                                                               double huber_a, int points_var,
                                                                               double* __restrict__ part_cost,
                                                                               double* __restrict__ part_gmax,
                                                                               const IntrVarRec* __restrict__ ivar) {
  const int slot = blockIdx.x * kEllThreads + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int g = slot >> 5;
  double cost = 0.0, gmax = 0.0;
  if (g < ell.n_groups) {
    const int pt = ell.pt[slot];
    const int mylen = ell.len[slot];
    const int r0 = ell.row0[g], nrow = ell.row0[g + 1] - r0;   // warp-uniform
    double X0 = 0, X1 = 0, X2 = 0;
    if (pt >= 0) {
      X0 = points[3 * (size_t)pt]; X1 = points[3 * (size_t)pt + 1]; X2 = points[3 * (size_t)pt + 2];
    }
    double V[6] = {0, 0, 0, 0, 0, 0}, gp[3] = {0, 0, 0};
#if B200_E1_PIPE
    // software pipeline in registers: while observation j is computed, the camera record of j + 1 and the index / pixel
    // of j + 2 are already in flight (they are issued BEFORE the arithmetic of j in program order; the A_o stores of j
    // cannot be reordered with later loads by the compiler, so without this the warp sees every latency in sequence)
    int camB = 0;
    double2 xyA = make_double2(0, 0), xyB = xyA;
    double4 qA = make_double4(0, 0, 0, 1), tA = make_double4(0, 0, 0, 0);
    if (mylen > 0) {
      const size_t i0 = (size_t)r0 * 32 + lane;
      const int camA = ld_stream(ell.cam + i0);
      xyA = ld_stream(ell.xy + i0);
      if (mylen > 1) {
        camB = ld_stream(ell.cam + i0 + 32);
        xyB = ld_stream(ell.xy + i0 + 32);
      }
      qA = ld_rec32(cam_rec + (size_t)camA * kCamRec);
      tA = ld_rec32(cam_rec + (size_t)camA * kCamRec + 4);
    }
#if B200_E1_PIPE >= 2   // experiment: records two observations ahead (index three ahead)
    double4 qB2 = qA, tB2 = tA;
    int camC2 = 0;
    if (mylen > 1) {
      qB2 = ld_rec32(cam_rec + (size_t)camB * kCamRec);
      tB2 = ld_rec32(cam_rec + (size_t)camB * kCamRec + 4);
    }
    if (mylen > 2) camC2 = ld_stream(ell.cam + (size_t)r0 * 32 + lane + 64);
#endif
    for (int j = 0; j < nrow; ++j) {
      if (j >= mylen) break;   // tracks are sorted by length inside a window: a lane is done when its own track is
      const size_t idx = ((size_t)r0 + j) * 32 + lane;
#if B200_E1_PIPE >= 2
      double4 qB = qB2, tB = tB2;          // record of j + 1 (gathered during j - 1)
      double4 qC = qB2, tC = tB2;
      int camC = 0, camD = 0;
      double2 xyC = xyB;
      if (j + 2 < mylen) {
        qC = ld_rec32(cam_rec + (size_t)camC2 * kCamRec);
        tC = ld_rec32(cam_rec + (size_t)camC2 * kCamRec + 4);
        xyC = ld_stream(ell.xy + idx + 64);
      }
      if (j + 3 < mylen) camD = ld_stream(ell.cam + idx + 96);
      (void)camC;
#else
      double4 qB = qA, tB = tA;
      int camC = 0;
      double2 xyC = xyB;
      if (j + 1 < mylen) {
        qB = ld_rec32(cam_rec + (size_t)camB * kCamRec);
        tB = ld_rec32(cam_rec + (size_t)camB * kCamRec + 4);
      }
      if (j + 2 < mylen) {
        camC = ld_stream(ell.cam + idx + 64);
        xyC = ld_stream(ell.xy + idx + 64);
      }
#endif
      const double* sr = ell.sensor ? v.sensor_rec + (size_t)ell.sensor[idx] * kSensorRec : nullptr;
      const int blk = obs_intr_idx(tA, sr);
      const double* ir = intr_rec + (size_t)blk * kIntrRec;
      ObsCore o;
      obs_core(qA, tA, ir, sr, X0, X1, X2, xyA, huber_a, o);
      cost += 0.5 * o.rho0;
      if (points_var) {
        double Jp[6], A[6], b[3];
        obs_point_blocks(o, Jp, A, b);
        double* row = ell.A + ((size_t)r0 + j) * (6 * 32) + lane;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          st_stream(row + 32 * k, A[k]);
          V[k] += A[k];
        }
        gp[0] += b[0]; gp[1] += b[1]; gp[2] += b[2];
        if (NK > 0) {   // B_o = rho' J_pt^T J_k next to A_o
          constexpr int NKK = NK > 0 ? NK : 1;
          double Jk[2][NKK], Bo[3 * NKK];
          obs_intr_rows<NK>(o, ld_intr(ir), ivar[blk], Jp, Jk, Bo);
          double* rowB = ell.B + ((size_t)r0 + j) * (3 * NK * 32) + lane;
#pragma unroll
          for (int k = 0; k < 3 * NK; ++k) st_stream(rowB + 32 * k, Bo[k]);
        }
      }
#if B200_E1_PIPE >= 2
      qA = qB; tA = tB; qB2 = qC; tB2 = tC; xyA = xyB; xyB = xyC; camC2 = camD;
#else
      qA = qB; tA = tB; xyA = xyB; xyB = xyC; camB = camC;
#endif
    }
#else
#pragma unroll 2
    for (int j = 0; j < nrow; ++j) {
      if (j >= mylen) continue;
      const size_t idx = ((size_t)r0 + j) * 32 + lane;
      const int cam = ld_stream(ell.cam + idx);
      const double2 xy = ld_stream(ell.xy + idx);
      const double4 q4 = ld_rec32(cam_rec + (size_t)cam * kCamRec);
      const double4 t4 = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
      const double* sr = ell.sensor ? v.sensor_rec + (size_t)ell.sensor[idx] * kSensorRec : nullptr;
      const int blk = obs_intr_idx(t4, sr);
      const double* ir = intr_rec + (size_t)blk * kIntrRec;
      ObsCore o;
      obs_core(q4, t4, ir, sr, X0, X1, X2, xy, huber_a, o);
      cost += 0.5 * o.rho0;
      if (points_var) {
        double Jp[6], A[6], b[3];
        obs_point_blocks(o, Jp, A, b);
        double* row = ell.A + ((size_t)r0 + j) * (6 * 32) + lane;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          st_stream(row + 32 * k, A[k]);
          V[k] += A[k];
        }
        gp[0] += b[0]; gp[1] += b[1]; gp[2] += b[2];
        if (NK > 0) {
          constexpr int NKK = NK > 0 ? NK : 1;
          double Jk[2][NKK], Bo[3 * NKK];
          obs_intr_rows<NK>(o, ld_intr(ir), ivar[blk], Jp, Jk, Bo);
          double* rowB = ell.B + ((size_t)r0 + j) * (3 * NK * 32) + lane;
#pragma unroll
          for (int k = 0; k < 3 * NK; ++k) st_stream(rowB + 32 * k, Bo[k]);
        }
      }
    }
#endif
    if (points_var && pt >= 0) {
#pragma unroll
      for (int k = 0; k < 6; ++k) v.V[6 * (size_t)pt + k] = V[k];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        v.gp[3 * (size_t)pt + k] = gp[k];
        gmax = fmax(gmax, fabs(gp[k]));
      }
    }
  }
  // one partial per warp (slot >> 5 == global warp index; the padding warps of the last CTA write zeros)
  cost = warp_sum(cost);
  gmax = warp_max(gmax);
  if (lane == 0) {
    part_cost[slot >> 5] = cost;
    part_gmax[slot >> 5] = gmax;
  }
}

// cost only (trial point of the LM step), same traversal: per-CTA partial costs
__global__ void __launch_bounds__(kEllThreads) ba3_cost(BAView v, EllView ell, const double* __restrict__ cam_rec,
                                                         const double* __restrict__ intr_rec,
                                                         const double* __restrict__ points, double huber_a,
                                                         double* __restrict__ part_cost) {
  __shared__ double scratch[32];
  const int slot = blockIdx.x * kEllThreads + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const int g = slot >> 5;
  double cost = 0.0;
  if (g < ell.n_groups) {
    const int pt = ell.pt[slot];
    const int mylen = ell.len[slot];
    const int r0 = ell.row0[g], nrow = ell.row0[g + 1] - r0;
    double X0 = 0, X1 = 0, X2 = 0;
    if (pt >= 0) {
      X0 = points[3 * (size_t)pt]; X1 = points[3 * (size_t)pt + 1]; X2 = points[3 * (size_t)pt + 2];
    }
#pragma unroll 2
    for (int j = 0; j < nrow; ++j) {
      if (j >= mylen) continue;
      const size_t idx = ((size_t)r0 + j) * 32 + lane;
      const int cam = ld_stream(ell.cam + idx);
      const double2 xy = ld_stream(ell.xy + idx);
      const double4 q4 = ld_rec32(cam_rec + (size_t)cam * kCamRec);
      const double4 t4 = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
      const double* sr = ell.sensor ? v.sensor_rec + (size_t)ell.sensor[idx] * kSensorRec : nullptr;
      const double* ir = intr_rec + (size_t)obs_intr_idx(t4, sr) * kIntrRec;
      const double q[4] = {q4.x, q4.y, q4.z, q4.w};
      double R[9];
      quat_to_R(q, R);
      double xc = R[0] * X0 + R[1] * X1 + R[2] * X2 + t4.x;
      double yc = R[3] * X0 + R[4] * X1 + R[5] * X2 + t4.y;
      double zc = R[6] * X0 + R[7] * X1 + R[8] * X2 + t4.z;
      if (sr) sensor_apply(sr, xc, yc, zc);
      if (zc > kZEps) {
        double px, py;
        project_only(ir, xc, yc, zc, px, py);
        const double e0 = px - xy.x, e1 = py - xy.y;
        double rho0, rho1;
        huber(e0 * e0 + e1 * e1, huber_a, rho0, rho1);
        cost += 0.5 * rho0;
      }
    }
  }
  cost = block_sum(cost, scratch);
  if (threadIdx.x == 0) part_cost[blockIdx.x] = cost;
}

// out[0] = sum part_a (fixed order), out[1] = max part_b (optional)   -- single CTA
__global__ void __launch_bounds__(1024) ba3_reduce_partials(int n, const double* __restrict__ part_a,
                                                           const double* __restrict__ part_b, double* __restrict__ out_sum,
                                                           double* __restrict__ out_max) {
  __shared__ double scratch[32];
  double s = 0.0, m = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    s += part_a[i];
    if (part_b) m = fmax(m, part_b[i]);
  }
  s = block_sum(s, scratch);
  if (threadIdx.x == 0) *out_sum = s;
  if (part_b) {
    m = block_max(m, scratch);
    if (threadIdx.x == 0) *out_max = m;
  }
}

// ---- pass A, point side of the implicit-Schur mat-vec --------------------------------------------------------------
//   s_p = [g_p] + sum_o A_o v_o,  v_o = x'_t - 2 X_p x x'_r (xp = packed R^T x rows);  z_p = Vinv s_p
//   MODE 0: z -> z4[P][4]                      (mat-vec)
//   MODE 2: back-substitution epilogue (points_new, per-CTA partial step scalars bscal[cta][4])
template <int MODE, int NK>
__global__ void __launch_bounds__(kEllThreads, MODE == 0 ? B200_EA_MIN_CTAS : B200_EA2_MIN_CTAS) ba3_pass_a(
    BAView v, EllView ell, BAViewV2 v2, const double* __restrict__ xp, const double* __restrict__ points,
    double* __restrict__ points_new, double radius, double* __restrict__ bscal, const PcgCtl* __restrict__ ctl) {
  __shared__ double scratch[32];
  if (ctl && ctl->done) return;   // the PCG stopping rule has fired: the queued iterations are no-ops
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
#pragma unroll 4
    for (int j = 0; j < nrow; ++j) {
      if (j >= mylen) continue;
      const size_t idx = ((size_t)r0 + j) * 32 + lane;
      const int cam = ld_stream(ell.cam + idx);
      const double* row = ell.A + ((size_t)r0 + j) * (6 * 32) + lane;
      const double a0 = ld_stream(row), a1 = ld_stream(row + 32), a2 = ld_stream(row + 64);
      const double a3 = ld_stream(row + 96), a4 = ld_stream(row + 128), a5 = ld_stream(row + 160);
      double xr0, xr1, xr2, xt0;
      ld_nc_256(xp + (size_t)cam * kXqStride, xr0, xr1, xr2, xt0);
      double4 xt;   // {x_t1, x_t2, x_k0, x_k1}: the intrinsics increments ride in the spare doubles of the row
      if (NK > 0) {
        xt = ld_rec32(xp + (size_t)cam * kXqStride + 4);
      } else {
        const double2 xt12 = __ldg(reinterpret_cast<const double2*>(xp + (size_t)cam * kXqStride + 4));
        xt = make_double4(xt12.x, xt12.y, 0.0, 0.0);
      }
      const double w0 = xt0 - 2.0 * (X1 * xr2 - X2 * xr1);
      const double w1 = xt.x - 2.0 * (X2 * xr0 - X0 * xr2);
      const double w2 = xt.y - 2.0 * (X0 * xr1 - X1 * xr0);
      s0 += a0 * w0 + a1 * w1 + a2 * w2;
      s1 += a1 * w0 + a3 * w1 + a4 * w2;
      s2 += a2 * w0 + a4 * w1 + a5 * w2;
      if (NK > 0) {   // + B_o x_k
        const double* rowB = ell.B + ((size_t)r0 + j) * (3 * NK * 32) + lane;
        const double xk[2] = {xt.z, xt.w};
#pragma unroll
        for (int k = 0; k < NK; ++k) {
          s0 += ld_stream(rowB + 32 * (3 * k)) * xk[k];
          s1 += ld_stream(rowB + 32 * (3 * k + 1)) * xk[k];
          s2 += ld_stream(rowB + 32 * (3 * k + 2)) * xk[k];
        }
      }
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
      if (MODE == 0) st_keep4(v2.z4 + 4 * p, make_double4(z[0], z[1], z[2], 0.0), l2_policy_evict_last());
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

}  // namespace b200
