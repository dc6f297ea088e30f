// ra_kernels.cuh -- rotation-averaging kernels (sm_90a).
//
// Replaces the arithmetic of glomap::RotationEstimator
// (reference: glomap/estimators/global_rotation_averaging.cc:479-772, 3-DoF
// frames with trivial rigs): per-edge SO(3) residual, IRLS / L1-ADMM weights,
// and the normal equations A^T W A, which for the reference's first-order
// A (rows -I at image 1, +I at image 2, .cc:396-415) are the weighted graph
// Laplacian (x) I3 plus the gauge block -- solved here by PCG with one
// edge-parallel Laplacian mat-vec per iteration instead of CHOLMOD (.cc:547-611).
//
// Layout: edges SoA  ei[E], ej[E] (int32), Rrel[E][9], w_edge[E]; the 3 gauge
// rows (.cc:455-460) are carried as one pseudo-edge with ei = -1 (identity, no
// scatter), ej = fixed frame, Rrel = R_fixed(initial), weight 1.
// Node vectors [n][3] are replicated on every rank; edges are sharded.
#pragma once
#include "common.cuh"
#include "pcg.cuh"

namespace b200 {

constexpr double kRaEps = 1e-12;   // glomap/types.h EPS

struct RAView {
  int n;
  long long E;            // local edges including the gauge pseudo-edge (rank 0)
  const int* ei;
  const int* ej;
  const double* Rrel;     // [E][9] row-major (gravity-aligned when use_gravity, .cc:311-326)
  const double* w_edge;   // [E] weights_ (.cc:466-472)
  // use_gravity (1-DoF frames, .cc:207-217): frames with gravity keep theta = (0, phi, 0) and
  // only their y slot is an unknown; pairs of two gravity frames carry ONE row (.cc:387-394)
  const unsigned char* node_grav;   // [n] or nullptr
  const double* angle_rel;          // [E] y angle of R_rel (both-gravity pairs / gravity gauge), or nullptr
  const double* xz_err;             // [E] x^2 + z^2 of log(R_rel) (.cc:330-337), or nullptr
  // unknown cam_from_rig rotations (.cc:173-245): nodes [n_frames, n) are the sensors that are not calibrated yet; an
  // edge adds -I at eci and +I at ecj (.cc:425-440) and its residual uses R_k = R_cam R_frame (.cc:726-736)
  int n_frames;                     // == n without unknown cameras
  const int* eci;                   // [E] node of image 1's camera, -1: calibrated / reference sensor; nullptr: none
  const int* ecj;                   // [E]
};

// which rows / coefficients an edge has
struct EdgeRows {
  bool gi, gj, y_only;
};
__device__ __forceinline__ EdgeRows edge_rows(const RAView& v, int i, int j) {
  EdgeRows r;
  r.gi = v.node_grav && i >= 0 && v.node_grav[i];
  r.gj = v.node_grav && v.node_grav[j];
  r.y_only = (i >= 0) ? (r.gi && r.gj) : r.gj;   // gauge rows: 1 row if the fixed frame has gravity (.cc:449-453)
  return r;
}
__device__ __forceinline__ double coef(bool grav, int k) { return (!grav || k == 1) ? 1.0 : 0.0; }

// AngleAxisToRotation (math/rigid3d.cc:45-63): first-order fallback below EPS
__device__ __forceinline__ void aa_to_R(const double v[3], double R[9]) {
  const double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (n > kRaEps) {
    const double inv = 1.0 / n;
    const double x = v[0] * inv, y = v[1] * inv, z = v[2] * inv;
    double s, c;
    sincos(n, &s, &c);
    const double t = 1.0 - c;
    // Eigen AngleAxis::toRotationMatrix
    R[0] = t * x * x + c;
    R[1] = t * x * y - s * z;
    R[2] = t * x * z + s * y;
    R[3] = t * x * y + s * z;
    R[4] = t * y * y + c;
    R[5] = t * y * z - s * x;
    R[6] = t * x * z - s * y;
    R[7] = t * y * z + s * x;
    R[8] = t * z * z + c;
  } else {
    R[0] = 1; R[1] = -v[2]; R[2] = v[1];
    R[3] = v[2]; R[4] = 1; R[5] = -v[0];
    R[6] = -v[1]; R[7] = v[0]; R[8] = 1;
  }
}

// RotationToAngleAxis (math/rigid3d.cc:39-43): Eigen Matrix3 -> Quaternion -> AngleAxis
__device__ __forceinline__ void R_to_aa(const double R[9], double v[3]) {
  double q[4];   // x y z w
  const double t = R[0] + R[4] + R[8];
  if (t > 0.0) {
    double tt = sqrt(t + 1.0);
    q[3] = 0.5 * tt;
    tt = 0.5 / tt;
    q[0] = (R[7] - R[5]) * tt;
    q[1] = (R[2] - R[6]) * tt;
    q[2] = (R[3] - R[1]) * tt;
  } else {
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double tt = sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0);
    q[i] = 0.5 * tt;
    tt = 0.5 / tt;
    q[3] = (R[3 * k + j] - R[3 * j + k]) * tt;
    q[j] = (R[3 * j + i] + R[3 * i + j]) * tt;
    q[k] = (R[3 * k + i] + R[3 * i + k]) * tt;
  }
  const double nv = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  if (nv > 0.0) {
    const double ang = 2.0 * atan2(nv, fabs(q[3]));
    const double f = (q[3] < 0.0 ? -ang : ang) / nv;
    v[0] = q[0] * f;
    v[1] = q[1] * f;
    v[2] = q[2] * f;
  } else {
    v[0] = v[1] = v[2] = 0.0;
  }
}

__device__ __forceinline__ void mat3_mul(const double A[9], const double B[9], double C[9]) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ __forceinline__ void mat3_tmul(const double A[9], const double B[9], double C[9]) {   // A^T B
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}

// ComputeResiduals (.cc:696-756) + the weight of each edge for the next solve.
//   mode 0: w_out = w_edge                       (L1 stage rows, .cc:488-489,506)
//   mode 1: w_out = w_edge * sigma^2/(e^2+sigma^2)^2   GEMAN_MCCLURE (.cc:583-585)
//   mode 2: w_out = w_edge * (e^2)^(-0.75)              HALF_NORM (.cc:587)
// flags[0] |= 1 on NaN weight (.cc:590-593)
__global__ void ra_residuals(RAView v, const double* __restrict__ theta, int mode, double sigma2,
                             double* __restrict__ res, double* __restrict__ w_out, int* __restrict__ flags) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= v.E) return;
  const int i = v.ei[e], j = v.ej[e];
  const EdgeRows er = edge_rows(v, i, j);
  if (er.y_only) {
    // RelAngleError (.cc:19-36; the rand() jitter near +-pi is not reproduced) / gravity gauge row (.cc:746-749)
    const double pi_ = 3.14159265358979323846;
    double est = theta[3 * (size_t)j + 1] - (i >= 0 ? theta[3 * (size_t)i + 1] : 0.0) - v.angle_rel[e];
    if (i >= 0) {
      while (est >= pi_) est -= 2 * pi_;
      while (est < -pi_) est += 2 * pi_;
    }
    res[3 * e] = 0.0;
    res[3 * e + 1] = est;
    res[3 * e + 2] = 0.0;
    double wgt = v.w_edge[e];
    if (i >= 0 && mode != 0) {
      const double e2 = est * est + v.xz_err[e];
      double wi;
      if (mode == 1) {
        const double tmp = e2 + sigma2;
        wi = sigma2 / (tmp * tmp);
      } else {
        wi = pow(e2, (0.5 - 2.0) / 2.0);
      }
      if (isnan(wi)) atomicOr(flags, 1);
      wgt *= wi;
    }
    w_out[e] = wgt;
    return;
  }
  double Rrel[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) Rrel[k] = v.Rrel[9 * e + k];
  double Rj[9], T[9], M[9], r[3];
  const double tj[3] = {theta[3 * (size_t)j], theta[3 * (size_t)j + 1], theta[3 * (size_t)j + 2]};
  aa_to_R(tj, Rj);
  const int ci = (v.eci && i >= 0) ? v.eci[e] : -1, cj = (v.ecj && i >= 0) ? v.ecj[e] : -1;
  if (cj >= 0) {   // R_2 = R_cam2 R_frame2 (.cc:733-736)
    const double tc[3] = {theta[3 * (size_t)cj], theta[3 * (size_t)cj + 1], theta[3 * (size_t)cj + 2]};
    double Rc[9], P[9];
    aa_to_R(tc, Rc);
    mat3_mul(Rc, Rj, P);
#pragma unroll
    for (int k = 0; k < 9; ++k) Rj[k] = P[k];
  }
  if (i >= 0) {
    const double ti[3] = {theta[3 * (size_t)i], theta[3 * (size_t)i + 1], theta[3 * (size_t)i + 2]};
    double Ri[9];
    aa_to_R(ti, Ri);
    if (ci >= 0) {   // R_1 = R_cam1 R_frame1 (.cc:726-730)
      const double tc[3] = {theta[3 * (size_t)ci], theta[3 * (size_t)ci + 1], theta[3 * (size_t)ci + 2]};
      double Rc[9], P[9];
      aa_to_R(tc, Rc);
      mat3_mul(Rc, Ri, P);
#pragma unroll
      for (int k = 0; k < 9; ++k) Ri[k] = P[k];
    }
    mat3_mul(Rrel, Ri, T);
  } else {
#pragma unroll
    for (int k = 0; k < 9; ++k) T[k] = Rrel[k];
  }
  mat3_tmul(Rj, T, M);      // R_j^T R_rel R_i
  R_to_aa(M, r);
  res[3 * e] = -r[0];
  res[3 * e + 1] = -r[1];
  res[3 * e + 2] = -r[2];
  double w = v.w_edge[e];
  if (i >= 0 && mode != 0) {
    const double e2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    double wi;
    if (mode == 1) {
      const double tmp = e2 + sigma2;
      wi = sigma2 / (tmp * tmp);
    } else {
      wi = pow(e2, (0.5 - 2.0) / 2.0);
    }
    if (isnan(wi)) atomicOr(flags, 1);
    w *= wi;
  }
  w_out[e] = w;
}

// out += A^T diag(w^p) vec  (p = 1 or 2); deg += w^p at both ends (Laplacian diagonal)
__global__ void ra_scatter(RAView v, const double* __restrict__ w, int square, const double* __restrict__ vec,
                           double* __restrict__ out, double* __restrict__ deg) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= v.E) return;
  const int i = v.ei[e], j = v.ej[e];
  double we = w[e];
  if (square) we *= we;
  const EdgeRows er = edge_rows(v, i, j);
  const int nci = (v.eci && i >= 0) ? v.eci[e] : -1, ncj = (v.ecj && i >= 0) ? v.ecj[e] : -1;
  const bool same_frame = i == j;   // only with unknown cameras: the -I and +I on the frame cancel (.cc:300-304 keeps the pair)
  const bool same_cam = nci == ncj;   // one unknown sensor in both images: its -I and +I cancel too (.cc:425-440 sums them)
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (er.y_only && k != 1) continue;
    const double a = we * vec[3 * e + k];
    const double cj = coef(er.gj, k);
    if (cj != 0.0 && !same_frame) {
      atomicAdd(&out[3 * (size_t)j + k], a);
      if (deg) atomicAdd(&deg[3 * (size_t)j + k], we);
    }
    if (i >= 0 && coef(er.gi, k) != 0.0 && !same_frame) {
      atomicAdd(&out[3 * (size_t)i + k], -a);
      if (deg) atomicAdd(&deg[3 * (size_t)i + k], we);
    }
    if (ncj >= 0 && !same_cam) {
      atomicAdd(&out[3 * (size_t)ncj + k], a);
      if (deg) atomicAdd(&deg[3 * (size_t)ncj + k], we);
    }
    if (nci >= 0 && !same_cam) {
      atomicAdd(&out[3 * (size_t)nci + k], -a);
      if (deg) atomicAdd(&deg[3 * (size_t)nci + k], we);
    }
  }
}

// y += L(w^p) x :  t = w (x_j - x_i); y_j += t; y_i -= t
__global__ void ra_laplacian(RAView v, const double* __restrict__ w, int square, const double* __restrict__ x,
                             double* __restrict__ y, const PcgCtl* __restrict__ ctl) {
  if (ctl && ctl->done) return;   // the PCG stopping rule has fired: the queued iterations are no-ops
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= v.E) return;
  const int i = v.ei[e], j = v.ej[e];
  double we = w[e];
  if (square) we *= we;
  const EdgeRows er = edge_rows(v, i, j);
  const int nci = (v.eci && i >= 0) ? v.eci[e] : -1, ncj = (v.ecj && i >= 0) ? v.ecj[e] : -1;
  const bool same_frame = i == j;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (er.y_only && k != 1) continue;
    const double cj = same_frame ? 0.0 : coef(er.gj, k), ci = (i >= 0 && !same_frame) ? coef(er.gi, k) : 0.0;
    double t = cj * x[3 * (size_t)j + k];
    if (ci != 0.0) t -= x[3 * (size_t)i + k];
    if (ncj >= 0) t += x[3 * (size_t)ncj + k];
    if (nci >= 0) t -= x[3 * (size_t)nci + k];
    t *= we;
    if (cj != 0.0) atomicAdd(&y[3 * (size_t)j + k], t);
    if (ci != 0.0) atomicAdd(&y[3 * (size_t)i + k], -t);
    if (ncj >= 0) atomicAdd(&y[3 * (size_t)ncj + k], t);
    if (nci >= 0) atomicAdd(&y[3 * (size_t)nci + k], -t);
  }
}

// ---------------------------------------------------------------------------
// CSR-by-node form of the same operators (3-DoF frames without gravity): every node owns the list of its incident
// edges, so the weighted Laplacian is a GATHER -- one warp per node, register accumulation, one store per node, no
// atomics (the edge-parallel ra_laplacian costs 6 FP64 RED per edge and ran at 0.12 of the HBM roofline).  The
// incidence list is sorted (node, edge id): the summation order is fixed, results are run-to-run identical.
//   inc_val[s] = edge id | (1u << 31 if the node is the edge's image 1, whose block in A is -I);  inc_other[s] = the
//   node at the other end (-1: the gauge pseudo-edge, which has no other end);  w_inc[s] = w_e^p in incidence order
//   (refreshed once per linear system by ra_node_setup, so the mat-vec streams 12 B per incidence).
// ---------------------------------------------------------------------------
struct RACsr {
  int n;
  const int* begin;        // [n + 1]
  const unsigned* val;     // [n_inc]
  const int* other;        // [n_inc]
  double* w_inc;           // [n_inc]
};

__global__ void ra_csr_count(long long E, const int* __restrict__ ei, const int* __restrict__ ej, int n,
                             int* __restrict__ cnt, int* __restrict__ keys, unsigned* __restrict__ vals) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int i = ei[e], j = ej[e];
  atomicAdd(&cnt[j], 1);
  keys[2 * e] = j;
  vals[2 * e] = (unsigned)e;
  if (i >= 0) {
    atomicAdd(&cnt[i], 1);
    keys[2 * e + 1] = i;
    vals[2 * e + 1] = (unsigned)e | 0x80000000u;
  } else {
    keys[2 * e + 1] = n;   // sorts behind every real node
    vals[2 * e + 1] = 0;
  }
}
__global__ void ra_csr_other(int n_inc, const unsigned* __restrict__ val, const int* __restrict__ ei,
                             const int* __restrict__ ej, int* __restrict__ other) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_inc) return;
  const unsigned v = val[s];
  const unsigned e = v & 0x7fffffffu;
  other[s] = (v >> 31) ? ej[e] : ei[e];
}

// per linear system: w_inc, Laplacian diagonal deg[n][3], rhs = A^T diag(w^p) vec   (replaces ra_scatter)
__global__ void __launch_bounds__(128) ra_node_setup(RACsr c, const double* __restrict__ w, int square,
                                                     const double* __restrict__ vec, double* __restrict__ rhs,
                                                     double* __restrict__ deg) {
  const int node = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (node >= c.n) return;
  const int b = c.begin[node], e = c.begin[node + 1];
  double d = 0, r0 = 0, r1 = 0, r2 = 0;
  for (int s = b + lane; s < e; s += 32) {
    const unsigned v = c.val[s];
    const unsigned ed = v & 0x7fffffffu;
    double we = w[ed];
    if (square) we *= we;
    c.w_inc[s] = we;
    d += we;
    const double sg = (v >> 31) ? -we : we;
    r0 += sg * vec[3 * (size_t)ed];
    r1 += sg * vec[3 * (size_t)ed + 1];
    r2 += sg * vec[3 * (size_t)ed + 2];
  }
  d = warp_sum(d); r0 = warp_sum(r0); r1 = warp_sum(r1); r2 = warp_sum(r2);
  if (lane == 0) {
    deg[3 * (size_t)node] = deg[3 * (size_t)node + 1] = deg[3 * (size_t)node + 2] = d;
    rhs[3 * (size_t)node] = r0; rhs[3 * (size_t)node + 1] = r1; rhs[3 * (size_t)node + 2] = r2;
  }
}

// y_n = sum_{e ~ n} w_e (x_n - x_other)
__global__ void __launch_bounds__(128) ra_laplacian_csr(RACsr c, const double* __restrict__ x, double* __restrict__ y,
                                                        const PcgCtl* __restrict__ ctl) {
  if (ctl && ctl->done) return;   // the PCG stopping rule has fired: the queued iterations are no-ops
  const int node = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (node >= c.n) return;
  const int b = c.begin[node], e = c.begin[node + 1];
  const double x0 = x[3 * (size_t)node], x1 = x[3 * (size_t)node + 1], x2 = x[3 * (size_t)node + 2];
  double a0 = 0, a1 = 0, a2 = 0;
#pragma unroll 2
  for (int s = b + lane; s < e; s += 32) {
    const double we = ld_stream(c.w_inc + s);
    const int o = ld_stream(c.other + s);
    double o0 = 0, o1 = 0, o2 = 0;
    if (o >= 0) { o0 = x[3 * (size_t)o]; o1 = x[3 * (size_t)o + 1]; o2 = x[3 * (size_t)o + 2]; }
    a0 += we * (x0 - o0);
    a1 += we * (x1 - o1);
    a2 += we * (x2 - o2);
  }
  a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
  if (lane == 0) { y[3 * (size_t)node] = a0; y[3 * (size_t)node + 1] = a1; y[3 * (size_t)node + 2] = a2; }
}

// ---------------------------------------------------------------------------
// Two-level preconditioner for the weighted Laplacian (3-DoF frames without gravity, large graphs):
//     M^-1 = D^-1 + P (P^T L P)^-1 P^T,     P = piecewise-constant prolongation over aggregates of ~256 nodes
// (greedy breadth-first clusters, built once per problem on the host: the graph does not change between the linear
// systems, only the weights do).  Jacobi alone needs O(graph diameter) iterations -- 350 at forcing tolerance 1e-2 on the
// 100 k-frame lattice of config 5, 24.5 k per rotation-averaging solve (VERDICT r1 weak #10); the coarse space
// removes the smooth error components and brings that to ~17 (measured with the same construction in scipy).
// The coarse matrix (n_c <= 1024, dense) is re-assembled and inverted in place whenever the weights change
// (Gauss-Jordan, one elimination kernel + one pivot kernel per column); its application is a dense mat-vec.
// ---------------------------------------------------------------------------
struct RACoarse {
  int nc;
  const int* agg_of;      // [n]
  const int* agg_begin;   // [nc + 1]
  const int* agg_nodes;   // [n] nodes grouped by aggregate
  double* Ac;             // [nc][nc]  coarse matrix, then its inverse
  double* rc;             // [nc][3]
  double* zc;             // [nc][3]
};

__global__ void ra_coarse_assemble(long long E, const int* __restrict__ ei, const int* __restrict__ ej,
                                   const double* __restrict__ w, int square, const int* __restrict__ agg_of, int nc,
                                   double* __restrict__ Ac) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int i = ei[e], j = ej[e];
  double we = w[e];
  if (square) we *= we;
  const int b = agg_of[j];
  if (i < 0) {   // gauge rows: + w on the fixed frame
    atomicAdd(&Ac[(size_t)b * nc + b], we);
    return;
  }
  const int a = agg_of[i];
  if (a == b) return;   // the edge lives inside one aggregate: P^T L P sees nothing of it
  atomicAdd(&Ac[(size_t)a * nc + a], we);
  atomicAdd(&Ac[(size_t)b * nc + b], we);
  atomicAdd(&Ac[(size_t)a * nc + b], -we);
  atomicAdd(&Ac[(size_t)b * nc + a], -we);
}
// in-place Gauss-Jordan inversion of the SPD coarse matrix, column k:  (1) every entry outside row / column k
__global__ void ra_gj_eliminate(int nc, int k, double* __restrict__ A) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j >= nc || i == k || j == k) return;
  A[(size_t)i * nc + j] -= A[(size_t)i * nc + k] * A[(size_t)k * nc + j] / A[(size_t)k * nc + k];
}
//   (2) row k, column k and the pivot   (single CTA)
__global__ void ra_gj_pivot(int nc, int k, double* __restrict__ A) {
  const double p = A[(size_t)k * nc + k];
  __syncthreads();
  for (int t = threadIdx.x; t < nc; t += blockDim.x) {
    if (t == k) continue;
    A[(size_t)k * nc + t] /= p;
    A[(size_t)t * nc + k] /= -p;
  }
  if (threadIdx.x == 0) A[(size_t)k * nc + k] = 1.0 / p;
}
// rc = P^T r   (one warp per aggregate)
__global__ void __launch_bounds__(128) ra_coarse_restrict(RACoarse c, const double* __restrict__ r,
                                                          const PcgCtl* __restrict__ ctl) {
  if (ctl && ctl->done) return;
  const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (a >= c.nc) return;
  double s0 = 0, s1 = 0, s2 = 0;
  for (int t = c.agg_begin[a] + lane; t < c.agg_begin[a + 1]; t += 32) {
    const size_t node = (size_t)c.agg_nodes[t];
    s0 += r[3 * node]; s1 += r[3 * node + 1]; s2 += r[3 * node + 2];
  }
  s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
  if (lane == 0) { c.rc[3 * a] = s0; c.rc[3 * a + 1] = s1; c.rc[3 * a + 2] = s2; }
}
// zc = Ac^-1 rc (one warp per row); part[blockIdx.x] = this CTA's share of rc . zc (= r . P zc, the coarse part of r.z)
__global__ void __launch_bounds__(128) ra_coarse_solve(RACoarse c, double* __restrict__ part_rz_extra,
                                                       const PcgCtl* __restrict__ ctl) {
  __shared__ double sh[4];
  if (ctl && ctl->done) return;
  const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double dot = 0.0;
  if (a < c.nc) {
    double s0 = 0, s1 = 0, s2 = 0;
    const double* row = c.Ac + (size_t)a * c.nc;
    for (int b = lane; b < c.nc; b += 32) {
      const double m = row[b];
      s0 += m * c.rc[3 * b]; s1 += m * c.rc[3 * b + 1]; s2 += m * c.rc[3 * b + 2];
    }
    s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
    if (lane == 0) {
      c.zc[3 * a] = s0; c.zc[3 * a + 1] = s1; c.zc[3 * a + 2] = s2;
      dot = s0 * c.rc[3 * a] + s1 * c.rc[3 * a + 1] + s2 * c.rc[3 * a + 2];
    }
  }
  if (lane == 0) sh[wid] = dot;
  __syncthreads();
  if (threadIdx.x == 0) part_rz_extra[blockIdx.x] = sh[0] + sh[1] + sh[2] + sh[3];
}
// z += P zc
__global__ void ra_coarse_prolong(int n, RACoarse c, double* __restrict__ z, const PcgCtl* __restrict__ ctl) {
  if (ctl && ctl->done) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int a = c.agg_of[i];
  z[3 * (size_t)i] += c.zc[3 * a];
  z[3 * (size_t)i + 1] += c.zc[3 * a + 1];
  z[3 * (size_t)i + 2] += c.zc[3 * a + 2];
}

// ---------------------------------------------------------------------------
// Fused two-level PCG iteration (one GPU, CSR Laplacian): four kernels instead of seven
//   ra2_direction      stopping rule + p = (z + P zc) + beta p   -- the prolongation is never materialised in z;
//                      also writes the 32-B padded copy p4 the Laplacian gathers as one 32-B record per incidence
//   ra2_laplacian_dot  q = L p and the per-CTA partials of p.q    (replaces ra_laplacian_csr + pcg_apply_diag)
//   pcg_update<3>      unchanged
//   ra2_coarse         rc = P^T r, grid barrier, zc = Ac^-1 rc + coarse part of r.z   (replaces restrict + solve)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kPcgThreads) ra2_direction(int n, int nblk, int it, double rel_tol,
                                                             const double* __restrict__ z, double* __restrict__ p,
                                                             double* __restrict__ p4, const double* __restrict__ zc,
                                                             const int* __restrict__ agg_of,
                                                             const double* __restrict__ dots_pp,
                                                             const double* __restrict__ part_rz,
                                                             const double* __restrict__ part_rr,
                                                             const double* __restrict__ part_ref,
                                                             double* __restrict__ dots_pub, PcgCtl* __restrict__ ctl) {
  __shared__ double sh3[3];
  double beta;
  if (!pcg_direction_head(nblk, it, 0, rel_tol, dots_pp, part_rz, part_rr, part_ref, dots_pub, ctl, sh3, beta)) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  const int a = agg_of[c];
  double pv[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const size_t i = 3 * (size_t)c + k;
    const double zf = z[i] + zc[3 * a + k];
    pv[k] = (it == 1) ? zf : zf + beta * p[i];
    p[i] = pv[k];
  }
  st_rec32(p4 + 4 * (size_t)c, pv[0], pv[1], pv[2], 0.0);
}

// CTA b owns the nodes [128 b, 128 b + 128) -- the same split as the vector kernels, so part_pq has one entry per PCG block --
// but runs kLapThreads = 512 threads: 16 warps of 8 nodes each, lanes over incidences (with 4 warps of 32 nodes per CTA the SM held
// too few warps to cover the gathers and the fused solve was slower than the unfused one)
constexpr int kLapThreads = 512;
constexpr int kLapNodesPerWarp = kPcgThreads / (kLapThreads / 32);
__global__ void __launch_bounds__(kLapThreads) ra2_laplacian_dot(RACsr c, const double* __restrict__ p4, double* __restrict__ q,
                                                                 double* __restrict__ part_pq, const PcgCtl* __restrict__ ctl) {
  __shared__ double shw[kLapThreads / 32];
  if (ctl && ctl->done) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int node0 = blockIdx.x * kPcgThreads + wid * kLapNodesPerWarp;
  double dot = 0.0;
  for (int j = 0; j < kLapNodesPerWarp; ++j) {
    const int node = node0 + j;
    if (node >= c.n) break;
    const int b = c.begin[node], e = c.begin[node + 1];
    const double4 xs = ld_rec32(p4 + 4 * (size_t)node);
    double a0 = 0, a1 = 0, a2 = 0;
#pragma unroll 2
    for (int s = b + lane; s < e; s += 32) {
      const double we = ld_stream(c.w_inc + s);
      const int o = ld_stream(c.other + s);
      double4 xo = make_double4(0, 0, 0, 0);
      if (o >= 0) xo = ld_rec32(p4 + 4 * (size_t)o);
      a0 += we * (xs.x - xo.x);
      a1 += we * (xs.y - xo.y);
      a2 += we * (xs.z - xo.z);
    }
    a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
    if (lane == 0) {
      q[3 * (size_t)node] = a0; q[3 * (size_t)node + 1] = a1; q[3 * (size_t)node + 2] = a2;
      dot += xs.x * a0 + xs.y * a1 + xs.z * a2;
    }
  }
  if (lane == 0) shw[wid] = dot;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kLapThreads / 32; ++w) s += shw[w];
    part_pq[blockIdx.x] = s;
  }
}

// restriction + coarse solve in one launch: every CTA restricts its 4 aggregates, all CTAs meet at a grid barrier (the
// grid is <= 256 CTAs of 128 threads: co-resident on 132 SMs), then every warp applies one row of the coarse inverse.
// bar[0] = arrival counter, bar[1] = generation (sense reversal: safe across launches, also across skipped ones)
__global__ void __launch_bounds__(128) ra2_coarse(RACoarse c, const double* __restrict__ r, double* __restrict__ part_rz_extra,
                                                  unsigned* __restrict__ bar, const PcgCtl* __restrict__ ctl) {
  __shared__ double sh[4];
  if (ctl && ctl->done) return;   // set by an earlier launch only: every CTA of this grid takes the same branch
  const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (a < c.nc) {
    double s0 = 0, s1 = 0, s2 = 0;
    for (int t = c.agg_begin[a] + lane; t < c.agg_begin[a + 1]; t += 32) {
      const size_t node = (size_t)c.agg_nodes[t];
      s0 += r[3 * node]; s1 += r[3 * node + 1]; s2 += r[3 * node + 2];
    }
    s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
    if (lane == 0) { c.rc[3 * a] = s0; c.rc[3 * a + 1] = s1; c.rc[3 * a + 2] = s2; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    volatile unsigned* vb = bar;
    const unsigned gen = vb[1];
    __threadfence();
    if (atomicAdd(bar, 1u) == gridDim.x - 1) {
      vb[0] = 0;
      __threadfence();
      atomicAdd(bar + 1, 1u);
    } else {
      while (vb[1] == gen) {}
    }
    __threadfence();
  }
  __syncthreads();
  double dot = 0.0;
  if (a < c.nc) {
    double s0 = 0, s1 = 0, s2 = 0;
    const double* row = c.Ac + (size_t)a * c.nc;
    const volatile double* rc = c.rc;   // written by other CTAs of this launch
    for (int b = lane; b < c.nc; b += 32) {
      const double m = row[b];
      s0 += m * rc[3 * b]; s1 += m * rc[3 * b + 1]; s2 += m * rc[3 * b + 2];
    }
    s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
    if (lane == 0) {
      c.zc[3 * a] = s0; c.zc[3 * a + 1] = s1; c.zc[3 * a + 2] = s2;
      dot = s0 * rc[3 * a] + s1 * rc[3 * a + 1] + s2 * rc[3 * a + 2];
    }
  }
  if (lane == 0) sh[wid] = dot;
  __syncthreads();
  if (threadIdx.x == 0) part_rz_extra[blockIdx.x] = sh[0] + sh[1] + sh[2] + sh[3];
}

// Minv (packed 3x3 diagonal) = 1/deg ; nodes without edges get identity
__global__ void ra_build_precond(int n, const double* __restrict__ deg, double* __restrict__ Minv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double d0 = deg[3 * (size_t)i], d1 = deg[3 * (size_t)i + 1], d2 = deg[3 * (size_t)i + 2];
  double* m = Minv + 6 * (size_t)i;
  m[0] = d0 > 0.0 ? 1.0 / d0 : 1.0; m[1] = 0; m[2] = 0; m[3] = d1 > 0.0 ? 1.0 / d1 : 1.0; m[4] = 0; m[5] = d2 > 0.0 ? 1.0 / d2 : 1.0;
}

// b = w * r  (row-weighted residual of the L1 stage); norms[0] += |b|^2
__global__ void ra_weighted_rhs(RAView v, const double* __restrict__ w, const double* __restrict__ res,
                                double* __restrict__ b, double* __restrict__ norms) {
  __shared__ double scratch[32];
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double s = 0.0;
  if (e < v.E) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double t = w[e] * res[3 * e + k];
      b[3 * e + k] = t;
      s += t * t;
    }
  }
  s = block_sum(s, scratch);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(&norms[0], s);
}

// One ADMM iteration after the x-update (colmap LeastAbsoluteDeviationSolver,
// rho = alpha = 1):  a = A_w x; z = shrink(a - b + u, 1/rho); u += a - z - b;
//   norms[1] += |a - z - b|^2, norms[2] += |a|^2, norms[3] += |z|^2
//   rhs  += A_w^T (b + z - u)      (next x-update)
//   svec += A_w^T (z - z_old)      (dual residual)
//   uvec += A_w^T u                (dual tolerance)
__global__ void ra_admm_step(RAView v, const double* __restrict__ w, const double* __restrict__ x,
                             const double* __restrict__ b, double* __restrict__ z, double* __restrict__ u, double rho,
                             double* __restrict__ rhs, double* __restrict__ svec, double* __restrict__ uvec,
                             double* __restrict__ norms) {
  __shared__ double scratch[32];
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double n1 = 0, n2 = 0, n3 = 0;
  if (e < v.E) {
    const int i = v.ei[e], j = v.ej[e];
    const double we = w[e];
    const double kappa = 1.0 / rho;
    const EdgeRows er = edge_rows(v, i, j);
    const int nci = (v.eci && i >= 0) ? v.eci[e] : -1, ncj = (v.ecj && i >= 0) ? v.ecj[e] : -1;
    const bool same_frame = i == j;   // unknown cameras only: the frame coefficients cancel
    double r3[3] = {0, 0, 0}, s3[3] = {0, 0, 0}, u3[3] = {0, 0, 0};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (er.y_only && k != 1) continue;   // this row does not exist
      double a = same_frame ? 0.0 : coef(er.gj, k) * x[3 * (size_t)j + k];
      if (i >= 0 && !same_frame) a -= coef(er.gi, k) * x[3 * (size_t)i + k];
      if (ncj >= 0) a += x[3 * (size_t)ncj + k];
      if (nci >= 0) a -= x[3 * (size_t)nci + k];
      a *= we;
      const double bo = b[3 * e + k], zo = z[3 * e + k], uo = u[3 * e + k];
      const double vv = a - bo + uo;
      const double zn = fmax(0.0, vv - kappa) - fmax(0.0, -vv - kappa);
      const double un = uo + a - zn - bo;
      z[3 * e + k] = zn;
      u[3 * e + k] = un;
      const double pr = a - zn - bo;
      n1 += pr * pr;
      n2 += a * a;
      n3 += zn * zn;
      r3[k] = we * (bo + zn - un);
      s3[k] = we * (zn - zo);
      u3[k] = we * un;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (er.y_only && k != 1) continue;
      if (coef(er.gj, k) != 0.0 && !same_frame) {
        atomicAdd(&rhs[3 * (size_t)j + k], r3[k]);
        atomicAdd(&svec[3 * (size_t)j + k], s3[k]);
        atomicAdd(&uvec[3 * (size_t)j + k], u3[k]);
      }
      if (i >= 0 && coef(er.gi, k) != 0.0 && !same_frame) {
        atomicAdd(&rhs[3 * (size_t)i + k], -r3[k]);
        atomicAdd(&svec[3 * (size_t)i + k], -s3[k]);
        atomicAdd(&uvec[3 * (size_t)i + k], -u3[k]);
      }
      if (ncj >= 0) {
        atomicAdd(&rhs[3 * (size_t)ncj + k], r3[k]);
        atomicAdd(&svec[3 * (size_t)ncj + k], s3[k]);
        atomicAdd(&uvec[3 * (size_t)ncj + k], u3[k]);
      }
      if (nci >= 0) {
        atomicAdd(&rhs[3 * (size_t)nci + k], -r3[k]);
        atomicAdd(&svec[3 * (size_t)nci + k], -s3[k]);
        atomicAdd(&uvec[3 * (size_t)nci + k], -u3[k]);
      }
    }
  }
  n1 = block_sum(n1, scratch);
  n2 = block_sum(n2, scratch);
  n3 = block_sum(n3, scratch);
  if (threadIdx.x == 0) {
    atomicAdd(&norms[1], n1);
    atomicAdd(&norms[2], n2);
    atomicAdd(&norms[3], n3);
  }
}

// UpdateGlobalRotations (.cc:631-640): theta <- log(exp(theta) exp(-step));
// sums[0] += |step_i| (ComputeAverageStepSize .cc:758-772), sums[1] += |step|^2,
// sums[2] = NaN flag
__global__ void ra_update(int n, int n_frames, double* __restrict__ theta, const double* __restrict__ step,
                          double* __restrict__ sums, const unsigned char* __restrict__ node_grav) {
  __shared__ double scratch[32];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double s1 = 0, s2 = 0, bad = 0;
  if (i >= n_frames && i < n) {   // unknown-camera node: updated by ra_update_cams; only |step|^2 / NaN are accounted here
    const double d[3] = {step[3 * (size_t)i], step[3 * (size_t)i + 1], step[3 * (size_t)i + 2]};
    s2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    if (isnan(s2)) bad = 1.0;
  }
  if (i < n_frames) {
    const double d[3] = {step[3 * (size_t)i], step[3 * (size_t)i + 1], step[3 * (size_t)i + 2]};
    const double nd[3] = {-d[0], -d[1], -d[2]};
    const double t[3] = {theta[3 * (size_t)i], theta[3 * (size_t)i + 1], theta[3 * (size_t)i + 2]};
    double R[9], Rd[9], M[9], out[3];
    if (node_grav && node_grav[i]) {       // 1-DoF frame: phi -= step (.cc:641-643)
      out[0] = 0.0;
      out[1] = t[1] - d[1];
      out[2] = 0.0;
    } else {
      aa_to_R(t, R);
      aa_to_R(nd, Rd);
      mat3_mul(R, Rd, M);
      R_to_aa(M, out);
    }
    theta[3 * (size_t)i] = out[0];
    theta[3 * (size_t)i + 1] = out[1];
    theta[3 * (size_t)i + 2] = out[2];
    const double sq = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    s1 = sqrt(sq);
    s2 = sq;
    if (isnan(sq)) bad = 1.0;
  }
  s1 = block_sum(s1, scratch);
  s2 = block_sum(s2, scratch);
  bad = block_sum(bad, scratch);
  if (threadIdx.x == 0) {
    atomicAdd(&sums[0], s1);
    atomicAdd(&sums[1], s2);
    if (bad > 0) atomicAdd(&sums[2], bad);
  }
}

// colmap::AverageQuaternions with unit weights (UPSTREAM-UNVERIFIED restatement), in two halves shared by ra_update_cams
// and rig_init_kernels.cuh: the packed symmetric 4x4 sum q q^T (10 entries, row by row) and its dominant eigenvector.
__device__ __forceinline__ void quat_outer_acc(double M[10], const double q[4]) {
  int idx = 0;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = a; b < 4; ++b) M[idx++] += q[a] * q[b];
}
// dominant eigenvector by cyclic Jacobi, a fixed 8 sweeps over the 6 planes (quadratic convergence: the off-diagonal
// mass is at rounding level after 4-5 on a 4x4, so the result is exact to about eps / relative gap however close the
// second eigenvalue is; a power iteration would need ~ log(eps) / log(lambda2 / lambda1) steps); the sign follows q0
__device__ __forceinline__ void quat_avg_eig(const double M[10], const double q0[4], double v[4]) {
  double A[4][4] = {{M[0], M[1], M[2], M[3]}, {M[1], M[4], M[5], M[6]}, {M[2], M[5], M[7], M[8]}, {M[3], M[6], M[8], M[9]}};
  double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sweep = 0; sweep < 8; ++sweep) {
#pragma unroll
    for (int pq = 0; pq < 6; ++pq) {
      const int p = pq < 3 ? 0 : (pq < 5 ? 1 : 2), q = pq < 3 ? pq + 1 : (pq < 5 ? pq - 1 : 3);
      const double apq = A[p][q];
      if (apq == 0.0) continue;
      const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
      const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
      for (int k = 0; k < 4; ++k) {   // A <- J^T A J, J = rotation in (p, q)
        const double akp = A[k][p], akq = A[k][q];
        A[k][p] = c * akp - s * akq;
        A[k][q] = s * akp + c * akq;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const double apk = A[p][k], aqk = A[q][k];
        A[p][k] = c * apk - s * aqk;
        A[q][k] = s * apk + c * aqk;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const double vkp = V[k][p], vkq = V[k][q];
        V[k][p] = c * vkp - s * vkq;
        V[k][q] = s * vkp + c * vkq;
      }
    }
  }
  int m = 0;
#pragma unroll
  for (int k = 1; k < 4; ++k)
    if (A[k][k] > A[m][m]) m = k;
  const double dot = V[0][m] * q0[0] + V[1][m] * q0[1] + V[2][m] * q0[2] + V[3][m] * q0[3];
  const double sg = dot < 0.0 ? -1.0 : 1.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = sg * V[k][m];
}

// Unknown cam_from_rig rotations (.cc:646-693): for every frame f that holds an image of camera c the updated rotation
// is R_c R_f exp(-step_c) R_f^T (R_f = the frame's ALREADY UPDATED rotation); the new R_c is the quaternion average
// (colmap::AverageQuaternions, unit weights: dominant eigenvector of sum q q^T) over those frames.  One warp per camera.
__global__ void __launch_bounds__(128) ra_update_cams(int n_frames, int n_cams, double* __restrict__ theta,
                                                      const double* __restrict__ step, const int* __restrict__ cf_begin,
                                                      const int* __restrict__ cf_list) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= n_cams) return;
  const size_t node = (size_t)n_frames + c;
  const double tc[3] = {theta[3 * node], theta[3 * node + 1], theta[3 * node + 2]};
  const double ns[3] = {-step[3 * node], -step[3 * node + 1], -step[3 * node + 2]};
  double Rc[9], Ru[9];
  aa_to_R(tc, Rc);
  aa_to_R(ns, Ru);
  double M[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // packed symmetric 4x4 of sum q q^T
  double q0[4] = {0, 0, 0, 1};
  bool have0 = false;
  for (int s = cf_begin[c] + lane; s < cf_begin[c + 1]; s += 32) {
    const int f = cf_list[s];
    const double tf[3] = {theta[3 * (size_t)f], theta[3 * (size_t)f + 1], theta[3 * (size_t)f + 2]};
    double Rf[9], A[9], B[9], P[9];
    aa_to_R(tf, Rf);
    mat3_mul(Rc, Rf, A);        // R_c R_f
    mat3_mul(A, Ru, B);         // R_c R_f R_upd
#pragma unroll
    for (int i = 0; i < 3; ++i)   // P = B R_f^T
#pragma unroll
      for (int j = 0; j < 3; ++j) P[3 * i + j] = B[3 * i] * Rf[3 * j] + B[3 * i + 1] * Rf[3 * j + 1] + B[3 * i + 2] * Rf[3 * j + 2];
    double q[4];   // Eigen::Quaterniond(Matrix3d)
    const double t = P[0] + P[4] + P[8];
    if (t > 0.0) {
      double tt = sqrt(t + 1.0);
      q[3] = 0.5 * tt;
      tt = 0.5 / tt;
      q[0] = (P[7] - P[5]) * tt; q[1] = (P[2] - P[6]) * tt; q[2] = (P[3] - P[1]) * tt;
    } else {
      int i = 0;
      if (P[4] > P[0]) i = 1;
      if (P[8] > P[4 * i]) i = 2;
      const int j = (i + 1) % 3, k = (i + 2) % 3;
      double tt = sqrt(P[4 * i] - P[4 * j] - P[4 * k] + 1.0);
      q[i] = 0.5 * tt;
      tt = 0.5 / tt;
      q[3] = (P[3 * k + j] - P[3 * j + k]) * tt; q[j] = (P[3 * j + i] + P[3 * i + j]) * tt; q[k] = (P[3 * k + i] + P[3 * i + k]) * tt;
    }
    quat_outer_acc(M, q);
    if (!have0) { q0[0] = q[0]; q0[1] = q[1]; q0[2] = q[2]; q0[3] = q[3]; have0 = true; }
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) M[k] = warp_sum(M[k]);
  if (lane != 0 || cf_begin[c + 1] == cf_begin[c]) return;
  double v[4];
  quat_avg_eig(M, q0, v);
  double R[9], out[3];
  quat_to_R(v, R);
  R_to_aa(R, out);
  theta[3 * node] = out[0]; theta[3 * node + 1] = out[1]; theta[3 * node + 2] = out[2];
}

// |a|^2, |b|^2 of node vectors: per-CTA partials (deterministic two-stage sum)
__global__ void __launch_bounds__(256) ra_norm2_partial(int n3, const double* __restrict__ a, const double* __restrict__ b,
                                                        double* __restrict__ part_a, double* __restrict__ part_b) {
  __shared__ double scratch[32];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double s0 = 0, s1 = 0;
  if (i < n3) {
    s0 = a[i] * a[i];
    s1 = b[i] * b[i];
  }
  s0 = block_sum(s0, scratch);
  s1 = block_sum(s1, scratch);
  if (threadIdx.x == 0) {
    part_a[blockIdx.x] = s0;
    part_b[blockIdx.x] = s1;
  }
}
__global__ void ra_norm2_final(int nblk, const double* __restrict__ part_a, const double* __restrict__ part_b,
                               double* __restrict__ out) {
  __shared__ double scratch[32];
  double s0 = 0, s1 = 0;
  for (int i = threadIdx.x; i < nblk; i += blockDim.x) {
    s0 += part_a[i];
    s1 += part_b[i];
  }
  s0 = block_sum(s0, scratch);
  s1 = block_sum(s1, scratch);
  if (threadIdx.x == 0) {
    out[0] = s0;
    out[1] = s1;
  }
}

// Warm-started PCG initialisation: x is kept, Ax holds L x (all-reduced):
//   r = b - Ax; z = Minv r; p = z; Ax <- 0; partial r.z, r.r, b.b
// Minv is the packed 3x3 diagonal of ra_build_precond: a gravity frame's slots differ (1, 1/d_y, 1), so each slot
// takes its own entry, as pcg_init / pcg_update apply it
__global__ void __launch_bounds__(128) ra_pcg_init_warm(int nb, const double* __restrict__ Minv,
                                                        const double* __restrict__ b, double* __restrict__ Ax,
                                                        double* __restrict__ r, double* __restrict__ z,
                                                        double* __restrict__ p, double* __restrict__ part_bb,
                                                        double* __restrict__ part_rz, double* __restrict__ part_rr) {
  __shared__ double scratch[32];
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  double rz = 0, rr = 0, bb = 0;
  if (c < nb) {
    const double minv[3] = {Minv[6 * (size_t)c], Minv[6 * (size_t)c + 3], Minv[6 * (size_t)c + 5]};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const size_t i = 3 * (size_t)c + k;
      const double bv = b[i];
      const double rv = bv - Ax[i];
      Ax[i] = 0.0;
      const double zv = minv[k] * rv;
      r[i] = rv;
      z[i] = zv;
      p[i] = zv;
      rz += rv * zv;
      rr += rv * rv;
      bb += bv * bv;
    }
  }
  rz = block_sum(rz, scratch);
  rr = block_sum(rr, scratch);
  bb = block_sum(bb, scratch);
  if (threadIdx.x == 0) {
    part_rz[blockIdx.x] = rz;
    part_rr[blockIdx.x] = rr;
    part_bb[blockIdx.x] = bb;
  }
}
__global__ void __launch_bounds__(128) ra_publish_warm(int nblk, const double* __restrict__ part_bb,
                                                       const double* __restrict__ part_rz,
                                                       const double* __restrict__ part_rr, double* __restrict__ dots0) {
  __shared__ double scratch[32];
  double a = 0, b = 0, c = 0;
  for (int i = threadIdx.x; i < nblk; i += blockDim.x) {
    a += part_bb[i];
    b += part_rz[i];
    c += part_rr[i];
  }
  a = block_sum(a, scratch);
  b = block_sum(b, scratch);
  c = block_sum(c, scratch);
  if (threadIdx.x == 0) {
    dots0[0] = 0.0;
    dots0[1] = b;
    dots0[2] = c;
    dots0[3] = a;   // |b|^2: the convergence reference of a warm-started solve
  }
}

}  // namespace b200
