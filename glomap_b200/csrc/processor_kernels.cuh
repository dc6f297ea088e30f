// processor_kernels.cuh -- the two per-element processors that sit between the solvers in the mapper, on the arrays a
// resident BA problem already holds (SURVEY.md 8(f) item 2):
//   * NormalizeReconstruction (glomap/processors/reconstruction_normalizer.cc:5-104): robust (p0..p1 percentile of the
//     FLOAT coordinates, sorted per axis) bounding box and trimmed mean of the projection centres -> similarity with
//     identity rotation; applied to the frame poses (colmap::TransformCameraWorld), the cam_from_rig translations and the
//     points.  The mapper calls it between the BA solves (controllers/global_mapper.cc:185,232,336): on a resident
//     problem that is three small kernels instead of a download / upload of the whole state.
//   * UndistortImages (glomap/processors/image_undistorter.cc:7-53): pixel -> unit bearing per observation,
//     CamFromImg(xy).homogeneous().normalized().  Radial models are inverted on the radius with a safeguarded Newton
//     iteration, the same steps as the host restatement (glomap_b200/synthetic.py bearings_from_pixels).
#pragma once
#include "ba_kernels.cuh"

namespace b200 {

// projection centre of every image as float: trivial frames -> n = C images; rigs -> n images (frame img_frame[i] seen
// through sensor img_sensor[i]), or with null tables the dense layout of n = F x S images (frame-major)
__global__ void proc_image_centres(int n, int S, const int* __restrict__ img_frame, const int* __restrict__ img_sensor,
                                   const double* __restrict__ quat, const double* __restrict__ trans,
                                   const double* __restrict__ sens_q, const double* __restrict__ sens_t,
                                   float* __restrict__ cx, float* __restrict__ cy, float* __restrict__ cz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = S > 0 ? (img_frame ? img_frame[i] : i / S) : i;
  const double q[4] = {quat[4 * (size_t)f], quat[4 * (size_t)f + 1], quat[4 * (size_t)f + 2], quat[4 * (size_t)f + 3]};
  double R[9];
  quat_to_R(q, R);
  double t[3] = {trans[3 * (size_t)f], trans[3 * (size_t)f + 1], trans[3 * (size_t)f + 2]};
  if (S > 0) {   // cam_from_world = cam_from_rig o rig_from_world
    const int s = img_sensor ? img_sensor[i] : i % S;
    const double qs[4] = {sens_q[4 * s], sens_q[4 * s + 1], sens_q[4 * s + 2], sens_q[4 * s + 3]};
    double Rs[9], Rc[9], tc[3];
    quat_to_R(qs, Rs);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) Rc[3 * r + c] = Rs[3 * r] * R[c] + Rs[3 * r + 1] * R[3 + c] + Rs[3 * r + 2] * R[6 + c];
      tc[r] = Rs[3 * r] * t[0] + Rs[3 * r + 1] * t[1] + Rs[3 * r + 2] * t[2] + sens_t[3 * s + r];
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = Rc[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) t[k] = tc[k];
  }
  // centre = -R^T t
  cx[i] = (float)(-(R[0] * t[0] + R[3] * t[1] + R[6] * t[2]));
  cy[i] = (float)(-(R[1] * t[0] + R[4] * t[1] + R[7] * t[2]));
  cz[i] = (float)(-(R[2] * t[0] + R[5] * t[1] + R[8] * t[2]));
}

// out[0..2] = sorted[P0], out[3..5] = sorted[P1], out[6..8] = sum_{i = P0..P1} sorted[i] (double accumulation); one CTA
__global__ void __launch_bounds__(256) proc_trimmed_stats(int P0, int P1, const float* __restrict__ sx, const float* __restrict__ sy,
                                                          const float* __restrict__ sz, double* __restrict__ out) {
  __shared__ double scratch[32];
  const float* srt[3] = {sx, sy, sz};
  for (int a = 0; a < 3; ++a) {
    double s = 0.0;
    for (int i = P0 + threadIdx.x; i <= P1; i += blockDim.x) s += (double)srt[a][i];
    s = block_sum(s, scratch);
    if (threadIdx.x == 0) {
      out[a] = (double)srt[a][P0];
      out[3 + a] = (double)srt[a][P1];
      out[6 + a] = s;
    }
    __syncthreads();
  }
}

// TransformCameraWorld for a similarity with identity rotation: rotation unchanged, t' = scale t - R tr
__global__ void proc_transform_frames(int F, double scale, double t0, double t1, double t2, const double* __restrict__ quat,
                                      double* __restrict__ trans) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const double q[4] = {quat[4 * (size_t)f], quat[4 * (size_t)f + 1], quat[4 * (size_t)f + 2], quat[4 * (size_t)f + 3]};
  double R[9];
  quat_to_R(q, R);
#pragma unroll
  for (int r = 0; r < 3; ++r)
    trans[3 * (size_t)f + r] = scale * trans[3 * (size_t)f + r] - (R[3 * r] * t0 + R[3 * r + 1] * t1 + R[3 * r + 2] * t2);
}
// y = scale y + (t0, t1, t2)  over n 3-vectors (points: the similarity; cam_from_rig translations: scale only, t = 0)
__global__ void proc_scale_shift3(long long n, double scale, double t0, double t1, double t2, double* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  y[3 * i] = scale * y[3 * i] + t0;
  y[3 * i + 1] = scale * y[3 * i + 1] + t1;
  y[3 * i + 2] = scale * y[3 * i + 2] + t2;
}

// Radial undistortion on the radius: the r in [0, r_fold] with g(r) = r (1 + k1 r^2 + k2 r^4) = rd, returned as the
// scale r / rd (1 at rd = 0).  g increases from 0 up to its fold r_fold, the first root of g'(r) = 1 + 3 k1 r^2 + 5 k2 r^4
// (none: g increases for good, and the root is below 2.25 rd because d(r^2) > 4/9 there).  Newton from r = rd inside the
// bracket [lo, hi] that the signs of g - rd maintain, a bisection where a step leaves it; stops when a step no longer
// moves r, or after kUndistortMaxIters.  Past the fold (rd > g(r_fold)) there is no inverse and the result, r_fold at
// most, is not meant to be used.  The host restatement (synthetic.undistort_radius_scale) takes the same steps.
constexpr int kUndistortMaxIters = 100;
__device__ __forceinline__ double undistort_radius_scale(double k1, double k2, double rd) {
  if (!(rd > 0.0)) return 1.0;
  // smallest positive root s of 1 + 3 k1 s + 5 k2 s^2 (s = r^2), or none
  double s_fold = -1.0;
  if (k2 == 0.0) {
    if (k1 < 0.0) s_fold = -1.0 / (3.0 * k1);
  } else {
    const double disc = 9.0 * k1 * k1 - 20.0 * k2;
    if (disc >= 0.0) {
      const double q = -0.5 * (3.0 * k1 + copysign(sqrt(disc), k1));   // roots q / (5 k2) and 1 / q
      const double a = q / (5.0 * k2), b = 1.0 / q;
      if (a > 0.0) s_fold = a;
      if (b > 0.0 && (s_fold < 0.0 || b < s_fold)) s_fold = b;
    }
  }
  double lo = 0.0, hi = s_fold > 0.0 ? sqrt(s_fold) : 2.25 * rd;
  double r = fmin(rd, hi);
  for (int it = 0; it < kUndistortMaxIters; ++it) {
    const double s = r * r;
    const double f = r * (1.0 + s * (k1 + k2 * s)) - rd;
    if (f < 0.0) lo = r; else hi = r;
    const double df = 1.0 + s * (3.0 * k1 + 5.0 * k2 * s);
    double rn = r - f / df;
    if (!(rn >= lo && rn <= hi)) rn = 0.5 * (lo + hi);   // outside the bracket, or df <= 0 / NaN
    if (rn == r) break;
    r = rn;
  }
  return r / rd;
}

// CamFromImg(xy).homogeneous().normalized() of one pixel for camera model m (0-3) with parameters p; writes out[0..2].
// Shared by UndistortImages below and the per-feature bearings of ImagePairsInlierCount (pair_kernels.cuh).
__device__ __forceinline__ void bearing_from_pixel(int m, const double* __restrict__ p, double2 xy, double* __restrict__ out) {
  double u, v;
  if (m == 0) {          // SIMPLE_PINHOLE f cx cy
    u = (xy.x - p[1]) / p[0]; v = (xy.y - p[2]) / p[0];
  } else if (m == 1) {   // PINHOLE fx fy cx cy
    u = (xy.x - p[2]) / p[0]; v = (xy.y - p[3]) / p[1];
  } else {               // SIMPLE_RADIAL f cx cy k / RADIAL f cx cy k1 k2
    const double ud = (xy.x - p[1]) / p[0], vd = (xy.y - p[2]) / p[0];
    const double sc = undistort_radius_scale(p[3], (m == 3) ? p[4] : 0.0, sqrt(ud * ud + vd * vd));
    u = ud * sc; v = vd * sc;
  }
  const double inv = 1.0 / sqrt(u * u + v * v + 1.0);
  out[0] = u * inv;
  out[1] = v * inv;
  out[2] = inv;
}

// unit bearing of every observation (caller's point-order indexing), from the CURRENT intrinsics
__global__ void proc_undistort(long long N, int S, const int* __restrict__ obs_cam, const unsigned short* __restrict__ obs_sensor,
                               const int* __restrict__ cam_intr, const int* __restrict__ sensor_intr,
                               const int* __restrict__ intr_model, const double* __restrict__ intr /*[K][12]*/,
                               const double2* __restrict__ obs_xy, double* __restrict__ out) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= N) return;
  const int blk = S > 0 ? sensor_intr[obs_sensor[o]] : cam_intr[obs_cam[o]];
  bearing_from_pixel(intr_model[blk], intr + (size_t)blk * 12, obs_xy[o], out + 3 * o);
}

}  // namespace b200
