// processor_kernels.cuh -- the two per-element processors that sit between the solvers in the mapper, on the arrays a
// resident BA problem already holds (SURVEY.md 8(f) item 2):
//   * NormalizeReconstruction (glomap/processors/reconstruction_normalizer.cc:5-104): robust (p0..p1 percentile of the
//     FLOAT coordinates, sorted per axis) bounding box and trimmed mean of the projection centres -> similarity with
//     identity rotation; applied to the frame poses (colmap::TransformCameraWorld), the cam_from_rig translations and the
//     points.  The mapper calls it between the BA solves (controllers/global_mapper.cc:185,232,336): on a resident
//     problem that is three small kernels instead of a download / upload of the whole state.
//   * UndistortImages (glomap/processors/image_undistorter.cc:7-53): pixel -> unit bearing per observation,
//     CamFromImg(xy).homogeneous().normalized().  Radial models are inverted with the 50-step fixed-point iteration of the
//     host restatement (glomap_b200/synthetic.py bearings_from_scene; colmap iterates Newton steps to the same point).
#pragma once
#include "ba_kernels.cuh"

namespace b200 {

// projection centre of every image as float: trivial frames -> C images; rigs -> F x S images (frame-major)
__global__ void proc_image_centres(int F, int S, const double* __restrict__ quat, const double* __restrict__ trans,
                                   const double* __restrict__ sens_q, const double* __restrict__ sens_t,
                                   float* __restrict__ cx, float* __restrict__ cy, float* __restrict__ cz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = S > 0 ? F * S : F;
  if (i >= n) return;
  const int f = S > 0 ? i / S : i;
  const double q[4] = {quat[4 * (size_t)f], quat[4 * (size_t)f + 1], quat[4 * (size_t)f + 2], quat[4 * (size_t)f + 3]};
  double R[9];
  quat_to_R(q, R);
  double t[3] = {trans[3 * (size_t)f], trans[3 * (size_t)f + 1], trans[3 * (size_t)f + 2]};
  if (S > 0) {   // cam_from_world = cam_from_rig o rig_from_world
    const int s = i % S;
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
    const double k1 = p[3], k2 = (m == 3) ? p[4] : 0.0;
    u = ud; v = vd;
    for (int it = 0; it < 50; ++it) {
      const double r2 = u * u + v * v;
      const double dd = 1.0 + k1 * r2 + k2 * r2 * r2;
      u = ud / dd; v = vd / dd;
    }
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
