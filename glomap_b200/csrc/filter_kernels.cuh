// filter_kernels.cuh -- track filters on the device-resident BA arrays
// (SURVEY.md 8(f) item 1).  Reference: glomap/processors/track_filter.cc
//   FilterTracksByReprojection   :7-52   (pixel space, in_normalized_image = false)
//   FilterTracksByAngle          :54-90
//   FilterTrackTriangulationAngle:92-127
// They run between every BA call of the mapper (controllers/global_mapper.cc:164-186,
// 243-276,309-337) on exactly the arrays the BA problem keeps in HBM; the kernels
// write a keep-mask per observation (or per track) and count the changed tracks,
// the host compacts Track::observations.
#pragma once
#include "ba_kernels.cuh"

namespace b200 {

constexpr double kFilterEps = 1e-12;   // glomap/types.h EPS

// keep[o] = 1 iff z >= EPS and |ImgFromCam(R X + t) - xy| < max_err   (track_filter.cc:19-42)
// one thread per observation; changed[pt] = 1 when any observation of the track is dropped
__global__ void filter_reprojection(BAView v, const double* __restrict__ cam_rec, const double* __restrict__ intr_rec,
                                    const double* __restrict__ points, double max_err,
                                    unsigned char* __restrict__ keep, int* __restrict__ changed) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= v.N) return;
  const int pt = v.obs_pt[o], cam = v.obs_cam[o];
  const double2 xy = v.obs_xy[o];
  const double4 q4 = ld_rec32(cam_rec + (size_t)cam * kCamRec);
  const double4 t4 = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
  const double q[4] = {q4.x, q4.y, q4.z, q4.w};
  double R[9];
  quat_to_R(q, R);
  const double X0 = points[3 * (size_t)pt], X1 = points[3 * (size_t)pt + 1], X2 = points[3 * (size_t)pt + 2];
  double xc = R[0] * X0 + R[1] * X1 + R[2] * X2 + t4.x;
  double yc = R[3] * X0 + R[4] * X1 + R[5] * X2 + t4.y;
  double zc = R[6] * X0 + R[7] * X1 + R[8] * X2 + t4.z;
  const double* sr = sensor_of_obs(v, o);
  if (sr) sensor_apply(sr, xc, yc, zc);   // cam_from_world = cam_from_rig * rig_from_world
  bool k = false;
  if (!(zc < kFilterEps)) {
    double px, py;
    project_only(intr_rec + (size_t)obs_intr_idx(t4, sr) * kIntrRec, xc, yc, zc, px, py);
    const double dx = px - xy.x, dy = py - xy.y;
    k = sqrt(dx * dx + dy * dy) < max_err;
  }
  keep[o] = k ? 1 : 0;
  if (!k) changed[pt] = 1;
}

// keep[o] = 1 iff z >= EPS and normalized(R X + t) . bearing > cos(max_angle [* 2 if uncalibrated])
// (track_filter.cc:61-80)
__global__ void filter_angle(BAView v, const double* __restrict__ cam_rec, const double* __restrict__ points,
                             const double* __restrict__ bearings, const unsigned char* __restrict__ calibrated,
                             double thres, double thres_uncalib, unsigned char* __restrict__ keep,
                             int* __restrict__ changed) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= v.N) return;
  const int pt = v.obs_pt[o], cam = v.obs_cam[o];
  const double4 q4 = ld_rec32(cam_rec + (size_t)cam * kCamRec);
  const double4 t4 = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
  const double q[4] = {q4.x, q4.y, q4.z, q4.w};
  double R[9];
  quat_to_R(q, R);
  const double X0 = points[3 * (size_t)pt], X1 = points[3 * (size_t)pt + 1], X2 = points[3 * (size_t)pt + 2];
  double xc = R[0] * X0 + R[1] * X1 + R[2] * X2 + t4.x;
  double yc = R[3] * X0 + R[4] * X1 + R[5] * X2 + t4.y;
  double zc = R[6] * X0 + R[7] * X1 + R[8] * X2 + t4.z;
  const double* sr = sensor_of_obs(v, o);
  if (sr) sensor_apply(sr, xc, yc, zc);
  bool k = false;
  if (!(zc < kFilterEps)) {
    const double inv = 1.0 / sqrt(xc * xc + yc * yc + zc * zc);
    const double d = (xc * bearings[3 * o] + yc * bearings[3 * o + 1] + zc * bearings[3 * o + 2]) * inv;
    // the prior-focal flag belongs to the camera: per image without rigs, per sensor with rigs
    const int ci = v.S > 0 ? (int)v.obs_sensor[o] : cam;
    const double th = (calibrated == nullptr || calibrated[ci]) ? thres : thres_uncalib;
    k = d > th;
  }
  keep[o] = k ? 1 : 0;
  if (!k) changed[pt] = 1;
}

// keep[o] = 1 iff z >= EPS and | (X_c.xy / X_c.z) - b.xy / (b.z + EPS) | < max_err, b = features_undist
// (track_filter.cc:24-31, in_normalized_image = true -- the variant the mapper calls, controllers/global_mapper.cc:176-181,254-259)
__global__ void filter_reprojection_normalized(BAView v, const double* __restrict__ cam_rec,
                                               const double* __restrict__ points, const double* __restrict__ bearings,
                                               double max_err, unsigned char* __restrict__ keep,
                                               int* __restrict__ changed) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= v.N) return;
  const int pt = v.obs_pt[o], cam = v.obs_cam[o];
  const double4 q4 = ld_rec32(cam_rec + (size_t)cam * kCamRec);
  const double4 t4 = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
  const double q[4] = {q4.x, q4.y, q4.z, q4.w};
  double R[9];
  quat_to_R(q, R);
  const double X0 = points[3 * (size_t)pt], X1 = points[3 * (size_t)pt + 1], X2 = points[3 * (size_t)pt + 2];
  double xc = R[0] * X0 + R[1] * X1 + R[2] * X2 + t4.x;
  double yc = R[3] * X0 + R[4] * X1 + R[5] * X2 + t4.y;
  double zc = R[6] * X0 + R[7] * X1 + R[8] * X2 + t4.z;
  const double* sr = sensor_of_obs(v, o);
  if (sr) sensor_apply(sr, xc, yc, zc);
  bool k = false;
  if (!(zc < kFilterEps)) {
    const double bz = bearings[3 * o + 2] + kFilterEps;
    const double dx = xc / zc - bearings[3 * o] / bz, dy = yc / zc - bearings[3 * o + 1] / bz;
    k = sqrt(dx * dx + dy * dy) < max_err;
  }
  keep[o] = k ? 1 : 0;
  if (!k) changed[pt] = 1;
}

// keep_track[p] = 1 iff some pair of viewing rays (X - c_i) has an angle larger than min_angle
// (track_filter.cc:98-122).  One warp per track; O(L^2) pair test spread over the lanes.
__global__ void filter_triangulation_angle(BAView v, const double* __restrict__ cam_rec,
                                           const double* __restrict__ points, double thres,
                                           unsigned char* __restrict__ keep_track, int* __restrict__ removed) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= v.P) return;
  const unsigned b = v.pt_begin[warp], e = v.pt_begin[warp + 1];
  const int L = (int)(e - b);
  const double X0 = points[3 * (size_t)warp], X1 = points[3 * (size_t)warp + 1], X2 = points[3 * (size_t)warp + 2];
  bool status = false;
  // rays recomputed on the fly: pairs (i, j), i < j, enumerated over the lanes
  const long long npairs = (long long)L * (L - 1) / 2;
  for (long long pidx = lane; pidx < npairs && !status; pidx += 32) {
    // invert pidx -> (i, j)
    int i = (int)((2.0 * L - 1 - sqrt((2.0 * L - 1) * (2.0 * L - 1) - 8.0 * (double)pidx)) / 2.0);
    while ((long long)i * (2 * L - i - 1) / 2 > pidx) --i;
    while ((long long)(i + 1) * (2 * L - i - 2) / 2 <= pidx) ++i;
    const int j = (int)(pidx - (long long)i * (2 * L - i - 1) / 2) + i + 1;
    double ray[2][3];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const unsigned oo = b + (s == 0 ? i : j);
      const int cam = v.obs_cam[oo];
      const double4 q4 = ld_rec32(cam_rec + (size_t)cam * kCamRec);
      const double4 t4 = ld_rec32(cam_rec + (size_t)cam * kCamRec + 4);
      const double q[4] = {q4.x, q4.y, q4.z, q4.w};
      double R[9];
      quat_to_R(q, R);
      // centre c = -R^T t ; ray = normalized(X - c).  Known rig: the image centre in the rig frame is
      // -R_cr^T t_cr, so t_f is replaced by t_f + R_cr^T t_cr.
      double tx = t4.x, ty = t4.y, tz = t4.z;
      const double* sr = sensor_of_obs(v, oo);
      if (sr) {
        tx += sr[0] * sr[9] + sr[3] * sr[10] + sr[6] * sr[11];
        ty += sr[1] * sr[9] + sr[4] * sr[10] + sr[7] * sr[11];
        tz += sr[2] * sr[9] + sr[5] * sr[10] + sr[8] * sr[11];
      }
      const double c0 = -(R[0] * tx + R[3] * ty + R[6] * tz);
      const double c1 = -(R[1] * tx + R[4] * ty + R[7] * tz);
      const double c2 = -(R[2] * tx + R[5] * ty + R[8] * tz);
      const double d0 = X0 - c0, d1 = X1 - c1, d2 = X2 - c2;
      // Eigen's normalized() leaves a zero vector as it is: a point on a camera centre gives a zero ray, whose dot
      // product 0 counts as a wide pair
      const double n2 = d0 * d0 + d1 * d1 + d2 * d2;
      const double inv = n2 > 0.0 ? 1.0 / sqrt(n2) : 0.0;
      ray[s][0] = d0 * inv; ray[s][1] = d1 * inv; ray[s][2] = d2 * inv;
    }
    if (ray[0][0] * ray[1][0] + ray[0][1] * ray[1][1] + ray[0][2] * ray[1][2] < thres) status = true;
  }
  status = __any_sync(0xffffffffu, status);
  if (lane == 0) {
    keep_track[warp] = status ? 1 : 0;
    if (!status) atomicAdd(removed, 1);
  }
}

__global__ void count_flags(int n, const int* __restrict__ flags, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int v = (i < n && flags[i]) ? 1 : 0;
  v = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(out, v);
}

}  // namespace b200
