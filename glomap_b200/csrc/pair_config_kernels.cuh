// pair_config_kernels.cuh -- device side of ViewGraphManipulater::UpdateImagePairsConfig
// (processors/view_graph_manipulation.cc:178-237), the first half of stage 0 of GlobalMapper::Solve
// (controllers/global_mapper.cc:22-34):
//   pass 1, one thread per pair: a valid pair whose two cameras both have a prior focal adds 1 to `total` of both cameras
//     when it is CALIBRATED or UNCALIBRATED, and 1 to `calibrated` of both when it is CALIBRATED.  A pair inside one camera
//     counts twice for it, as the reference's two increments do.  Integer atomics: the counts do not depend on order.
//   camera validity: calibrated * 1. / total > 0.5 in FP64, strict; a camera no pair counted is not valid (the reference's
//     camera_validity[id] default-constructs to false).
//   pass 2, one thread per pair: a valid UNCALIBRATED pair whose two cameras are valid becomes CALIBRATED and gets
//     F = K2^-T [t]x R K1^-1 (FundamentalFromMotionAndCameras, math/two_view_geometry.cc:38-55, with Camera::GetK,
//     scene/camera.h:34-39: fx = fy = f for the SIMPLE_* models).  R is Eigen's toRotationMatrix of the pair's
//     cam2_from_cam1 quaternion as stored (not normalised, as Eigen does not), t its translation.  K^-1 is taken in closed
//     form, [[1/fx, 0, -cx/fx], [0, 1/fy, -cy/fy], [0, 0, 1]], and the products are explicitly rounded FP64 operations
//     (no FMA contraction) in the host restatement's order, so the device F equals it bit for bit.
// Pass 2 writes device copies only; the host buffers are written when no index was out of range and no promoted pair has
// a camera model outside 0-3.
#pragma once
#include "context.cuh"

namespace b200 {

// flags[0]: a camera index out of range; flags[1]: a promoted pair's camera has a model outside 0-3; flags[2]: promoted
__global__ void pc_count(long long E, int K, const int* __restrict__ cam1, const int* __restrict__ cam2,
                         const unsigned char* __restrict__ valid, const int* __restrict__ config,
                         const unsigned char* __restrict__ prior, int* __restrict__ total, int* __restrict__ calibrated,
                         int* __restrict__ flags) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int a = cam1[e], b = cam2[e];
  if (a < 0 || a >= K || b < 0 || b >= K) {
    flags[0] = 1;
    return;
  }
  if (!valid[e] || !prior[a] || !prior[b]) return;
  const int c = config[e];
  if (c == B200SFM_TWO_VIEW_CALIBRATED) {
    atomicAdd(&total[a], 1);
    atomicAdd(&total[b], 1);
    atomicAdd(&calibrated[a], 1);
    atomicAdd(&calibrated[b], 1);
  } else if (c == B200SFM_TWO_VIEW_UNCALIBRATED) {
    atomicAdd(&total[a], 1);
    atomicAdd(&total[b], 1);
  }
}

__device__ __forceinline__ bool pc_camera_valid(const int* __restrict__ total, const int* __restrict__ calibrated, int k) {
  const int t = total[k];
  return t > 0 && (double)calibrated[k] / (double)t > 0.5;
}

// fx, fy, cx, cy of Camera::GetK for models 0-3; false for any other model
__device__ __forceinline__ bool pc_pinhole(int model, const double* __restrict__ p, double& fx, double& fy, double& cx,
                                           double& cy) {
  if (model == B200SFM_PINHOLE) {
    fx = p[0]; fy = p[1]; cx = p[2]; cy = p[3];
    return true;
  }
  if (model == B200SFM_SIMPLE_PINHOLE || model == B200SFM_SIMPLE_RADIAL || model == B200SFM_RADIAL) {
    fx = fy = p[0]; cx = p[1]; cy = p[2];
    return true;
  }
  return false;
}

__global__ void pc_promote(long long E, int K, const int* __restrict__ cam1, const int* __restrict__ cam2,
                           const unsigned char* __restrict__ valid, const int* __restrict__ total,
                           const int* __restrict__ calibrated, const int* __restrict__ model, const double* __restrict__ intr,
                           const double* __restrict__ quat, const double* __restrict__ trans, int* __restrict__ config,
                           double* __restrict__ F, int* __restrict__ flags) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool promoted = false;
  if (e < E && valid[e] && config[e] == B200SFM_TWO_VIEW_UNCALIBRATED) {
    const int a = cam1[e], b = cam2[e];   // pc_count flags an index out of range; it is skipped here
    if (a >= 0 && a < K && b >= 0 && b < K && pc_camera_valid(total, calibrated, a) && pc_camera_valid(total, calibrated, b)) {
      double fx1, fy1, cx1, cy1, fx2, fy2, cx2, cy2;
      if (!pc_pinhole(model[a], intr + (size_t)a * B200SFM_INTR_STRIDE, fx1, fy1, cx1, cy1) ||
          !pc_pinhole(model[b], intr + (size_t)b * B200SFM_INTR_STRIDE, fx2, fy2, cx2, cy2)) {
        flags[1] = 1;
      } else {
        promoted = true;
        config[e] = B200SFM_TWO_VIEW_CALIBRATED;
        // Eigen's Quaternion::toRotationMatrix (Geometry/Quaternion.h); every product and sum rounded on its own, in the
        // order of view_graph_manipulation.fundamental_from_motion_and_cameras, so that the two agree bit for bit
        const double x = quat[4 * e], y = quat[4 * e + 1], z = quat[4 * e + 2], w = quat[4 * e + 3];
        const double tx = __dmul_rn(2.0, x), ty = __dmul_rn(2.0, y), tz = __dmul_rn(2.0, z);
        const double twx = __dmul_rn(tx, w), twy = __dmul_rn(ty, w), twz = __dmul_rn(tz, w), txx = __dmul_rn(tx, x),
                     txy = __dmul_rn(ty, x), txz = __dmul_rn(tz, x), tyy = __dmul_rn(ty, y), tyz = __dmul_rn(tz, y),
                     tzz = __dmul_rn(tz, z);
        const double R[9] = {__dsub_rn(1.0, __dadd_rn(tyy, tzz)), __dsub_rn(txy, twz), __dadd_rn(txz, twy),
                             __dadd_rn(txy, twz), __dsub_rn(1.0, __dadd_rn(txx, tzz)), __dsub_rn(tyz, twx),
                             __dsub_rn(txz, twy), __dadd_rn(tyz, twx), __dsub_rn(1.0, __dadd_rn(txx, tyy))};
        const double t0 = trans[3 * e], t1 = trans[3 * e + 1], t2 = trans[3 * e + 2];
        const double T[9] = {0.0, -t2, t1, t2, 0.0, -t0, -t1, t0, 0.0};   // EssentialFromMotion: [t]x R
        double Em[9];
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c)
            Em[3 * r + c] = __dadd_rn(__dadd_rn(__dmul_rn(T[3 * r], R[c]), __dmul_rn(T[3 * r + 1], R[3 + c])),
                                      __dmul_rn(T[3 * r + 2], R[6 + c]));
        // M = E K1^-1: column 0 / fx1, column 1 / fy1, column 2 - cx1/fx1 col 0 - cy1/fy1 col 1
        const double ia = __ddiv_rn(1.0, fx1), ib = __ddiv_rn(1.0, fy1), ua = __ddiv_rn(-cx1, fx1), ub = __ddiv_rn(-cy1, fy1);
        double M[9];
        for (int r = 0; r < 3; ++r) {
          M[3 * r] = __dmul_rn(Em[3 * r], ia);
          M[3 * r + 1] = __dmul_rn(Em[3 * r + 1], ib);
          M[3 * r + 2] = __dadd_rn(__dadd_rn(__dmul_rn(Em[3 * r], ua), __dmul_rn(Em[3 * r + 1], ub)), Em[3 * r + 2]);
        }
        // F = K2^-T M: K2^-T = [[1/fx2, 0, 0], [0, 1/fy2, 0], [-cx2/fx2, -cy2/fy2, 1]]
        const double ja = __ddiv_rn(1.0, fx2), jb = __ddiv_rn(1.0, fy2), va = __ddiv_rn(-cx2, fx2), vb = __ddiv_rn(-cy2, fy2);
        double* f = F + 9 * e;
        for (int c = 0; c < 3; ++c) {
          f[c] = __dmul_rn(M[c], ja);
          f[3 + c] = __dmul_rn(M[3 + c], jb);
          f[6 + c] = __dadd_rn(__dadd_rn(__dmul_rn(M[c], va), __dmul_rn(M[3 + c], vb)), M[6 + c]);
        }
      }
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, promoted);   // one atomic per warp with a promoted pair
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&flags[2], __popc(m));
}

// Returns 0 on success, 1 when a camera index is out of range, 2 when a promoted pair's camera has a model outside 0-3
// (the host buffers are then untouched).  Arguments validated by the caller: E >= 1, K >= 1, null pointers.
inline int update_image_pairs_config(b200sfm_ctx* ctx, int K, const int* h_model, const double* h_intr, const unsigned char* h_prior,
                                     long long E, const int* h_cam1, const int* h_cam2, const unsigned char* h_valid,
                                     const double* h_quat, const double* h_trans, int* h_config, double* h_F,
                                     long long* num_promoted) {
  cudaStream_t s = ctx->stream;
  DevBuf<int> model, cam1, cam2, config, total, calibrated, flags;
  DevBuf<unsigned char> prior, valid;
  DevBuf<double> intr, quat, trans, F;
  model.alloc(K); intr.alloc((size_t)K * B200SFM_INTR_STRIDE); prior.alloc(K); total.alloc(K); calibrated.alloc(K);
  cam1.alloc(E); cam2.alloc(E); valid.alloc(E); config.alloc(E); quat.alloc(4 * (size_t)E); trans.alloc(3 * (size_t)E);
  F.alloc(9 * (size_t)E); flags.alloc(4);
  model.upload(h_model, K, s); intr.upload(h_intr, (size_t)K * B200SFM_INTR_STRIDE, s); prior.upload(h_prior, K, s);
  cam1.upload(h_cam1, E, s); cam2.upload(h_cam2, E, s); valid.upload(h_valid, E, s); config.upload(h_config, E, s);
  quat.upload(h_quat, 4 * (size_t)E, s); trans.upload(h_trans, 3 * (size_t)E, s); F.upload(h_F, 9 * (size_t)E, s);
  total.zero(s); calibrated.zero(s); flags.zero(s);
  B200_LAUNCH(ctx, pc_count, cdiv(E, 256), 256, 0, E, K, cam1.p, cam2.p, valid.p, config.p, prior.p, total.p, calibrated.p, flags.p);
  B200_LAUNCH(ctx, pc_promote, cdiv(E, 256), 256, 0, E, K, cam1.p, cam2.p, valid.p, total.p, calibrated.p, model.p, intr.p, quat.p,
              trans.p, config.p, F.p, flags.p);
  int h[4];
  B200_CUDA_OK(cudaMemcpyAsync(h, flags.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  B200_CUDA_OK(cudaStreamSynchronize(s));
  if (h[0]) return 1;
  if (h[1]) return 2;
  config.download(h_config, E, s);
  F.download(h_F, 9 * (size_t)E, s);
  B200_CUDA_OK(cudaStreamSynchronize(s));
  *num_promoted = h[2];
  return 0;
}

}  // namespace b200
