// rig_init_kernels.cuh -- device side of ConvertRotationsFromImageToRig (glomap/estimators/rotation_initializer.cc:7-125):
// per-image cam_from_world rotations -> the unknown cameras' cam_from_rig rotations and the frames' rig_from_world
// rotations.  Flat arrays in sorted-id order; the rules are stated with b200sfm_rig_rotations_from_images
// (include/b200sfm.h).  Layout:
//   1. one stable radix sort of the keys frame(i) (unregistered images last) carrying the image index: the frame
//      segments, images in ascending index inside each
//   2. one thread per frame: the reference image (the first of its segment whose camera is the frame's reference camera)
//   3. one thread per image: its camera sample q_i conj(q_ref), keyed by camera (no sample: key K); one stable radix sort
//      gives the camera segments, samples in ascending image index inside each
//   4. one warp per camera segment, then one warp per frame segment: the 10 packed entries of sum q q^T accumulated
//      lane-strided and reduced by warp_sum (a fixed order: repeated calls are bit-identical, no floating-point atomics);
//      lane 0 takes the dominant eigenvector (quat_avg_eig, shared with ra_update_cams)
#pragma once
#include <cub/cub.cuh>

#include <vector>

#include "context.cuh"
#include "ra_kernels.cuh"      // quat_outer_acc, quat_avg_eig
#include "track_kernels.cuh"   // trk_iota

namespace b200 {

__device__ __forceinline__ void rig_qnorm(const double* __restrict__ q, double o[4]) {
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  o[0] = q[0] / n; o[1] = q[1] / n; o[2] = q[2] / n; o[3] = q[3] / n;
}
// o = a (x) b, xyzw (Eigen's quaternion product)
__device__ __forceinline__ void rig_qmul(const double a[4], const double b[4], double o[4]) {
  o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  o[1] = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
  o[2] = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
  o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}

__global__ void rig_frame_keys(int I, int F, const int* __restrict__ img_frame, int* __restrict__ key) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < I) key[i] = img_frame[i] >= 0 ? img_frame[i] : F;
}
// with the keys sorted: the segment [lo, hi) of every key below nkey (lo = hi = 0 beforehand: empty)
__global__ void rig_segments(int n, int nkey, const int* __restrict__ skey, int* __restrict__ lo, int* __restrict__ hi) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int v = skey[p];
  if (v >= nkey) return;
  if (p == 0 || skey[p - 1] != v) lo[v] = p;
  if (p == n - 1 || skey[p + 1] != v) hi[v] = p + 1;
}
// rule 1: the registered image of smallest index whose camera is the frame's reference camera, or -1
__global__ void rig_ref_images(int F, const int* __restrict__ lo, const int* __restrict__ hi, const int* __restrict__ simg,
                               const int* __restrict__ img_cam, const int* __restrict__ ref_cam, int* __restrict__ ref) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int r = -1;
  for (int p = lo[f]; p < hi[f]; ++p)
    if (img_cam[simg[p]] == ref_cam[f]) { r = simg[p]; break; }
  ref[f] = r;
}
// rule 2: the camera sample of image i, q_i conj(q_r), keyed by camera; key K when i gives none
__global__ void rig_cam_samples(int I, int K, const int* __restrict__ img_frame, const int* __restrict__ img_cam,
                                const unsigned char* __restrict__ est, const double* __restrict__ q_img,
                                const int* __restrict__ ref, const int* __restrict__ ref_cam,
                                const unsigned char* __restrict__ known, int* __restrict__ key, double* __restrict__ sq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= I) return;
  const int f = img_frame[i], c = img_cam[i];
  int k = K;
  if (f >= 0) {
    const int r = ref[f];
    if (r >= 0 && c != ref_cam[f] && !known[c] && est[i] && est[r]) {
      double qi[4], qr[4], s[4];
      rig_qnorm(q_img + 4 * (size_t)i, qi);
      rig_qnorm(q_img + 4 * (size_t)r, qr);
      qr[0] = -qr[0]; qr[1] = -qr[1]; qr[2] = -qr[2];
      rig_qmul(qi, qr, s);
      rig_qnorm(s, sq + 4 * (size_t)i);
      k = c;
    }
  }
  key[i] = k;
}
// the average of the samples handed out by `sample`, visited in segment order [lo, hi): q0 is the first one
template <class Sample>
__device__ __forceinline__ int rig_warp_average(int lo, int hi, int lane, Sample&& sample, double out[4]) {
  double M[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  double q0[4] = {0, 0, 0, 1};
  bool have0 = false;
  int n = 0;
  for (int base = lo; base < hi; base += 32) {
    double q[4] = {0, 0, 0, 1};
    const bool ok = base + lane < hi && sample(base + lane, q);
    const unsigned ball = __ballot_sync(0xffffffffu, ok);
    if (ok) quat_outer_acc(M, q);
    if (!have0 && ball) {   // the first sample in segment order
      const int src = __ffs(ball) - 1;
#pragma unroll
      for (int a = 0; a < 4; ++a) q0[a] = __shfl_sync(0xffffffffu, q[a], src);
      have0 = true;
    }
    n += __popc(ball);
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) M[k] = warp_sum(M[k]);
  if (n == 1) {   // a single sample is returned as it is
#pragma unroll
    for (int a = 0; a < 4; ++a) out[a] = q0[a];
  } else if (n > 1) {
    quat_avg_eig(M, q0, out);
  }
  if (n > 0 && out[3] < 0.0)   // canonical sign
#pragma unroll
    for (int a = 0; a < 4; ++a) out[a] = -out[a];
  return n;
}
// rule 3: one warp per camera; an unknown camera with samples gets their average and becomes usable (avail)
__global__ void __launch_bounds__(128) rig_cam_average(int K, const int* __restrict__ lo, const int* __restrict__ hi,
                                                       const int* __restrict__ simg, const double* __restrict__ sq,
                                                       const unsigned char* __restrict__ known, double* __restrict__ cam_q,
                                                       int* __restrict__ cam_n, unsigned char* __restrict__ avail) {
  const int c = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (c >= K) return;
  double avg[4];
  const int n = rig_warp_average(lo[c], hi[c], lane, [&](int p, double q[4]) {
    const double* s = sq + 4 * (size_t)simg[p];
    q[0] = s[0]; q[1] = s[1]; q[2] = s[2]; q[3] = s[3];
    return true;
  }, avg);
  if (lane != 0) return;
  cam_n[c] = n;
  if (n > 0)
    for (int a = 0; a < 4; ++a) cam_q[4 * (size_t)c + a] = avg[a];
  avail[c] = known[c] || n > 0;
}
// rule 4: one warp per frame over its registered, estimated images
__global__ void __launch_bounds__(128) rig_frame_average(int F, const int* __restrict__ lo, const int* __restrict__ hi,
                                                         const int* __restrict__ simg, const int* __restrict__ img_cam,
                                                         const unsigned char* __restrict__ est,
                                                         const double* __restrict__ q_img, const int* __restrict__ ref,
                                                         const unsigned char* __restrict__ avail,
                                                         const double* __restrict__ cam_q, double* __restrict__ frame_q,
                                                         int* __restrict__ frame_n) {
  const int f = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (f >= F) return;
  const int r = ref[f];
  double avg[4];
  const int n = rig_warp_average(lo[f], hi[f], lane, [&](int p, double q[4]) {
    const int i = simg[p];
    if (!est[i]) return false;
    double qi[4];
    rig_qnorm(q_img + 4 * (size_t)i, qi);
    if (i == r) {
      q[0] = qi[0]; q[1] = qi[1]; q[2] = qi[2]; q[3] = qi[3];
      return true;
    }
    const int c = img_cam[i];
    if (!avail[c]) return false;
    double qc[4], s[4];
    rig_qnorm(cam_q + 4 * (size_t)c, qc);
    qc[0] = -qc[0]; qc[1] = -qc[1]; qc[2] = -qc[2];
    rig_qmul(qc, qi, s);
    rig_qnorm(s, q);
    return true;
  }, avg);
  if (lane != 0) return;
  frame_n[f] = n;
  if (n > 0)
    for (int a = 0; a < 4; ++a) frame_q[4 * (size_t)f + a] = avg[a];
}

struct RigInitStats {
  int num_ref_frames = 0, num_cam_samples = 0, num_cams_averaged = 0, num_frame_samples = 0, num_frames_averaged = 0;
};

struct RigInitRunner {
  b200sfm_ctx* ctx;
  DevBuf<unsigned char> tmp;
  explicit RigInitRunner(b200sfm_ctx* c) : ctx(c) {}

  template <class F>
  void cub_call(F&& f) {   // size query, grow the scratch, run
    size_t need = 0;
    B200_CUDA_OK(f((void*)nullptr, need));
    if (need > tmp.n) tmp.alloc(need);
    size_t nb = tmp.n;
    B200_CUDA_OK(f((void*)tmp.p, nb));
  }
  static int key_bits(int v) { return std::max(1, 32 - __builtin_clz((unsigned)v)); }

  // Arguments validated by the caller: I, F, K >= 1, indices in range.  est may be null (every image estimated).
  void run(int I, int F, int K, const int* h_frame, const int* h_cam, const unsigned char* h_est, const double* h_q,
           const int* h_ref_cam, const unsigned char* h_known, double* h_cam_q, int* h_cam_n, double* h_frame_q,
           int* h_frame_n, RigInitStats& st) {
    cudaStream_t s = ctx->stream;
    DevBuf<int> frame, cam, ref_cam, key, iota, skey, simg, lo, hi, ref, cam_n, frame_n;
    DevBuf<unsigned char> est, known, avail;
    DevBuf<double> q, sq, cam_q, frame_q;
    frame.alloc(I); cam.alloc(I); key.alloc(I); iota.alloc(I); skey.alloc(I); simg.alloc(I); est.alloc(I);
    q.alloc(4 * (size_t)I); sq.alloc(4 * (size_t)I);
    ref_cam.alloc(F); lo.alloc(std::max(F, K)); hi.alloc(std::max(F, K)); ref.alloc(F); frame_n.alloc(F); frame_q.alloc(4 * (size_t)F);
    known.alloc(K); avail.alloc(K); cam_n.alloc(K); cam_q.alloc(4 * (size_t)K);
    frame.upload(h_frame, I, s); cam.upload(h_cam, I, s); q.upload(h_q, 4 * (size_t)I, s);
    if (h_est) {
      est.upload(h_est, I, s);
    } else {
      B200_CUDA_OK(cudaMemsetAsync(est.p, 1, I, s));
    }
    ref_cam.upload(h_ref_cam, F, s); frame_q.upload(h_frame_q, 4 * (size_t)F, s);
    known.upload(h_known, K, s); cam_q.upload(h_cam_q, 4 * (size_t)K, s);
    // 1. frame segments
    B200_LAUNCH(ctx, rig_frame_keys, cdiv(I, 256), 256, 0, I, F, frame.p, key.p);
    B200_LAUNCH(ctx, trk_iota, cdiv(I, 256), 256, 0, (long long)I, iota.p);
    cub_call([&](void* p, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(p, nb, key.p, skey.p, iota.p, simg.p, I, 0, key_bits(F), s);
    });
    lo.zero(s); hi.zero(s);
    B200_LAUNCH(ctx, rig_segments, cdiv(I, 256), 256, 0, I, F, skey.p, lo.p, hi.p);
    // 2. reference images
    B200_LAUNCH(ctx, rig_ref_images, cdiv(F, 256), 256, 0, F, lo.p, hi.p, simg.p, cam.p, ref_cam.p, ref.p);
    // 3. camera samples and their segments (the frame segments stay in skey / simg; the camera ones reuse key / iota)
    B200_LAUNCH(ctx, rig_cam_samples, cdiv(I, 256), 256, 0, I, K, frame.p, cam.p, est.p, q.p, ref.p, ref_cam.p, known.p,
                key.p, sq.p);
    DevBuf<int> ckey, cimg, clo, chi;
    ckey.alloc(I); cimg.alloc(I); clo.alloc(K); chi.alloc(K);
    B200_LAUNCH(ctx, trk_iota, cdiv(I, 256), 256, 0, (long long)I, iota.p);
    cub_call([&](void* p, size_t& nb) {
      return cub::DeviceRadixSort::SortPairs(p, nb, key.p, ckey.p, iota.p, cimg.p, I, 0, key_bits(K), s);
    });
    clo.zero(s); chi.zero(s);
    B200_LAUNCH(ctx, rig_segments, cdiv(I, 256), 256, 0, I, K, ckey.p, clo.p, chi.p);
    // 4. averages
    B200_LAUNCH(ctx, rig_cam_average, cdiv(32LL * K, 128), 128, 0, K, clo.p, chi.p, cimg.p, sq.p, known.p, cam_q.p, cam_n.p, avail.p);
    B200_LAUNCH(ctx, rig_frame_average, cdiv(32LL * F, 128), 128, 0, F, lo.p, hi.p, simg.p, cam.p, est.p, q.p, ref.p, avail.p,
                cam_q.p, frame_q.p, frame_n.p);
    std::vector<int> h_ref(F), cn(K), fn(F);
    ref.download(h_ref.data(), F, s);
    cam_n.download(cn.data(), K, s);
    frame_n.download(fn.data(), F, s);
    cam_q.download(h_cam_q, 4 * (size_t)K, s);
    frame_q.download(h_frame_q, 4 * (size_t)F, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    for (int f = 0; f < F; ++f) {
      st.num_ref_frames += h_ref[f] >= 0;
      st.num_frame_samples += fn[f];
      st.num_frames_averaged += fn[f] > 0;
    }
    for (int c = 0; c < K; ++c) {
      st.num_cam_samples += cn[c];
      st.num_cams_averaged += cn[c] > 0;
    }
    if (h_cam_n) std::copy(cn.begin(), cn.end(), h_cam_n);
    if (h_frame_n) std::copy(fn.begin(), fn.end(), h_frame_n);
  }
};

}  // namespace b200
