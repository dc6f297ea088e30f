// view_graph_kernels.cuh -- device side of the two view-graph passes GlobalMapper::Solve runs after each rotation
// averaging (controllers/global_mapper.cc:91-115):
//   RelPoseFilter::FilterRotations (processors/relpose_filter.cc:7-33): one thread per pair.  A valid pair whose two images
//     are registered gets q_calc = q2 * conj(q1) from the images' cam_from_world rotations and the angle of Eigen's
//     angularDistance against its cam2_from_cam1 rotation, d = q_calc * conj(q_rel), 2 atan2(|d.vec|, |d.w|), in degrees
//     (math/rigid3d.cc:7-9, the Rigid3d overload of CalcAngle).  angle > max_angle invalidates the pair; a NaN angle does
//     not.  Eigen's inverse() and Rigid3d's normalisation of the product scale a quaternion by a positive factor, which
//     the angle does not depend on, so the conjugate stands for the inverse and the product is not normalised.  The
//     products use explicitly rounded FP64 operations (no FMA contraction), in Eigen's quat_product term order.
//   ViewGraph::KeepLargestConnectedComponents (scene/view_graph.cc:56-97) in frame space: the nodes are the frames of the
//     valid pairs (CreateFrameAdjacencyList, :140-150; a pair inside one frame makes that frame a node of its own).
//     Components by hook-and-compress: rounds of atomicMin hooking over the valid pairs' frame labels, each followed by a
//     full compression (every label walks to its root), until a hooking pass changes nothing.  A label only ever moves to
//     a smaller frame of the same component, so at the end every frame's label is the smallest frame of its component.
//     The largest component is the one maximal in (size << 32 | ~smallest frame): ties go to the component holding the
//     smallest frame index (the reference's choice depends on hash-map order; rotation_averager.largest_component and
//     prune_kernels.cuh use the same rule).  Then every frame is deregistered except those of that component, every pair
//     with an image outside it invalidated, and the number of registered images returned (:75-96).  Without a valid pair
//     nothing changes and 0 is returned (:71).
// Integer work only in the component pass and no floating-point atomics anywhere: results are exact and reproducible.
// Every index is range-checked on the device before it is dereferenced; a bad one sets a flag and the call reports it.
#pragma once
#include <vector>

#include "context.cuh"

namespace b200 {

// Eigen's quat_product (Geometry/Quaternion.h), xyzw storage, every product and sum rounded on its own
__device__ __forceinline__ void vg_qmul(const double a[4], const double b[4], double c[4]) {
  const double ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
  c[3] = __dsub_rn(__dsub_rn(__dsub_rn(__dmul_rn(aw, bw), __dmul_rn(ax, bx)), __dmul_rn(ay, by)), __dmul_rn(az, bz));
  c[0] = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(aw, bx), __dmul_rn(ax, bw)), __dmul_rn(ay, bz)), __dmul_rn(az, by));
  c[1] = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(aw, by), __dmul_rn(ay, bw)), __dmul_rn(az, bx)), __dmul_rn(ax, bz));
  c[2] = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(aw, bz), __dmul_rn(az, bw)), __dmul_rn(ax, by)), __dmul_rn(ay, bx));
}

// flags[0]: an index out of range; flags[1]: invalidated pairs / hooking changed something; flags[2]: registered images
__global__ void vg_filter_rotations(long long E, int I, const double* __restrict__ q_img, const unsigned char* __restrict__ img_reg,
                                    const int* __restrict__ img1, const int* __restrict__ img2, const double* __restrict__ q_rel,
                                    double max_angle_deg, unsigned char* __restrict__ valid, int* __restrict__ flags) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool cut = false;
  if (e < E) {
    const int a = img1[e], b = img2[e];
    if (a < 0 || a >= I || b < 0 || b >= I) {
      flags[0] = 1;
    } else if (valid[e] && (!img_reg || (img_reg[a] && img_reg[b]))) {
      const double q1i[4] = {-q_img[4 * (size_t)a], -q_img[4 * (size_t)a + 1], -q_img[4 * (size_t)a + 2], q_img[4 * (size_t)a + 3]};
      const double q2[4] = {q_img[4 * (size_t)b], q_img[4 * (size_t)b + 1], q_img[4 * (size_t)b + 2], q_img[4 * (size_t)b + 3]};
      const double* r = q_rel + 4 * (size_t)e;
      const double rc[4] = {-r[0], -r[1], -r[2], r[3]};
      double qc[4], d[4];
      vg_qmul(q2, q1i, qc);
      vg_qmul(qc, rc, d);
      const double vn = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
      const double angle = __ddiv_rn(__dmul_rn(__dmul_rn(2.0, atan2(vn, fabs(d[3]))), 180.0), 3.14159265358979323846);
      if (angle > max_angle_deg) {   // false for NaN
        valid[e] = 0;
        cut = true;
      }
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, cut);   // one atomic per warp with a cut pair
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&flags[1], __popc(m));
}

// image -> frame range check
__global__ void vg_check_frames(int I, const int* __restrict__ image_frame, int F, int* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < I && (image_frame[i] < 0 || image_frame[i] >= F)) flags[0] = 1;
}
// frames of every pair ((-1, -1) when an index is bad); the frames of the valid pairs are the nodes
__global__ void vg_pair_frames(long long E, int I, int F, const int* __restrict__ img1, const int* __restrict__ img2,
                               const int* __restrict__ image_frame, const unsigned char* __restrict__ valid, int2* __restrict__ ends,
                               unsigned char* __restrict__ node, int* __restrict__ flags) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int a = img1[e], b = img2[e];
  int fa = -1, fb = -1;
  if (a < 0 || a >= I || b < 0 || b >= I) {
    flags[0] = 1;
  } else {
    fa = image_frame[a];
    fb = image_frame[b];
    if (fa < 0 || fa >= F || fb < 0 || fb >= F) fa = fb = -1;   // flagged by vg_check_frames
  }
  ends[e] = make_int2(fa, fb);
  if (fa >= 0 && valid[e]) {
    node[fa] = 1;
    node[fb] = 1;
  }
}
__global__ void vg_iota(int n, int* __restrict__ a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = i;
}
// hooking: the larger of the two labels of a valid pair takes the smaller one
__global__ void vg_hook(long long E, const int2* __restrict__ ends, const unsigned char* __restrict__ valid, int* __restrict__ label,
                        int* __restrict__ flags) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E || !valid[e]) return;
  const int2 f = ends[e];
  if (f.x < 0) return;
  const int la = label[f.x], lb = label[f.y];
  if (la == lb) return;
  atomicMin(&label[max(la, lb)], min(la, lb));
  flags[1] = 1;
}
// compression: every label walks to its root (labels point to smaller frames, so the walk ends; a concurrent write only
// replaces a label by one of its ancestors)
__global__ void vg_compress(int F, int* __restrict__ label) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int r = label[f];
  while (true) {
    const int p = label[r];
    if (p == r) break;
    r = p;
  }
  label[f] = r;
}
// component sizes by root (the smallest frame of the component), node frames only
__global__ void vg_comp_size(int F, const int* __restrict__ label, const unsigned char* __restrict__ node, int* __restrict__ size) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F && node[f]) atomicAdd(&size[label[f]], 1);
}
// the largest component, ties to the smallest root: max of (size << 32 | ~root); 0 when there is no node
__global__ void vg_largest(int F, const int* __restrict__ size, unsigned long long* __restrict__ best) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F && size[f] > 0) atomicMax(best, ((unsigned long long)size[f] << 32) | (0xffffffffu - (unsigned)f));
}
__global__ void vg_register(int F, const int* __restrict__ label, const unsigned char* __restrict__ node,
                            const unsigned long long* __restrict__ best, unsigned char* __restrict__ reg) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int r = (int)(0xffffffffu - (unsigned)(*best & 0xffffffffull));
  reg[f] = node[f] && label[f] == r;
}
// every pair with an image outside the registered frames becomes invalid (:85-90)
__global__ void vg_invalidate(long long E, const int2* __restrict__ ends, const unsigned char* __restrict__ reg,
                              unsigned char* __restrict__ valid) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int2 f = ends[e];
  if (f.x < 0) return;
  if (!reg[f.x] || !reg[f.y]) valid[e] = 0;
}
// registered images (:92-95): one atomic per warp
__global__ void vg_count_images(int I, const int* __restrict__ image_frame, int F, const unsigned char* __restrict__ reg,
                                int* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool r = false;
  if (i < I) {
    const int f = image_frame[i];
    r = f >= 0 && f < F && reg[f];
  }
  const unsigned m = __ballot_sync(0xffffffffu, r);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&flags[2], __popc(m));
}

struct ViewGraphRunner {
  b200sfm_ctx* ctx;
  cudaStream_t s;
  explicit ViewGraphRunner(b200sfm_ctx* c) : ctx(c), s(c->stream) {}

  void read_flags(const int* d, int* h, int n) {
    B200_CUDA_OK(cudaMemcpyAsync(h, d, n * sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }

  // Returns false when an index is out of range (the host buffers are then untouched).  Arguments validated by the
  // caller: E >= 1, null pointers, sizes.
  bool filter_rotations(int I, const double* h_q_img, const unsigned char* h_reg, long long E, const int* h_img1, const int* h_img2,
                        const double* h_q_rel, double max_angle_deg, unsigned char* h_valid, long long* num_invalidated) {
    DevBuf<double> q_img, q_rel;
    DevBuf<unsigned char> reg, valid;
    DevBuf<int> img1, img2, flags;
    q_img.alloc(4 * (size_t)I); q_rel.alloc(4 * (size_t)E); img1.alloc(E); img2.alloc(E); valid.alloc(E); flags.alloc(4);
    q_img.upload(h_q_img, 4 * (size_t)I, s);
    if (h_reg) { reg.alloc(I); reg.upload(h_reg, I, s); }
    img1.upload(h_img1, E, s); img2.upload(h_img2, E, s); q_rel.upload(h_q_rel, 4 * (size_t)E, s); valid.upload(h_valid, E, s);
    flags.zero(s);
    B200_LAUNCH(ctx, vg_filter_rotations, cdiv(E, 256), 256, 0, E, I, q_img.p, reg.p, img1.p, img2.p, q_rel.p, max_angle_deg, valid.p,
                flags.p);
    int h[4];
    read_flags(flags.p, h, 4);
    if (h[0]) return false;
    valid.download(h_valid, E, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    *num_invalidated = h[1];
    return true;
  }

  // Same contract.  frame_reg [F] and valid [E] are only written when there is a valid pair.
  bool keep_largest_component(int F, int I, const int* h_image_frame, long long E, const int* h_img1, const int* h_img2,
                              unsigned char* h_valid, unsigned char* h_frame_reg, int* num_registered_images) {
    DevBuf<int> image_frame, img1, img2, label, size, flags;
    DevBuf<int2> ends;
    DevBuf<unsigned char> valid, node, reg;
    DevBuf<unsigned long long> best;
    image_frame.alloc(std::max(I, 1)); img1.alloc(E); img2.alloc(E); valid.alloc(E); ends.alloc(E); flags.alloc(4);
    node.alloc(std::max(F, 1)); label.alloc(std::max(F, 1)); size.alloc(std::max(F, 1)); reg.alloc(std::max(F, 1)); best.alloc(1);
    image_frame.upload(h_image_frame, I, s);
    img1.upload(h_img1, E, s); img2.upload(h_img2, E, s); valid.upload(h_valid, E, s);
    flags.zero(s); node.zero(s); size.zero(s); best.zero(s);
    if (I > 0) B200_LAUNCH(ctx, vg_check_frames, cdiv(I, 256), 256, 0, I, image_frame.p, F, flags.p);
    B200_LAUNCH(ctx, vg_pair_frames, cdiv(E, 256), 256, 0, E, I, F, img1.p, img2.p, image_frame.p, valid.p, ends.p, node.p, flags.p);
    img1.release(); img2.release();
    int h[4];
    read_flags(flags.p, h, 4);
    if (h[0]) return false;
    *num_registered_images = 0;
    if (F == 0) return true;
    B200_LAUNCH(ctx, vg_iota, cdiv(F, 256), 256, 0, F, label.p);
    do {
      B200_CUDA_OK(cudaMemsetAsync(flags.p + 1, 0, sizeof(int), s));
      B200_LAUNCH(ctx, vg_hook, cdiv(E, 256), 256, 0, E, ends.p, valid.p, label.p, flags.p);
      B200_LAUNCH(ctx, vg_compress, cdiv(F, 256), 256, 0, F, label.p);
      read_flags(flags.p, h, 4);
    } while (h[1]);
    B200_LAUNCH(ctx, vg_comp_size, cdiv(F, 256), 256, 0, F, label.p, node.p, size.p);
    B200_LAUNCH(ctx, vg_largest, cdiv(F, 256), 256, 0, F, size.p, best.p);
    unsigned long long h_best = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&h_best, best.p, sizeof(h_best), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    if (h_best == 0) return true;                      // no valid pair: nothing changes (:71)
    B200_LAUNCH(ctx, vg_register, cdiv(F, 256), 256, 0, F, label.p, node.p, best.p, reg.p);
    B200_LAUNCH(ctx, vg_invalidate, cdiv(E, 256), 256, 0, E, ends.p, reg.p, valid.p);
    if (I > 0) B200_LAUNCH(ctx, vg_count_images, cdiv(I, 256), 256, 0, I, image_frame.p, F, reg.p, flags.p);
    read_flags(flags.p, h, 4);
    reg.download(h_frame_reg, F, s);
    valid.download(h_valid, E, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    *num_registered_images = h[2];
    return true;
  }
};

}  // namespace b200
