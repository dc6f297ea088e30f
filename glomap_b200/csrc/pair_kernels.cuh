// pair_kernels.cuh -- device side of ImagePairsInlierCount (glomap/processors/image_pair_inliers.cc:200-213; the scorers
// ScoreErrorEssential / Fundamental / Homography :20-198 and the two-view arithmetic of math/two_view_geometry.cc):
//   1. pair_bearings  -- unit bearing of every feature of the images that appear in a CALIBRATED pair, once per feature
//                        (UndistortImages, the same arithmetic as proc_undistort through bearing_from_pixel)
//   2. pair_setup     -- one 256-B record per pair: E = [t]x R, epipoles, F epipole, squared threshold
//   3. pair_score     -- one warp per pair, 32 matches per step: gather, r2 and the decision flags, per-lane sums, then
//                        a fixed-order shuffle reduction (no atomics: the outputs are reproducible bit for bit).  F pairs
//                        take a second loop over their mask once the signum majority is known.
// Match indices are checked against the feature counts of their images; an index out of range sets *err and is never
// dereferenced.
#pragma once
#include <cmath>

#include "context.cuh"
#include "processor_kernels.cuh"

namespace b200 {

constexpr double kTwoViewEps = 1e-12;   // glomap EPS (types.h:14)

struct alignas(16) PairRec {
  double M[9];              // E (CALIBRATED), F (UNCALIBRATED) or H (PLANAR / PANORAMIC / PLANAR_OR_PANORAMIC), row-major
  double R[9];              // cam2_from_cam1 rotation (E)
  double t[3];              // cam2_from_cam1 translation (E)
  double e12[3], e21[3];    // E: epipoles, z made non-negative (image_pair_inliers.cc:26-31)
  double ep[3];             // F: epipole used by GetOrientationSignum (:99-110)
  double thr2;              // squared threshold of the pair's model
  int kind;                 // 0: no inliers, 1: E, 2: F, 3: H
  int pad;
};
static_assert(sizeof(PairRec) == 256, "one pair record is 256 B");

__global__ void pair_bearings(int I, const long long* __restrict__ feature_begin, const unsigned char* __restrict__ need,
                              const int* __restrict__ image_intr, const int* __restrict__ intr_model,
                              const double* __restrict__ intr /*[K][12]*/, const double2* __restrict__ xy,
                              double* __restrict__ bear /*[nf][3]*/) {
  const int img = blockIdx.x;
  if (img >= I || !need[img]) return;
  const int blk = image_intr[img];
  const int m = intr_model[blk];
  const double* p = intr + (size_t)blk * 12;
  for (long long f = feature_begin[img] + threadIdx.x; f < feature_begin[img + 1]; f += blockDim.x)
    bearing_from_pixel(m, p, xy[f], bear + 3 * f);
}

// config values: colmap::TwoViewGeometry::ConfigurationType (include/b200sfm.h, B200SFM_TWO_VIEW_*)
__global__ void pair_setup(long long E, const int* __restrict__ config, const double* __restrict__ quat,
                           const double* __restrict__ trans, const double* __restrict__ Fm, const double* __restrict__ Hm,
                           const int* __restrict__ img1, const int* __restrict__ img2, const int* __restrict__ image_intr,
                           const int* __restrict__ intr_model, const double* __restrict__ intr, double err_E, double err_F,
                           double err_H, PairRec* __restrict__ rec) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  PairRec r{};
  const int c = config[e];
  if (c == 2) {   // CALIBRATED: EssentialFromMotion (two_view_geometry.cc:41-45)
    const double q[4] = {quat[4 * e], quat[4 * e + 1], quat[4 * e + 2], quat[4 * e + 3]};
    quat_to_R(q, r.R);
    const double t0 = trans[3 * e], t1 = trans[3 * e + 1], t2 = trans[3 * e + 2];
    r.t[0] = t0; r.t[1] = t1; r.t[2] = t2;
    const double tx[9] = {0.0, -t2, t1, t2, 0.0, -t0, -t1, t0, 0.0};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) r.M[3 * i + j] = tx[3 * i] * r.R[j] + tx[3 * i + 1] * r.R[3 + j] + tx[3 * i + 2] * r.R[6 + j];
    const double s12 = t2 < 0 ? -1.0 : 1.0;
    r.e12[0] = s12 * t0; r.e12[1] = s12 * t1; r.e12[2] = s12 * t2;
    double e21[3];   // Inverse(cam2_from_cam1).translation = -R^T t
#pragma unroll
    for (int i = 0; i < 3; ++i) e21[i] = -(r.R[i] * t0 + r.R[3 + i] * t1 + r.R[6 + i] * t2);
    const double s21 = e21[2] < 0 ? -1.0 : 1.0;
    r.e21[0] = s21 * e21[0]; r.e21[1] = s21 * e21[1]; r.e21[2] = s21 * e21[2];
    // Camera::Focal() = (fx + fy) / 2 (scene/camera.h:28); fx = fy = params[0] except for PINHOLE
    double foc[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int blk = image_intr[k == 0 ? img1[e] : img2[e]];
      const double* p = intr + (size_t)blk * 12;
      foc[k] = intr_model[blk] == 1 ? (p[0] + p[1]) / 2.0 : (p[0] + p[0]) / 2.0;
    }
    const double thr = err_E * 0.5 * (1. / foc[0] + 1. / foc[1]);
    r.thr2 = thr * thr;
    r.kind = 1;
  } else if (c == 3) {   // UNCALIBRATED
#pragma unroll
    for (int k = 0; k < 9; ++k) r.M[k] = Fm[9 * e + k];
    const double* F = r.M;
    double ep[3] = {F[1] * F[8] - F[2] * F[7], F[2] * F[6] - F[0] * F[8], F[0] * F[7] - F[1] * F[6]};   // row 0 x row 2
    if (!(ep[0] > kTwoViewEps || ep[0] < -kTwoViewEps || ep[1] > kTwoViewEps || ep[1] < -kTwoViewEps || ep[2] > kTwoViewEps ||
          ep[2] < -kTwoViewEps)) {   // row 1 x row 2
      ep[0] = F[4] * F[8] - F[5] * F[7]; ep[1] = F[5] * F[6] - F[3] * F[8]; ep[2] = F[3] * F[7] - F[4] * F[6];
    }
    r.ep[0] = ep[0]; r.ep[1] = ep[1]; r.ep[2] = ep[2];
    r.thr2 = err_F * err_F;
    r.kind = 2;
  } else if (c == 4 || c == 5 || c == 6) {   // PLANAR, PANORAMIC, PLANAR_OR_PANORAMIC
#pragma unroll
    for (int k = 0; k < 9; ++k) r.M[k] = Hm[9 * e + k];
    r.thr2 = err_H * err_H;
    r.kind = 3;
  }
  rec[e] = r;
}

__device__ __forceinline__ int warp_isum(int v) { return (int)__reduce_add_sync(0xffffffffu, (unsigned)v); }

// One warp per pair.  mask[k]: 1 = inlier.  F pairs first store 1 / 2 (pre-inlier with non-positive / positive signum)
// and rewrite the mask in a second loop over the same k of the same lane.
__global__ void __launch_bounds__(128) pair_score(long long E, const PairRec* __restrict__ rec, const int* __restrict__ img1,
                                                  const int* __restrict__ img2, const long long* __restrict__ feature_begin,
                                                  const long long* __restrict__ match_begin, const int2* __restrict__ matches,
                                                  const double* __restrict__ bear, const double2* __restrict__ xy,
                                                  double cos_epipole_thr, unsigned char* __restrict__ mask,
                                                  int* __restrict__ num_inliers, double* __restrict__ score, int* __restrict__ err) {
  const long long e = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= E) return;
  const int kind = rec[e].kind;
  const double thr2 = rec[e].thr2;
  const long long k0 = match_begin[e], k1 = match_begin[e + 1];
  const long long fb1 = feature_begin[img1[e]], fb2 = feature_begin[img2[e]];
  const long long n1 = feature_begin[img1[e] + 1] - fb1, n2 = feature_begin[img2[e] + 1] - fb2;
  double M[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) M[i] = rec[e].M[i];
  int cnt = 0, npos = 0, nneg = 0, bad = 0;
  double s = 0.0, s_pos = 0.0, s_neg = 0.0;   // F: s = thresholds of the non-pre-inliers, s_pos / s_neg = r2 of the pre-inliers
  for (long long k = k0 + lane; k < k1; k += 32) {
    const int2 m = matches[k];
    if (m.x < 0 || m.x >= n1 || m.y < 0 || m.y >= n2) {
      bad = 1;
      mask[k] = 0;
      continue;
    }
    unsigned char out = 0;
    if (kind == 1) {   // ScoreErrorEssential (image_pair_inliers.cc:20-92) on features_undist
      const double* b1 = bear + 3 * (fb1 + m.x);
      const double* b2 = bear + 3 * (fb2 + m.y);
      const double x1[3] = {b1[0], b1[1], b1[2]}, x2[3] = {b2[0], b2[1], b2[2]};
      // SampsonError, 3-vector form (two_view_geometry.cc:71-83)
      const double d1 = kTwoViewEps + x1[2], d2 = kTwoViewEps + x2[2];
      double Ex1[3], Etx2[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        Ex1[i] = (M[3 * i] * x1[0] + M[3 * i + 1] * x1[1] + M[3 * i + 2] * x1[2]) / d1;
        Etx2[i] = (M[i] * x2[0] + M[3 + i] * x2[1] + M[6 + i] * x2[2]) / d2;
      }
      const double C = Ex1[0] * x2[0] + Ex1[1] * x2[1] + Ex1[2] * x2[2];
      const double r2 = C * C / ((Ex1[0] * Ex1[0] + Ex1[1] * Ex1[1]) + (Etx2[0] * Etx2[0] + Etx2[1] * Etx2[1]));
      bool inl = false;
      if (r2 < thr2) {
        const PairRec& p = rec[e];
        // CheckCheirality(pose, x1, x2, 1e-2, 100) (two_view_geometry.cc:5-29)
        double Rx1[3], Rtx2[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          Rx1[i] = p.R[3 * i] * x1[0] + p.R[3 * i + 1] * x1[1] + p.R[3 * i + 2] * x1[2];
          Rtx2[i] = p.R[i] * x2[0] + p.R[3 + i] * x2[1] + p.R[6 + i] * x2[2];
        }
        const double a = -(Rx1[0] * x2[0] + Rx1[1] * x2[1] + Rx1[2] * x2[2]);
        const double b1v = -(Rx1[0] * p.t[0] + Rx1[1] * p.t[1] + Rx1[2] * p.t[2]);
        const double b2v = x2[0] * p.t[0] + x2[1] * p.t[1] + x2[2] * p.t[2];
        const double l1 = b1v - a * b2v, l2 = -a * b1v + b2v;
        const double min_d = 1e-2 * (1 - a * a), max_d = 100. * (1 - a * a);
        const bool cheir = l1 > min_d && l2 > min_d && l1 < max_d && l2 < max_d;
        const double diff_angle = x1[0] * Rtx2[0] + x1[1] * Rtx2[1] + x1[2] * Rtx2[2];
        const double dep1 = x1[0] * p.e21[0] + x1[1] * p.e21[1] + x1[2] * p.e21[2];
        const double dep2 = x2[0] * p.e12[0] + x2[1] * p.e12[1] + x2[2] * p.e12[2];
        inl = cheir && diff_angle < 1.0 + 1e-6 && dep1 < cos_epipole_thr && dep2 < cos_epipole_thr;
      }
      out = inl;
      s += inl ? r2 : thr2;
      cnt += inl;
    } else if (kind == 2) {   // ScoreErrorFundamental (:94-164), first loop
      const double2 x1 = xy[fb1 + m.x], x2 = xy[fb2 + m.y];
      double Fx1[3], Ftx2[3];   // SampsonError, 2-vector form (two_view_geometry.cc:57-69)
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        Fx1[i] = M[3 * i] * x1.x + M[3 * i + 1] * x1.y + M[3 * i + 2];
        Ftx2[i] = M[i] * x2.x + M[3 + i] * x2.y + M[6 + i];
      }
      const double C = Fx1[0] * x2.x + Fx1[1] * x2.y + Fx1[2];
      const double r2 = C * C / ((Fx1[0] * Fx1[0] + Fx1[1] * Fx1[1]) + (Ftx2[0] * Ftx2[0] + Ftx2[1] * Ftx2[1]));
      if (r2 < thr2) {   // GetOrientationSignum (two_view_geometry.cc:31-39)
        const PairRec& p = rec[e];
        const double sg = (M[0] * x2.x + M[3] * x2.y + M[6]) * (p.ep[1] - p.ep[2] * x1.y);
        if (sg > 0) { out = 2; ++npos; s_pos += r2; }
        else { out = 1; ++nneg; s_neg += r2; }
      } else {
        s += thr2;
      }
    } else if (kind == 3) {   // ScoreErrorHomography (:166-198), HomographyError (two_view_geometry.cc:85-93)
      const double2 x1 = xy[fb1 + m.x], x2 = xy[fb2 + m.y];
      const double h0 = M[0] * x1.x + M[1] * x1.y + M[2];
      const double h1 = M[3] * x1.x + M[4] * x1.y + M[5];
      const double h2 = M[6] * x1.x + M[7] * x1.y + M[8];
      const double dx = h0 / (kTwoViewEps + h2) - x2.x, dy = h1 / (kTwoViewEps + h2) - x2.y;
      const double r2 = dx * dx + dy * dy;
      const bool inl = r2 < thr2;
      out = inl;
      s += inl ? r2 : thr2;
      cnt += inl;
    }
    mask[k] = out;
  }
  bad = warp_isum(bad);
  if (bad && lane == 0) *err = 1;
  s = warp_sum(s);
  if (kind == 2) {
    npos = warp_isum(npos);
    nneg = warp_isum(nneg);
    s_pos = warp_sum(s_pos);
    s_neg = warp_sum(s_neg);
    const bool tie = npos == nneg;   // the pair cannot be oriented: no inliers, score 0 (:147-150)
    const unsigned char keep = npos > nneg ? 2 : 1;
    for (long long k = k0 + lane; k < k1; k += 32) mask[k] = !tie && mask[k] == keep;
    cnt = tie ? 0 : (npos > nneg ? npos : nneg);
    // rejected pre-inliers add the threshold (:154-162)
    s = tie ? 0.0 : s + (npos > nneg ? s_pos + (double)nneg * thr2 : s_neg + (double)npos * thr2);
  } else {
    cnt = warp_isum(cnt);
  }
  if (lane == 0) {
    num_inliers[e] = cnt;
    score[e] = s;
  }
}

// ImagePairsInlierCount on the device (b200sfm_image_pairs_inlier_count); arguments validated by the caller except the
// match indices, which are checked by pair_score.  Returns false when a match index is out of range.
inline bool image_pairs_inlier_count(b200sfm_ctx* ctx, int I, long long nf, const int64_t* h_feature_begin,
                                          const double* h_features, const int32_t* h_image_intr, int K,
                                          const int32_t* h_intr_model, const double* h_intr, long long E, const int32_t* h_img1,
                                          const int32_t* h_img2, const int32_t* h_config, const double* h_quat,
                                          const double* h_trans, const double* h_F, const double* h_H,
                                          const int64_t* h_match_begin, const int32_t* h_matches, double err_E, double err_F,
                                          double err_H, const unsigned char* h_need_bearings, uint8_t* h_mask,
                                          int32_t* h_num_inliers, double* h_score) {
  cudaStream_t s = ctx->stream;
  const long long M = h_match_begin[E];
  DevBuf<long long> feature_begin, match_begin;
  DevBuf<double2> xy;
  DevBuf<double> bear, intr, quat, trans, Fm, Hm, score;
  DevBuf<int> image_intr, intr_model, img1, img2, config, num_inliers, err;
  DevBuf<unsigned char> need, mask;
  DevBuf<int2> matches;
  DevBuf<PairRec> rec;
  feature_begin.alloc((size_t)I + 1); feature_begin.upload(reinterpret_cast<const long long*>(h_feature_begin), (size_t)I + 1, s);
  xy.alloc(std::max(nf, 1LL)); xy.upload(reinterpret_cast<const double2*>(h_features), nf, s);
  image_intr.alloc(std::max(I, 1)); image_intr.upload(h_image_intr, I, s);
  intr_model.alloc(std::max(K, 1)); intr_model.upload(h_intr_model, K, s);
  intr.alloc((size_t)std::max(K, 1) * 12); intr.upload(h_intr, (size_t)K * 12, s);
  img1.alloc(E); img1.upload(h_img1, E, s);
  img2.alloc(E); img2.upload(h_img2, E, s);
  config.alloc(E); config.upload(h_config, E, s);
  quat.alloc(4 * E); quat.upload(h_quat, 4 * E, s);
  trans.alloc(3 * E); trans.upload(h_trans, 3 * E, s);
  Fm.alloc(9 * E); Fm.upload(h_F, 9 * E, s);
  Hm.alloc(9 * E); Hm.upload(h_H, 9 * E, s);
  match_begin.alloc(E + 1); match_begin.upload(reinterpret_cast<const long long*>(h_match_begin), E + 1, s);
  matches.alloc(std::max(M, 1LL)); matches.upload(reinterpret_cast<const int2*>(h_matches), M, s);
  mask.alloc(std::max(M, 1LL));
  rec.alloc(E); num_inliers.alloc(E); score.alloc(E);
  err.alloc(1); err.zero(s);
  bool any_bearings = false;
  for (int i = 0; i < I && !any_bearings; ++i) any_bearings = h_need_bearings[i] != 0;
  if (any_bearings) {
    need.alloc(I); need.upload(h_need_bearings, I, s);
    bear.alloc((size_t)std::max(nf, 1LL) * 3);
    B200_LAUNCH(ctx, pair_bearings, I, 128, 0, I, feature_begin.p, need.p, image_intr.p, intr_model.p, intr.p, xy.p, bear.p);
  }
  B200_LAUNCH(ctx, pair_setup, cdiv(E, 128), 128, 0, E, config.p, quat.p, trans.p, Fm.p, Hm.p, img1.p, img2.p, image_intr.p, intr_model.p,
              intr.p, err_E, err_F, err_H, rec.p);
  // cos(DegToRad(3)) + 1e-6 (image_pair_inliers.cc:54-57; colmap::DegToRad multiplies by this constant)
  const double cos_epipole_thr = std::cos(3.0 * 0.0174532925199432954743716805978692718953) + 1e-6;
  B200_LAUNCH(ctx, pair_score, cdiv(E, 4), 128, 0, E, rec.p, img1.p, img2.p, feature_begin.p, match_begin.p, matches.p, bear.p, xy.p,
              cos_epipole_thr, mask.p, num_inliers.p, score.p, err.p);
  int h_err = 0;
  B200_CUDA_OK(cudaMemcpyAsync(&h_err, err.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  mask.download(h_mask, M, s);
  num_inliers.download(h_num_inliers, E, s);
  score.download(h_score, E, s);
  B200_CUDA_OK(cudaStreamSynchronize(s));
  return h_err == 0;
}

}  // namespace b200
