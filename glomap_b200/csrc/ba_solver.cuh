// ba_solver.cuh -- host-side driver of the device BA: problem residency,
// Ceres-semantics Levenberg-Marquardt loop (trust_region_minimizer.cc /
// levenberg_marquardt_strategy.cc, restated in oracle/ceres_lm.py) with the
// reduced camera system solved by implicit-Schur PCG on the device.
// Reference path replaced: glomap/estimators/bundle_adjustment.cc:11-106.
#pragma once
#include <cub/cub.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <vector>

#include "../../include/b200sfm_testing.h"
#include "ba_kernels.cuh"
#include "ba_kernels_v2.cuh"
#include "ba_kernels_v3.cuh"
#include "ba_kernels_ext.cuh"
#include "filter_kernels.cuh"
#include "processor_kernels.cuh"
#include "context.cuh"
#include "pcg.cuh"

namespace b200 {

// ---- structure-building kernels ----------------------------------------------
// largest share of L2 that one point slice's 32-B records (z4 / pts4) may fill in the camera-order passes: 8 slices at
// config 4 on an H100 (64 MB of records, 50 MB of L2), where the slice-count sweep of DESIGN §6 flattens; one at config 2
constexpr double kSliceL2Share = 1.0 / 6.0;

__global__ void k_expand_obs_pt(int P, const unsigned* __restrict__ pt_begin, int* __restrict__ obs_pt) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  for (unsigned o = pt_begin[p]; o < pt_begin[p + 1]; ++o) obs_pt[o] = p;
}
// sort key = bucket (camera half, point slice, "virtual camera"): ((half * n_slices + pt / slice_pts) * VC + vc, where
// vc = frame * smul + sensor (smul = 1, sensor = 0 without rigs) and half = frame >= half_frame.  Excluded observations
// get the key n_buckets, past every bucket.  One slice and half_frame past the last frame: the key is vc.
__global__ void k_cam_keys(long long N, int VC, int smul, int min_views, int slice_pts, int n_slices, int half_frame,
                           int n_buckets, const int* __restrict__ obs_cam, const unsigned short* __restrict__ obs_sensor,
                           const int* __restrict__ obs_pt, const unsigned* __restrict__ pt_begin,
                           int* __restrict__ keys, int* __restrict__ vals, int* __restrict__ bucket_count,
                           int* __restrict__ bad) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= N) return;
  const int pt = obs_pt[o];
  const bool valid = (int)(pt_begin[pt + 1] - pt_begin[pt]) >= min_views;
  const int cam = obs_cam[o] * smul + (obs_sensor ? (int)obs_sensor[o] : 0);
  // caller-supplied camera index out of range: flag it (-> B200SFM_ERR_INVALID_ARG) instead of writing out of bounds
  const bool in_range = obs_cam[o] >= 0 && cam < VC;
  if (!in_range) *bad = 1;
  const int bucket = ((obs_cam[o] >= half_frame ? n_slices : 0) + pt / slice_pts) * VC + cam;
  keys[o] = (valid && in_range) ? bucket : n_buckets;
  vals[o] = (int)o;
  if (valid && in_range) atomicAdd(&bucket_count[bucket], 1);
}
__global__ void k_seg_counts(int n_buckets, const int* __restrict__ bucket_count, int* __restrict__ seg_count) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n_buckets) seg_count[c] = seg_split(bucket_count[c]);
}
// the seg_split(n) equal segments of one bucket (k_cam_keys): bucket c belongs to virtual camera c % VC
__global__ void k_fill_segs(int n_buckets, int VC, int smul, const int* __restrict__ cam_begin, const int* __restrict__ seg_off,
                            const int* __restrict__ cam_intr, const int* __restrict__ sensor_intr,
                            int* __restrict__ seg_cam, int* __restrict__ seg_sensor, int* __restrict__ seg_intr,
                            int* __restrict__ seg_begin, int* __restrict__ seg_end) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_buckets) return;
  const int b = cam_begin[c], e = cam_begin[c + 1];
  const int vc = c % VC;
  const int frame = vc / smul, sensor = vc - frame * smul;
  const int blk = sensor_intr ? sensor_intr[sensor] : (cam_intr ? cam_intr[frame] : 0);
  const int n = e - b, ns = seg_split(n);
  for (int j = 0; j < ns; ++j) {
    const int s = seg_off[c] + j;
    seg_cam[s] = frame;
    if (seg_sensor) seg_sensor[s] = sensor;
    if (seg_intr) seg_intr[s] = blk;
    seg_begin[s] = b + (int)((long long)n * j / ns);
    seg_end[s] = b + (int)((long long)n * (j + 1) / ns);
  }
}
__global__ void k_gather_camorder(int Nv, const int* __restrict__ camord_obs, const int* __restrict__ obs_pt,
                                  const double2* __restrict__ obs_xy, int* __restrict__ pt_c,
                                  double2* __restrict__ xy_c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Nv) return;
  const int o = camord_obs[i];
  pt_c[i] = obs_pt[o];
  xy_c[i] = obs_xy[o];
}
__global__ void k_gather_int(int n, const int* __restrict__ idx, const int* __restrict__ src, int* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}
// blk_used[b] = 1: block b (frame f | C + intrinsics k | C + K + sensor s) has an observation of a kept track, i.e. it
// is a parameter block of the problem whatever its curvature (plain stores of the same value: the races are benign)
__global__ void k_block_used(int VC, int n_groups, int smul, int C, int K, const int* __restrict__ bucket_count,
                             const int* __restrict__ cam_intr, const int* __restrict__ sensor_intr,
                             double* __restrict__ blk_used) {
  const int vc = blockIdx.x * blockDim.x + threadIdx.x;
  if (vc >= VC) return;
  int n = 0;   // observations of vc over its n_groups buckets (camera half x point slice)
  for (int g = 0; g < n_groups; ++g) n += bucket_count[(size_t)g * VC + vc];
  if (n == 0) return;
  const int f = vc / smul, s = vc - f * smul;
  blk_used[f] = 1.0;
  blk_used[C + (sensor_intr ? sensor_intr[s] : cam_intr[f])] = 1.0;
  if (sensor_intr) blk_used[C + K + s] = 1.0;
}
__global__ void k_eff_mask(int C, const unsigned char* __restrict__ base, int fix_rot, int fix_trn,
                           unsigned char* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) out[c] = (unsigned char)((base ? base[c] : 0) | (fix_rot ? 1 : 0) | (fix_trn ? 2 : 0));
}
__global__ void k_normalize_quat(int C, double* __restrict__ q) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double n = sqrt(q[4 * c] * q[4 * c] + q[4 * c + 1] * q[4 * c + 1] + q[4 * c + 2] * q[4 * c + 2] +
                        q[4 * c + 3] * q[4 * c + 3]);
  if (n > 0) {
    const double inv = 1.0 / n;
    for (int k = 0; k < 4; ++k) q[4 * c + k] *= inv;
  }
}
// b = -(gc + y); fixed (optional, one entry per block of bs): b = 0 on the blocks with fixed < 0
__global__ void k_rhs(int n, const double* __restrict__ gc, const double* __restrict__ y, double* __restrict__ b,
                      const double* __restrict__ fixed = nullptr, int bs = 1) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) b[i] = (fixed && fixed[i / bs] < 0.0) ? 0.0 : -(gc[i] + (y ? y[i] : 0.0));
}

}  // namespace b200

struct b200sfm_ba_problem {
  using BAView = b200::BAView;
  template <class T>
  using DevBuf = b200::DevBuf<T>;

  b200sfm_ctx* ctx = nullptr;
  int C = 0, P = 0, K = 0;
  long long N = 0;
  int Nv = 0, n_tiles = 0, n_segs = 0, min_views = 3;
  int seg_mid = 0;   // first camera-order segment of a camera >= C / 2 (split all-reduce of the multi-GPU mat-vec)
  int n_slices = 1, slice_pts = 0;   // camera-order observations are grouped by point slices of slice_pts points (create())
  long long n_obs_used = 0;

  // structure
  DevBuf<int> obs_cam, obs_pt, tile_pt_begin, camord_obs, pt_c, seg_cam, seg_begin, seg_end, cam_intr, intr_model;
  // known rigs (S > 0): see BAView
  int S = 0;
  DevBuf<unsigned short> obs_sensor;
  DevBuf<int> seg_sensor, seg_intr, sensor_intr;
  DevBuf<double> sensor_rec;
  DevBuf<double2> obs_xy, xy_c;
  DevBuf<int4> tile_desc;
  DevBuf<unsigned> pt_begin;
  DevBuf<unsigned char> cam_mask_base, cam_mask;
  DevBuf<double> blk_used;   // [CB] > 0: the block is a parameter block of the problem (k_block_used; summed over the ranks)
  // state + candidate + snapshot
  DevBuf<double> quat[2], trans[2], points[2], intr, intr_cand, quat_saved, trans_saved, points_saved, intr_saved;
  // extended path (ba_kernels_ext.cuh): intrinsics blocks and unknown cam_from_rig poses as pseudo-camera blocks
  // appended to the frames: block f | C + k | C + K + s;  CB = C + K + S.  nbk = blocks in the current solve.
  int CB = 0, nbk = 0;
  bool ext = false, ext_k = false, ext_s = false;
  std::vector<int> h_intr_model;
  std::vector<b200::IntrVarRec> h_ivar;
  DevBuf<b200::IntrVarRec> ivar;
  std::vector<unsigned char> h_sensor_var;       // [S] caller's request (b200sfm_ba_problem_set_sensor_variable)
  DevBuf<unsigned char> sensor_var;
  DevBuf<double> sens_q[2], sens_t[2], sens_q_saved, sens_t_saved;   // cam_from_rig state (indexed like quat/trans by cur)
  b200::ExtView ext_view() {
    b200::ExtView e;
    e.C = C; e.K = K; e.S = S; e.ivar = ivar.p; e.sensor_var = (ext_s && S > 0) ? sensor_var.p : nullptr;
    return e;
  }
  // design v2 (compact rows, camera-order second pass)
  bool use_v2 = false;
  // point side of v2 in the ELL-32 layout (ba_kernels_v3.cuh): one thread per point
  bool use_ell = false;
  int ell_groups = 0, ell_ctas = 0, ell_bpart_rows = 0;
  long long ell_rows = 0;
  DevBuf<int> ell_row0, ell_pt, ell_len, ell_slot, ell_cam;
  DevBuf<double2> ell_xy;
  DevBuf<unsigned short> ell_sensor;
  DevBuf<double> ell_A, ell_part;
  b200::EllView ell_view() {
    b200::EllView e;
    e.n_groups = ell_groups; e.row0 = ell_row0.p; e.pt = ell_pt.p; e.len = ell_len.p; e.cam = ell_cam.p; e.xy = ell_xy.p;
    e.sensor = S > 0 ? ell_sensor.p : nullptr; e.A = ell_A.p; e.B = kfast ? ell_B.p : nullptr;
    return e;
  }
  DevBuf<double> z4, pts4, xq, bpart, bpart2;
  size_t smem_k3v2 = 0;
  // stored-row intrinsics path (ba_kernels_v2.cuh): <= 2 variable parameters per camera, no unknown cam_from_rig
  bool kfast = false;
  int nk = 0;
  DevBuf<double> ell_B, Ufk;
  b200::BAViewV2 view2() {
    b200::BAViewV2 w;
    w.Ap = W.p; w.z4 = z4.p; w.pts4 = pts4.p;
    w.Ufk = kfast ? Ufk.p : nullptr; w.ivar = ivar.p; w.C = C;
    return w;
  }
  int cur = 0;
  DevBuf<double> cam_rec, intr_rec;
  // linear system
  DevBuf<double> W, V, Vinv, gp, lin /* U | gc | cost */, Sd, Minv, jscale_c, jscale_p, Dc;
  // pcg
  DevBuf<double> px, pr, pz, pp, pq, yw, bvec;
  DevBuf<double> scal;   // [0] cost [1] gmax | [2..5] bscal | [6] cand cost | [8..12] cscal
  b200::EventTimer timer_lin, timer_mv;
  size_t smem_k1 = 0, smem_k3 = 0;

  // lin = U[CB][21] | gc[CB][6] | cost | one max|g_p| slot per rank  (fixed layout; a solve uses the first nbk blocks)
  double* U() { return lin.p; }
  double* gc() { return lin.p + (size_t)CB * 21; }
  double* cost_ptr() { return lin.p + (size_t)CB * 27; }

  BAView view() {
    BAView v;
    v.C = C; v.P = P; v.K = K; v.N = N; v.n_tiles = n_tiles; v.n_segs = n_segs; v.min_views = min_views;
    v.obs_cam = obs_cam.p; v.obs_pt = obs_pt.p; v.obs_xy = obs_xy.p; v.pt_begin = pt_begin.p;
    v.tile_pt_begin = tile_pt_begin.p; v.tile_desc = tile_desc.p; v.camord_obs = camord_obs.p; v.pt_c = pt_c.p; v.xy_c = xy_c.p;
    v.seg_cam = seg_cam.p; v.seg_begin = seg_begin.p; v.seg_end = seg_end.p;
    v.S = S; v.obs_sensor = obs_sensor.p; v.seg_sensor = seg_sensor.p; v.seg_intr = seg_intr.p; v.sensor_rec = sensor_rec.p;
    v.W = W.p; v.V = V.p; v.Vinv = Vinv.p; v.gp = gp.p; v.U = U(); v.gc = gc(); v.Sd = Sd.p; v.Minv = Minv.p;
    v.jscale_c = jscale_c.p; v.jscale_p = jscale_p.p; v.Dc = Dc.p;
    return v;
  }

  // -------------------------------------------------------------------------
  void create(b200sfm_ctx* c, int C_, int P_, long long N_, int K_, const int64_t* h_pt_begin, const int32_t* h_obs_cam,
              const double* h_obs_xy, const int32_t* h_cam_intr, const int32_t* h_intr_model,
              const uint8_t* h_cam_mask, int min_views_, b200sfm_lm_stats* st, int S_ = 0,
              const uint16_t* h_obs_sensor = nullptr, const double* h_sensor_q = nullptr,
              const double* h_sensor_t = nullptr, const int32_t* h_sensor_intr = nullptr) {
    using namespace b200;
    ctx = c; C = C_; P = P_; N = N_; K = K_; min_views = min_views_; S = S_;
    CB = C + K + S;
    nbk = C;
    const int smul = std::max(S, 1);
    const int VC = C * smul;
    cudaStream_t s = ctx->stream;
    // host: CSR offsets -> uint32, greedy tiling of whole points into <= kTile observations
    std::vector<unsigned> ptb((size_t)P + 1);
    std::vector<int> tiles;
    tiles.reserve((size_t)(N / 200) + 16);
    tiles.push_back(0);
    long long tile_obs = 0;
    int tile_pts = 0;
    n_obs_used = 0;
    for (int p = 0; p < P; ++p) {
      ptb[p] = (unsigned)h_pt_begin[p];
      const long long len = h_pt_begin[p + 1] - h_pt_begin[p];
      if (len < 0) throw InvalidInput{"pt_obs_begin must be non-decreasing"};
      if (len >= min_views) n_obs_used += len;
      if (tile_pts > 0 && (tile_obs + len > kTile || tile_pts >= kTilePts)) {
        tiles.push_back(p);
        tile_obs = 0;
        tile_pts = 0;
      }
      tile_obs += len;
      ++tile_pts;
    }
    ptb[P] = (unsigned)h_pt_begin[P];
    tiles.push_back(P);
    n_tiles = (int)tiles.size() - 1;

    obs_cam.alloc(N); obs_pt.alloc(N); obs_xy.alloc(N); pt_begin.alloc((size_t)P + 1);
    tile_pt_begin.alloc(tiles.size()); cam_intr.alloc(C); intr_model.alloc(K);
    cam_mask_base.alloc(CB); cam_mask.alloc(CB);   // the extra blocks carry no mask (zero)
    cam_mask_base.zero(s); cam_mask.zero(s);
    obs_cam.upload(h_obs_cam, N, s);
    obs_xy.upload(reinterpret_cast<const double2*>(h_obs_xy), N, s);
    pt_begin.upload(ptb.data(), (size_t)P + 1, s);
    tile_pt_begin.upload(tiles.data(), tiles.size(), s);
    std::vector<int4> descs((size_t)n_tiles);
    for (int t = 0; t < n_tiles; ++t) {
      const int a = tiles[t], b = tiles[t + 1];
      descs[t] = make_int4(a, b - a, (int)ptb[a], (int)(ptb[b] - ptb[a]));
    }
    tile_desc.alloc(descs.size());
    tile_desc.upload(descs.data(), descs.size(), s);
    if (S > 0) {
      // constant sensor records: R_cam_from_rig row-major, t_cam_from_rig, intrinsics block
      std::vector<double> rec((size_t)S * kSensorRec, 0.0);
      for (int i = 0; i < S; ++i) {
        const double* q = h_sensor_q + 4 * (size_t)i;
        const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
        const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
        double* r = rec.data() + (size_t)i * kSensorRec;
        r[0] = 1 - 2 * (y * y + z * z); r[1] = 2 * (x * y - z * w); r[2] = 2 * (x * z + y * w);
        r[3] = 2 * (x * y + z * w); r[4] = 1 - 2 * (x * x + z * z); r[5] = 2 * (y * z - x * w);
        r[6] = 2 * (x * z - y * w); r[7] = 2 * (y * z + x * w); r[8] = 1 - 2 * (x * x + y * y);
        r[9] = h_sensor_t[3 * (size_t)i]; r[10] = h_sensor_t[3 * (size_t)i + 1]; r[11] = h_sensor_t[3 * (size_t)i + 2];
        r[12] = (double)h_sensor_intr[i];
      }
      sensor_rec.alloc(rec.size());
      sensor_rec.upload(rec.data(), rec.size(), s);
      sensor_intr.alloc(S);
      sensor_intr.upload(h_sensor_intr, S, s);
      for (int i = 0; i < 2; ++i) { sens_q[i].alloc((size_t)S * 4); sens_t[i].alloc((size_t)S * 3); }
      sens_q[0].upload(h_sensor_q, (size_t)S * 4, s);
      sens_t[0].upload(h_sensor_t, (size_t)S * 3, s);
      B200_LAUNCH(ctx, b200::k_normalize_quat, b200::cdiv(S, 256), 256, 0, S, sens_q[0].p);
      sensor_var.alloc(S);
      sensor_var.zero(s);
      h_sensor_var.assign(S, 0);
      obs_sensor.alloc(N);
      obs_sensor.upload(h_obs_sensor, N, s);
      B200_CUDA_OK(cudaStreamSynchronize(s));   // rec is a local
      // cam_intr is unused with rigs (the intrinsics block belongs to the sensor); keep it defined
      std::vector<int> zeros(C, 0);
      cam_intr.upload(zeros.data(), C, s);
      B200_CUDA_OK(cudaStreamSynchronize(s));
    } else {
      for (int c2 = 0; c2 < C; ++c2)
        if (h_cam_intr[c2] < 0 || h_cam_intr[c2] >= K) throw InvalidInput{"cam_intr out of range"};
      cam_intr.upload(h_cam_intr, C, s);
    }
    intr_model.upload(h_intr_model, K, s);
    this->h_intr_model.assign(h_intr_model, h_intr_model + K);
    if (h_cam_mask) cam_mask_base.upload(h_cam_mask, C, s);
    if (st) st->h2d_bytes += N * 20 + ((long long)P + 1) * 4 + (long long)tiles.size() * 4 + (long long)C * 5 + K * 4;

    B200_LAUNCH(ctx, k_expand_obs_pt, cdiv(P, 256), 256, 0, P, pt_begin.p, obs_pt.p);
    // camera order, grouped by point slice.  Every camera-order kernel gathers one per-point record per observation
    // (z4 / pts4: 32 B, Vinv: 48 B) at a random address.  CTAs start roughly in blockIdx order, so with the rows of
    // one point slice together the resident warps gather from that slice's records only, and those stay in L2.
    // Slices start on ELL windows; there are as many as it takes for a slice's 32-B records to fill at most
    // kSliceL2Share of L2 (one slice, the plain camera order, when they all fit).  B200SFM_PT_SLICES=n asks for n.
    {
      int want = 1;
      if (getenv("B200SFM_PT_SLICES")) {
        want = std::max(1, atoi(getenv("B200SFM_PT_SLICES")));
      } else {
        int l2 = 0;
        B200_CUDA_OK(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, ctx->device));
        want = std::max(1, cdiv((long long)P * 32, std::max(1ll, (long long)(l2 * kSliceL2Share))));
      }
      want = std::min(want, std::max(1, (INT_MAX - 1) / (2 * VC)));   // bucket keys stay ints
      slice_pts = std::max(1, cdiv(cdiv(P, want), kEllWindow)) * kEllWindow;
      n_slices = std::max(1, cdiv(P, slice_pts));
    }
    // buckets (camera half, point slice, virtual camera): the halves split at frame C/2, so that every camera below
    // C/2 is complete after segment seg_mid (split all-reduce of the multi-GPU mat-vec); within a bucket the stable
    // sort keeps point order
    const int n_groups = 2 * n_slices, n_buckets = n_groups * VC;
    DevBuf<int> keys, vals, keys_out, cam_count, seg_count, cam_begin, seg_off, bad;
    keys.alloc(N); vals.alloc(N); keys_out.alloc(N); camord_obs.alloc(N);
    cam_count.alloc((size_t)n_buckets + 1); seg_count.alloc((size_t)n_buckets + 1); cam_begin.alloc((size_t)n_buckets + 1);
    seg_off.alloc((size_t)n_buckets + 1);
    bad.alloc(1);
    cam_count.zero(s); seg_count.zero(s); bad.zero(s);
    B200_LAUNCH(ctx, k_cam_keys, cdiv(N, 256), 256, 0, N, VC, smul, min_views, slice_pts, n_slices, C / 2, n_buckets,
                obs_cam.p, S > 0 ? obs_sensor.p : nullptr, obs_pt.p, pt_begin.p, keys.p, vals.p, cam_count.p, bad.p);
    int end_bit = 1;
    while ((1ll << end_bit) <= n_buckets) ++end_bit;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys.p, keys_out.p, vals.p, camord_obs.p, (int)N, 0, end_bit, s);
    size_t scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cam_count.p, cam_begin.p, n_buckets + 1, s);
    DevBuf<unsigned char> tmp;
    tmp.alloc(std::max(tmp_bytes, scan_bytes) + 16);
    size_t tb = tmp.bytes();
    cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.p, keys_out.p, vals.p, camord_obs.p, (int)N, 0, end_bit, s);
    ctx->launches += 8;
    tb = tmp.bytes();
    cub::DeviceScan::ExclusiveSum(tmp.p, tb, cam_count.p, cam_begin.p, n_buckets + 1, s);
    B200_LAUNCH(ctx, k_seg_counts, cdiv(n_buckets, 256), 256, 0, n_buckets, cam_count.p, seg_count.p);
    blk_used.alloc(CB);
    blk_used.zero(s);
    B200_LAUNCH(ctx, k_block_used, cdiv(VC, 256), 256, 0, VC, n_groups, smul, C, K, cam_count.p, cam_intr.p,
                S > 0 ? sensor_intr.p : nullptr, blk_used.p);
    ctx->allreduce_sum(blk_used.p, CB);   // a block observed on any rank is a block of the problem on every rank
    tb = tmp.bytes();
    cub::DeviceScan::ExclusiveSum(tmp.p, tb, seg_count.p, seg_off.p, n_buckets + 1, s);
    ctx->launches += 4;
    int h_tot[4];
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[0], cam_begin.p + n_buckets, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[1], seg_off.p + n_buckets, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[2], bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[3], seg_off.p + (size_t)n_slices * VC, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    if (h_tot[2]) throw InvalidInput{"obs_cam out of range [0, C)"};
    Nv = h_tot[0];
    n_segs = h_tot[1];
    seg_mid = h_tot[3];   // the first segment of the upper camera half
    seg_cam.alloc(std::max(n_segs, 1)); seg_begin.alloc(std::max(n_segs, 1)); seg_end.alloc(std::max(n_segs, 1));
    seg_sensor.alloc(std::max(n_segs, 1)); seg_intr.alloc(std::max(n_segs, 1));
    pt_c.alloc(std::max(Nv, 1)); xy_c.alloc(std::max(Nv, 1));
    B200_LAUNCH(ctx, k_fill_segs, cdiv(n_buckets, 256), 256, 0, n_buckets, VC, smul, cam_begin.p, seg_off.p, cam_intr.p,
                S > 0 ? sensor_intr.p : nullptr, seg_cam.p, seg_sensor.p, seg_intr.p, seg_begin.p, seg_end.p);
    if (Nv > 0)
      B200_LAUNCH(ctx, k_gather_camorder, cdiv(Nv, 256), 256, 0, Nv, camord_obs.p, obs_pt.p, obs_xy.p, pt_c.p, xy_c.p);

    // ELL-32 point-order structure (ba_kernels_v3.cuh): windows of 1024 points sorted by track length, 32 per group
    {
      using Sort = cub::BlockRadixSort<unsigned, kEllWindow, 1, int>;
      const int n_win = cdiv(P, kEllWindow);
      ell_groups = n_win * (kEllWindow / 32);
      ell_ctas = cdiv((long long)ell_groups * 32, kEllThreads);
      ell_pt.alloc((size_t)ell_groups * 32); ell_len.alloc((size_t)ell_groups * 32); ell_slot.alloc(P);
      ell_row0.alloc((size_t)ell_groups + 1);
      DevBuf<int> grows;
      grows.alloc((size_t)ell_groups + 1);
      grows.zero(s);
      B200_LAUNCH(ctx, (ell_sort_window<Sort>), n_win, kEllWindow, 0, P, min_views, pt_begin.p, ell_pt.p, ell_len.p, ell_slot.p, grows.p);
      size_t need = 0;
      cub::DeviceScan::ExclusiveSum(nullptr, need, grows.p, ell_row0.p, ell_groups + 1, s);
      DevBuf<unsigned char> tmp3;
      tmp3.alloc(need + 16);
      size_t tb3 = tmp3.bytes();
      cub::DeviceScan::ExclusiveSum(tmp3.p, tb3, grows.p, ell_row0.p, ell_groups + 1, s);
      ctx->launches += 1;
      int h_rows = 0;
      B200_CUDA_OK(cudaMemcpyAsync(&h_rows, ell_row0.p + ell_groups, sizeof(int), cudaMemcpyDeviceToHost, s));
      B200_CUDA_OK(cudaStreamSynchronize(s));
      ell_rows = h_rows;
      const size_t cells = (size_t)std::max<long long>(ell_rows, 1) * 32;
      ell_cam.alloc(cells); ell_xy.alloc(cells); ell_A.alloc(cells * 6);
      if (S > 0) ell_sensor.alloc(cells);
      ell_part.alloc((size_t)ell_ctas * (kEllThreads / 32) * 2 + 8);
      ell_bpart_rows = ell_ctas;
      B200_LAUNCH(ctx, ell_scatter_obs, cdiv(N, 256), 256, 0, N, min_views, obs_pt.p, pt_begin.p, obs_cam.p, obs_xy.p,
                  S > 0 ? obs_sensor.p : nullptr, ell_slot.p, ell_row0.p, ell_cam.p, ell_xy.p, S > 0 ? ell_sensor.p : nullptr);
      B200_CUDA_OK(cudaStreamSynchronize(s));   // temporaries go out of scope
    }
    for (int i = 0; i < 2; ++i) {
      quat[i].alloc((size_t)C * 4); trans[i].alloc((size_t)C * 3); points[i].alloc((size_t)P * 3);
    }
    intr.alloc((size_t)K * B200SFM_INTR_STRIDE);
    intr_cand.alloc((size_t)K * B200SFM_INTR_STRIDE);
    cam_rec.alloc((size_t)C * kCamRec); intr_rec.alloc((size_t)K * kIntrRec);
    W.alloc((size_t)N * kWDoubles); V.alloc((size_t)P * 6); Vinv.alloc((size_t)P * 6); gp.alloc((size_t)P * 3);
    lin.alloc((size_t)CB * 27 + 1 + (size_t)ctx->world);   // U | gc | cost | one max|g_p| slot per rank
    Sd.alloc((size_t)CB * 27);                              // Schur-Jacobi blocks | right-hand-side accumulator (one all-reduce for both)
    Minv.alloc((size_t)CB * 21);
    jscale_c.alloc((size_t)CB * 6); jscale_p.alloc((size_t)P * 3); Dc.alloc((size_t)CB * 6);
    px.alloc((size_t)CB * 6); pr.alloc((size_t)CB * 6); pz.alloc((size_t)CB * 6); pp.alloc((size_t)CB * 6);
    pq.alloc((size_t)CB * 6); yw.alloc((size_t)CB * 6); bvec.alloc((size_t)CB * 6);
    ivar.alloc(K);
    scal.alloc(16);
    smem_k1 = sizeof(K1Smem) + 128;
    smem_k3 = sizeof(K3Smem) + 128;
    B200_CUDA_OK(cudaFuncSetAttribute(ba_linearize_points<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k1));
    B200_CUDA_OK(cudaFuncSetAttribute(ba_linearize_points<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k1));
    B200_CUDA_OK(cudaFuncSetAttribute(ba_schur_pass<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k3));
    B200_CUDA_OK(cudaFuncSetAttribute(ba_schur_pass<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k3));
    B200_CUDA_OK(cudaFuncSetAttribute(ba_schur_pass<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k3));
    // several 50-KB CTAs per SM: ask for the full shared-memory carve-out
    // shared-memory carve-out of the tiled kernels: 75 % leaves ~60 KB of L1 for the camera-record / R^T x gathers
    // (100 % = max shared starves the gathers of L1, 25 % halves the resident CTAs)
    const int carve = getenv("B200SFM_CARVEOUT") ? atoi(getenv("B200SFM_CARVEOUT")) : 75;
    B200_CUDA_OK(cudaFuncSetAttribute(ba_linearize_points<false>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    B200_CUDA_OK(cudaFuncSetAttribute(ba_linearize_points<true>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    B200_CUDA_OK(cudaFuncSetAttribute(ba_schur_pass<0>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    B200_CUDA_OK(cudaFuncSetAttribute(ba_schur_pass<1>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    B200_CUDA_OK(cudaFuncSetAttribute(ba_schur_pass<2>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    smem_k3v2 = sizeof(K3v2Smem) + 128;
    B200_CUDA_OK(cudaFuncSetAttribute(ba2_pass_a<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k3v2));
    B200_CUDA_OK(cudaFuncSetAttribute(ba2_pass_a<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k3v2));
    B200_CUDA_OK(cudaFuncSetAttribute(ba2_pass_a<0>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    B200_CUDA_OK(cudaFuncSetAttribute(ba2_pass_a<2>, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    z4.alloc((size_t)P * 4); pts4.alloc((size_t)P * 4); xq.alloc((size_t)C * kXqStride);
    bpart.alloc((size_t)std::max(std::max(n_tiles, ell_bpart_rows), 1) * 4);
    bpart2.alloc(296 * 4);
    B200_CUDA_OK(cudaStreamSynchronize(s));   // temporaries go out of scope
  }

  void set_state(const double* h_intr, const double* h_quat, const double* h_trans, const double* h_points,
                 b200sfm_lm_stats* st) {
    cudaStream_t s = ctx->stream;
    intr.upload(h_intr, (size_t)K * B200SFM_INTR_STRIDE, s);
    quat[cur].upload(h_quat, (size_t)C * 4, s);
    trans[cur].upload(h_trans, (size_t)C * 3, s);
    points[cur].upload(h_points, (size_t)P * 3, s);
    B200_LAUNCH(ctx, b200::k_normalize_quat, b200::cdiv(C, 256), 256, 0, C, quat[cur].p);
    if (st) st->h2d_bytes += ((long long)K * B200SFM_INTR_STRIDE + (long long)C * 7 + (long long)P * 3) * 8;
  }
  void get_state(double* h_intr, double* h_quat, double* h_trans, double* h_points, b200sfm_lm_stats* st) {
    cudaStream_t s = ctx->stream;
    if (h_intr) intr.download(h_intr, (size_t)K * B200SFM_INTR_STRIDE, s);
    if (h_quat) quat[cur].download(h_quat, (size_t)C * 4, s);
    if (h_trans) trans[cur].download(h_trans, (size_t)C * 3, s);
    if (h_points) points[cur].download(h_points, (size_t)P * 3, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    if (st) st->d2h_bytes += ((long long)K * B200SFM_INTR_STRIDE + (long long)C * 7 + (long long)P * 3) * 8;
  }
  void save_state() {
    cudaStream_t s = ctx->stream;
    if (!quat_saved.p) {
      quat_saved.alloc((size_t)C * 4); trans_saved.alloc((size_t)C * 3); points_saved.alloc((size_t)P * 3);
      intr_saved.alloc((size_t)K * B200SFM_INTR_STRIDE);
      if (S > 0) { sens_q_saved.alloc((size_t)S * 4); sens_t_saved.alloc((size_t)S * 3); }
    }
    if (S > 0) {
      B200_CUDA_OK(cudaMemcpyAsync(sens_q_saved.p, sens_q[cur].p, sens_q_saved.bytes(), cudaMemcpyDeviceToDevice, s));
      B200_CUDA_OK(cudaMemcpyAsync(sens_t_saved.p, sens_t[cur].p, sens_t_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    }
    B200_CUDA_OK(cudaMemcpyAsync(quat_saved.p, quat[cur].p, quat_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(trans_saved.p, trans[cur].p, trans_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(points_saved.p, points[cur].p, points_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(intr_saved.p, intr.p, intr_saved.bytes(), cudaMemcpyDeviceToDevice, s));
  }
  bool restore_state() {
    if (!quat_saved.p) return false;
    cudaStream_t s = ctx->stream;
    B200_CUDA_OK(cudaMemcpyAsync(quat[cur].p, quat_saved.p, quat_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(trans[cur].p, trans_saved.p, trans_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(points[cur].p, points_saved.p, points_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(intr.p, intr_saved.p, intr_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    if (S > 0) {
      B200_CUDA_OK(cudaMemcpyAsync(sens_q[cur].p, sens_q_saved.p, sens_q_saved.bytes(), cudaMemcpyDeviceToDevice, s));
      B200_CUDA_OK(cudaMemcpyAsync(sens_t[cur].p, sens_t_saved.p, sens_t_saved.bytes(), cudaMemcpyDeviceToDevice, s));
      B200_LAUNCH(ctx, b200::bax_build_sensor_rec, b200::cdiv(S, 256), 256, 0, S, sens_q[cur].p, sens_t[cur].p, sensor_intr.p, sensor_rec.p);
    }
    return true;
  }

  // -------------------------------------------------------------------------
  void build_records(int which) {
    using namespace b200;
    B200_LAUNCH(ctx, ba_build_records, cdiv(std::max(C, K), 256), 256, 0, C, K, quat[which].p, trans[which].p,
                cam_intr.p, cam_mask.p, (which == cur ? intr.p : intr_cand.p), intr_model.p, cam_rec.p, intr_rec.p);
    // cam_from_rig poses: constant unless a sensor is an unknown of this solve; the records are rebuilt either way
    // (S is small) so that a state accepted by an earlier optimize_rig_poses solve stays in effect
    if (S > 0)
      B200_LAUNCH(ctx, bax_build_sensor_rec, cdiv(S, 256), 256, 0, S, sens_q[which].p, sens_t[which].p,
                  sensor_intr.p, sensor_rec.p);
  }
  void set_sensor_variable(const uint8_t* h_var) {
    h_sensor_var.assign(h_var, h_var + S);
    sensor_var.upload(h_sensor_var.data(), S, ctx->stream);
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
  }
  void get_sensor_poses(double* h_q, double* h_t) {
    if (h_q) sens_q[cur].download(h_q, (size_t)S * 4, ctx->stream);
    if (h_t) sens_t[cur].download(h_t, (size_t)S * 3, ctx->stream);
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
  }

  // robust cost of points[which] under the current records -> scal[6] (this rank's shard)
  void launch_cost(int which, double huber_a) {
    using namespace b200;
    if (use_ell) {
      B200_LAUNCH(ctx, ba3_cost, ell_ctas, kEllThreads, 0, view(), ell_view(), cam_rec.p, intr_rec.p, points[which].p, huber_a, ell_part.p);
      B200_LAUNCH(ctx, ba3_reduce_partials, 1, 256, 0, ell_ctas, ell_part.p, nullptr, scal.p + 6, nullptr);
    } else {
      const int grid = std::min(cdiv(N, 256), ctx->num_sms * 8);
      B200_LAUNCH(ctx, ba_cost, grid, 256, 0, view(), cam_rec.p, intr_rec.p, points[which].p, huber_a, scal.p + 6);
    }
  }

  // robust cost of state `which` -> host (synchronises)
  double eval_cost(int which, double huber_a) {
    using namespace b200;
    build_records(which);
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 6, 0, sizeof(double), ctx->stream));
    launch_cost(which, huber_a);
    ctx->allreduce_sum(scal.p + 6, 1);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal, scal.p + 6, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return ctx->h_scal[0];
  }

  // Jacobian + Schur blocks at the current state.  Returns (cost, max|g|).
  void linearize(double huber_a, bool points_var, bool first, bool profile, double& cost, double& gmax) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    build_records(cur);
    lin.zero(s);
    B200_CUDA_OK(cudaMemsetAsync(scal.p, 0, 2 * sizeof(double), s));
    BAView v = view();
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (profile) {
      e0 = timer_lin.next();
      e1 = timer_lin.next();
      B200_CUDA_OK(cudaEventRecord(e0, s));
    }
    if (use_ell) {
      const int nwp = ell_ctas * (kEllThreads / 32);   // one partial per warp
#define B200_LIN_P(NKV)                                                                                                   \
  B200_LAUNCH(ctx, ba3_linearize_points<NKV>, ell_ctas, kEllThreads, 0, v, ell_view(), cam_rec.p, intr_rec.p, points[cur].p, \
              huber_a, points_var ? 1 : 0, ell_part.p, ell_part.p + nwp, ivar.p)
      if (kfast && nk == 2) B200_LIN_P(2);
      else if (kfast && nk == 1) B200_LIN_P(1);
      else B200_LIN_P(0);
#undef B200_LIN_P
      B200_LAUNCH(ctx, ba3_reduce_partials, 1, 1024, 0, nwp, ell_part.p, ell_part.p + nwp, scal.p, scal.p + 1);
    } else if (use_v2)
      B200_LAUNCH(ctx, ba_linearize_points<true>, n_tiles, kTile, smem_k1, v, cam_rec.p, intr_rec.p, points[cur].p, huber_a,
                  points_var ? 1 : 0, scal.p);
    else
      B200_LAUNCH(ctx, ba_linearize_points<false>, n_tiles, kTile, smem_k1, v, cam_rec.p, intr_rec.p, points[cur].p, huber_a,
                  points_var ? 1 : 0, scal.p);
    if (profile) B200_CUDA_OK(cudaEventRecord(e1, s));
    if (n_segs > 0) {
      const int sgrid = cdiv((long long)n_segs * 32, 128);
      if (kfast) {
        Ufk.zero(s);
        B200_LAUNCH(ctx, ba2_pad_points, cdiv(P, 256), 256, 0, P, points[cur].p, pts4.p);
        if (nk == 2) B200_LAUNCH(ctx, ba2_linearize_cams<2>, sgrid, 128, 0, v, view2(), cam_rec.p, intr_rec.p, huber_a);
        else B200_LAUNCH(ctx, ba2_linearize_cams<1>, sgrid, 128, 0, v, view2(), cam_rec.p, intr_rec.p, huber_a);
      } else if (ext) {
        B200_LAUNCH(ctx, bax_linearize_blocks<0>, sgrid, 128, 0, v, ext_view(), cam_rec.p, intr_rec.p, points[cur].p, huber_a);
        if (ext_k) B200_LAUNCH(ctx, bax_linearize_blocks<1>, sgrid, 128, 0, v, ext_view(), cam_rec.p, intr_rec.p, points[cur].p, huber_a);
        if (ext_s) B200_LAUNCH(ctx, bax_linearize_blocks<2>, sgrid, 128, 0, v, ext_view(), cam_rec.p, intr_rec.p, points[cur].p, huber_a);
      } else if (use_v2) {
        B200_LAUNCH(ctx, ba2_pad_points, cdiv(P, 256), 256, 0, P, points[cur].p, pts4.p);
        B200_LAUNCH(ctx, ba2_linearize_cams<0>, sgrid, 128, 0, v, view2(), cam_rec.p, intr_rec.p, huber_a);
      } else {
        B200_LAUNCH(ctx, ba_linearize_cams, sgrid, 128, 0, v, cam_rec.p, intr_rec.p, points[cur].p, huber_a);
      }
    }
    // cost and this rank's max|g_p| (own slot, zeros elsewhere) travel with U|gc through ONE sum all-reduce
    B200_CUDA_OK(cudaMemcpyAsync(cost_ptr(), scal.p, sizeof(double), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(cost_ptr() + 1 + ctx->rank, scal.p + 1, sizeof(double), cudaMemcpyDeviceToDevice, s));
    ctx->allreduce_sum(lin.p, (size_t)CB * 27 + 1 + (size_t)ctx->world);
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 1, 0, sizeof(double), s));
    B200_LAUNCH(ctx, ba_finalize_cams, cdiv(nbk, 128), 128, 0, nbk, U(), gc(), cam_mask.p, jscale_c.p, first ? 1 : 0,
                scal.p, cost_ptr() + 1, ctx->world);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal, cost_ptr(), sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal + 1, scal.p + 1, sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    cost = ctx->h_scal[0];
    gmax = ctx->h_scal[1];
  }

  // ---- processors on the resident arrays (processor_kernels.cuh) ---------------------------------
  DevBuf<double> bear_res;   // unit bearings of all observations [N][3], filled by undistort()
  // UndistortImages (image_undistorter.cc:7-53) from the current intrinsics; h_out [N][3] may be null
  void undistort(double* h_out) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    if (bear_res.n < (size_t)N * 3) bear_res.alloc((size_t)std::max<long long>(N, 1) * 3);
    if (N > 0)
      B200_LAUNCH(ctx, proc_undistort, cdiv(N, 256), 256, 0, N, S, obs_cam.p, S > 0 ? obs_sensor.p : nullptr, cam_intr.p,
                  S > 0 ? sensor_intr.p : nullptr, intr_model.p, intr.p, obs_xy.p, bear_res.p);
    if (h_out) bear_res.download(h_out, (size_t)N * 3, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }
  // NormalizeReconstruction (reconstruction_normalizer.cc:5-104) on the current state; returns the similarity
  // X' = scale X + t (identity rotation)
  void normalize(bool fixed_scale, double extent, double p0, double p1, double* scale_out, double* t_out) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    const int n_img = S > 0 ? C * S : C;
    double scale = 1.0, t[3] = {0, 0, 0};
    if (n_img > 0) {
      DevBuf<float> c_in, c_out;
      DevBuf<double> stats;
      c_in.alloc((size_t)n_img * 3); c_out.alloc((size_t)n_img * 3); stats.alloc(9);
      B200_LAUNCH(ctx, proc_image_centres, cdiv(n_img, 256), 256, 0, C, S, quat[cur].p, trans[cur].p, S > 0 ? sens_q[cur].p : nullptr,
                  S > 0 ? sens_t[cur].p : nullptr, c_in.p, c_in.p + n_img, c_in.p + 2 * (size_t)n_img);
      size_t need = 0;
      cub::DeviceRadixSort::SortKeys(nullptr, need, c_in.p, c_out.p, n_img, 0, 32, s);
      DevBuf<unsigned char> tmp;
      tmp.alloc(need);
      for (int a = 0; a < 3; ++a) {   // per-axis sort of the float coordinates (.cc:31-33)
        size_t nb = need;
        cub::DeviceRadixSort::SortKeys(tmp.p, nb, c_in.p + (size_t)a * n_img, c_out.p + (size_t)a * n_img, n_img, 0, 32, s);
      }
      const size_t P0 = (size_t)((n_img > 3) ? p0 * (n_img - 1) : 0);                     // .cc:35-38
      const size_t P1 = (size_t)((n_img > 3) ? p1 * (n_img - 1) : n_img - 1);
      B200_LAUNCH(ctx, proc_trimmed_stats, 1, 256, 0, (int)P0, (int)P1, c_out.p, c_out.p + n_img, c_out.p + 2 * (size_t)n_img, stats.p);
      double h[9];
      B200_CUDA_OK(cudaMemcpyAsync(h, stats.p, sizeof(h), cudaMemcpyDeviceToHost, s));
      B200_CUDA_OK(cudaStreamSynchronize(s));
      double mean[3];
      for (int a = 0; a < 3; ++a) mean[a] = h[6 + a] / (double)(P1 - P0 + 1);
      if (!fixed_scale) {
        const double d0 = h[3] - h[0], d1 = h[4] - h[1], d2 = h[5] - h[2];
        const double old_extent = std::sqrt(d0 * d0 + d1 * d1 + d2 * d2);
        if (old_extent >= 2.220446049250313e-16) scale = extent / old_extent;             // .cc:54-60
      }
      for (int a = 0; a < 3; ++a) t[a] = -scale * mean[a];
      B200_LAUNCH(ctx, proc_transform_frames, cdiv(C, 256), 256, 0, C, scale, t[0], t[1], t[2], quat[cur].p, trans[cur].p);
      if (S > 0) B200_LAUNCH(ctx, proc_scale_shift3, cdiv(S, 256), 256, 0, (long long)S, scale, 0.0, 0.0, 0.0, sens_t[cur].p);   // .cc:70-79
      if (P > 0) B200_LAUNCH(ctx, proc_scale_shift3, cdiv(P, 256), 256, 0, (long long)P, scale, t[0], t[1], t[2], points[cur].p);  // .cc:81-83
      B200_CUDA_OK(cudaStreamSynchronize(s));   // the scratch buffers go out of scope
    }
    if (scale_out) *scale_out = scale;
    if (t_out) { t_out[0] = t[0]; t_out[1] = t[1]; t_out[2] = t[2]; }
  }

  // ---- track filters on the resident arrays (glomap/processors/track_filter.cc) -----------------
  // mode 0: reprojection (pixels), 1: angle (needs bearings), 2: triangulation angle (per track),
  // 3: reprojection in the normalised image plane (needs bearings)
  long long run_filter(int mode, double thr, const double* h_bearings, const uint8_t* h_calibrated, uint8_t* h_keep) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    B200_LAUNCH(ctx, k_eff_mask, cdiv(C, 256), 256, 0, C, cam_mask_base.p, 0, 0, cam_mask.p);
    build_records(cur);
    BAView v = view();
    const double kPi = 3.14159265358979323846;
    DevBuf<int> changed, counter;
    DevBuf<unsigned char> keep;
    counter.alloc(1);
    counter.zero(s);
    long long result = 0;
    if (mode == 2) {
      keep.alloc(P);
      B200_LAUNCH(ctx, filter_triangulation_angle, cdiv((long long)P * 32, 256), 256, 0, v, cam_rec.p, points[cur].p,
                  std::cos(thr * kPi / 180.0), keep.p, counter.p);
      keep.download(h_keep, P, s);
    } else {
      keep.alloc(N);
      changed.alloc(P);
      changed.zero(s);
      if (mode == 0) {
        B200_LAUNCH(ctx, filter_reprojection, cdiv(N, 256), 256, 0, v, cam_rec.p, intr_rec.p, points[cur].p, thr, keep.p, changed.p);
      } else {
        DevBuf<double> bear_up;
        DevBuf<unsigned char> cal;
        const double* bear_p;
        if (h_bearings) {
          bear_up.alloc((size_t)N * 3);
          bear_up.upload(h_bearings, (size_t)N * 3, s);
          bear_p = bear_up.p;
        } else {   // no host bearings: the resident ones of undistort() (computed now if they are not there yet)
          if (bear_res.n < (size_t)N * 3) undistort(nullptr);
          bear_p = bear_res.p;
        }
        const int ncal = S > 0 ? S : C;
        if (h_calibrated) { cal.alloc(ncal); cal.upload(h_calibrated, ncal, s); }
        if (mode == 3)
          B200_LAUNCH(ctx, filter_reprojection_normalized, cdiv(N, 256), 256, 0, v, cam_rec.p, points[cur].p, bear_p, thr,
                      keep.p, changed.p);
        else
          B200_LAUNCH(ctx, filter_angle, cdiv(N, 256), 256, 0, v, cam_rec.p, points[cur].p, bear_p, h_calibrated ? cal.p : nullptr,
                      std::cos(thr * kPi / 180.0), std::cos(2.0 * thr * kPi / 180.0), keep.p, changed.p);
        B200_CUDA_OK(cudaStreamSynchronize(s));   // bear_up / cal go out of scope
      }
      B200_LAUNCH(ctx, count_flags, cdiv(P, 256), 256, 0, P, changed.p, counter.p);
      keep.download(h_keep, N, s);
    }
    int h_cnt = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&h_cnt, counter.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    result = h_cnt;
    return result;
  }

  struct StepResult {
    double model_cost_change = 0, cand_cost = 0, step_norm = 0, x_norm = 0;
    int pcg_iters = 0;
    bool finite = true;
  };

  // mat-vec of the extended path: yw = (J^T J - W Vinv W^T) p over all nbk blocks (ba_kernels_ext.cuh); the damping
  // is added by pcg_apply_diag.  x == nullptr: right-hand-side mode (z4 already holds Vinv g_p).
  void ext_matvec(const double* x, double* y, double huber_a, double radius, bool points_var, const b200::PcgCtl* ctl) {
    using namespace b200;
    BAView v = view();
    ExtView ex = ext_view();
    const int sgrid = cdiv((long long)n_segs * 32, 128);
    if (x && points_var) {
#define B200_EXT_A(WK, WS)                                                                                              \
  B200_LAUNCH(ctx, (bax_pass_a<0, WK, WS>), ell_ctas, kEllThreads, 0, v, ell_view(), ex, view2(), cam_rec.p, intr_rec.p, x, \
              points[cur].p, nullptr, huber_a, radius, nullptr, ctl)
      if (ext_k && ext_s) B200_EXT_A(true, true);
      else if (ext_k) B200_EXT_A(true, false);
      else if (ext_s) B200_EXT_A(false, true);
      else B200_EXT_A(false, false);
#undef B200_EXT_A
    }
    if (n_segs > 0) {
#define B200_EXT_B(WK, WS)                                                                                              \
  B200_LAUNCH(ctx, (bax_pass_b<WK, WS>), sgrid, 128, 0, v, ex, view2(), cam_rec.p, intr_rec.p, points[cur].p, x, huber_a, y, ctl)
      if (ext_k && ext_s) B200_EXT_B(true, true);
      else if (ext_k) B200_EXT_B(true, false);
      else if (ext_s) B200_EXT_B(false, true);
      else B200_EXT_B(false, false);
#undef B200_EXT_B
    }
  }

  void launch_pass_b(const b200::BAView& v, double huber_a, double* y, const b200::PcgCtl* ctl, int seg_lo = 0,
                     int seg_hi = -1) {
    using namespace b200;
    if (seg_hi < 0) seg_hi = n_segs;
    if (seg_hi <= seg_lo) return;
    const int grid = cdiv((long long)(seg_hi - seg_lo) * 32, 128);
#define B200_PASS_B(NKV) \
  B200_LAUNCH(ctx, ba2_pass_b<NKV>, grid, 128, 0, v, view2(), cam_rec.p, intr_rec.p, huber_a, y, ctl, seg_lo, seg_hi)
    if (kfast && nk == 2) B200_PASS_B(2);
    else if (kfast) B200_PASS_B(1);
    else B200_PASS_B(0);
#undef B200_PASS_B
  }
  void launch_pass_a0(const b200::BAView& v, double radius, const b200::PcgCtl* ctl) {
    using namespace b200;
    if (kfast && nk == 2)
      B200_LAUNCH(ctx, (ba3_pass_a<0, 2>), ell_ctas, kEllThreads, 0, v, ell_view(), view2(), xq.p, points[cur].p, nullptr, radius, nullptr, ctl);
    else if (kfast)
      B200_LAUNCH(ctx, (ba3_pass_a<0, 1>), ell_ctas, kEllThreads, 0, v, ell_view(), view2(), xq.p, points[cur].p, nullptr, radius, nullptr, ctl);
    else
      B200_LAUNCH(ctx, (ba3_pass_a<0, 0>), ell_ctas, kEllThreads, 0, v, ell_view(), view2(), xq.p, points[cur].p, nullptr, radius, nullptr, ctl);
  }
  void launch_cross(const double* x, double* y, const b200::PcgCtl* ctl) {
    using namespace b200;
    if (nk == 2) B200_LAUNCH(ctx, ba2k_cross<2>, cdiv(C, 256), 256, 0, C, K, cam_rec.p, Ufk.p, x, y, ctl);
    else B200_LAUNCH(ctx, ba2k_cross<1>, cdiv(C, 256), 256, 0, C, K, cam_rec.p, Ufk.p, x, y, ctl);
  }

  // Schur-Jacobi blocks need the stored A_o rows of the fast path; the extended path preconditions with block-Jacobi
  bool matrix_free() const { return ext && !kfast; }   // matrix-free extended mat-vec (ba_kernels_ext.cuh); kfast: stored rows
  bool schur_jacobi_on(const b200sfm_ba_opts& o, bool points_var) const {
    return points_var && o.preconditioner == 1 && !matrix_free();   // kfast: frames Schur-Jacobi, intrinsics block-Jacobi
  }

  // Observation passes of one mat-vec of the reduced camera system S + D, then the all-reduce of y over the ranks.
  // They leave in y what pcg_apply_diag does not add: everything but the blocks U + D (the matrix-free extended
  // path: everything but D).  y must be zero on entry.  The v2 point pass reads x through its packed copy xq (filled by ba2_pcg_direction_pack, or by
  // ba2_pack_x + ba2k_pack_xk), the other kernels read x itself.
  void matvec(const double* x, double* y, const b200sfm_ba_opts& o, double radius, bool points_var, bool split_ar,
              bool profile, const b200::PcgCtl* ctl) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    BAView v = view();
    const int nB6 = nbk * 6;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (profile) {
      e0 = timer_mv.next();
      e1 = timer_mv.next();
      B200_CUDA_OK(cudaEventRecord(e0, s));
    }
    if (matrix_free()) {
      ext_matvec(x, y, o.thres_loss_function, radius, points_var, ctl);
    } else if (kfast && !points_var) {
      // constant points: no Schur term; U x = block diagonal (apply_diag) + the frame x intrinsics coupling
      launch_cross(x, y, ctl);
    } else if (use_v2) {
      if (use_ell)
        launch_pass_a0(v, radius, ctl);
      else
        B200_LAUNCH(ctx, ba2_pass_a<0>, n_tiles, kTile, smem_k3v2, v, view2(), xq.p, points[cur].p, nullptr, radius, nullptr, ctl);
      if (kfast) launch_cross(x, y, ctl);   // before pass B: its y_f updates are plain stores of the owning thread
      if (split_ar) {
        // cameras below C/2 are complete after the first half of the (camera-sorted) segments: their all-reduce
        // runs on the second stream while pass B works through the upper half
        launch_pass_b(v, o.thres_loss_function, y, ctl, 0, seg_mid);
        B200_CUDA_OK(cudaEventRecord(ctx->ev_half, s));
        B200_CUDA_OK(cudaStreamWaitEvent(ctx->comm_stream, ctx->ev_half, 0));
        ctx->allreduce_sum_on(ctx->comm_stream, y, (size_t)(C / 2) * 6);
        B200_CUDA_OK(cudaEventRecord(ctx->ev_comm, ctx->comm_stream));
        launch_pass_b(v, o.thres_loss_function, y, ctl, seg_mid, n_segs);
      } else if (n_segs > 0) {
        launch_pass_b(v, o.thres_loss_function, y, ctl);
      }
    } else {
      B200_LAUNCH(ctx, ba_schur_pass<0>, n_tiles, kTile, smem_k3, v, x, y, nullptr, nullptr, radius, nullptr, nullptr,
                  nullptr, 0, ctl);
    }
    if (profile) B200_CUDA_OK(cudaEventRecord(e1, s));
    if (split_ar) {
      ctx->allreduce_sum(y + (size_t)(C / 2) * 6, nB6 - (size_t)(C / 2) * 6);   // upper half + pseudo-camera blocks
      B200_CUDA_OK(cudaStreamWaitEvent(s, ctx->ev_comm, 0));
    } else {
      ctx->allreduce_sum(y, nB6);
    }
  }

  // One trust-region step at the current linearisation: damping, preconditioner,
  // PCG on the reduced camera system, back-substitution, candidate + its cost.
  StepResult compute_step(const b200sfm_ba_opts& o, double radius, bool points_var, bool set_jscale_p, bool profile) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    BAView v = view();
    const int nB6 = nbk * 6;
    if (points_var) B200_LAUNCH(ctx, ba_damp_points, cdiv(P, 256), 256, 0, P, V.p, jscale_p.p, set_jscale_p ? 1 : 0, radius, Vinv.p);
    B200_LAUNCH(ctx, ba_damp_cams, cdiv(nB6, 256), 256, 0, nbk, U(), jscale_c.p, radius, Dc.p);
    const bool recomp = matrix_free();
    const bool schur_jacobi = schur_jacobi_on(o, points_var);
    double* yrhs = Sd.p + (size_t)CB * 21;   // W Vinv g_p accumulates next to Sd so that both share one all-reduce
    Sd.zero(s);
    if (schur_jacobi && n_segs > 0) {
      if (use_v2)
        B200_LAUNCH(ctx, ba2_schur_diag, cdiv((long long)n_segs * 32, 128), 128, 0, v, view2(), cam_rec.p, intr_rec.p,
                    o.thres_loss_function);
      else B200_LAUNCH(ctx, ba_schur_diag, cdiv((long long)n_segs * 32, 128), 128, 0, v);
    }
    if (points_var) {
      if (use_v2) {
        B200_LAUNCH(ctx, ba2_point_rhs_z, cdiv(P, 256), 256, 0, v, view2());
        if (recomp) ext_matvec(nullptr, yrhs, o.thres_loss_function, radius, true, nullptr);
        else if (n_segs > 0) launch_pass_b(v, o.thres_loss_function, yrhs, nullptr);
      } else {
        B200_LAUNCH(ctx, ba_schur_pass<1>, n_tiles, kTile, smem_k3, v, nullptr, yrhs, nullptr, nullptr, radius, nullptr);
      }
    } else if (recomp) {
      z4.zero(s);   // constant points: no Schur term, pass B still applies J^T J
    }
    if (schur_jacobi || points_var) ctx->allreduce_sum(Sd.p, (size_t)CB * 27);
    B200_LAUNCH(ctx, ba_build_precond, cdiv(nbk, 128), 128, 0, nbk, U(), Dc.p, schur_jacobi ? Sd.p : nullptr, Minv.p);
    // right-hand side b = -(gc - W Vinv gp)   (W Vinv gp was accumulated above, next to Sd)
    B200_LAUNCH(ctx, k_rhs, cdiv(nB6, 256), 256, 0, nB6, gc(), points_var ? yrhs : nullptr, bvec.p);
    // ---- PCG (loop control on the device, iterations queued ahead of the read-back: pcg.cuh) --------
    const int max_it = std::max(1, o.pcg_max_iterations);
    const int nblk = cdiv(nbk, kPcgThreads);
    ctx->pcgh.ensure(max_it, (size_t)nblk * 3, ctx->world);
    double* part_pq = ctx->pcgh.d_part;
    double* part_rz = ctx->pcgh.d_part + nblk;
    double* part_rr = ctx->pcgh.d_part + 2 * (size_t)nblk;
    PcgCtl* ctl = ctx->pcgh.d_ctl;
    StepResult res;
    const size_t mv_ev0 = timer_mv.used;
    const bool has_mv = points_var || ext;   // an observation pass per iteration (else S = U + D is block diagonal)
    // several GPUs, opt-in (B200SFM_SPLIT_AR=1): split the per-iteration all-reduce at camera C/2 and overlap its first half
    // with pass B over the upper half.  It lost on 2 GPUs of another GPU generation (two NCCL launches and two event
    // hand-overs per iteration cost more than the overlap hides); not measured on H100, so it stays off by default.
    const bool split_ar = ctx->world > 1 && use_v2 && !recomp && points_var && C >= 64 &&
                          (getenv("B200SFM_SPLIT_AR") && atoi(getenv("B200SFM_SPLIT_AR")) == 1);
    if (split_ar) ctx->ensure_comm_stream();
    const bool pack_dir = points_var && use_v2 && !recomp;   // direction kernel also packs R^T p for pass A
    PcgResult pr_ = ctx->pcgh.run(
        s, max_it,
        [&]() { B200_LAUNCH(ctx, pcg_init<6>, nblk, kPcgThreads, 0, nbk, Minv.p, bvec.p, px.p, pr.p, pz.p, part_rz, part_rr); },
        [&](int it) {
          double* d_pp = ctx->pcgh.dots(it - 2);
          double* d_pub = ctx->pcgh.dots(it - 1);
          double* d_it = ctx->pcgh.dots(it);
          if (pack_dir) {
            B200_LAUNCH(ctx, ba2_pcg_direction_pack, nblk, kPcgThreads, 0, nbk, nblk, it, o.pcg_min_iterations, o.pcg_rel_tolerance,
                        pz.p, pp.p, yw.p, d_pp, part_rz, part_rr, d_pub, ctl, cam_rec.p, xq.p, C);
            if (kfast) B200_LAUNCH(ctx, ba2k_pack_xk, cdiv(C, 256), 256, 0, C, cam_rec.p, pp.p, xq.p, ctl);
          }
          else
            B200_LAUNCH(ctx, pcg_direction<6>, nblk, kPcgThreads, 0, nbk, nblk, it, o.pcg_min_iterations, o.pcg_rel_tolerance, pz.p,
                        pp.p, yw.p, d_pp, part_rz, part_rr, nullptr, d_pub, ctl);
          if (has_mv) matvec(pp.p, yw.p, o, radius, points_var, split_ar, profile, ctl);
          // extended path: J^T J is inside yw already, only the damping is added here
          B200_LAUNCH(ctx, pcg_apply_diag<6>, nblk, kPcgThreads, 0, nbk, recomp ? nullptr : U(), Dc.p, pp.p, has_mv ? yw.p : nullptr, pq.p,
                      part_pq, ctl);
          B200_LAUNCH(ctx, pcg_update<6>, nblk, kPcgThreads, 0, nbk, nblk, Minv.p, pp.p, pq.p, px.p, pr.p, pz.p, d_pub, part_pq, part_rz,
                      part_rr, d_it, ctl);
        },
        [&](int launched) { B200_LAUNCH(ctx, pcg_finalize, 1, kPcgThreads, 0, nblk, launched, part_rr, ctl); });
    res.finite = pr_.finite;
    // the queued-ahead iterations after the stopping rule fired were no-ops: keep only the real mat-vecs in the timer
    if (profile && has_mv) timer_mv.used = mv_ev0 + 2 * (size_t)std::min(pr_.iters, pr_.launched);
    res.pcg_iters = pr_.iters;
    // ---- back-substitution + candidate ------------------------------------------
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 2, 0, 14 * sizeof(double), s));
    const int nxt = cur ^ 1;
    if (ext) {
      B200_LAUNCH(ctx, bax_update_extras, cdiv(std::max(K + S, 1), 128), 128, 0, ext_view(), ivar.p, intr_model.p, intr.p, intr_cand.p,
                  S > 0 ? sens_q[cur].p : nullptr, S > 0 ? sens_t[cur].p : nullptr, S > 0 ? sens_q[nxt].p : nullptr,
                  S > 0 ? sens_t[nxt].p : nullptr, px.p, gc(), pr.p, Dc.p, jscale_c.p, blk_used.p, 1, scal.p + 8);
    } else {
      B200_CUDA_OK(cudaMemcpyAsync(intr_cand.p, intr.p, intr.bytes(), cudaMemcpyDeviceToDevice, s));
      if (S > 0) {   // the cam_from_rig poses follow `cur` like the frame poses: the candidate buffer mirrors them
        B200_CUDA_OK(cudaMemcpyAsync(sens_q[nxt].p, sens_q[cur].p, sens_q[cur].bytes(), cudaMemcpyDeviceToDevice, s));
        B200_CUDA_OK(cudaMemcpyAsync(sens_t[nxt].p, sens_t[cur].p, sens_t[cur].bytes(), cudaMemcpyDeviceToDevice, s));
      }
    }
    if (points_var && use_v2) {
      const int nrow_part = use_ell ? ell_ctas : n_tiles;
      if (recomp) {
        ExtView ex = ext_view();
#define B200_EXT_A2(WK, WS)                                                                                                  \
  B200_LAUNCH(ctx, (bax_pass_a<2, WK, WS>), ell_ctas, kEllThreads, 0, v, ell_view(), ex, view2(), cam_rec.p, intr_rec.p, px.p, \
              points[cur].p, points[nxt].p, o.thres_loss_function, radius, bpart.p, nullptr)
        if (ext_k && ext_s) B200_EXT_A2(true, true);
        else if (ext_k) B200_EXT_A2(true, false);
        else if (ext_s) B200_EXT_A2(false, true);
        else B200_EXT_A2(false, false);
#undef B200_EXT_A2
      } else {
        B200_LAUNCH(ctx, ba2_pack_x, cdiv(C, 256), 256, 0, C, px.p, cam_rec.p, xq.p);
        if (kfast) B200_LAUNCH(ctx, ba2k_pack_xk, cdiv(C, 256), 256, 0, C, cam_rec.p, px.p, xq.p, nullptr);
        if (use_ell && kfast && nk == 2)
          B200_LAUNCH(ctx, (ba3_pass_a<2, 2>), ell_ctas, kEllThreads, 0, v, ell_view(), view2(), xq.p, points[cur].p, points[nxt].p, radius,
                      bpart.p, nullptr);
        else if (use_ell && kfast)
          B200_LAUNCH(ctx, (ba3_pass_a<2, 1>), ell_ctas, kEllThreads, 0, v, ell_view(), view2(), xq.p, points[cur].p, points[nxt].p, radius,
                      bpart.p, nullptr);
        else if (use_ell)
          B200_LAUNCH(ctx, (ba3_pass_a<2, 0>), ell_ctas, kEllThreads, 0, v, ell_view(), view2(), xq.p, points[cur].p, points[nxt].p, radius,
                      bpart.p, nullptr);
        else
          B200_LAUNCH(ctx, ba2_pass_a<2>, n_tiles, kTile, smem_k3v2, v, view2(), xq.p, points[cur].p, points[nxt].p, radius, bpart.p, nullptr);
      }
      const int nb = std::min(cdiv(nrow_part, 256), 296);
      B200_LAUNCH(ctx, ba2_sum4_stage1, nb, 256, 0, nrow_part, bpart.p, bpart2.p);
      B200_LAUNCH(ctx, ba_colsum, 4, 256, 0, nb, 4, bpart2.p, scal.p + 2);
    } else if (points_var) {
      B200_LAUNCH(ctx, ba_schur_pass<2>, n_tiles, kTile, smem_k3, v, px.p, nullptr, points[cur].p, points[nxt].p, radius,
                  scal.p + 2);
    } else {
      B200_CUDA_OK(cudaMemcpyAsync(points[nxt].p, points[cur].p, points[cur].bytes(), cudaMemcpyDeviceToDevice, s));
    }
    B200_LAUNCH(ctx, ba_update_cams, cdiv(C, 128), 128, 0, C, quat[cur].p, trans[cur].p, px.p, gc(), pr.p, Dc.p, jscale_c.p,
                blk_used.p, cam_mask.p, quat[nxt].p, trans[nxt].p, scal.p + 8);
    build_records(nxt);
    launch_cost(nxt, o.thres_loss_function);
    // bscal[0..3] + cand cost are per-shard partial sums; cscal[8..12] is replicated but summed
    // with atomics (rank-dependent rounding): all-reduce everything and average the replicated
    // part so that every rank takes bit-identical accept/reject decisions.
    ctx->allreduce_sum(scal.p + 2, 11);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal, scal.p, 16 * sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    double* h = ctx->h_scal;
    for (int k = 8; k <= 12; ++k) h[k] /= (double)ctx->world;
    const double g_dot_d = h[8] + h[2];
    const double dDd = h[10] + h[3];
    res.model_cost_change = 0.5 * (-g_dot_d + h[9] + dDd);
    res.cand_cost = h[6];
    res.step_norm = std::sqrt(h[11] + h[4]);
    res.x_norm = std::sqrt(h[12] + h[5]);
    if (!std::isfinite(res.model_cost_change) || !std::isfinite(res.cand_cost)) res.finite = false;
    return res;
  }

  // Which parameter blocks beyond the frame poses are unknowns of a solve with options `o`, and which kernel
  // paths it takes (v1 / v2 tile / ELL, stored-row intrinsics, matrix-free extended); sizes their buffers.
  void select_paths(const b200sfm_ba_opts& o) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    // intrinsics (bundle_adjustment.cc:273-293): optimize_principal_point -> no manifold is set at all, EVERY parameter
    // of every camera is variable; else optimize_intrinsics -> SubsetManifold holding the principal point; else constant
    {
      static const int nfoc[4][3] = {{0, -1, -1}, {0, 1, -1}, {0, 3, -1}, {0, 3, 4}};   // focal + distortion parameter indices
      static const int pp[4][2] = {{1, 2}, {2, 3}, {1, 2}, {1, 2}};                      // principal point indices
      h_ivar.assign(K, b200::IntrVarRec{});
      ext_k = false;
      const bool all_var = o.optimize_principal_point != 0, foc_var = o.optimize_intrinsics != 0 || all_var;
      for (int k = 0; k < K; ++k) {
        std::vector<int> idx;
        if (foc_var)
          for (int j = 0; j < 3; ++j)
            if (nfoc[h_intr_model[k]][j] >= 0) idx.push_back(nfoc[h_intr_model[k]][j]);
        if (all_var) { idx.push_back(pp[h_intr_model[k]][0]); idx.push_back(pp[h_intr_model[k]][1]); }
        std::sort(idx.begin(), idx.end());
        h_ivar[k].col0 = 0;
        h_ivar[k].mb = (int)idx.size();
        for (size_t j = 0; j < idx.size(); ++j) h_ivar[k].pidx[j] = idx[j];
        ext_k = ext_k || !idx.empty();
      }
      B200_CUDA_OK(cudaMemcpyAsync(ivar.p, h_ivar.data(), K * sizeof(b200::IntrVarRec), cudaMemcpyHostToDevice, s));
    }
    // unknown cam_from_rig (optimize_rig_poses, bundle_adjustment.cc:162-180,296-308): the sensors the caller marked
    // (b200sfm_ba_problem_set_sensor_variable; the reference: every non-reference sensor)
    ext_s = false;
    if (o.optimize_rig_poses && S > 0)
      for (int i = 0; i < S; ++i) ext_s = ext_s || h_sensor_var[i] != 0;
    ext = ext_k || ext_s;
    nbk = ext ? CB : C;
    B200_CUDA_OK(cudaStreamSynchronize(s));   // h_ivar upload
    use_v2 = ext || (o.design != 1);          // v1 (W blocks + atomics) only on request, constant intrinsics
    use_ell = use_v2 && (ext || !(getenv("B200SFM_ELL") && atoi(getenv("B200SFM_ELL")) == 0));   // point side: one thread per point
    // intrinsics with <= 2 variable parameters per camera and no unknown cam_from_rig: stored B_o rows instead of the
    // recomputed Jacobians of the extended path (B200SFM_KFAST=0 forces the matrix-free path, for comparison)
    nk = 0;
    if (ext_k)
      for (int k = 0; k < K; ++k) nk = std::max(nk, h_ivar[k].mb);
    // (S == 0: with rigs an image is a (frame, sensor) pair, and the cross block / x_k packing below are per frame)
    kfast = ext_k && !ext_s && S == 0 && nk <= 2 && !(getenv("B200SFM_KFAST") && atoi(getenv("B200SFM_KFAST")) == 0);
    if (kfast) {
      const size_t cells = (size_t)std::max<long long>(ell_rows, 1) * 32;
      if (ell_B.n < cells * 3 * nk) ell_B.alloc(cells * 3 * nk);
      if (Ufk.n < (size_t)C * 6 * nk) Ufk.alloc((size_t)C * 6 * nk);
    }
  }
  // effective per-camera mask: the caller's mask | optimize_rotations / optimize_translation off
  void launch_eff_mask(const b200sfm_ba_opts& o) {
    B200_LAUNCH(ctx, b200::k_eff_mask, b200::cdiv(C, 256), 256, 0, C, cam_mask_base.p, o.optimize_rotations ? 0 : 1,
                o.optimize_translation ? 0 : 1, cam_mask.p);
  }

  // A step that is not accepted: compute_step ended by building the records of the candidate (for its cost); the next
  // step works on the same linearisation, whose stored rows and Jacobians belong to the current state's records (and
  // the camera-order kernels rebuild A_o from those records and pts4, which still holds points[cur]).
  void reject_step() { build_records(cur); }

  // The LM loop, Ceres order of checks (see oracle/ceres_lm.py).
  int solve(const b200sfm_ba_opts& o, b200sfm_lm_stats* st) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    select_paths(o);
    // v2: keep z4 (written by pass A, gathered by pass B) in the persisting part of L2 when it fits there
    const bool l2_persist = use_v2 && !(getenv("B200SFM_L2_PERSIST") && atoi(getenv("B200SFM_L2_PERSIST")) == 0) &&
                            l2_persist_window(s, ctx->device, z4.p, z4.bytes());
    const long long launches0 = ctx->launches;
    timer_lin.reset();
    timer_mv.reset();
    cudaEvent_t ev0, ev1;
    B200_CUDA_OK(cudaEventCreate(&ev0));
    B200_CUDA_OK(cudaEventCreate(&ev1));
    B200_CUDA_OK(cudaEventRecord(ev0, s));
    const bool points_var = o.optimize_points != 0;
    const bool profile = o.profile_kernels != 0;
    launch_eff_mask(o);
    double cost = 0, gmax = 0;
    linearize(o.thres_loss_function, points_var, true, profile, cost, gmax);
    b200sfm_lm_stats local{};
    local.initial_cost = cost;
    local.usable = 1;
    local.num_observations = n_obs_used;
    double radius = 1e4, decrease = 2.0;
    int invalid = 0, it = 0, term = B200SFM_TERM_NONE;
    bool set_jscale_p = true;
    const bool fixed = o.fixed_num_iterations > 0;
    const int max_it = fixed ? o.fixed_num_iterations : o.max_num_iterations;
    if (!fixed && gmax <= o.gradient_tolerance) term = B200SFM_TERM_GRADIENT_TOLERANCE;
    while (term == B200SFM_TERM_NONE) {
      if (it >= max_it) { term = B200SFM_TERM_MAX_ITERATIONS; break; }
      if (radius < 1e-32) { term = B200SFM_TERM_MIN_RADIUS; break; }
      ++it;
      StepResult r = compute_step(o, radius, points_var, set_jscale_p, profile);
      set_jscale_p = false;
      local.pcg_iterations += r.pcg_iters;
      if (!r.finite || !(r.model_cost_change > 0.0)) {
        if (++invalid >= 5) { term = B200SFM_TERM_INVALID_STEPS; local.usable = 0; break; }
        reject_step();
        radius /= decrease;
        decrease *= 2;
        continue;
      }
      invalid = 0;
      if (!fixed) {
        if (r.step_norm <= o.parameter_tolerance * (r.x_norm + o.parameter_tolerance)) { term = B200SFM_TERM_PARAMETER_TOLERANCE; break; }
        if (std::fabs(cost - r.cand_cost) <= o.function_tolerance * cost) { term = B200SFM_TERM_FUNCTION_TOLERANCE; break; }
      }
      const double rel = (cost - r.cand_cost) / r.model_cost_change;
      if (rel > 1e-3) {
        cur ^= 1;
        std::swap(intr.p, intr_cand.p);   // the candidate intrinsics become current (buffers have equal size)
        ++local.num_successful_steps;
        linearize(o.thres_loss_function, points_var, false, profile, cost, gmax);
        radius = std::min(1e16, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rel - 1.0, 3)));
        decrease = 2.0;
        if (!fixed && gmax <= o.gradient_tolerance) { term = B200SFM_TERM_GRADIENT_TOLERANCE; break; }
      } else {
        reject_step();
        radius /= decrease;
        decrease *= 2;
      }
    }
    B200_CUDA_OK(cudaEventRecord(ev1, s));
    B200_CUDA_OK(cudaEventSynchronize(ev1));
    if (l2_persist) l2_persist_clear(s);
    float ms = 0;
    B200_CUDA_OK(cudaEventElapsedTime(&ms, ev0, ev1));
    cudaEventDestroy(ev0);
    cudaEventDestroy(ev1);
    local.iterations = it;
    local.termination = term;
    local.final_cost = cost;
    local.ms_total = ms;
    for (size_t i = 0; i + 1 < timer_lin.used; i += 2) {
      float t;
      B200_CUDA_OK(cudaEventElapsedTime(&t, timer_lin.ev[i], timer_lin.ev[i + 1]));
      local.ms_linearize += t;
      ++local.n_linearize;
    }
    for (size_t i = 0; i + 1 < timer_mv.used; i += 2) {
      float t;
      B200_CUDA_OK(cudaEventElapsedTime(&t, timer_mv.ev[i], timer_mv.ev[i + 1]));
      local.ms_matvec += t;
      ++local.n_matvec;
    }
    local.kernel_launches = ctx->launches - launches0;
    if (st) {
      local.h2d_bytes = st->h2d_bytes; local.d2h_bytes = st->d2h_bytes; local.ms_h2d = st->ms_h2d; local.ms_d2h = st->ms_d2h;
      local.kernel_launches += st->kernel_launches;
      *st = local;
    }
    return B200SFM_OK;
  }

  // ---- test probe (include/b200sfm_testing.h) ----------------------------------------------------------------------
  b200sfm_ba_opts probe_opts{};
  double probe_radius = 0;
  bool probe_ready = false;

  // the first LM iteration of solve() up to the candidate and its cost, without accepting it; with first_radius > 0 the
  // step at `radius` is the second one, after a step at first_radius that was not accepted (same linearisation)
  void test_step(const b200sfm_ba_opts& o, double first_radius, double radius, b200sfm_test_ba_step_out* out) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    select_paths(o);
    launch_eff_mask(o);
    const bool points_var = o.optimize_points != 0;
    double cost = 0, gmax = 0;
    linearize(o.thres_loss_function, points_var, true, false, cost, gmax);
    if (first_radius > 0.0) {
      compute_step(o, first_radius, points_var, true, false);
      reject_step();
    }
    const StepResult r = compute_step(o, radius, points_var, !(first_radius > 0.0), false);
    reject_step();
    probe_opts = o;
    probe_radius = radius;
    probe_ready = true;
    const int nxt = cur ^ 1;
    const size_t nb6 = (size_t)nbk * 6;
    if (out->U) B200_CUDA_OK(cudaMemcpyAsync(out->U, U(), (size_t)nbk * 21 * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (out->g_c) B200_CUDA_OK(cudaMemcpyAsync(out->g_c, gc(), nb6 * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (out->jscale_c) jscale_c.download(out->jscale_c, nb6, s);
    if (out->V) V.download(out->V, (size_t)P * 6, s);
    if (out->g_p) gp.download(out->g_p, (size_t)P * 3, s);
    if (out->jscale_p) jscale_p.download(out->jscale_p, (size_t)P * 3, s);
    if (out->Dc) Dc.download(out->Dc, nb6, s);
    if (out->Minv) Minv.download(out->Minv, (size_t)nbk * 21, s);
    if (out->b) bvec.download(out->b, nb6, s);
    if (out->px) px.download(out->px, nb6, s);
    if (out->cand_points) points[nxt].download(out->cand_points, (size_t)P * 3, s);
    if (out->cand_quat) quat[nxt].download(out->cand_quat, (size_t)C * 4, s);
    if (out->cand_trans) trans[nxt].download(out->cand_trans, (size_t)C * 3, s);
    if (out->cand_intr) intr_cand.download(out->cand_intr, (size_t)K * B200SFM_INTR_STRIDE, s);
    if (S > 0 && out->cand_sensor_quat) sens_q[nxt].download(out->cand_sensor_quat, (size_t)S * 4, s);
    if (S > 0 && out->cand_sensor_trans) sens_t[nxt].download(out->cand_sensor_trans, (size_t)S * 3, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    out->cost = cost;
    out->gmax = gmax;
    out->model_cost_change = r.model_cost_change;
    out->cand_cost = r.cand_cost;
    out->step_norm = r.step_norm;
    out->x_norm = r.x_norm;
    out->pcg_iterations = r.pcg_iters;
    out->use_v2 = use_v2; out->use_ell = use_ell; out->kfast = kfast; out->nk = nk;
    out->ext = ext; out->ext_k = ext_k; out->ext_s = ext_s;
    out->schur_jacobi = schur_jacobi_on(o, points_var);
    out->nbk = nbk;
  }

  // y = (S + D) x at the linearisation and damping of the last test_step, through the mat-vec chain of a PCG iteration
  void test_apply(const double* h_x, double* h_y) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    const bool points_var = probe_opts.optimize_points != 0;
    const int nblk = cdiv(nbk, kPcgThreads);
    PcgCtl* ctl = ctx->pcgh.d_ctl;
    B200_CUDA_OK(cudaMemsetAsync(ctl, 0, sizeof(PcgCtl), s));   // every kernel of the chain returns early once ctl->done is set
    pp.upload(h_x, (size_t)nbk * 6, s);
    yw.zero(s);
    if (points_var && use_v2 && !matrix_free()) {   // what ba2_pcg_direction_pack does inside PCG
      B200_LAUNCH(ctx, ba2_pack_x, cdiv(C, 256), 256, 0, C, pp.p, cam_rec.p, xq.p);
      if (kfast) B200_LAUNCH(ctx, ba2k_pack_xk, cdiv(C, 256), 256, 0, C, cam_rec.p, pp.p, xq.p, ctl);
    }
    const bool has_mv = points_var || ext;
    if (has_mv) matvec(pp.p, yw.p, probe_opts, probe_radius, points_var, false, false, ctl);
    B200_LAUNCH(ctx, pcg_apply_diag<6>, nblk, kPcgThreads, 0, nbk, matrix_free() ? nullptr : U(), Dc.p, pp.p,
                has_mv ? yw.p : nullptr, pq.p, ctx->pcgh.d_part, ctl);
    pq.download(h_y, (size_t)nbk * 6, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }
};
