// gp_solver.cuh -- host-side driver of the device global positioner: problem
// residency and the Ceres-semantics LM loop with box bounds on the scales
// (projection in Plus + projected Armijo line search; restated in
// oracle/ceres_lm.py).  Reference path replaced:
// glomap/estimators/global_positioning.cc:28-93 (the ceres::Solve at :83).
#pragma once
#include "ba_solver.cuh"
#include "gp_kernels.cuh"

struct b200sfm_gp_problem {
  template <class T>
  using DevBuf = b200::DevBuf<T>;
  using GPView = b200::GPView;

  b200sfm_ctx* ctx = nullptr;
  int C = 0, P = 0;
  long long N = 0, n_obs_used = 0, first_valid_obs = -1;
  int Nv = 0, n_tiles = 0, n_segs = 0, min_views = 3;
  DevBuf<int> obs_cam, obs_pt, tile_pt_begin, camord_obs, pt_c, seg_cam, seg_begin, seg_end;
  DevBuf<unsigned> pt_begin;
  DevBuf<double> obs_dir, obs_off;
  DevBuf<unsigned char> obs_cal;
  DevBuf<unsigned char> calibrated, cam_const_base, cam_const;
  bool has_calibrated = false;
  // unknown cam_from_rig centres (RigUnknownBATA): S_u pseudo-camera blocks behind the C frames; CB = C + S_u
  int n_us = 0, CB = 0;
  DevBuf<int> obs_us;
  DevBuf<double> frame_rot, ucen[2], ucen_saved, off_static, off_dyn;
  // state / candidate / snapshot
  DevBuf<double> centers[2], points[2], scales[2], centers_saved, points_saved, scales_saved;
  int cur = 0;
  DevBuf<double> cen4;
  // linear system
  DevBuf<double> M, bw, graw, jscale_s, Vinv, gX, Dp, jscale_p, out16, U, gc, Dc, Minv, jscale_c;
  DevBuf<double> px, pr, pz, pp, pq, yw, bvec, dX, ds, scal;
  b200::EventTimer timer_lin, timer_mv;
  size_t smem_g1 = 0, smem_g3 = 0;

  GPView view(bool scales_var) {
    GPView v;
    v.C = C; v.P = P; v.N = N; v.n_tiles = n_tiles; v.n_segs = n_segs; v.min_views = min_views;
    v.const_obs = (ctx->rank == 0) ? first_valid_obs : -1;
    v.scales_var = scales_var ? 1 : 0;
    v.obs_cam = obs_cam.p; v.obs_pt = obs_pt.p; v.obs_dir = obs_dir.p; v.pt_begin = pt_begin.p;
    v.obs_off = n_us > 0 ? off_dyn.p : obs_off.p; v.obs_cal = obs_cal.p;
    v.n_us = n_us; v.obs_us = obs_us.p; v.frame_rot = frame_rot.p;
    v.tile_pt_begin = tile_pt_begin.p; v.camord_obs = camord_obs.p; v.pt_c = pt_c.p;
    v.seg_cam = seg_cam.p; v.seg_begin = seg_begin.p; v.seg_end = seg_end.p;
    v.M = M.p; v.bw = bw.p; v.jscale_s = jscale_s.p; v.Vinv = Vinv.p; v.gX = gX.p; v.Dp = Dp.p; v.jscale_p = jscale_p.p;
    v.graw = graw.p;
    return v;
  }

  // known rigs: constant per-observation offset (and the camera's prior-focal flag); nullptr clears
  void set_rig_terms(const double* h_off, const uint8_t* h_cal) {
    cudaStream_t s = ctx->stream;
    if (h_off) { obs_off.alloc((size_t)N * 3); obs_off.upload(h_off, (size_t)N * 3, s); }
    else obs_off.release();
    if (h_cal) { obs_cal.alloc(N); obs_cal.upload(h_cal, N, s); }
    else obs_cal.release();
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }

  // unknown cam_from_rig: h_obs_us[N] (-1: the observing image's sensor is the reference sensor / calibrated),
  // h_frame_rot[C][9] rig_from_world rotations, h_ucen[S_u][3] initial centres.  Re-sizes the camera-block arrays.
  void set_rig_unknown(int S_u, const int32_t* h_obs_us, const double* h_frame_rot, const double* h_ucen) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    n_us = S_u;
    CB = C + n_us;
    obs_us.alloc(N); obs_us.upload(h_obs_us, N, s);
    frame_rot.alloc((size_t)C * 9); frame_rot.upload(h_frame_rot, (size_t)C * 9, s);
    for (int i = 0; i < 2; ++i) ucen[i].alloc((size_t)n_us * 3);
    ucen[cur].upload(h_ucen, (size_t)n_us * 3, s);
    off_dyn.alloc((size_t)N * 3);
    alloc_blocks();
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }
  void get_rig_unknown(double* h_ucen) {
    ucen[cur].download(h_ucen, (size_t)n_us * 3, ctx->stream);
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
  }
  // fold -R_rw^T u_s of state `which` into the per-observation offsets
  void dyn_offsets(int which) {
    using namespace b200;
    if (n_us > 0)
      B200_LAUNCH(ctx, gp_dyn_offsets, cdiv(N, 256), 256, 0, N, obs_cam.p, obs_us.p, frame_rot.p, ucen[which].p,
                  obs_off.p /* static known-rig offsets or nullptr */, off_dyn.p);
  }
  // per-block arrays of the reduced system (CB blocks of 3)
  void alloc_blocks() {
    cudaStream_t s = ctx->stream;
    out16.alloc((size_t)CB * b200::kOutW + 1 + (size_t)ctx->world);   // per block kOutW | cost | one max|g| slot per rank
    U.alloc((size_t)CB * 6); gc.alloc((size_t)CB * 3); Dc.alloc((size_t)CB * 3);
    Minv.alloc((size_t)CB * 6); jscale_c.alloc(CB);
    px.alloc((size_t)CB * 3); pr.alloc((size_t)CB * 3); pz.alloc((size_t)CB * 3); pp.alloc((size_t)CB * 3);
    pq.alloc((size_t)CB * 3); yw.alloc((size_t)CB * 3); bvec.alloc((size_t)CB * 3);
    cam_const.alloc(CB);   // [0, C): frames (k_eff_mask); the unknown-sensor blocks are always variable (.cc:440-453)
    cam_const.zero(s);
  }

  void create(b200sfm_ctx* c, int C_, int P_, long long N_, const int64_t* h_pt_begin, const int32_t* h_obs_cam,
              const double* h_obs_dir, const uint8_t* h_calibrated, const uint8_t* h_cam_const, int min_views_) {
    using namespace b200;
    ctx = c; C = C_; P = P_; N = N_; min_views = min_views_;
    cudaStream_t s = ctx->stream;
    std::vector<unsigned> ptb((size_t)P + 1);
    std::vector<int> tiles;
    tiles.reserve((size_t)(N / 100) + 16);
    tiles.push_back(0);
    long long tile_obs = 0;
    int tile_pts = 0;
    n_obs_used = 0;
    first_valid_obs = -1;
    for (int p = 0; p < P; ++p) {
      ptb[p] = (unsigned)h_pt_begin[p];
      const long long len = h_pt_begin[p + 1] - h_pt_begin[p];
      if (len < 0) throw InvalidInput{"pt_obs_begin must be non-decreasing"};
      if (len >= min_views) {
        if (first_valid_obs < 0) first_valid_obs = h_pt_begin[p];
        n_obs_used += len;
      }
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
    obs_cam.alloc(N); obs_pt.alloc(N); obs_dir.alloc((size_t)N * 3); pt_begin.alloc((size_t)P + 1);
    tile_pt_begin.alloc(tiles.size()); calibrated.alloc(C); cam_const_base.alloc(C);
    obs_cam.upload(h_obs_cam, N, s);
    obs_dir.upload(h_obs_dir, (size_t)N * 3, s);
    pt_begin.upload(ptb.data(), (size_t)P + 1, s);
    tile_pt_begin.upload(tiles.data(), tiles.size(), s);
    has_calibrated = h_calibrated != nullptr;
    if (h_calibrated) calibrated.upload(h_calibrated, C, s);
    if (h_cam_const) cam_const_base.upload(h_cam_const, C, s);
    else cam_const_base.zero(s);
    B200_LAUNCH(ctx, k_expand_obs_pt, cdiv(P, 256), 256, 0, P, pt_begin.p, obs_pt.p);
    DevBuf<int> keys, vals, keys_out, cam_count, seg_count, cam_begin, seg_off, bad;
    keys.alloc(N); vals.alloc(N); keys_out.alloc(N); camord_obs.alloc(N);
    cam_count.alloc((size_t)C + 1); seg_count.alloc((size_t)C + 1); cam_begin.alloc((size_t)C + 1); seg_off.alloc((size_t)C + 1);
    bad.alloc(1);
    cam_count.zero(s); seg_count.zero(s); bad.zero(s);
    // plain camera order: one point slice, no camera halves (keys = camera)
    B200_LAUNCH(ctx, k_cam_keys, cdiv(N, 256), 256, 0, N, C, 1, min_views, std::max(P, 1), 1, C, C, obs_cam.p, nullptr, obs_pt.p,
                pt_begin.p, keys.p, vals.p, cam_count.p, bad.p);
    int end_bit = 1;
    while ((1ll << end_bit) <= C) ++end_bit;
    size_t tmp_bytes = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys.p, keys_out.p, vals.p, camord_obs.p, (int)N, 0, end_bit, s);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cam_count.p, cam_begin.p, C + 1, s);
    DevBuf<unsigned char> tmp;
    tmp.alloc(std::max(tmp_bytes, scan_bytes) + 16);
    size_t tb = tmp.bytes();
    cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.p, keys_out.p, vals.p, camord_obs.p, (int)N, 0, end_bit, s);
    tb = tmp.bytes();
    cub::DeviceScan::ExclusiveSum(tmp.p, tb, cam_count.p, cam_begin.p, C + 1, s);
    B200_LAUNCH(ctx, k_seg_counts, cdiv(C, 256), 256, 0, C, cam_count.p, seg_count.p);
    tb = tmp.bytes();
    cub::DeviceScan::ExclusiveSum(tmp.p, tb, seg_count.p, seg_off.p, C + 1, s);
    ctx->launches += 12;
    int h_tot[3];
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[0], cam_begin.p + C, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[1], seg_off.p + C, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[2], bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    if (h_tot[2]) throw InvalidInput{"obs_cam out of range [0, C)"};
    Nv = h_tot[0];
    n_segs = h_tot[1];
    seg_cam.alloc(std::max(n_segs, 1)); seg_begin.alloc(std::max(n_segs, 1)); seg_end.alloc(std::max(n_segs, 1));
    pt_c.alloc(std::max(Nv, 1));
    B200_LAUNCH(ctx, k_fill_segs, cdiv(C, 256), 256, 0, C, C, 1, cam_begin.p, seg_off.p, nullptr, nullptr, seg_cam.p, nullptr, nullptr,
                seg_begin.p, seg_end.p);
    if (Nv > 0) B200_LAUNCH(ctx, k_gather_int, cdiv(Nv, 256), 256, 0, Nv, camord_obs.p, obs_pt.p, pt_c.p);
    for (int i = 0; i < 2; ++i) {
      centers[i].alloc((size_t)C * 3); points[i].alloc((size_t)P * 3); scales[i].alloc(N);
    }
    cen4.alloc((size_t)C * 4);
    M.alloc((size_t)N * kMDoubles); bw.alloc((size_t)N * 4); graw.alloc((size_t)N * 3); jscale_s.alloc(N);
    Vinv.alloc((size_t)P * 6); gX.alloc((size_t)P * 3); Dp.alloc(P); jscale_p.alloc(P);
    CB = C;
    alloc_blocks();
    dX.alloc((size_t)P * 3); ds.alloc(N); scal.alloc(16);
    smem_g1 = sizeof(G1Smem) + 128;
    smem_g3 = sizeof(G3Smem) + 128;
    const int carve = (int)cudaSharedmemCarveoutMaxShared;
    B200_CUDA_OK(cudaFuncSetAttribute(gp_linearize_points, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g1));
    B200_CUDA_OK(cudaFuncSetAttribute(gp_linearize_points, cudaFuncAttributePreferredSharedMemoryCarveout, carve));
    B200_CUDA_OK(cudaFuncSetAttribute(gp_schur_pass<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g3));
    B200_CUDA_OK(cudaFuncSetAttribute((gp_schur_pass<0, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g3));
    B200_CUDA_OK(cudaFuncSetAttribute(gp_schur_pass<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g3));
    B200_CUDA_OK(cudaFuncSetAttribute(gp_schur_pass<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_g3));
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }

  void set_state(const double* h_centers, const double* h_points, const double* h_scales) {
    cudaStream_t s = ctx->stream;
    centers[cur].upload(h_centers, (size_t)C * 3, s);
    points[cur].upload(h_points, (size_t)P * 3, s);
    scales[cur].upload(h_scales, N, s);
  }
  void get_state(double* h_centers, double* h_points, double* h_scales) {
    cudaStream_t s = ctx->stream;
    if (h_centers) centers[cur].download(h_centers, (size_t)C * 3, s);
    if (h_points) points[cur].download(h_points, (size_t)P * 3, s);
    if (h_scales) scales[cur].download(h_scales, N, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }
  void save_state() {
    cudaStream_t s = ctx->stream;
    if (!centers_saved.p) { centers_saved.alloc((size_t)C * 3); points_saved.alloc((size_t)P * 3); scales_saved.alloc(N); }
    B200_CUDA_OK(cudaMemcpyAsync(centers_saved.p, centers[cur].p, centers_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(points_saved.p, points[cur].p, points_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(scales_saved.p, scales[cur].p, scales_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    if (n_us > 0) {
      if (!ucen_saved.p) ucen_saved.alloc((size_t)n_us * 3);
      B200_CUDA_OK(cudaMemcpyAsync(ucen_saved.p, ucen[cur].p, ucen_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    }
  }
  bool restore_state() {
    if (!centers_saved.p) return false;
    cudaStream_t s = ctx->stream;
    B200_CUDA_OK(cudaMemcpyAsync(centers[cur].p, centers_saved.p, centers_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(points[cur].p, points_saved.p, points_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(scales[cur].p, scales_saved.p, scales_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    if (n_us > 0 && ucen_saved.p)
      B200_CUDA_OK(cudaMemcpyAsync(ucen[cur].p, ucen_saved.p, ucen_saved.bytes(), cudaMemcpyDeviceToDevice, s));
    return true;
  }

  double eval_cost(int which, const GPView& v, double huber_a) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    B200_LAUNCH(ctx, gp_build_records, cdiv(C, 256), 256, 0, C, centers[which].p, has_calibrated ? calibrated.p : nullptr, cen4.p);
    dyn_offsets(which);
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 6, 0, sizeof(double), s));
    const int grid = std::min(cdiv(N, 256), ctx->num_sms * 8);
    B200_LAUNCH(ctx, gp_cost, grid, 256, 0, v, cen4.p, points[which].p, scales[which].p, huber_a, scal.p + 6);
    ctx->allreduce_sum(scal.p + 6, 1);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal + 32, scal.p + 6, sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return ctx->h_scal[32];
  }

  struct StepResult {
    double cost = 0, gmax = 0, model_cost_change = 0, g_dot_delta = 0;
    int pcg_iters = 0;
    bool finite = true;
  };

  // Linearise at the current state with damping `radius`, solve for the step
  // (dc in px, dX, ds).  Everything is recomputed: M_o depends on the radius
  // through the eliminated scale's damping.
  StepResult compute_step(const b200sfm_gp_opts& o, const GPView& v, double radius, bool first, bool points_var,
                          bool profile) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    const int nC3 = CB * 3;   // frames + unknown-sensor blocks
    B200_LAUNCH(ctx, gp_build_records, cdiv(C, 256), 256, 0, C, centers[cur].p, has_calibrated ? calibrated.p : nullptr, cen4.p);
    dyn_offsets(cur);
    B200_CUDA_OK(cudaMemsetAsync(scal.p, 0, 16 * sizeof(double), s));
    out16.zero(s);
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (profile) {
      e0 = timer_lin.next(); e1 = timer_lin.next();
      B200_CUDA_OK(cudaEventRecord(e0, s));
    }
    B200_LAUNCH(ctx, gp_linearize_points, n_tiles, kTile, smem_g1, v, cen4.p, points[cur].p, scales[cur].p,
                o.thres_loss_function, radius, first ? 1 : 0, points_var ? 1 : 0, scal.p);
    if (profile) B200_CUDA_OK(cudaEventRecord(e1, s));
    // Schur-Jacobi blocks only without unknown sensors (their frame / sensor cross terms are not block diagonal)
    const bool schur_jacobi = points_var && o.preconditioner == 1 && n_us == 0;
    if (n_segs > 0)
      B200_LAUNCH(ctx, gp_linearize_cams, cdiv((long long)n_segs * 32, 128), 128, 0, v, schur_jacobi ? 1 : 0, out16.p);
    if (n_us > 0) B200_LAUNCH(ctx, gp_linearize_sensors, cdiv(N, 256), 256, 0, v, out16.p);
    // cost and this rank's max|g_X| (own slot) travel with the camera blocks through ONE sum all-reduce
    B200_CUDA_OK(cudaMemcpyAsync(out16.p + (size_t)CB * b200::kOutW, scal.p, sizeof(double), cudaMemcpyDeviceToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(out16.p + (size_t)CB * b200::kOutW + 1 + ctx->rank, scal.p + 1, sizeof(double), cudaMemcpyDeviceToDevice, s));
    ctx->allreduce_sum(out16.p, (size_t)CB * b200::kOutW + 1 + (size_t)ctx->world);
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 1, 0, sizeof(double), s));
    B200_LAUNCH(ctx, gp_finalize_cams, cdiv(CB, 128), 128, 0, CB, out16.p, cam_const.p, jscale_c.p, first ? 1 : 0, radius,
                schur_jacobi ? 1 : 0, U.p, gc.p, Dc.p, Minv.p, scal.p, out16.p + (size_t)CB * b200::kOutW + 1, ctx->world);
    // rhs  (constant points have Vinv = 0 from G1, so the same passes apply)
    {
      yw.zero(s);
      B200_LAUNCH(ctx, gp_schur_pass<1>, n_tiles, kTile, smem_g3, v, nullptr, yw.p, nullptr, nullptr, nullptr, 0.0, radius,
                  nullptr, nullptr, nullptr);
      ctx->allreduce_sum(yw.p, nC3);
    }
    // constant blocks (jscale_c < 0) are identity rows with b = 0, here and in pcg_apply_diag: PCG leaves their dc at 0,
    // so the back-substitution and the step scalars see the reduced program without them
    B200_LAUNCH(ctx, k_rhs, cdiv(nC3, 256), 256, 0, nC3, gc.p, yw.p, bvec.p, jscale_c.p, 3);
    // PCG (3x3 blocks; loop control on the device, pcg.cuh)
    const int max_it = std::max(1, o.pcg_max_iterations);
    const int nblk = cdiv(CB, kPcgThreads);
    ctx->pcgh.ensure(max_it, (size_t)nblk * 3, ctx->world);
    double *part_pq = ctx->pcgh.d_part, *part_rz = ctx->pcgh.d_part + nblk, *part_rr = ctx->pcgh.d_part + 2 * (size_t)nblk;
    PcgCtl* ctl = ctx->pcgh.d_ctl;
    StepResult res;
    const size_t mv_ev0 = timer_mv.used;
    PcgResult pr_ = ctx->pcgh.run(
        s, max_it,
        [&]() { B200_LAUNCH(ctx, pcg_init<3>, nblk, kPcgThreads, 0, CB, Minv.p, bvec.p, px.p, pr.p, pz.p, part_rz, part_rr); },
        [&](int it) {
          double* d_pub = ctx->pcgh.dots(it - 1);
          B200_LAUNCH(ctx, pcg_direction<3>, nblk, kPcgThreads, 0, CB, nblk, it, o.pcg_min_iterations, o.pcg_rel_tolerance, pz.p,
                      pp.p, yw.p, ctx->pcgh.dots(it - 2), part_rz, part_rr, nullptr, d_pub, ctl);
          matvec(v, pp.p, yw.p, part_pq, ctl, profile);
          B200_LAUNCH(ctx, pcg_update<3>, nblk, kPcgThreads, 0, CB, nblk, Minv.p, pp.p, pq.p, px.p, pr.p, pz.p, d_pub, part_pq,
                      part_rz, part_rr, ctx->pcgh.dots(it), ctl);
        },
        [&](int launched) { B200_LAUNCH(ctx, pcg_finalize, 1, kPcgThreads, 0, nblk, launched, part_rr, ctl); });
    if (profile) timer_mv.used = mv_ev0 + 2 * (size_t)std::min(pr_.iters, pr_.launched);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal + 8, out16.p + (size_t)CB * b200::kOutW, sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal + 9, scal.p + 1, sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    res.cost = ctx->h_scal[8];
    res.gmax = ctx->h_scal[9];
    res.finite = pr_.finite;
    const int it = pr_.iters;
    res.pcg_iters = it;
    // back-substitution (dX, ds) + step scalars
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 2, 0, 14 * sizeof(double), s));
    B200_LAUNCH(ctx, gp_schur_pass<2>, n_tiles, kTile, smem_g3, v, px.p, nullptr, cen4.p, points[cur].p, scales[cur].p,
                o.thres_loss_function, radius, dX.p, ds.p, scal.p + 2);
    B200_LAUNCH(ctx, gp_cam_scalars, cdiv(nC3, 256), 256, 0, CB, px.p, pr.p, Dc.p, jscale_c.p, scal.p + 8);
    ctx->allreduce_sum(scal.p + 2, 8);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal, scal.p, 16 * sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    double* h = ctx->h_scal;
    h[8] /= ctx->world;
    h[9] /= ctx->world;
    const double g_dot = h[2];
    res.g_dot_delta = g_dot;
    res.model_cost_change = 0.5 * (-g_dot + h[8] + h[3] + h[9]);
    if (!std::isfinite(res.model_cost_change)) res.finite = false;
    return res;
  }

  // q = (S + D) p through the kernels of one PCG iteration: the implicit Schur pass (the SPEC variant when iterations
  // are queued ahead of the read-back), the all-reduce, then the block diagonal.  y must be zero on entry; the pass
  // accumulates into it.  Constant blocks (jscale_c < 0) are identity rows.
  void matvec(const GPView& v, const double* p, double* y, double* part_pq, const b200::PcgCtl* ctl, bool profile) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    cudaEvent_t m0 = nullptr, m1 = nullptr;
    if (profile) {
      m0 = timer_mv.next(); m1 = timer_mv.next();
      B200_CUDA_OK(cudaEventRecord(m0, s));
    }
    if (ctx->pcgh.depth > 1)   // iterations are queued ahead of the read-back: the pass tests the stopping flag
      B200_LAUNCH(ctx, (gp_schur_pass<0, true>), n_tiles, kTile, smem_g3, v, p, y, nullptr, nullptr, nullptr, 0.0, 0.0,
                  nullptr, nullptr, nullptr, ctl);
    else
      B200_LAUNCH(ctx, gp_schur_pass<0>, n_tiles, kTile, smem_g3, v, p, y, nullptr, nullptr, nullptr, 0.0, 0.0,
                  nullptr, nullptr, nullptr, nullptr);
    if (profile) B200_CUDA_OK(cudaEventRecord(m1, s));
    ctx->allreduce_sum(y, (size_t)CB * 3);
    // unknown sensors: the pass already applied the direct term per observation (A = nullptr)
    B200_LAUNCH(ctx, pcg_apply_diag<3>, cdiv(CB, kPcgThreads), kPcgThreads, 0, CB, n_us > 0 ? nullptr : U.p, Dc.p, p, y, pq.p,
                part_pq, ctl, jscale_c.p);
  }

  // candidate = Project(x + alpha delta) into the other buffer; returns (cost, step_norm, x_norm)
  void make_candidate(const GPView& v, double alpha, double huber_a, bool points_var, double& cand_cost, double& step_norm,
                      double& x_norm) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    const int nxt = cur ^ 1;
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 12, 0, 2 * sizeof(double), s));
    const long long nthreads = std::max<long long>(N, std::max<long long>((long long)P * 3, (long long)CB * 3));
    B200_LAUNCH(ctx, gp_apply_step, cdiv(nthreads, 256), 256, 0, v, alpha, centers[cur].p, points[cur].p, scales[cur].p, px.p,
                dX.p, ds.p, jscale_c.p, ctx->rank == 0 ? 1 : 0, points_var ? 1 : 0, centers[nxt].p, points[nxt].p, scales[nxt].p, scal.p + 12,
                n_us > 0 ? ucen[cur].p : nullptr, n_us > 0 ? ucen[nxt].p : nullptr);
    cand_cost = eval_cost(nxt, v, huber_a);
    // points/scales norms are per-shard, camera norms replicated: reduce the former only approximately matters
    ctx->allreduce_sum(scal.p + 12, 2);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal + 40, scal.p + 12, 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    step_norm = std::sqrt(ctx->h_scal[40]);
    x_norm = std::sqrt(ctx->h_scal[41]);
  }

  int solve(const b200sfm_gp_opts& o, b200sfm_lm_stats* st) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    const long long launches0 = ctx->launches;
    timer_lin.reset();
    timer_mv.reset();
    cudaEvent_t ev0, ev1;
    B200_CUDA_OK(cudaEventCreate(&ev0));
    B200_CUDA_OK(cudaEventCreate(&ev1));
    B200_CUDA_OK(cudaEventRecord(ev0, s));
    const bool points_var = o.optimize_points != 0;
    const bool scales_var = o.optimize_scales != 0;
    const bool profile = o.profile_kernels != 0;
    B200_LAUNCH(ctx, k_eff_mask, cdiv(C, 256), 256, 0, C, cam_const_base.p, o.optimize_positions ? 0 : 1, 0, cam_const.p);
    GPView v = view(scales_var);
    b200sfm_lm_stats local{};
    local.usable = 1;
    local.num_observations = n_obs_used;
    double radius = 1e4, decrease = 2.0;
    int invalid = 0, it = 0, term = B200SFM_TERM_NONE;
    const bool fixed = o.fixed_num_iterations > 0;
    const int max_it = fixed ? o.fixed_num_iterations : o.max_num_iterations;
    bool first = true;
    double cost = 0;
    while (term == B200SFM_TERM_NONE) {
      if (it >= max_it) { term = B200SFM_TERM_MAX_ITERATIONS; break; }
      if (radius < 1e-32) { term = B200SFM_TERM_MIN_RADIUS; break; }
      StepResult r = compute_step(o, v, radius, first, points_var, profile);
      cost = r.cost;
      if (first) local.initial_cost = cost;
      first = false;
      local.pcg_iterations += r.pcg_iters;
      if (!fixed && r.gmax <= o.gradient_tolerance) { term = B200SFM_TERM_GRADIENT_TOLERANCE; break; }
      ++it;
      if (!r.finite || !(r.model_cost_change > 0.0)) {
        if (++invalid >= 5) { term = B200SFM_TERM_INVALID_STEPS; local.usable = 0; break; }
        radius /= decrease;
        decrease *= 2;
        continue;
      }
      invalid = 0;
      double alpha = 1.0, cand = 0, step_norm = 0, x_norm = 0;
      make_candidate(v, alpha, o.thres_loss_function, points_var, cand, step_norm, x_norm);
      if (scales_var && o.max_num_line_search_step_size_iterations > 0) {
        // projected Armijo line search (trust_region_minimizer.cc DoLineSearch; oracle/ceres_lm.py)
        const double g0 = r.g_dot_delta;
        double pa = 0, pf = 0, ca = 0, cf = 0;
        bool have_prev = false, have_cur = false, ok = false;
        double a = 1.0, fa = cand;
        for (int ls = 0; ls <= o.max_num_line_search_step_size_iterations; ++ls) {
          if (std::isfinite(fa) && fa <= cost + 1e-4 * g0 * a) { ok = true; break; }
          if (have_cur) { pa = ca; pf = cf; have_prev = true; }
          ca = a; cf = fa; have_cur = true;
          double lo = 1e-3 * a, hi = 0.6 * a, an;
          if (!std::isfinite(fa)) {
            an = lo; have_prev = have_cur = false;
          } else if (!have_prev) {
            const double c2 = (cf - cost - g0 * ca) / (ca * ca);
            an = (c2 > 0) ? -g0 / (2 * c2) : hi;
          } else {
            // cubic through (0, cost, g0), (ca, cf), (pa, pf)
            const double r1 = cf - cost - g0 * ca, r2 = pf - cost - g0 * pa;
            const double det = ca * ca * ca * pa * pa - pa * pa * pa * ca * ca;
            double a3 = 0, a2 = r1 / (ca * ca);
            if (std::fabs(det) > 0) {
              a3 = (r1 * pa * pa - r2 * ca * ca) / det;
              a2 = (ca * ca * ca * r2 - pa * pa * pa * r1) / det;
            }
            an = hi;
            double best = cost + g0 * hi + a2 * hi * hi + a3 * hi * hi * hi;
            auto consider = [&](double x) {
              x = std::min(std::max(x, lo), hi);
              const double f = cost + g0 * x + a2 * x * x + a3 * x * x * x;
              if (f < best) { best = f; an = x; }
            };
            consider(lo);
            if (std::fabs(a3) > 0) {
              const double disc = 4 * a2 * a2 - 12 * a3 * g0;
              if (disc >= 0) {
                consider((-2 * a2 + std::sqrt(disc)) / (6 * a3));
                consider((-2 * a2 - std::sqrt(disc)) / (6 * a3));
              }
            } else if (a2 != 0) {
              consider(-g0 / (2 * a2));
            }
          }
          a = std::min(std::max(an, lo), hi);
          if (a < 1e-12) break;
          make_candidate(v, a, o.thres_loss_function, points_var, fa, step_norm, x_norm);
        }
        if (ok) { alpha = a; cand = fa; }
        else if (a != 1.0) make_candidate(v, 1.0, o.thres_loss_function, points_var, cand, step_norm, x_norm);
      }
      if (!fixed) {
        if (step_norm <= o.parameter_tolerance * (x_norm + o.parameter_tolerance)) { term = B200SFM_TERM_PARAMETER_TOLERANCE; break; }
        if (std::fabs(cost - cand) <= o.function_tolerance * cost) { term = B200SFM_TERM_FUNCTION_TOLERANCE; break; }
      }
      const double rel = (cost - cand) / r.model_cost_change;
      if (rel > 1e-3) {
        cur ^= 1;
        cost = cand;
        ++local.num_successful_steps;
        radius = std::min(1e16, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rel - 1.0, 3)));
        decrease = 2.0;
      } else {
        radius /= decrease;
        decrease *= 2;
      }
    }
    B200_CUDA_OK(cudaEventRecord(ev1, s));
    B200_CUDA_OK(cudaEventSynchronize(ev1));
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
    if (st) *st = local;
    return B200SFM_OK;
  }

  // ---- test probe (include/b200sfm_testing.h) ----------------------------------------------------------------------
  bool probe_ready = false;
  bool probe_scales_var = true;

  // the first LM iteration of solve() up to the candidate and its cost, without accepting it; with first_radius > 0 the
  // step at `radius` is the second one and reuses the Jacobi scales of the step at first_radius
  void test_step(const b200sfm_gp_opts& o, double first_radius, double radius, double alpha, b200sfm_test_gp_step_out* out) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    const bool points_var = o.optimize_points != 0;
    probe_scales_var = o.optimize_scales != 0;
    B200_LAUNCH(ctx, k_eff_mask, cdiv(C, 256), 256, 0, C, cam_const_base.p, o.optimize_positions ? 0 : 1, 0, cam_const.p);
    GPView v = view(probe_scales_var);
    if (first_radius > 0.0) compute_step(o, v, first_radius, true, points_var, false);
    const StepResult r = compute_step(o, v, radius, !(first_radius > 0.0), points_var, false);
    double cand = 0, step_norm = 0, x_norm = 0;
    make_candidate(v, alpha, o.thres_loss_function, points_var, cand, step_norm, x_norm);
    probe_ready = true;
    const int nxt = cur ^ 1;
    const size_t nb3 = (size_t)CB * 3;
    if (out->M) M.download(out->M, (size_t)N * 6, s);
    if (out->bw) bw.download(out->bw, (size_t)N * 4, s);
    if (out->jscale_s) jscale_s.download(out->jscale_s, N, s);
    if (out->ds) ds.download(out->ds, N, s);
    if (out->Vinv) Vinv.download(out->Vinv, (size_t)P * 6, s);
    if (out->gX) gX.download(out->gX, (size_t)P * 3, s);
    if (out->Dp) Dp.download(out->Dp, P, s);
    if (out->jscale_p) jscale_p.download(out->jscale_p, P, s);
    if (out->dX) dX.download(out->dX, (size_t)P * 3, s);
    if (out->U) U.download(out->U, (size_t)CB * 6, s);
    if (out->gc) gc.download(out->gc, nb3, s);
    if (out->Dc) Dc.download(out->Dc, nb3, s);
    if (out->Minv) Minv.download(out->Minv, (size_t)CB * 6, s);
    if (out->jscale_c) jscale_c.download(out->jscale_c, CB, s);
    if (out->b) bvec.download(out->b, nb3, s);
    if (out->px) px.download(out->px, nb3, s);
    if (out->resid) pr.download(out->resid, nb3, s);
    if (out->cand_centers) centers[nxt].download(out->cand_centers, (size_t)C * 3, s);
    if (out->cand_points) points[nxt].download(out->cand_points, (size_t)P * 3, s);
    if (out->cand_scales) scales[nxt].download(out->cand_scales, N, s);
    if (n_us > 0 && out->cand_ucen) ucen[nxt].download(out->cand_ucen, (size_t)n_us * 3, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    out->cost = r.cost;
    out->gmax = r.gmax;
    out->g_dot_delta = r.g_dot_delta;
    out->model_cost_change = r.model_cost_change;
    out->cand_cost = cand;
    out->step_norm = step_norm;
    out->x_norm = x_norm;
    out->pcg_iterations = r.pcg_iters;
    out->schur_jacobi = (points_var && o.preconditioner == 1 && n_us == 0) ? 1 : 0;
    out->CB = CB;
    out->n_us = n_us;
    out->pcg_depth = ctx->pcgh.depth;
  }

  // y = (S + D) x at the linearisation and damping of the last test_step, through matvec()
  void test_apply(const double* h_x, double* h_y) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    PcgCtl* ctl = ctx->pcgh.d_ctl;
    B200_CUDA_OK(cudaMemsetAsync(ctl, 0, sizeof(PcgCtl), s));   // every kernel of the chain returns early once ctl->done is set
    pp.upload(h_x, (size_t)CB * 3, s);
    yw.zero(s);
    matvec(view(probe_scales_var), pp.p, yw.p, ctx->pcgh.d_part, ctl, false);
    pq.download(h_y, (size_t)CB * 3, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }
};
