// vgc_solver.cuh -- host-side driver of the device view-graph calibrator: upload, incidence CSR, the Ceres-semantics LM
// loop with the focal lower bound (projection in Plus + projected Armijo line search, as gp_solver.cuh and
// oracle/ceres_lm.py), then the reference's copy-back and pair filter.  Reference path replaced:
// glomap/estimators/view_graph_calibration.cc:11-185 (the ceres::Solve at :38).
//
// The reference factors the K x K normal matrix exactly (DENSE / SPARSE_NORMAL_CHOLESKY, .cc:21-24).  Here it is solved
// by Jacobi-preconditioned CG whose loop control stays on the device (pcg.cuh, B = 1); the default relative tolerance
// (1e-12) is tight enough that the LM trajectory is the exact solver's (DESIGN.md section 6).
#pragma once
#include <cub/cub.cuh>

#include <cmath>
#include <vector>

#include "../../include/b200sfm.h"
#include "context.cuh"
#include "vgc_kernels.cuh"

namespace b200 {

struct VgcSolver {
  b200sfm_ctx* ctx = nullptr;
  int K = 0, n_inc = 0, n_seg = 0, cur = 0;
  long long E = 0;
  int nblk_e = 0, nblk_k = 0, nblk_w = 0;   // CTAs of the per-pair, per-camera and warp-per-camera kernels
  DevBuf<int> ci, cj, inc_begin, inc_other, seg_off, seg_begin, seg_end;
  DevBuf<unsigned> inc_val;
  DevBuf<unsigned char> var, valid;
  DevBuf<double> pp, F, d, x[2], jscale, A_s, D, Minv, bvec, g, dx, off, mv_part, res, part, scal;
  DevBuf<double> px, pr, pz, ppv, pq, yw;
  DevBuf<double4> jd;
  DevBuf<double2> seg_part;
  EventTimer timer_lin, timer_mv;
  double b = 0, c = 0;   // Cauchy b = a^2, c = 1 / b

  VGCView view() const {
    VGCView v;
    v.E = E; v.K = K; v.ci = ci.p; v.cj = cj.p; v.d = d.p; v.var = var.p;
    return v;
  }
  double* part_a() const { return part.p; }
  double* part_b() const { return part.p + std::max(nblk_e, std::max(nblk_k, nblk_w)); }

  // upload, Fetzer constants, incidence CSR and segments.  Returns the H2D time (CUDA events) in *ms_h2d.
  void create(b200sfm_ctx* c_, int K_, long long E_, const double* h_pp, const double* h_focal, const uint8_t* h_var,
              const int32_t* h_c1, const int32_t* h_c2, const double* h_F, double* ms_h2d) {
    ctx = c_; K = K_; E = E_;
    cudaStream_t s = ctx->stream;
    nblk_e = cdiv(E, kVgcThreads);
    nblk_k = cdiv(K, kVgcThreads);
    nblk_w = cdiv((long long)K * 32, 128);
    ci.alloc(E); cj.alloc(E); F.alloc((size_t)E * 9); pp.alloc((size_t)K * 2); var.alloc(K);
    for (int i = 0; i < 2; ++i) x[i].alloc(K);
    cudaEvent_t h0, h1;
    B200_CUDA_OK(cudaEventCreate(&h0));
    B200_CUDA_OK(cudaEventCreate(&h1));
    B200_CUDA_OK(cudaEventRecord(h0, s));
    ci.upload(h_c1, E, s); cj.upload(h_c2, E, s); F.upload(h_F, (size_t)E * 9, s);
    pp.upload(h_pp, (size_t)K * 2, s); var.upload(h_var, K, s); x[0].upload(h_focal, K, s);
    B200_CUDA_OK(cudaEventRecord(h1, s));
    d.alloc((size_t)E * 8);
    B200_LAUNCH(ctx, vgc_setup, nblk_e, kVgcThreads, 0, E, F.p, pp.p, ci.p, cj.p, d.p);
    // incidence lists by camera (device radix sort on (camera, 2 e + side): a fixed summation order)
    DevBuf<int> cnt, keys, keys_out, seg_count;
    DevBuf<unsigned> vals;
    cnt.alloc((size_t)K + 1); keys.alloc((size_t)2 * E); keys_out.alloc((size_t)2 * E); vals.alloc((size_t)2 * E);
    inc_val.alloc((size_t)2 * E); inc_begin.alloc((size_t)K + 1); seg_count.alloc((size_t)K + 1); seg_off.alloc((size_t)K + 1);
    cnt.zero(s); seg_count.zero(s);
    B200_LAUNCH(ctx, vgc_inc_keys, nblk_e, kVgcThreads, 0, view(), cnt.p, keys.p, vals.p);
    int end_bit = 1;
    while ((1ll << end_bit) <= K) ++end_bit;
    size_t sort_bytes = 0, scan_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys.p, keys_out.p, vals.p, inc_val.p, (int)(2 * E), 0, end_bit, s);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cnt.p, inc_begin.p, K + 1, s);
    DevBuf<unsigned char> tmp;
    tmp.alloc(std::max(sort_bytes, scan_bytes) + 16);
    size_t tb = tmp.bytes();
    cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.p, keys_out.p, vals.p, inc_val.p, (int)(2 * E), 0, end_bit, s);
    tb = tmp.bytes();
    cub::DeviceScan::ExclusiveSum(tmp.p, tb, cnt.p, inc_begin.p, K + 1, s);
    B200_LAUNCH(ctx, vgc_seg_counts, nblk_k, kVgcThreads, 0, K, inc_begin.p, seg_count.p);
    tb = tmp.bytes();
    cub::DeviceScan::ExclusiveSum(tmp.p, tb, seg_count.p, seg_off.p, K + 1, s);
    ctx->launches += 4;
    int h_tot[2];
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[0], inc_begin.p + K, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaMemcpyAsync(&h_tot[1], seg_off.p + K, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    float ms = 0;
    B200_CUDA_OK(cudaEventElapsedTime(&ms, h0, h1));
    cudaEventDestroy(h0);
    cudaEventDestroy(h1);
    *ms_h2d = ms;
    n_inc = h_tot[0];
    n_seg = h_tot[1];
    inc_other.alloc(std::max(n_inc, 1)); seg_begin.alloc(std::max(n_seg, 1)); seg_end.alloc(std::max(n_seg, 1));
    if (n_inc > 0) B200_LAUNCH(ctx, vgc_inc_other, cdiv(n_inc, 256), 256, 0, n_inc, view(), inc_val.p, inc_other.p);
    if (n_seg > 0) B200_LAUNCH(ctx, vgc_fill_segs, cdiv(n_seg, 256), 256, 0, n_seg, K, seg_off.p, inc_begin.p, seg_begin.p, seg_end.p);
    jscale.alloc(K); A_s.alloc(K); D.alloc(K); Minv.alloc(K); bvec.alloc(K); g.alloc(K); dx.alloc(K);
    px.alloc(K); pr.alloc(K); pz.alloc(K); ppv.alloc(K); pq.alloc(K); yw.alloc(K);
    jd.alloc(E); off.alloc(E); seg_part.alloc(std::max(n_seg, 1)); mv_part.alloc(std::max(n_seg, 1));
    part.alloc(2 * (size_t)std::max(nblk_e, std::max(nblk_k, nblk_w)));
    scal.alloc(16);
    B200_CUDA_OK(cudaStreamSynchronize(s));   // sort temporaries go out of scope
    F.release();
  }

  void reduce(const double* p, int n, int mode, int slot) {
    B200_LAUNCH(ctx, vgc_reduce, 1, 1024, 0, p, n, mode, scal.p + slot);
  }
  void read_scal(int n) {
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal, scal.p, n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
  }

  struct StepResult {
    double cost = 0, gmax = 0, model_cost_change = 0, g_dot_delta = 0, dx_max = 0;
    int pcg_iters = 0;
    bool finite = true;
  };

  // linearise at x[cur] with damping 1 / radius, solve for the step dx, its model cost change and g . dx
  StepResult compute_step(const b200sfm_vgc_opts& o, double radius, bool first, bool profile) {
    cudaStream_t s = ctx->stream;
    const VGCView v = view();
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (profile) {
      e0 = timer_lin.next(); e1 = timer_lin.next();
      B200_CUDA_OK(cudaEventRecord(e0, s));
    }
    B200_LAUNCH(ctx, vgc_linearize, nblk_e, kVgcThreads, 0, v, x[cur].p, b, c, jd.p, off.p, part_a());
    if (profile) B200_CUDA_OK(cudaEventRecord(e1, s));
    reduce(part_a(), nblk_e, 0, 0);
    B200_LAUNCH(ctx, vgc_seg_sums, cdiv((long long)n_seg * 32, 128), 128, 0, n_seg, seg_begin.p, seg_end.p, inc_val.p, jd.p,
                seg_part.p);
    B200_LAUNCH(ctx, vgc_cam_system, nblk_w, 128, 0, K, seg_off.p, seg_part.p, var.p, x[cur].p, first ? 1 : 0, radius, jscale.p,
                A_s.p, D.p, Minv.p, bvec.p, g.p, part_b());
    reduce(part_b(), nblk_w, 1, 1);
    // Jacobi-preconditioned CG on the scaled system (loop control on the device, pcg.cuh)
    const int max_it = std::max(1, o.pcg_max_iterations);
    const int nblk = cdiv(K, kPcgThreads);
    ctx->pcgh.ensure(max_it, (size_t)nblk * 3, 1);
    double *part_pq = ctx->pcgh.d_part, *part_rz = ctx->pcgh.d_part + nblk, *part_rr = ctx->pcgh.d_part + 2 * (size_t)nblk;
    PcgCtl* ctl = ctx->pcgh.d_ctl;
    const size_t mv_ev0 = timer_mv.used;
    PcgResult pr_ = ctx->pcgh.run(
        s, max_it,
        [&]() { B200_LAUNCH(ctx, pcg_init<1>, nblk, kPcgThreads, 0, K, Minv.p, bvec.p, px.p, pr.p, pz.p, part_rz, part_rr); },
        [&](int it) {
          double* d_pub = ctx->pcgh.dots(it - 1);
          B200_LAUNCH(ctx, pcg_direction<1>, nblk, kPcgThreads, 0, K, nblk, it, o.pcg_min_iterations, o.pcg_rel_tolerance, pz.p,
                      ppv.p, nullptr, ctx->pcgh.dots(it - 2), part_rz, part_rr, nullptr, d_pub, ctl);
          cudaEvent_t m0 = nullptr, m1 = nullptr;
          if (profile) {
            m0 = timer_mv.next(); m1 = timer_mv.next();
            B200_CUDA_OK(cudaEventRecord(m0, s));
          }
          B200_LAUNCH(ctx, vgc_mv_seg, cdiv((long long)n_seg * 32, 128), 128, 0, n_seg, seg_begin.p, seg_end.p, inc_val.p,
                      inc_other.p, off.p, jscale.p, ppv.p, mv_part.p, ctl);
          B200_LAUNCH(ctx, vgc_mv_cam, nblk_w, 128, 0, K, seg_off.p, mv_part.p, jscale.p, yw.p, ctl);
          if (profile) B200_CUDA_OK(cudaEventRecord(m1, s));
          // q = (A_s + D) p + yw (the off-diagonal part)
          B200_LAUNCH(ctx, pcg_apply_diag<1>, nblk, kPcgThreads, 0, K, A_s.p, D.p, ppv.p, yw.p, pq.p, part_pq, ctl);
          B200_LAUNCH(ctx, pcg_update<1>, nblk, kPcgThreads, 0, K, nblk, Minv.p, ppv.p, pq.p, px.p, pr.p, pz.p, d_pub, part_pq,
                      part_rz, part_rr, ctx->pcgh.dots(it), ctl);
        },
        [&](int launched) { B200_LAUNCH(ctx, pcg_finalize, 1, kPcgThreads, 0, nblk, launched, part_rr, ctl); });
    if (profile) timer_mv.used = mv_ev0 + 2 * (size_t)std::min(pr_.iters, pr_.launched);
    StepResult res_;
    res_.finite = pr_.finite;
    res_.pcg_iters = pr_.iters;
    B200_LAUNCH(ctx, vgc_step, nblk_k, kVgcThreads, 0, K, px.p, jscale.p, g.p, dx.p, part_a(), part_b());
    reduce(part_a(), nblk_k, 0, 2);
    reduce(part_b(), nblk_k, 1, 3);
    B200_LAUNCH(ctx, vgc_model, nblk_e, kVgcThreads, 0, v, x[cur].p, dx.p, b, c, part_a());
    reduce(part_a(), nblk_e, 0, 4);
    read_scal(5);
    const double* h = ctx->h_scal;
    res_.cost = h[0];
    res_.gmax = h[1];
    res_.g_dot_delta = h[2];
    res_.dx_max = h[3];
    res_.model_cost_change = h[4];
    if (!std::isfinite(res_.model_cost_change)) res_.finite = false;
    return res_;
  }

  // candidate x[cur ^ 1] = Project(x + alpha dx): its cost, |step| and |x|
  void make_candidate(double alpha, double& cand_cost, double& step_norm, double& x_norm) {
    const int nxt = cur ^ 1;
    B200_LAUNCH(ctx, vgc_candidate, nblk_k, kVgcThreads, 0, K, alpha, var.p, x[cur].p, dx.p, x[nxt].p, part_a(), part_b());
    reduce(part_a(), nblk_k, 0, 5);
    reduce(part_b(), nblk_k, 0, 6);
    B200_LAUNCH(ctx, vgc_cost, nblk_e, kVgcThreads, 0, view(), x[nxt].p, b, c, part_a());
    reduce(part_a(), nblk_e, 0, 7);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal + 5, scal.p + 5, 3 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    step_norm = std::sqrt(ctx->h_scal[5]);
    x_norm = std::sqrt(ctx->h_scal[6]);
    cand_cost = ctx->h_scal[7];
  }

  // value-only Armijo step of the line search (oracle/ceres_lm.py _interp_step): minimiser over [lo, hi] of the
  // quadratic through (0, f0, g0), (ca, cf), or of the cubic through those and (pa, pf)
  static double interp_step(double f0, double g0, bool have_prev, double pa, double pf, double ca, double cf, double lo, double hi) {
    double a2 = 0, a3 = 0;
    double cands[4] = {lo, hi, 0, 0};
    int n = 2;
    if (!have_prev) {
      a2 = (cf - f0 - g0 * ca) / (ca * ca);
      if (a2 > 0) cands[n++] = -g0 / (2 * a2);
    } else {
      const double r1 = cf - f0 - g0 * ca, r2 = pf - f0 - g0 * pa;
      const double det = ca * ca * ca * pa * pa - pa * pa * pa * ca * ca;
      if (det != 0) {
        a3 = (r1 * pa * pa - r2 * ca * ca) / det;
        a2 = (ca * ca * ca * r2 - pa * pa * pa * r1) / det;
      } else {
        a2 = r1 / (ca * ca);
      }
      if (a3 != 0) {
        const double disc = 4 * a2 * a2 - 12 * a3 * g0;
        if (disc >= 0) {
          cands[n++] = (-2 * a2 + std::sqrt(disc)) / (6 * a3);
          cands[n++] = (-2 * a2 - std::sqrt(disc)) / (6 * a3);
        }
      } else if (a2 != 0) {
        cands[n++] = -g0 / (2 * a2);
      }
    }
    double best = 0, best_f = 0;
    for (int i = 0; i < n; ++i) {
      const double xx = std::min(std::max(cands[i], lo), hi);
      const double f = f0 + g0 * xx + a2 * xx * xx + a3 * xx * xx * xx;
      if (i == 0 || f < best_f) { best = xx; best_f = f; }
    }
    return best;
  }

  void solve(const b200sfm_vgc_opts& o, b200sfm_lm_stats& st) {
    cudaStream_t s = ctx->stream;
    const long long launches0 = ctx->launches;
    timer_lin.reset();
    timer_mv.reset();
    const bool profile = o.profile_kernels != 0;
    b = o.thres_loss_function * o.thres_loss_function;
    c = 1.0 / b;
    cudaEvent_t ev0, ev1;
    B200_CUDA_OK(cudaEventCreate(&ev0));
    B200_CUDA_OK(cudaEventCreate(&ev1));
    B200_CUDA_OK(cudaEventRecord(ev0, s));
    double radius = 1e4, decrease = 2.0;
    int invalid = 0, it = 0, term = B200SFM_TERM_NONE;
    bool first = true;
    double cost = 0;
    st.usable = 1;
    while (term == B200SFM_TERM_NONE) {
      if (it >= o.max_num_iterations) { term = B200SFM_TERM_MAX_ITERATIONS; break; }
      if (radius < 1e-32) { term = B200SFM_TERM_MIN_RADIUS; break; }
      StepResult r = compute_step(o, radius, first, profile);
      cost = r.cost;
      if (first) {
        st.initial_cost = cost;
        // the initial evaluation failed (a non-finite F): Ceres stops with FAILURE, the parameters untouched
        if (!std::isfinite(cost)) { st.usable = 0; break; }
      }
      first = false;
      st.pcg_iterations += r.pcg_iters;
      if (r.gmax <= o.gradient_tolerance) { term = B200SFM_TERM_GRADIENT_TOLERANCE; break; }
      ++it;
      if (!r.finite || !(r.model_cost_change > 0.0)) {
        if (++invalid >= 5) { term = B200SFM_TERM_INVALID_STEPS; st.usable = 0; break; }
        radius /= decrease;
        decrease *= 2;
        continue;
      }
      invalid = 0;
      double cand = 0, step_norm = 0, x_norm = 0;
      make_candidate(1.0, cand, step_norm, x_norm);
      if (o.max_num_line_search_step_size_iterations > 0) {
        // projected Armijo line search (trust_region_minimizer.cc DoLineSearch; oracle/ceres_lm.py)
        const double g0 = r.g_dot_delta;
        double pa = 0, pf = 0, ca = 0, cf = 0, a = 1.0, fa = cand;
        bool have_prev = false, have_cur = false, ok = false;
        for (int ls = 0; ls <= o.max_num_line_search_step_size_iterations; ++ls) {
          if (ls > 0) make_candidate(a, fa, step_norm, x_norm);
          if (std::isfinite(fa) && fa <= cost + 1e-4 * g0 * a) { ok = true; break; }
          if (have_cur) { pa = ca; pf = cf; have_prev = true; }
          ca = a; cf = fa; have_cur = true;
          if (!std::isfinite(fa)) {
            a *= 1e-3;
            have_prev = have_cur = false;
          } else {
            a = interp_step(cost, g0, have_prev, pa, pf, ca, cf, 1e-3 * a, 0.6 * a);
          }
          if (a * r.dx_max < 1e-9) break;
        }
        if (ok) cand = fa;
        else if (a != 1.0) make_candidate(1.0, cand, step_norm, x_norm);
      }
      if (step_norm <= o.parameter_tolerance * (x_norm + o.parameter_tolerance)) { term = B200SFM_TERM_PARAMETER_TOLERANCE; break; }
      if (std::fabs(cost - cand) <= o.function_tolerance * cost) { term = B200SFM_TERM_FUNCTION_TOLERANCE; break; }
      const double rel = (cost - cand) / r.model_cost_change;
      if (rel > 1e-3) {
        cur ^= 1;
        cost = cand;
        ++st.num_successful_steps;
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
    st.iterations = it;
    st.termination = term;
    st.final_cost = cost;
    st.ms_total = ms;
    for (size_t i = 0; i + 1 < timer_lin.used; i += 2) {
      float t;
      B200_CUDA_OK(cudaEventElapsedTime(&t, timer_lin.ev[i], timer_lin.ev[i + 1]));
      st.ms_linearize += t;
      ++st.n_linearize;
    }
    for (size_t i = 0; i + 1 < timer_mv.used; i += 2) {
      float t;
      B200_CUDA_OK(cudaEventElapsedTime(&t, timer_mv.ev[i], timer_mv.ev[i + 1]));
      st.ms_matvec += t;
      ++st.n_matvec;
    }
    st.kernel_launches = ctx->launches - launches0;
  }

  // unlossed residuals and the pair mask at the final focals; downloads focal, pair_valid and (optionally) residuals
  void finish(double thres_two_view_error, double* h_focal, uint8_t* h_valid, double* h_res, double* ms_d2h) {
    cudaStream_t s = ctx->stream;
    res.alloc((size_t)E * 2);
    valid.alloc(E);
    B200_LAUNCH(ctx, vgc_filter, nblk_e, kVgcThreads, 0, view(), x[cur].p, thres_two_view_error * thres_two_view_error, res.p,
                valid.p);
    cudaEvent_t h0, h1;
    B200_CUDA_OK(cudaEventCreate(&h0));
    B200_CUDA_OK(cudaEventCreate(&h1));
    B200_CUDA_OK(cudaEventRecord(h0, s));
    x[cur].download(h_focal, K, s);
    valid.download(h_valid, E, s);
    if (h_res) res.download(h_res, (size_t)E * 2, s);
    B200_CUDA_OK(cudaEventRecord(h1, s));
    B200_CUDA_OK(cudaEventSynchronize(h1));
    float ms = 0;
    B200_CUDA_OK(cudaEventElapsedTime(&ms, h0, h1));
    cudaEventDestroy(h0);
    cudaEventDestroy(h1);
    *ms_d2h = ms;
  }
};

}  // namespace b200
