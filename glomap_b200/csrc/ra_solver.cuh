// ra_solver.cuh -- host-side driver of the device rotation averaging
// (reference: glomap/estimators/global_rotation_averaging.cc:40-85, the
// SetupLinearSystem / SolveL1Regression / SolveIRLS sequence; the L1 solver is
// colmap::LeastAbsoluteDeviationSolver restated in oracle/ra_oracle.py).
#pragma once
#include <cub/cub.cuh>

#include "../../include/b200sfm_testing.h"
#include "context.cuh"
#include "pcg.cuh"
#include "ra_kernels.cuh"

struct b200sfm_ra_problem {
  template <class T>
  using DevBuf = b200::DevBuf<T>;
  b200sfm_ctx* ctx = nullptr;
  int n = 0;              // nodes: frames followed by the unknown cam_from_rig rotations
  int n_frames = 0, n_cams = 0;
  DevBuf<int> eci, ecj, cf_begin, cf_list;
  long long E = 0;        // local edges (+1 gauge pseudo-edge on rank 0)
  long long E_real = 0;
  long long E_total = 0;  // valid edges over all ranks
  int fixed = 0;
  DevBuf<int> ei, ej, flags;
  DevBuf<unsigned char> node_grav;
  DevBuf<double> angle_rel, xz_err;
  bool has_grav = false;
  long long rows_total = 0;
  DevBuf<double> Rrel, w_edge, theta, res, w, b, z, u;
  DevBuf<double> deg, Minv, Azero, Dzero, rhs, svec, uvec, px, pr, pz, pp, pq, yw, part, scal;
  // CSR-by-node incidence lists (3-DoF frames without gravity): gather form of the Laplacian, see ra_kernels.cuh
  bool use_csr = false;
  int n_inc = 0;
  DevBuf<int> inc_begin, inc_other;
  DevBuf<unsigned> inc_val;
  DevBuf<double> w_inc;
  // two-level preconditioner (ra_kernels.cuh): aggregates built on the host at create()
  bool use_2lvl = false, coarse_l1_valid = false;
  int nc = 0, nblk_c = 0;
  DevBuf<int> agg_of, agg_begin, agg_nodes;
  DevBuf<double> Ac, rc, zc, p4;   // p4: 32-B padded copy of the PCG direction for the Laplacian gathers (fused iteration)
  DevBuf<unsigned> gbar;           // grid barrier of ra2_coarse: {arrivals, generation}
  b200::RACoarse coarse() {
    b200::RACoarse c;
    c.nc = nc; c.agg_of = agg_of.p; c.agg_begin = agg_begin.p; c.agg_nodes = agg_nodes.p; c.Ac = Ac.p; c.rc = rc.p; c.zc = zc.p;
    return c;
  }
  b200::RACsr csr() {
    b200::RACsr c;
    c.n = n; c.begin = inc_begin.p; c.val = inc_val.p; c.other = inc_other.p; c.w_inc = w_inc.p;
    return c;
  }

  b200::RAView view() {
    b200::RAView v;
    v.n = n; v.E = E; v.ei = ei.p; v.ej = ej.p; v.Rrel = Rrel.p; v.w_edge = w_edge.p;
    v.node_grav = has_grav ? node_grav.p : nullptr;
    v.angle_rel = has_grav ? angle_rel.p : nullptr;
    v.xz_err = has_grav ? xz_err.p : nullptr;
    v.n_frames = n_frames; v.eci = n_cams > 0 ? eci.p : nullptr; v.ecj = n_cams > 0 ? ecj.p : nullptr;
    return v;
  }

  void create(b200sfm_ctx* c, int n_, long long E_, const int32_t* h_ei, const int32_t* h_ej, const double* h_Rrel,
              const double* h_w, int use_weight, int fixed_, const double* h_theta, const uint8_t* h_grav = nullptr,
              int n_cams_ = 0, const int32_t* h_eci = nullptr, const int32_t* h_ecj = nullptr,
              const int32_t* h_cf_begin = nullptr, const int32_t* h_cf_list = nullptr) {
    using namespace b200;
    ctx = c; n = n_; E_real = E_; fixed = fixed_;
    n_cams = n_cams_;
    n_frames = n - n_cams;
    cudaStream_t s = ctx->stream;
    const bool gauge_here = ctx->rank == 0;
    E = E_real + (gauge_here ? 1 : 0);
    std::vector<int> hi(h_ei, h_ei + E_real), hj(h_ej, h_ej + E_real);
    std::vector<double> hr(h_Rrel, h_Rrel + 9 * E_real), hw((size_t)E_real, 1.0);
    if (use_weight && h_w)
      for (long long e = 0; e < E_real; ++e) hw[e] = h_w[e] >= 0 ? h_w[e] : 1.0;   // .cc:390-393,417-421
    if (gauge_here) {
      // gauge rows (.cc:455-460): pseudo-edge (identity -> fixed frame) with R_rel = R_fixed(initial)
      hi.push_back(-1);
      hj.push_back(fixed);
      const double* t = h_theta + 3 * (size_t)fixed;
      const double nn = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
      double R[9];
      if (nn > 1e-12) {
        const double x = t[0] / nn, y = t[1] / nn, zc = t[2] / nn, sn = std::sin(nn), cs = std::cos(nn), tt = 1 - cs;
        const double Rm[9] = {tt * x * x + cs, tt * x * y - sn * zc, tt * x * zc + sn * y,
                              tt * x * y + sn * zc, tt * y * y + cs, tt * y * zc - sn * x,
                              tt * x * zc - sn * y, tt * y * zc + sn * x, tt * zc * zc + cs};
        std::copy(Rm, Rm + 9, R);
      } else {
        const double Rm[9] = {1, -t[2], t[1], t[2], 1, -t[0], -t[1], t[0], 1};
        std::copy(Rm, Rm + 9, R);
      }
      hr.insert(hr.end(), R, R + 9);
      hw.push_back(1.0);
    }
    // use_gravity: y angle / xz error of the (gravity-aligned) relative rotations (.cc:328-337)
    has_grav = h_grav != nullptr;
    std::vector<double> h_ang((size_t)E, 0.0), h_xz((size_t)E, 0.0);
    long long rows_local = 0;
    for (long long e = 0; e < E; ++e) {
      const int i = hi[e], j = hj[e];
      const bool gi = has_grav && i >= 0 && h_grav[i], gj = has_grav && h_grav[j];
      const bool y_only = (i >= 0) ? (gi && gj) : gj;
      rows_local += y_only ? 1 : 3;
      if (!y_only) continue;
      if (i < 0) { h_ang[e] = h_theta[3 * (size_t)j + 1]; continue; }   // gauge: phi_fixed(initial)
      const double* R = &hr[9 * (size_t)e];
      // Eigen matrix -> quaternion -> angle-axis (math/rigid3d.cc:39-43)
      double q[4];
      const double t = R[0] + R[4] + R[8];
      if (t > 0.0) {
        double tt = std::sqrt(t + 1.0);
        q[3] = 0.5 * tt; tt = 0.5 / tt;
        q[0] = (R[7] - R[5]) * tt; q[1] = (R[2] - R[6]) * tt; q[2] = (R[3] - R[1]) * tt;
      } else {
        int a = 0;
        if (R[4] > R[0]) a = 1;
        if (R[8] > R[4 * a]) a = 2;
        const int b2 = (a + 1) % 3, c2 = (a + 2) % 3;
        double tt = std::sqrt(R[4 * a] - R[4 * b2] - R[4 * c2] + 1.0);
        q[a] = 0.5 * tt; tt = 0.5 / tt;
        q[3] = (R[3 * c2 + b2] - R[3 * b2 + c2]) * tt; q[b2] = (R[3 * b2 + a] + R[3 * a + b2]) * tt; q[c2] = (R[3 * c2 + a] + R[3 * a + c2]) * tt;
      }
      const double nv = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
      double aa[3] = {0, 0, 0};
      if (nv > 0) {
        const double ang = 2.0 * std::atan2(nv, std::fabs(q[3]));
        const double f = (q[3] < 0 ? -ang : ang) / nv;
        aa[0] = q[0] * f; aa[1] = q[1] * f; aa[2] = q[2] * f;
      }
      h_ang[e] = aa[1];
      h_xz[e] = aa[0] * aa[0] + aa[2] * aa[2];
    }
    const size_t Ea = (size_t)std::max<long long>(E, 1);
    if (has_grav) {
      node_grav.alloc(n); angle_rel.alloc(Ea); xz_err.alloc(Ea);
      node_grav.upload(h_grav, n, s); angle_rel.upload(h_ang.data(), E, s); xz_err.upload(h_xz.data(), E, s);
    }
    if (n_cams > 0) {
      std::vector<int> hci(h_eci, h_eci + E_real), hcj(h_ecj, h_ecj + E_real);
      if (gauge_here) { hci.push_back(-1); hcj.push_back(-1); }
      eci.alloc(Ea); ecj.alloc(Ea);
      eci.upload(hci.data(), E, s); ecj.upload(hcj.data(), E, s);
      cf_begin.alloc((size_t)n_cams + 1);
      cf_begin.upload(h_cf_begin, (size_t)n_cams + 1, s);
      const int n_cf = h_cf_begin[n_cams];
      cf_list.alloc((size_t)std::max(n_cf, 1));
      cf_list.upload(h_cf_list, n_cf, s);
      B200_CUDA_OK(cudaStreamSynchronize(s));   // hci / hcj are locals
    }
    ei.alloc(Ea); ej.alloc(Ea); Rrel.alloc(Ea * 9); w_edge.alloc(Ea); flags.alloc(4);
    ei.upload(hi.data(), E, s); ej.upload(hj.data(), E, s); Rrel.upload(hr.data(), (size_t)E * 9, s); w_edge.upload(hw.data(), E, s);
    theta.alloc((size_t)n * 3);
    theta.upload(h_theta, (size_t)n * 3, s);
    res.alloc(Ea * 3); w.alloc(Ea); b.alloc(Ea * 3); z.alloc(Ea * 3); u.alloc(Ea * 3);
    deg.alloc((size_t)n * 3); Minv.alloc((size_t)n * 6); Azero.alloc((size_t)n * 6); Dzero.alloc((size_t)n * 3);
    rhs.alloc((size_t)n * 9);   // rhs | svec | uvec contiguous for one all-reduce
    px.alloc((size_t)n * 3); pr.alloc((size_t)n * 3); pz.alloc((size_t)n * 3); pp.alloc((size_t)n * 3);
    pq.alloc((size_t)n * 3); yw.alloc((size_t)n * 3); scal.alloc(16);
    Azero.zero(s); Dzero.zero(s);
    {
      const double cnt[2] = {(double)E_real, (double)rows_local};
      B200_CUDA_OK(cudaMemcpyAsync(scal.p, cnt, 2 * sizeof(double), cudaMemcpyHostToDevice, s));
      ctx->allreduce_sum(scal.p, 2);
      double tot[2] = {0, 0};
      B200_CUDA_OK(cudaMemcpyAsync(tot, scal.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
      B200_CUDA_OK(cudaStreamSynchronize(s));
      E_total = (long long)(tot[0] + 0.5);
      rows_total = (long long)(tot[1] + 0.5);
    }
    // aggregates of the two-level preconditioner: greedy breadth-first clusters over the LOCAL edge list (all ranks hold
    // the same list only when world == 1: the coarse space is used by single-process contexts)
    {
      const char* env = getenv("B200SFM_RA_2LVL");
      const int min_nodes = env ? (atoi(env) > 0 ? 0 : 1 << 30) : 20000;   // default: large graphs only; =1 forces, =0 disables
      use_2lvl = !has_grav && n_cams == 0 && ctx->world == 1 && E_real > 0 && n >= std::max(min_nodes, 64);
    }
    if (use_2lvl) {
      const int target = std::max(32, (n + 399) / 400);   // ~400 aggregates, never more than 1024
      std::vector<int> deg_h((size_t)n + 1, 0);
      for (long long e = 0; e < E_real; ++e) { ++deg_h[hi[e] + 1]; ++deg_h[hj[e] + 1]; }
      for (int i = 0; i < n; ++i) deg_h[i + 1] += deg_h[i];
      std::vector<int> adj((size_t)deg_h[n]), fill(deg_h.begin(), deg_h.end() - 1);
      for (long long e = 0; e < E_real; ++e) { adj[fill[hi[e]]++] = hj[e]; adj[fill[hj[e]]++] = hi[e]; }
      std::vector<int> agg((size_t)n, -1), queue;
      queue.reserve(target + 8);
      int na = 0;
      for (int seed = 0; seed < n; ++seed) {
        if (agg[seed] >= 0) continue;
        queue.clear();
        queue.push_back(seed);
        agg[seed] = na;
        int cnt = 1;
        for (size_t head = 0; head < queue.size() && cnt < target; ++head) {
          const int u = queue[head];
          for (int t = deg_h[u]; t < deg_h[u + 1] && cnt < target; ++t) {
            const int v2 = adj[t];
            if (agg[v2] < 0) { agg[v2] = na; ++cnt; queue.push_back(v2); }
          }
        }
        ++na;
      }
      if (na > 1024 || na < 2) {
        use_2lvl = false;   // pathological graph (many tiny components): Jacobi only
      } else {
        nc = na;
        std::vector<int> ab((size_t)nc + 1, 0), an((size_t)n);
        for (int i = 0; i < n; ++i) ++ab[agg[i] + 1];
        for (int a = 0; a < nc; ++a) ab[a + 1] += ab[a];
        std::vector<int> f2(ab.begin(), ab.end() - 1);
        for (int i = 0; i < n; ++i) an[f2[agg[i]]++] = i;
        agg_of.alloc(n); agg_begin.alloc((size_t)nc + 1); agg_nodes.alloc(n);
        agg_of.upload(agg.data(), n, s); agg_begin.upload(ab.data(), (size_t)nc + 1, s); agg_nodes.upload(an.data(), n, s);
        Ac.alloc((size_t)nc * nc); rc.alloc((size_t)nc * 3); zc.alloc((size_t)nc * 3);
        nblk_c = cdiv((long long)nc * 32, 128);
        B200_CUDA_OK(cudaStreamSynchronize(s));   // host vectors are locals
      }
    }
    // incidence lists by node (device radix sort on (node, edge id): deterministic summation order)
    use_csr = !has_grav && n_cams == 0 && E > 0 && !(getenv("B200SFM_RA_CSR") && atoi(getenv("B200SFM_RA_CSR")) == 0);
    if (use_csr) {
      DevBuf<int> cnt, keys, keys_out;
      DevBuf<unsigned> vals;
      cnt.alloc((size_t)n + 1); keys.alloc((size_t)2 * E); keys_out.alloc((size_t)2 * E); vals.alloc((size_t)2 * E);
      inc_val.alloc((size_t)2 * E); inc_begin.alloc((size_t)n + 1);
      cnt.zero(s);
      B200_LAUNCH(ctx, ra_csr_count, cdiv(E, 256), 256, 0, E, ei.p, ej.p, n, cnt.p, keys.p, vals.p);
      int end_bit = 1;
      while ((1ll << end_bit) <= n) ++end_bit;
      size_t sort_bytes = 0, scan_bytes = 0;
      cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys.p, keys_out.p, vals.p, inc_val.p, (int)(2 * E), 0, end_bit, s);
      cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, cnt.p, inc_begin.p, n + 1, s);
      DevBuf<unsigned char> tmp;
      tmp.alloc(std::max(sort_bytes, scan_bytes) + 16);
      size_t tb = tmp.bytes();
      cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys.p, keys_out.p, vals.p, inc_val.p, (int)(2 * E), 0, end_bit, s);
      tb = tmp.bytes();
      cub::DeviceScan::ExclusiveSum(tmp.p, tb, cnt.p, inc_begin.p, n + 1, s);
      ctx->launches += 4;
      int h_inc = 0;
      B200_CUDA_OK(cudaMemcpyAsync(&h_inc, inc_begin.p + n, sizeof(int), cudaMemcpyDeviceToHost, s));
      B200_CUDA_OK(cudaStreamSynchronize(s));
      n_inc = h_inc;
      inc_other.alloc((size_t)std::max(n_inc, 1)); w_inc.alloc((size_t)std::max(n_inc, 1));
      B200_LAUNCH(ctx, ra_csr_other, cdiv(std::max(n_inc, 1), 256), 256, 0, n_inc, inc_val.p, ei.p, ej.p, inc_other.p);
      B200_CUDA_OK(cudaStreamSynchronize(s));   // sort temporaries go out of scope
    }
    B200_CUDA_OK(cudaStreamSynchronize(s));   // host vectors go out of scope
  }

  // y = L(w^p) x over this rank's edges (then all-reduced by the caller); weights as prepared by prepare_system
  void laplacian(const b200::RAView& v, int square, const double* x, double* y, const b200::PcgCtl* ctl) {
    using namespace b200;
    if (use_csr) {
      B200_LAUNCH(ctx, ra_laplacian_csr, cdiv((long long)n * 32, 128), 128, 0, csr(), x, y, ctl);
    } else if (E > 0) {
      B200_LAUNCH(ctx, ra_laplacian, cdiv(std::max<long long>(E, 1), 256), 256, 0, v, w.p, square, x, y, ctl);
    }
  }

  // fused iteration (ra_kernels.cuh: ra2_*): four kernels, the prolongation folded into the direction update.  Opt-in
  // (B200SFM_RA_FUSED=1): at config 5 on one H100 (700 W) it is within 2 % of the seven-kernel iteration (614 vs 624 ms
  // per solve) with 24 k instead of 37 k launches -- the launch count is not what bounds the iteration.  It reorders the
  // PCG arithmetic (the iteration count differs by one or two), so the default keeps the seven-kernel results.
  bool fused_iteration() const {
    return use_2lvl && use_csr && ctx->world == 1 && (getenv("B200SFM_RA_FUSED") && atoi(getenv("B200SFM_RA_FUSED")) == 1);
  }

  void fused_buffers() {
    if (p4.n < (size_t)n * 4) p4.alloc((size_t)n * 4);
    if (gbar.n < 2) { gbar.alloc(2); gbar.zero(ctx->stream); }
  }

  // x = L(w^p)^-1 rhs_vec by PCG (result in px); returns iterations.  Loop control on the device (pcg.cuh).
  int pcg_solve(const b200sfm_ra_opts& o, int square, const double* rhs_vec, bool& finite, bool warm = false) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    RAView v = view();
    const int nblk = cdiv(n, kPcgThreads);
    // partial sums: nblk per-CTA Jacobi partials followed by nblk_c coarse partials (r.z only; zero for p.q and r.r)
    const int nblk_t = nblk + (use_2lvl ? nblk_c : 0);
    const int max_it = std::max(1, o.pcg_max_iterations);
    ctx->pcgh.ensure(max_it, (size_t)nblk_t * 3, ctx->world);
    // a rotation-averaging PCG iteration is ~10 small kernels (~150 us at 100 k frames on an H100: 624 ms for 4 240
    // iterations): the read-back round trip is a sizeable part of it even on one GPU, so two iterations are always kept in
    // flight here
    if (!ctx->pcgh.depth_from_env) ctx->pcgh.depth = 2;
    double *part_pq = ctx->pcgh.d_part, *part_rz = ctx->pcgh.d_part + nblk_t, *part_rr = ctx->pcgh.d_part + 2 * (size_t)nblk_t;
    if (use_2lvl) B200_CUDA_OK(cudaMemsetAsync(ctx->pcgh.d_part, 0, (size_t)nblk_t * 3 * sizeof(double), s));
    PcgCtl* ctl = ctx->pcgh.d_ctl;
    if (fused_iteration()) {
      fused_buffers();
      PcgResult rf = ctx->pcgh.run(
          s, max_it,
          [&]() {
            if (warm) {
              yw.zero(s);
              laplacian(v, square, px.p, yw.p, nullptr);
              B200_LAUNCH(ctx, ra_pcg_init_warm, nblk, kPcgThreads, 0, n, Minv.p, rhs_vec, yw.p, pr.p, pz.p, pp.p, part_pq, part_rz, part_rr);
            } else {
              B200_LAUNCH(ctx, pcg_init<3>, nblk, kPcgThreads, 0, n, Minv.p, rhs_vec, px.p, pr.p, pz.p, part_rz, part_rr);
            }
            B200_LAUNCH(ctx, ra2_coarse, nblk_c, 128, 0, coarse(), pr.p, part_rz + nblk, gbar.p, nullptr);
          },
          [&](int it) {
            double* d_pub = ctx->pcgh.dots(it - 1);
            B200_LAUNCH(ctx, ra2_direction, nblk, kPcgThreads, 0, n, nblk_t, it, o.pcg_rel_tolerance, pz.p, pp.p, p4.p, zc.p, agg_of.p,
                        ctx->pcgh.dots(it - 2), part_rz, part_rr, (warm && it == 1) ? part_pq : nullptr, d_pub, ctl);
            B200_LAUNCH(ctx, ra2_laplacian_dot, nblk, kLapThreads, 0, csr(), p4.p, pq.p, part_pq, ctl);
            B200_LAUNCH(ctx, pcg_update<3>, nblk, kPcgThreads, 0, n, nblk_t, Minv.p, pp.p, pq.p, px.p, pr.p, pz.p, d_pub, part_pq, part_rz,
                        part_rr, ctx->pcgh.dots(it), ctl);
            B200_LAUNCH(ctx, ra2_coarse, nblk_c, 128, 0, coarse(), pr.p, part_rz + nblk, gbar.p, ctl);
          },
          [&](int launched) { B200_LAUNCH(ctx, pcg_finalize, 1, kPcgThreads, 0, nblk_t, launched, part_rr, ctl); });
      finite = rf.finite;
      return rf.iters;
    }
    PcgResult r = ctx->pcgh.run(
        s, max_it,
        [&]() {
          if (warm) {
            // r0 = b - L x_prev (ADMM x-updates change little between iterations); reference = |b|^2 (partials in part_pq)
            yw.zero(s);
            laplacian(v, square, px.p, yw.p, nullptr);
            ctx->allreduce_sum(yw.p, (size_t)n * 3);
            B200_LAUNCH(ctx, ra_pcg_init_warm, nblk, kPcgThreads, 0, n, Minv.p, rhs_vec, yw.p, pr.p, pz.p, pp.p, part_pq, part_rz, part_rr);
          } else {
            B200_LAUNCH(ctx, pcg_init<3>, nblk, kPcgThreads, 0, n, Minv.p, rhs_vec, px.p, pr.p, pz.p, part_rz, part_rr);
          }
          if (use_2lvl) coarse_correct(pr.p, pz.p, part_rz + nblk, nullptr);
        },
        [&](int it) {
          double* d_pub = ctx->pcgh.dots(it - 1);
          B200_LAUNCH(ctx, pcg_direction<3>, nblk, kPcgThreads, 0, n, nblk_t, it, 0, o.pcg_rel_tolerance, pz.p, pp.p, yw.p,
                      ctx->pcgh.dots(it - 2), part_rz, part_rr, (warm && it == 1) ? part_pq : nullptr, d_pub, ctl);
          laplacian(v, square, pp.p, yw.p, ctl);
          ctx->allreduce_sum(yw.p, (size_t)n * 3);
          B200_LAUNCH(ctx, pcg_apply_diag<3>, nblk, kPcgThreads, 0, n, Azero.p, Dzero.p, pp.p, yw.p, pq.p, part_pq, ctl);
          B200_LAUNCH(ctx, pcg_update<3>, nblk, kPcgThreads, 0, n, nblk_t, Minv.p, pp.p, pq.p, px.p, pr.p, pz.p, d_pub, part_pq, part_rz,
                      part_rr, ctx->pcgh.dots(it), ctl);
          if (use_2lvl) coarse_correct(pr.p, pz.p, part_rz + nblk, ctl);
        },
        [&](int launched) { B200_LAUNCH(ctx, pcg_finalize, 1, kPcgThreads, 0, nblk_t, launched, part_rr, ctl); });
    finite = r.finite;
    return r.iters;
  }

  // weights w -> Laplacian diagonal + preconditioner, rhs = A^T diag(w^p) vec
  void prepare_system(int square, const double* vec) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    RAView v = view();
    if (use_csr) {   // gather form: also refreshes the incidence-ordered weights the mat-vec streams
      B200_LAUNCH(ctx, ra_node_setup, cdiv((long long)n * 32, 128), 128, 0, csr(), w.p, square, vec, rhs.p, deg.p);
    } else {
      deg.zero(s);
      B200_CUDA_OK(cudaMemsetAsync(rhs.p, 0, (size_t)n * 3 * sizeof(double), s));
      if (E > 0) B200_LAUNCH(ctx, ra_scatter, cdiv(E, 256), 256, 0, v, w.p, square, vec, rhs.p, deg.p);
    }
    ctx->allreduce_sum(rhs.p, (size_t)n * 3);
    ctx->allreduce_sum(deg.p, (size_t)n * 3);
    B200_LAUNCH(ctx, ra_build_precond, cdiv(n, 256), 256, 0, n, deg.p, Minv.p);
    // coarse matrix P^T L(w^p) P, inverted in place.  The L1 stage keeps the weights of the rows fixed (w_edge, .cc:488-489):
    // its five outer iterations share one inverse
    if (use_2lvl && !(square == 1 && coarse_l1_valid)) {
      coarse_l1_valid = square == 1;
      Ac.zero(s);
      B200_LAUNCH(ctx, ra_coarse_assemble, cdiv(std::max<long long>(E, 1), 256), 256, 0, E, ei.p, ej.p, w.p, square, agg_of.p, nc, Ac.p);
      const dim3 g2(cdiv(nc, 128), nc);
      for (int k = 0; k < nc; ++k) {
        B200_LAUNCH(ctx, ra_gj_eliminate, g2, 128, 0, nc, k, Ac.p);
        B200_LAUNCH(ctx, ra_gj_pivot, 1, 256, 0, nc, k, Ac.p);
      }
    }
  }
  // z += P Ac^-1 P^T r and the coarse share of r.z (partials behind the nblk Jacobi partials)
  void coarse_correct(double* r, double* z, double* part_rz_extra, const b200::PcgCtl* ctl) {
    using namespace b200;
    B200_LAUNCH(ctx, ra_coarse_restrict, nblk_c, 128, 0, coarse(), r, ctl);
    B200_LAUNCH(ctx, ra_coarse_solve, nblk_c, 128, 0, coarse(), part_rz_extra, ctl);
    B200_LAUNCH(ctx, ra_coarse_prolong, cdiv(n, 256), 256, 0, n, coarse(), z, ctl);
  }

  // residuals at theta and the weights of the next system (ra_residuals: mode 0 L1 rows, 1 Geman-McClure, 2 half-norm)
  void residuals(int mode, double sigma2) {
    using namespace b200;
    if (E > 0) B200_LAUNCH(ctx, ra_residuals, cdiv(E, 256), 256, 0, view(), theta.p, mode, sigma2, res.p, w.p, flags.p);
  }

  // the L1 stage's linear system (.cc:479-541): b = W r, |b|^2 in scal[0], z = u = 0; ADMM on |A_w x - b|_1 with
  // A_w^T A_w = L(w^2): rhs = A^T W^2 r = A_w^T b, deg = sum w^2
  void l1_system() {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    B200_CUDA_OK(cudaMemsetAsync(scal.p, 0, 8 * sizeof(double), s));
    if (E > 0) B200_LAUNCH(ctx, ra_weighted_rhs, cdiv(E, 256), 256, 0, view(), w.p, res.p, b.p, scal.p);
    ctx->allreduce_sum(scal.p, 1);   // |b|^2 over all ranks
    z.zero(s);
    u.zero(s);
    prepare_system(1, res.p);
  }

  // one ADMM iteration after the x-update in px: z, u; rhs | svec | uvec (ra_admm_step); scal[1..3] = |A_w x - z - b|^2,
  // |A_w x|^2, |z|^2; scal[4..5] = |svec|^2, |uvec|^2
  void admm_step(double rho) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    B200_CUDA_OK(cudaMemsetAsync(rhs.p, 0, (size_t)n * 9 * sizeof(double), s));
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 1, 0, 3 * sizeof(double), s));
    if (E > 0)
      B200_LAUNCH(ctx, ra_admm_step, cdiv(E, 256), 256, 0, view(), w.p, px.p, b.p, z.p, u.p, rho, rhs.p, rhs.p + (size_t)n * 3,
                  rhs.p + (size_t)n * 6, scal.p);
    ctx->allreduce_sum(rhs.p, (size_t)n * 9);
    ctx->allreduce_sum(scal.p + 1, 3);
    const int nb2 = cdiv((long long)n * 3, 256);
    if (part.n < (size_t)nb2 * 2) part.alloc((size_t)nb2 * 2 + 3 * (size_t)cdiv(n, kPcgThreads));
    B200_LAUNCH(ctx, ra_norm2_partial, nb2, 256, 0, n * 3, rhs.p + (size_t)n * 3, rhs.p + (size_t)n * 6, part.p, part.p + nb2);
    B200_LAUNCH(ctx, ra_norm2_final, 1, 256, 0, nb2, part.p, part.p + nb2, scal.p + 4);
  }

  // theta <- theta (+) step(px); returns (avg step, |step|, nan?)
  void apply_step(double& avg, double& norm, bool& bad) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    B200_CUDA_OK(cudaMemsetAsync(scal.p + 8, 0, 4 * sizeof(double), s));
    B200_LAUNCH(ctx, ra_update, cdiv(n, 256), 256, 0, n, n_frames, theta.p, px.p, scal.p + 8, has_grav ? node_grav.p : nullptr);
    if (n_cams > 0)   // after the frames: the averaging uses the updated frame rotations (.cc:646-693)
      B200_LAUNCH(ctx, ra_update_cams, cdiv((long long)n_cams * 32, 128), 128, 0, n_frames, n_cams, theta.p, px.p, cf_begin.p, cf_list.p);
    B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal + 8, scal.p + 8, 4 * sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    avg = ctx->h_scal[8] / n_frames;   // ComputeAverageStepSize runs over the frames (.cc:758-772)
    norm = std::sqrt(ctx->h_scal[9]);
    bad = ctx->h_scal[10] > 0 || !std::isfinite(ctx->h_scal[9]);
  }

  // ---- test probe (include/b200sfm_testing.h) ----------------------------------------------------------------------
  void test_info(b200sfm_test_ra_info* info, int32_t* h_agg_of) {
    info->n = n; info->n_frames = n_frames; info->n_cams = n_cams; info->has_grav = has_grav;
    info->use_csr = use_csr; info->use_2lvl = use_2lvl; info->fused = fused_iteration(); info->nc = use_2lvl ? nc : 0;
    info->rows_total = rows_total; info->E_total = E_total;
    if (h_agg_of && use_2lvl) {
      agg_of.download(h_agg_of, n, ctx->stream);
      B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    }
  }

  // the system of an L1 outer iteration (square = 1) or of an IRLS iteration (square = 0) at the current theta
  void test_system(int mode, double sigma2, int square, b200sfm_test_ra_system_out* out) {
    cudaStream_t s = ctx->stream;
    residuals(mode, sigma2);
    if (square) l1_system();
    else prepare_system(0, res.p);
    if (out->res) res.download(out->res, (size_t)E * 3, s);
    if (out->w) w.download(out->w, E, s);
    if (out->b && square) b.download(out->b, (size_t)E * 3, s);
    if (out->rhs) rhs.download(out->rhs, (size_t)n * 3, s);
    if (out->deg) deg.download(out->deg, (size_t)n * 3, s);
    if (out->Minv) Minv.download(out->Minv, (size_t)n * 6, s);
    if (out->Ac && use_2lvl) Ac.download(out->Ac, (size_t)nc * nc, s);
    double bn = 0;
    if (square) B200_CUDA_OK(cudaMemcpyAsync(&bn, scal.p, sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    out->b_norm2 = bn;
  }

  // the PCG partials and control record as pcg_solve lays them out, reset
  double* test_pcg_parts(int& nblk, int& nblk_t) {
    nblk = b200::cdiv(n, b200::kPcgThreads);
    nblk_t = nblk + (use_2lvl ? nblk_c : 0);
    ctx->pcgh.ensure(1, (size_t)nblk_t * 3, ctx->world);
    B200_CUDA_OK(cudaMemsetAsync(ctx->pcgh.d_part, 0, (size_t)nblk_t * 3 * sizeof(double), ctx->stream));
    B200_CUDA_OK(cudaMemsetAsync(ctx->pcgh.d_ctl, 0, sizeof(b200::PcgCtl), ctx->stream));
    return ctx->pcgh.d_part;
  }

  // y = L x: the mat-vec of a PCG iteration (fused: ra2_laplacian_dot on the padded copy ra2_direction writes)
  void test_apply(int square, const double* h_x, double* h_y) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    int nblk, nblk_t;
    double* part_pq = test_pcg_parts(nblk, nblk_t);
    PcgCtl* ctl = ctx->pcgh.d_ctl;
    if (fused_iteration()) {
      fused_buffers();
      std::vector<double> x4((size_t)n * 4, 0.0);
      for (int i = 0; i < n; ++i) std::copy(h_x + 3 * (size_t)i, h_x + 3 * (size_t)i + 3, &x4[4 * (size_t)i]);
      p4.upload(x4.data(), (size_t)n * 4, s);
      B200_LAUNCH(ctx, ra2_laplacian_dot, nblk, kLapThreads, 0, csr(), p4.p, pq.p, part_pq, ctl);
      pq.download(h_y, (size_t)n * 3, s);
      B200_CUDA_OK(cudaStreamSynchronize(s));
      return;
    }
    pp.upload(h_x, (size_t)n * 3, s);
    yw.zero(s);
    laplacian(view(), square, pp.p, yw.p, ctl);
    ctx->allreduce_sum(yw.p, (size_t)n * 3);
    B200_LAUNCH(ctx, pcg_apply_diag<3>, nblk, kPcgThreads, 0, n, Azero.p, Dzero.p, pp.p, yw.p, pq.p, part_pq, ctl);
    pq.download(h_y, (size_t)n * 3, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }

  // z = M^-1 r as the first iteration of a cold solve applies it: pcg_init's Jacobi blocks, then the coarse correction
  // (fused: ra2_coarse, and the fold of P zc into the first direction by ra2_direction)
  void test_precond(const double* h_r, double* h_z) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    int nblk, nblk_t;
    double* part = test_pcg_parts(nblk, nblk_t);
    double *part_rz = part + nblk_t, *part_rr = part + 2 * (size_t)nblk_t;
    yw.upload(h_r, (size_t)n * 3, s);
    B200_LAUNCH(ctx, pcg_init<3>, nblk, kPcgThreads, 0, n, Minv.p, yw.p, px.p, pr.p, pz.p, part_rz, part_rr);
    if (fused_iteration()) {
      fused_buffers();
      B200_LAUNCH(ctx, ra2_coarse, nblk_c, 128, 0, coarse(), pr.p, part_rz + nblk, gbar.p, nullptr);
      B200_LAUNCH(ctx, ra2_direction, nblk, kPcgThreads, 0, n, nblk_t, 1, 0.0, pz.p, pp.p, p4.p, zc.p, agg_of.p,
                  ctx->pcgh.dots(-1), part_rz, part_rr, nullptr, ctx->pcgh.dots(0), ctx->pcgh.d_ctl);
      pp.download(h_z, (size_t)n * 3, s);
    } else {
      if (use_2lvl) coarse_correct(pr.p, pz.p, part_rz + nblk, nullptr);
      pz.download(h_z, (size_t)n * 3, s);
    }
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }

  // exactly k iterations of pcg_solve on rhs (tolerance 0), cold or warm-started from h_warm
  int test_pcg(int square, int k, const double* h_warm, double* h_x) {
    cudaStream_t s = ctx->stream;
    b200sfm_ra_opts o{};
    o.pcg_max_iterations = k;
    o.pcg_rel_tolerance = 0.0;
    if (h_warm) px.upload(h_warm, (size_t)n * 3, s);
    bool finite = true;
    const int it = pcg_solve(o, square, rhs.p, finite, h_warm != nullptr);
    px.download(h_x, (size_t)n * 3, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return it;
  }

  void test_admm_step(double rho, const double* h_x, const double* h_b, double* h_z, double* h_u, double* h_rsu,
                      double* h_norms) {
    cudaStream_t s = ctx->stream;
    px.upload(h_x, (size_t)n * 3, s);
    b.upload(h_b, (size_t)E * 3, s);
    z.upload(h_z, (size_t)E * 3, s);
    u.upload(h_u, (size_t)E * 3, s);
    admm_step(rho);
    z.download(h_z, (size_t)E * 3, s);
    u.download(h_u, (size_t)E * 3, s);
    rhs.download(h_rsu, (size_t)n * 9, s);
    B200_CUDA_OK(cudaMemcpyAsync(h_norms, scal.p + 1, 5 * sizeof(double), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
  }

  void test_update(const double* h_step, double* h_theta, double* sums) {
    px.upload(h_step, (size_t)n * 3, ctx->stream);
    double avg, norm;
    bool bad;
    apply_step(avg, norm, bad);
    theta.download(h_theta, (size_t)n * 3, ctx->stream);
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    sums[0] = avg; sums[1] = norm; sums[2] = bad ? 1.0 : 0.0;
  }

  int solve(const b200sfm_ra_opts& o, b200sfm_ra_stats* st) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    const long long launches0 = ctx->launches;
    cudaEvent_t ev0, ev1;
    B200_CUDA_OK(cudaEventCreate(&ev0));
    B200_CUDA_OK(cudaEventCreate(&ev1));
    B200_CUDA_OK(cudaEventRecord(ev0, s));
    b200sfm_ra_stats local{};
    local.usable = 1;
    local.num_edges = E_real;
    flags.zero(s);
    bool failed = false;
    // ---- L1 (.cc:479-541) ----------------------------------------------------------
    if (o.max_num_l1_iterations > 0) {
      residuals(0, 0.0);
      double last_norm = 0, curr_norm = 0;
      for (int it = 0; it < o.max_num_l1_iterations && !failed; ++it) {
        last_norm = curr_norm;
        l1_system();
        double b_norm2 = 0;
        const double eps_pri_thr = std::sqrt((double)rows_total) * o.l1_absolute_tolerance;   // sqrt(A.rows())
        const double eps_dual_thr = std::sqrt(3.0 * n) * o.l1_absolute_tolerance;
        for (int k = 0; k < o.l1_max_admm_iterations; ++k) {
          bool finite = true;
          local.pcg_iterations += pcg_solve(o, 1, rhs.p, finite, /*warm=*/k > 0);
          ++local.admm_iterations;
          if (!finite) { failed = true; break; }
          admm_step(o.l1_rho);
          B200_CUDA_OK(cudaMemcpyAsync(ctx->h_scal, scal.p, 8 * sizeof(double), cudaMemcpyDeviceToHost, s));
          B200_CUDA_OK(cudaStreamSynchronize(s));
          const double* h = ctx->h_scal;
          b_norm2 = h[0];
          const double r_norm = std::sqrt(h[1]), s_norm = o.l1_rho * std::sqrt(h[4]);
          const double eps_pri = eps_pri_thr + o.l1_relative_tolerance * std::sqrt(std::max(b_norm2, std::max(h[2], h[3])));
          const double eps_dual = eps_dual_thr + o.l1_relative_tolerance * o.l1_rho * std::sqrt(h[5]);
          if (r_norm < eps_pri && s_norm < eps_dual) break;
        }
        if (failed) break;
        double avg, norm;
        bool bad;
        apply_step(avg, norm, bad);                                    // UpdateGlobalRotations (.cc:523)
        if (bad) { failed = true; break; }                             // .cc:508-512
        curr_norm = norm;
        residuals(0, 0.0);                                             // .cc:524
        ++local.l1_iterations;
        if (avg < o.l1_step_convergence_threshold || std::fabs(last_norm - curr_norm) < kRaEps) break;   // .cc:528-535
      }
    }
    // ---- IRLS (.cc:543-625) --------------------------------------------------------
    if (!failed && o.max_num_irls_iterations > 0) {
      const double sigma = o.irls_loss_parameter_sigma * M_PI / 180.0;
      const int mode = (o.weight_type == 1) ? 2 : 1;
      for (int it = 0; it < o.max_num_irls_iterations; ++it) {
        residuals(mode, sigma * sigma);
        {
          int hflag = 0;
          B200_CUDA_OK(cudaMemcpyAsync(&hflag, flags.p, sizeof(int), cudaMemcpyDeviceToHost, s));
          B200_CUDA_OK(cudaStreamSynchronize(s));
          if (hflag) { failed = true; break; }                         // "nan weight!" .cc:590-593
        }
        prepare_system(0, res.p);                                      // A^T W A, A^T W r (.cc:603-611)
        bool finite = true;
        local.pcg_iterations += pcg_solve(o, 0, rhs.p, finite);
        if (!finite) { failed = true; break; }
        double avg, norm;
        bool bad;
        apply_step(avg, norm, bad);
        if (bad) { failed = true; break; }
        ++local.irls_iterations;
        if (avg < o.irls_step_convergence_threshold) break;            // .cc:616-620
      }
    }
    B200_CUDA_OK(cudaEventRecord(ev1, s));
    B200_CUDA_OK(cudaEventSynchronize(ev1));
    float ms = 0;
    B200_CUDA_OK(cudaEventElapsedTime(&ms, ev0, ev1));
    cudaEventDestroy(ev0);
    cudaEventDestroy(ev1);
    local.ms_total = ms;
    local.usable = failed ? 0 : 1;
    local.kernel_launches = ctx->launches - launches0;
    if (st) *st = local;
    return B200SFM_OK;
  }
};
