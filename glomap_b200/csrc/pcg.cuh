// pcg.cuh -- block-preconditioned conjugate gradients on the reduced camera
// system with the loop control ON THE DEVICE.  The reference factors this system
// with CHOLMOD (bundle_adjustment.cc:94-96, global_positioning.cc:551-559);
// north_star mandates PCG with one all-reduce per mat-vec.
//
// Control flow.  A PcgCtl record in device memory holds the convergence state.
// The first kernel of iteration `it` (pcg_direction) re-sums the partial inner
// products of iteration it-1 in a fixed order, evaluates the stopping rule and,
// when it fires, sets ctl->done; every later kernel of the solve starts with
// `if (ctl->done) return`.  The host therefore never has to wait for an
// iteration before it launches the next one: it keeps `depth` iterations queued
// ahead of the one whose control record it has read back (PcgHost::run), so the
// GPU does not idle on a device->host->device round trip per iteration (at 8
// GPUs, where the per-GPU work is small, that round trip dominates).  depth = 1 is
// the classic "synchronise every iteration" loop.
//
// All inner products are DETERMINISTIC: every CTA writes its partial sum to
// part[which][blockIdx.x] and the consuming kernel re-sums the partials in a
// fixed order.  With replicated camera-sized vectors alpha, beta and the
// stopping rule are bit-identical on every rank, all ranks set `done` in the
// same iteration and launch the same number of collectives.
//
// Scalars: dots[k][0] = p.q of iteration k, dots[k][1] = r.z and dots[k][2] =
// r.r after k iterations (k = 0: initial values).
#pragma once
#include <algorithm>

#include "common.cuh"

namespace b200 {

constexpr int kPcgThreads = 128;

struct PcgCtl {
  int done;     // 0 running, 1 converged, 2 non-finite residual, 3 iteration cap
  int iters;    // iterations whose update is part of x
  int pad0, pad1;
  double tol2;  // rel_tol^2 * reference
  double rr0;   // |r_0|^2
};

// fixed-order sum of n partials by the first warp of the CTA; result broadcast
// through shared memory to all threads.
__device__ __forceinline__ double sum_partials(const double* __restrict__ part, int n, double* sh) {
  if (threadIdx.x < 32) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 32) s += part[i];
    s = warp_sum(s);
    if (threadIdx.x == 0) *sh = s;
  }
  __syncthreads();
  return *sh;
}
// CTA-level deterministic sum -> part[blockIdx.x]
__device__ __forceinline__ void write_partial(double v, double* __restrict__ part, double* scratch) {
  v = block_sum(v, scratch);
  if (threadIdx.x == 0) part[blockIdx.x] = v;
}

// q_c = (A_c + diag(D_c)) p_c + yw_c ; part_pq[blk] = partial p.q
//   fixed (optional, one entry per block): blocks with fixed[c] < 0 are identity rows, q_c = p_c, whatever yw holds
template <int B>
__global__ void __launch_bounds__(kPcgThreads) pcg_apply_diag(int nb, const double* __restrict__ A,
                                                              const double* __restrict__ D,
                                                              const double* __restrict__ p,
                                                              const double* __restrict__ yw, double* __restrict__ q,
                                                              double* __restrict__ part_pq,
                                                              const PcgCtl* __restrict__ ctl,
                                                              const double* __restrict__ fixed = nullptr) {
  constexpr int NP = B * (B + 1) / 2;
  __shared__ double scratch[32];
  if (ctl->done) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  double pq = 0.0;
  if (c < nb && fixed && fixed[c] < 0.0) {
#pragma unroll
    for (int k = 0; k < B; ++k) {
      const double pv = p[(size_t)c * B + k];
      q[(size_t)c * B + k] = pv;
      pq += pv * pv;
    }
  } else if (c < nb) {
    double a[NP], pv[B], out[B];
#pragma unroll
    for (int k = 0; k < NP; ++k) a[k] = A ? A[(size_t)c * NP + k] : 0.0;   // A == nullptr: the mat-vec already holds A p
#pragma unroll
    for (int k = 0; k < B; ++k) pv[k] = p[(size_t)c * B + k];
    sym_packed_mul<B>(a, pv, out);
#pragma unroll
    for (int k = 0; k < B; ++k) {
      const double qv = out[k] + D[(size_t)c * B + k] * pv[k] + (yw ? yw[(size_t)c * B + k] : 0.0);
      q[(size_t)c * B + k] = qv;
      pq += qv * pv[k];
    }
  }
  write_partial(pq, part_pq, scratch);
}

// alpha = rz / pq; x += alpha p; r -= alpha q; z = Minv r; partial r.z, r.r
//   dots_prev = dots[it-1] (r.z published by pcg_direction of this iteration), dots_it = dots[it] (receives p.q)
template <int B>
__global__ void __launch_bounds__(kPcgThreads) pcg_update(int nb, int nblk, const double* __restrict__ Minv,
                                                          const double* __restrict__ p, const double* __restrict__ q,
                                                          double* __restrict__ x, double* __restrict__ r,
                                                          double* __restrict__ z, const double* __restrict__ dots_prev,
                                                          const double* __restrict__ part_pq,
                                                          double* __restrict__ part_rz, double* __restrict__ part_rr,
                                                          double* __restrict__ dots_it,
                                                          const PcgCtl* __restrict__ ctl) {
  constexpr int NP = B * (B + 1) / 2;
  __shared__ double scratch[32];
  __shared__ double sh;
  if (ctl->done) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const double pq = sum_partials(part_pq, nblk, &sh);
  const double rz = dots_prev[1];
  const double alpha = (pq > 0.0) ? rz / pq : 0.0;
  if (blockIdx.x == 0 && threadIdx.x == 0) dots_it[0] = pq;
  double rzn = 0.0, rr = 0.0;
  if (c < nb) {
    double m[NP], rv[B], zv[B];
#pragma unroll
    for (int k = 0; k < NP; ++k) m[k] = Minv[(size_t)c * NP + k];
#pragma unroll
    for (int k = 0; k < B; ++k) {
      const size_t i = (size_t)c * B + k;
      x[i] += alpha * p[i];
      rv[k] = r[i] - alpha * q[i];
      r[i] = rv[k];
      rr += rv[k] * rv[k];
    }
    sym_packed_mul<B>(m, rv, zv);
#pragma unroll
    for (int k = 0; k < B; ++k) {
      z[(size_t)c * B + k] = zv[k];
      rzn += rv[k] * zv[k];
    }
  }
  write_partial(rzn, part_rz, scratch);
  write_partial(rr, part_rr, scratch);
}

// Head of iteration `it` (>= 1), executed identically by every CTA: publish r.z / r.r after it-1 iterations, evaluate
// the stopping rule on them and return beta.  Returns false when the solve is over (ctl->done set by CTA 0).
//   dots_pub = dots[it-1]; dots_pp = dots[it-2] (it >= 2); part_ref: optional partials of the convergence reference
//   (warm-started solves measure against |b|^2 instead of |r_0|^2)
__device__ __forceinline__ bool pcg_direction_head(int nblk, int it, int min_it, double rel_tol,
                                                   const double* __restrict__ dots_pp,
                                                   const double* __restrict__ part_rz,
                                                   const double* __restrict__ part_rr,
                                                   const double* __restrict__ part_ref, double* __restrict__ dots_pub,
                                                   PcgCtl* __restrict__ ctl, double* sh3, double& beta) {
  if (ctl->done) return false;   // set by an earlier launch only (this launch decides below, identically in every CTA)
  const double rzn = sum_partials(part_rz, nblk, sh3);
  const double rr = sum_partials(part_rr, nblk, sh3 + 1);
  double tol2;
  bool stop;
  int code = 1;
  if (it == 1) {
    const double ref2 = part_ref ? sum_partials(part_ref, nblk, sh3 + 2) : rr;
    tol2 = rel_tol * rel_tol * ref2;
    stop = !(ref2 > 0.0) || !isfinite(rr) || (min_it <= 0 && rr <= tol2);
    if (!isfinite(rr)) code = 2;
    beta = 0.0;
  } else {
    tol2 = ctl->tol2;
    stop = !isfinite(rr) || (it - 1 >= min_it && rr <= tol2);
    if (!isfinite(rr)) code = 2;
    const double rz = dots_pp[1];
    beta = (rz > 0.0) ? rzn / rz : 0.0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    dots_pub[1] = rzn;
    dots_pub[2] = rr;
    if (it == 1) {
      ctl->tol2 = tol2;
      ctl->rr0 = rr;
    }
    if (stop) {
      ctl->iters = it - 1;
      ctl->done = code;
    }
  }
  return !stop;
}

// p = z + beta p (it == 1: p = z); clears the mat-vec accumulator yw
template <int B>
__global__ void __launch_bounds__(kPcgThreads) pcg_direction(int nb, int nblk, int it, int min_it, double rel_tol,
                                                             const double* __restrict__ z, double* __restrict__ p,
                                                             double* __restrict__ yw, const double* __restrict__ dots_pp,
                                                             const double* __restrict__ part_rz,
                                                             const double* __restrict__ part_rr,
                                                             const double* __restrict__ part_ref,
                                                             double* __restrict__ dots_pub, PcgCtl* __restrict__ ctl) {
  __shared__ double sh3[3];
  double beta;
  if (!pcg_direction_head(nblk, it, min_it, rel_tol, dots_pp, part_rz, part_rr, part_ref, dots_pub, ctl, sh3, beta)) return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < nb) {
#pragma unroll
    for (int k = 0; k < B; ++k) {
      const size_t i = (size_t)c * B + k;
      p[i] = (it == 1) ? z[i] : z[i] + beta * p[i];
      if (yw) yw[i] = 0.0;
    }
  }
}

// x = 0; r = b; z = Minv r; partial r.z, r.r   (p is set by pcg_direction of iteration 1)
template <int B>
__global__ void __launch_bounds__(kPcgThreads) pcg_init(int nb, const double* __restrict__ Minv,
                                                        const double* __restrict__ b, double* __restrict__ x,
                                                        double* __restrict__ r, double* __restrict__ z,
                                                        double* __restrict__ part_rz, double* __restrict__ part_rr) {
  constexpr int NP = B * (B + 1) / 2;
  __shared__ double scratch[32];
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  double rz = 0.0, rr = 0.0;
  if (c < nb) {
    double m[NP], rv[B], zv[B];
#pragma unroll
    for (int k = 0; k < NP; ++k) m[k] = Minv[(size_t)c * NP + k];
#pragma unroll
    for (int k = 0; k < B; ++k) {
      const size_t i = (size_t)c * B + k;
      rv[k] = b[i];
      x[i] = 0.0;
      r[i] = rv[k];
      rr += rv[k] * rv[k];
    }
    sym_packed_mul<B>(m, rv, zv);
#pragma unroll
    for (int k = 0; k < B; ++k) {
      const size_t i = (size_t)c * B + k;
      z[i] = zv[k];
      rz += rv[k] * zv[k];
    }
  }
  write_partial(rz, part_rz, scratch);
  write_partial(rr, part_rr, scratch);
}

// After the last launched iteration: the cap was reached without the stopping rule firing (single CTA).
__global__ void __launch_bounds__(kPcgThreads) pcg_finalize(int nblk, int launched, const double* __restrict__ part_rr,
                                                            PcgCtl* __restrict__ ctl) {
  __shared__ double sh;
  if (ctl->done) return;
  const double rr = sum_partials(part_rr, nblk, &sh);
  if (threadIdx.x == 0) {
    ctl->iters = launched;
    ctl->done = isfinite(rr) ? 3 : 2;
  }
}

// ---------------------------------------------------------------------------
// host side: speculative launch of the iterations
// ---------------------------------------------------------------------------
struct PcgResult {
  int iters = 0;
  int launched = 0;
  bool finite = true;
  double rr0 = 0;
};

struct PcgHost {
  static constexpr int kMaxDepth = 8;
  PcgCtl* h_slots = nullptr;   // pinned
  cudaEvent_t ev[kMaxDepth + 1] = {};
  PcgCtl* d_ctl = nullptr;
  double* d_dots = nullptr;
  double* d_part = nullptr;
  size_t n_dots = 0, n_part = 0;
  int depth = 2;
  bool depth_from_env = false;
  // Iterations queued ahead of the read-back.  One GPU: the mat-vec (1.6 ms at config 4 on an H100) dwarfs the round trip
  // and depth 2 gains nothing (127.0 vs 127.1 ms per config-4 solve, one H100 SXM at 700 W), so the loop synchronises every
  // iteration.  Several GPUs: the per-iteration work shrinks with
  // 1 / world while the round trip does not, and an all-reduce sits in every iteration -- two iterations are kept in flight.
  void configure(int world) {
    if (!depth_from_env) depth = world > 1 ? 2 : 1;
  }

  PcgHost() = default;
  PcgHost(const PcgHost&) = delete;
  PcgHost& operator=(const PcgHost&) = delete;
  ~PcgHost() {
    if (h_slots) cudaFreeHost(h_slots);
    for (auto e : ev)
      if (e) cudaEventDestroy(e);
    if (d_ctl) cudaFree(d_ctl);
    if (d_dots) cudaFree(d_dots);
    if (d_part) cudaFree(d_part);
  }
  // dots: (max_it + 2) x 4 doubles; part: n_part doubles (caller's layout)
  void ensure(int max_it, size_t part_doubles, int world = 1) {
    if (!h_slots) {
      B200_CUDA_OK(cudaMallocHost(&h_slots, sizeof(PcgCtl) * (kMaxDepth + 1)));
      for (auto& e : ev) B200_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      B200_CUDA_OK(cudaMalloc(&d_ctl, sizeof(PcgCtl)));
      const char* d = getenv("B200SFM_PCG_DEPTH");
      if (d) {
        depth = std::min(std::max(atoi(d), 1), (int)kMaxDepth);
        depth_from_env = true;
      }
    }
    configure(world);
    const size_t need = (size_t)(max_it + 2) * 4;
    if (n_dots < need) {
      if (d_dots) cudaFree(d_dots);
      B200_CUDA_OK(cudaMalloc(&d_dots, need * sizeof(double)));
      n_dots = need;
    }
    if (n_part < part_doubles) {
      if (d_part) cudaFree(d_part);
      B200_CUDA_OK(cudaMalloc(&d_part, part_doubles * sizeof(double)));
      n_part = part_doubles;
    }
  }
  double* dots(int k) const { return d_dots + (size_t)std::max(k, 0) * 4; }

  // init(): launches the kernels that leave r, z and the partial r.z / r.r of iteration 0;
  // iter(it): launches iteration it = direction(it), mat-vec (+ all-reduce), apply_diag, update(it);
  // final(launched): launches pcg_finalize.
  template <class Init, class Iter, class Final>
  PcgResult run(cudaStream_t s, int max_it, Init&& init, Iter&& iter, Final&& final) {
    B200_CUDA_OK(cudaMemsetAsync(d_ctl, 0, sizeof(PcgCtl), s));
    init();
    const int nslots = depth + 1;
    int launched = 0;
    for (int it = 1; it <= max_it; ++it) {
      if (it > depth) {
        const int slot = (it - depth) % nslots;
        B200_CUDA_OK(cudaEventSynchronize(ev[slot]));
        if (h_slots[slot].done) break;
      }
      iter(it);
      const int slot = it % nslots;
      B200_CUDA_OK(cudaMemcpyAsync(&h_slots[slot], d_ctl, sizeof(PcgCtl), cudaMemcpyDeviceToHost, s));
      B200_CUDA_OK(cudaEventRecord(ev[slot], s));
      launched = it;
    }
    final(launched);
    B200_CUDA_OK(cudaMemcpyAsync(&h_slots[0], d_ctl, sizeof(PcgCtl), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    PcgResult r;
    r.iters = h_slots[0].iters;
    r.launched = launched;
    r.finite = h_slots[0].done != 2;
    r.rr0 = h_slots[0].rr0;
    return r;
  }
};

}  // namespace b200
