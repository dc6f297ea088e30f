// common.cuh -- shared device helpers for the b200sfm kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

namespace b200 {

// Tunables of the point-order kernels (overridable with -D for sweeps)
#ifndef B200_TILE
#define B200_TILE 128
#endif
#ifndef B200_K1_MIN_CTAS
#define B200_K1_MIN_CTAS 5
#endif
#ifndef B200_K3_MIN_CTAS
#define B200_K3_MIN_CTAS 8
#endif
#ifndef B200_PA_MIN_CTAS   // v2 pass A: 12 CTAs x 128 threads (40 registers, no spills)
#define B200_PA_MIN_CTAS 12
#endif
#ifndef B200_LC_MIN_CTAS   // v2 camera-order linearisation
#define B200_LC_MIN_CTAS 3   // the register-pipelined kernel needs ~168 registers without spills (3 CTAs); 4 CTAs was slower on H100
#endif
#ifndef B200_PB_MIN_CTAS
#define B200_PB_MIN_CTAS 4   // pass B recomputes each observation: 126 registers at 4; 5 and 6 spilled and were slower (DESIGN §6)
#endif
#ifndef B200_SD_MIN_CTAS   // v2 camera-order Schur-Jacobi diagonal: 168 registers, no spills, 12 warps / SM
#define B200_SD_MIN_CTAS 3
#endif
#ifndef B200_E1_MIN_CTAS   // ELL point-side linearisation (one thread per point): CTAs of 128 threads per SM
#define B200_E1_MIN_CTAS 4   // with the register pipeline: ~122 registers, no spills, 16 warps / SM (H100 sweep: 3 equal, 5 slower)
#endif
#ifndef B200_E1_PIPE       // ELL linearisation: 1 = register software pipeline (next camera record / index in flight), 0 = plain loop
#define B200_E1_PIPE 1
#endif
#ifndef B200_EA_MIN_CTAS   // ELL pass A (mat-vec)
#define B200_EA_MIN_CTAS 8
#endif
#ifndef B200_EA2_MIN_CTAS  // ELL pass A, back-substitution epilogue
#define B200_EA2_MIN_CTAS 6
#endif
#ifndef B200_STREAM_HINTS  // evict-first loads/stores on the once-per-pass streams so the gathered arrays stay in L2
#define B200_STREAM_HINTS 1
#endif
constexpr int kTile = B200_TILE; // observations per point-order tile == threads per CTA
constexpr int kTilePts = 64;     // max points per tile (bounds the per-point shared-memory arrays)
constexpr int kWDoubles = 18;    // W block of one observation: 6x3 doubles, row-major
constexpr int kWBytes = kWDoubles * 8;

#define B200_CUDA_OK(expr)                                                                     \
  do {                                                                                         \
    cudaError_t err__ = (expr);                                                                \
    if (err__ != cudaSuccess) {                                                                \
      throw ::b200::CudaError(std::string(#expr) + ": " + cudaGetErrorString(err__), __LINE__); \
    }                                                                                          \
  } while (0)

struct CudaError {
  std::string msg;
  int line;
  CudaError(std::string m, int l) : msg(std::move(m)), line(l) {}
};
// caller-supplied indices out of range (found on the host or by a device-side check): B200SFM_ERR_INVALID_ARG
struct InvalidInput {
  std::string msg;
};

// ---------------------------------------------------------------------------
// TMA 1-D bulk copies (cp.async.bulk) + mbarrier.  The W tiles are contiguous
// arrays of 144-byte rows, so a plain bulk copy (SASS UBLKCP) moves a whole
// tile between HBM and shared memory without touching the LSU/L1 path.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared, completion signalled on the mbarrier (bytes % 16 == 0, 16-B aligned)
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// same, with an L2 evict-first policy: a once-per-pass stream must not push the gathered arrays out of L2
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void tma_load_1d_stream(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
#if B200_STREAM_HINTS
  const uint64_t pol = l2_policy_evict_first();
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
#else
  tma_load_1d(smem_dst, gsrc, bytes, bar);
#endif
}
// software prefetch into L1 (no register is tied up while the line travels): used one / two loop iterations ahead of
// the dependent index -> record gathers of the linearisation kernels
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
// 32-B read-only gather as two 128-bit loads (LDG.E.128.CONSTANT; sm_90 has no wider global access).  p must be 32-B
// aligned, so both halves fall in the same 32-B sector: the record still costs one sector of traffic.
__device__ __forceinline__ void ld_nc_256(const double* p, double& a, double& b, double& c, double& d) {
  asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(a), "=d"(b) : "l"(p));
  asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(c), "=d"(d) : "l"(p + 2));
}
// One 32-B read-only gather as a value.  p must be 32-B aligned.
#ifndef B200_REC_CG
#define B200_REC_CG 0
#endif
__device__ __forceinline__ double4 ld_rec32(const double* p) {
  double4 r;
#if B200_REC_CG   // experiment: cache the gathered records in L2 only
  asm("ld.global.cg.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
  asm("ld.global.cg.v2.f64 {%0, %1}, [%2];" : "=d"(r.z), "=d"(r.w) : "l"(p + 2));
#else
  asm("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p));
  asm("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(r.z), "=d"(r.w) : "l"(p + 2));
#endif
  return r;
}
// 32-B store as two 128-bit stores (p 32-B aligned)
__device__ __forceinline__ void st_rec32(double* p, double a, double b, double c, double d) {
  asm volatile("st.global.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(a), "d"(b) : "memory");
  asm volatile("st.global.v2.f64 [%0], {%1, %2};" ::"l"(p + 2), "d"(c), "d"(d) : "memory");
}
// streaming (evict-first) scalar accesses
template <class T>
__device__ __forceinline__ T ld_stream(const T* p) {
#if B200_STREAM_HINTS
  return __ldcs(p);
#else
  return *p;
#endif
}
template <class T>
__device__ __forceinline__ void st_stream(T* p, T v) {
#if B200_STREAM_HINTS
  __stcs(p, v);
#else
  *p = v;
#endif
}
// gathered-array accesses that should stay L2-resident between the passes (evict-last policy)
#ifndef B200_KEEP_HINTS
#define B200_KEEP_HINTS 0
#endif
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ double4 ld_keep4(const double* p, uint64_t pol) {
#if B200_KEEP_HINTS
  double4 v;
  asm volatile("ld.global.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(v.x), "=d"(v.y) : "l"(p), "l"(pol));
  asm volatile("ld.global.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(v.z), "=d"(v.w) : "l"(p + 2), "l"(pol));
  return v;
#else
  return ld_rec32(p);   // one 32-B gather (the array is written by the previous kernel, never by this one)
#endif
}
__device__ __forceinline__ void st_keep4(double* p, double4 v, uint64_t pol) {
#if B200_KEEP_HINTS
  asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v.x), "d"(v.y), "l"(pol) : "memory");
  asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p + 2), "d"(v.z), "d"(v.w), "l"(pol) : "memory");
#else
  st_rec32(p, v.x, v.y, v.z, v.w);
#endif
}
// shared -> global (bulk async group)
__device__ __forceinline__ void tma_store_1d(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// Reduce-scatter of K <= 32 per-lane values: the warp total of value k ends in lanes [k * S, (k + 1) * S), S =
// warp_rs_stride<K>(), so lane l returns the total of value l / S.  Recursive halving with partners at xor distances
// 16, 8, 4, 2, 1 (K padded with zeros to a power of two Kp; once one value is left the remaining distances are plain
// butterfly steps): Kp - 1 + (5 - log2 Kp) exchanges in place of warp_sum's 5 K.  Every partial is the sum of the same
// two operands warp_sum adds at that distance, so each total is bit-identical to warp_sum's.
template <int K>
__host__ __device__ constexpr int warp_rs_stride() {
  static_assert(K >= 1 && K <= 32, "warp_reduce_scatter takes 1..32 values");
  return K <= 1 ? 32 : K <= 2 ? 16 : K <= 4 ? 8 : K <= 8 ? 4 : K <= 16 ? 2 : 1;
}
// one level of warp_reduce_scatter: M values per lane, partner at xor distance D (a template per level, so that every
// index into a[] is a constant and the array stays in registers)
template <int M, int D>
__device__ __forceinline__ double warp_rs_level(double* a, int lane) {
  if constexpr (D == 0) {
    return a[0];
  } else if constexpr (M > 1) {   // keep the half of the values selected by lane bit D, send the other half
    const bool hi = lane & D;
#pragma unroll
    for (int j = 0; j < M / 2; ++j) {
      const double keep = hi ? a[M / 2 + j] : a[j], send = hi ? a[j] : a[M / 2 + j];
      a[j] = keep + __shfl_xor_sync(0xffffffffu, send, D);
    }
    return warp_rs_level<M / 2, D / 2>(a, lane);
  } else {
    a[0] += __shfl_xor_sync(0xffffffffu, a[0], D);
    return warp_rs_level<1, D / 2>(a, lane);
  }
}
template <int K>
__device__ __forceinline__ double warp_reduce_scatter(const double (&v)[K]) {
  constexpr int Kp = 32 / warp_rs_stride<K>();
  double a[Kp];
#pragma unroll
  for (int k = 0; k < Kp; ++k) a[k] = k < K ? v[k] : 0.0;
  return warp_rs_level<Kp, 16>(a, threadIdx.x & 31);
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Sum over the CTA; result valid in thread 0.  `scratch` holds >= 32 doubles.
__device__ __forceinline__ double block_sum(double v, double* scratch) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) scratch[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  v = (threadIdx.x < nw) ? scratch[threadIdx.x] : 0.0;
  if (w == 0) v = warp_sum(v);
  return v;
}
__device__ __forceinline__ double block_max(double v, double* scratch) {
  v = warp_max(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) scratch[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  v = (threadIdx.x < nw) ? scratch[threadIdx.x] : 0.0;
  if (w == 0) v = warp_max(v);
  return v;
}
// atomic max for non-negative doubles (bit pattern order == value order)
__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {
  atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

// ---------------------------------------------------------------------------
// small dense algebra
// ---------------------------------------------------------------------------
// symmetric 3x3 stored as (00,01,02,11,12,22); returns false if not invertible
__device__ __forceinline__ bool sym3_inverse(const double a[6], double inv[6]) {
  const double c00 = a[3] * a[5] - a[4] * a[4];
  const double c01 = a[2] * a[4] - a[1] * a[5];
  const double c02 = a[1] * a[4] - a[2] * a[3];
  const double det = a[0] * c00 + a[1] * c01 + a[2] * c02;
  if (!(fabs(det) > 0.0)) {
    inv[0] = inv[1] = inv[2] = inv[3] = inv[4] = inv[5] = 0.0;
    return false;
  }
  const double id = 1.0 / det;
  inv[0] = c00 * id;
  inv[1] = c01 * id;
  inv[2] = c02 * id;
  inv[3] = (a[0] * a[5] - a[2] * a[2]) * id;
  inv[4] = (a[1] * a[2] - a[0] * a[4]) * id;
  inv[5] = (a[0] * a[3] - a[1] * a[1]) * id;
  return true;
}
__device__ __forceinline__ void sym3_mul(const double a[6], const double v[3], double out[3]) {
  out[0] = a[0] * v[0] + a[1] * v[1] + a[2] * v[2];
  out[1] = a[1] * v[0] + a[3] * v[1] + a[4] * v[2];
  out[2] = a[2] * v[0] + a[4] * v[1] + a[5] * v[2];
}

// index of (i,j), i<=j, in the packed upper triangle of an n x n symmetric matrix
__host__ __device__ constexpr int sym_idx(int n, int i, int j) { return i * n - (i * (i - 1)) / 2 + (j - i); }

// Inverse of a symmetric positive-definite n x n matrix given as packed upper
// triangle, via Cholesky.  Non-positive pivots are replaced by 1 (the block
// then acts as identity on that dof) -- only reachable for dofs that carry no
// observation.
template <int n>
__device__ __forceinline__ void spd_inverse_packed(const double* a, double* inv) {
  double L[n][n];
#pragma unroll
  for (int i = 0; i < n; ++i)
#pragma unroll
    for (int j = 0; j < n; ++j) L[i][j] = 0.0;
#pragma unroll
  for (int j = 0; j < n; ++j) {
    double d = a[sym_idx(n, j, j)];
#pragma unroll
    for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
    const bool ok = d > 0.0;
    const double ljj = ok ? sqrt(d) : 1.0;
    L[j][j] = ljj;
    const double il = 1.0 / ljj;
#pragma unroll
    for (int i = j + 1; i < n; ++i) {
      double s = a[sym_idx(n, j, i)];
#pragma unroll
      for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
      L[i][j] = ok ? s * il : 0.0;
    }
  }
  // Linv (lower triangular)
  double Li[n][n];
#pragma unroll
  for (int i = 0; i < n; ++i)
#pragma unroll
    for (int j = 0; j < n; ++j) Li[i][j] = 0.0;
#pragma unroll
  for (int j = 0; j < n; ++j) {
    Li[j][j] = 1.0 / L[j][j];
#pragma unroll
    for (int i = j + 1; i < n; ++i) {
      double s = 0.0;
#pragma unroll
      for (int k = j; k < i; ++k) s -= L[i][k] * Li[k][j];
      Li[i][j] = s / L[i][i];
    }
  }
  // inv = Li^T Li
#pragma unroll
  for (int i = 0; i < n; ++i)
#pragma unroll
    for (int j = i; j < n; ++j) {
      double s = 0.0;
#pragma unroll
      for (int k = j; k < n; ++k) s += Li[k][i] * Li[k][j];
      inv[sym_idx(n, i, j)] = s;
    }
}

template <int n>
__device__ __forceinline__ void sym_packed_mul(const double* a, const double* v, double* out) {
#pragma unroll
  for (int i = 0; i < n; ++i) {
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < n; ++j) s += a[i <= j ? sym_idx(n, i, j) : sym_idx(n, j, i)] * v[j];
    out[i] = s;
  }
}

// ---------------------------------------------------------------------------
// SO(3)
// ---------------------------------------------------------------------------
// rotation matrix (row-major) of a unit quaternion (x,y,z,w)
__device__ __forceinline__ void quat_to_R(const double q[4], double R[9]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  R[0] = 1 - 2 * (y * y + z * z);
  R[1] = 2 * (x * y - z * w);
  R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);
  R[4] = 1 - 2 * (x * x + z * z);
  R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);
  R[7] = 2 * (y * z + x * w);
  R[8] = 1 - 2 * (x * x + y * y);
}

}  // namespace b200
