// prune_kernels.cuh -- device side of PruneWeaklyConnectedImages (glomap/processors/reconstruction_pruning.cc:6-131),
// stage 8 of GlobalMapper::Solve, with EstablishStrongClusters (processors/view_graph_manipulation.cc:70-176),
// KeepLargestConnectedComponents and MarkConnectedComponents (scene/view_graph.cc:56-126), all in frame space
// (frames 0..F-1).  Integer work only, no floating-point atomics, so the result is exact and reproducible:
//   1. per observation: range check of its frame; per-frame observation count over the tracks longer than 2 (:14-21)
//   2. covisibility: one 64-bit key lo * F + hi per (track, i < j) slot whose two frames differ (:22-34).  The global
//      slot range (prefix sum of L (L - 1) / 2 over the tracks longer than 2) is cut into passes of at most
//      max_pair_keys_per_pass slots, by slot index, so a track longer than a pass is split too.  Each pass radix-sorts
//      its keys over the significant bits only (end_bit = bit width of F^2 - 1) and run-length encodes them; the runs of
//      all passes are merged by one more sort + reduce-by-key
//   3. visibility edges: count >= 5 and both frames' observation counts >= min_num_observations (:38-60); median and
//      MAD of the edge weights by device sorts (:106-127)
//   4. union-find (track_kernels.cuh: trk_hook hooks the larger root under the smaller, so a set's root is its smallest
//      frame index and every component is named canonically) for the largest component (5a), the strong edges (5b),
//      the merge passes over root pairs (5c) and the final components of the surviving edges (5d-e)
#pragma once
#include <cub/cub.cuh>

#include <vector>

#include "context.cuh"
#include "track_kernels.cuh"

namespace b200 {

// 1. frame range check + per-frame observation counts of the tracks longer than 2
__global__ void prn_obs(long long n, int T, const long long* __restrict__ track_begin, const int* __restrict__ obs_frame, int F,
                        int* __restrict__ obs_count, int* __restrict__ bad) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n) return;
  const int f = obs_frame[o];
  if (f < 0 || f >= F) {
    *bad = 1;
    return;
  }
  int lo = 0, hi = T;                                  // track t with track_begin[t] <= o < track_begin[t + 1]
  while (hi - lo > 1) {
    const int mid = lo + ((hi - lo) >> 1);
    if (track_begin[mid] <= o) lo = mid; else hi = mid;
  }
  if (track_begin[lo + 1] - track_begin[lo] > 2) atomicAdd(&obs_count[f], 1);
}

// slots of track t: L (L - 1) / 2 index pairs when L > 2, none otherwise (the reference skips tracks of <= 2 observations)
__global__ void prn_slot_count(int T, const long long* __restrict__ track_begin, long long* __restrict__ slots) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > T) return;
  if (t == T) { slots[t] = 0; return; }
  const long long L = track_begin[t + 1] - track_begin[t];
  slots[t] = L > 2 ? L * (L - 1) / 2 : 0;
}

// 2. keys of the slots [s0, s0 + n): slot k of a track of length L is the k-th pair (i, j), i < j, in row-major order
__global__ void prn_pair_keys(long long s0, long long n, int T, const long long* __restrict__ slot_begin,
                              const long long* __restrict__ track_begin, const int* __restrict__ obs_frame,
                              unsigned long long F, unsigned long long* __restrict__ keys) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const long long s = s0 + q;
  int lo = 0, hi = T;                                  // track t with slot_begin[t] <= s < slot_begin[t + 1]
  while (hi - lo > 1) {
    const int mid = lo + ((hi - lo) >> 1);
    if (slot_begin[mid] <= s) lo = mid; else hi = mid;
  }
  const long long k = s - slot_begin[lo];
  const long long b = track_begin[lo], L = track_begin[lo + 1] - b;
  // row i holds the pairs (i, i+1..L-1); rows 0..i-1 hold before(i) = i (2L - i - 1) / 2 slots
  const double m = (double)(2 * L - 1);
  long long i = (long long)((m - sqrt(m * m - 8.0 * (double)k)) * 0.5);
  if (i < 0) i = 0;
  if (i > L - 2) i = L - 2;
  while (i > 0 && i * (2 * L - i - 1) / 2 > k) --i;
  while (i < L - 2 && (i + 1) * (2 * L - i - 2) / 2 <= k) ++i;
  const long long j = k - i * (2 * L - i - 1) / 2 + i + 1;
  const unsigned long long a = (unsigned)obs_frame[b + i], c = (unsigned)obs_frame[b + j];
  // same frame: no pair (:25); F^2 - 1 is never a pair key (the largest is (F - 2) F + F - 1) and sorts last
  keys[q] = a == c ? F * F - 1 : (a < c ? a * F + c : c * F + a);
}

// 3. visibility edges: flag, and split the kept keys into the endpoint array of trk_hook ([lo..., hi...])
__global__ void prn_edge_flags(long long R, const unsigned long long* __restrict__ keys, const int* __restrict__ counts,
                               const int* __restrict__ obs_count, int min_obs, unsigned long long F, int* __restrict__ min5,
                               unsigned char* __restrict__ edge) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int a = (int)(keys[r] / F), b = (int)(keys[r] % F);
  const bool c5 = counts[r] >= 5;
  min5[r] = c5;
  edge[r] = c5 && obs_count[a] >= min_obs && obs_count[b] >= min_obs;
}
__global__ void prn_split_keys(long long E, const unsigned long long* __restrict__ keys, unsigned long long F, int* __restrict__ ends) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  ends[e] = (int)(keys[e] / F);
  ends[E + e] = (int)(keys[e] % F);
}
__global__ void prn_abs_diff(long long E, const int* __restrict__ sorted, int median, int* __restrict__ diff) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < E) diff[e] = abs(sorted[e] - median);
}

// frames of the frame adjacency list (CreateFrameAdjacencyList): an endpoint of a selected edge, or a frame with an
// intra-frame (self-loop) edge
__global__ void prn_mark_ends(long long E, const int* __restrict__ ends, unsigned char* __restrict__ in_adj) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  in_adj[ends[e]] = 1;
  in_adj[ends[E + e]] = 1;
}
// after 5d the self-loops of the registered frames remain valid
__global__ void prn_registered_loops(int F, const unsigned char* __restrict__ self_loop, const unsigned char* __restrict__ reg,
                                     unsigned char* __restrict__ in_adj) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F) in_adj[f] = self_loop[f] && reg[f];
}
// component sizes by root (parent flattened); roots are the smallest frame of their set
__global__ void prn_comp_size(int F, const int* __restrict__ root, const unsigned char* __restrict__ in_adj, int* __restrict__ size) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F && in_adj[f]) atomicAdd(&size[root[f]], 1);
}
// 5a: the largest component, ties to the smallest root: max of (size << 32 | ~root)
__global__ void prn_largest(int F, const int* __restrict__ size, unsigned long long* __restrict__ best) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F && size[f] > 0) atomicMax(best, ((unsigned long long)size[f] << 32) | (0xffffffffu - (unsigned)f));
}
__global__ void prn_register(int F, const int* __restrict__ root, const unsigned char* __restrict__ in_adj,
                             const unsigned long long* __restrict__ best, unsigned char* __restrict__ reg) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int r = (int)(0xffffffffu - (unsigned)(*best & 0xffffffffull));
  reg[f] = in_adj[f] && root[f] == r;
}
// 5b (op 0): registered edges with weight > thr; 5c (op 1): registered edges with weight >= 0.75 thr joining two sets;
// 5d (op 2): registered edges inside one set
__global__ void prn_select_edges(long long E, const int* __restrict__ ends, const int* __restrict__ w, const unsigned char* __restrict__ reg,
                                 const int* __restrict__ root, double thr, int op, unsigned char* __restrict__ sel) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int a = ends[e], b = ends[E + e];
  bool s = reg[a] && reg[b];
  if (op == 0) s = s && w[e] > thr;
  else if (op == 1) s = s && !(w[e] < 0.75 * thr) && root[a] != root[b];
  else s = s && root[a] == root[b];
  sel[e] = s;
}
// 5c: unordered root pair of every selected edge (F^2 - 1 = not selected)
__global__ void prn_root_keys(long long E, const int* __restrict__ ends, const unsigned char* __restrict__ sel, const int* __restrict__ root,
                              unsigned long long F, unsigned long long* __restrict__ keys) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  if (!sel[e]) { keys[e] = F * F - 1; return; }
  const unsigned long long a = (unsigned)root[ends[e]], b = (unsigned)root[ends[E + e]];
  keys[e] = a < b ? a * F + b : b * F + a;
}
// root pairs counted >= 2 times; the sentinel run sorts last and is never selected
__global__ void prn_strong_pairs(long long R, const unsigned long long* __restrict__ keys, const int* __restrict__ counts,
                                 unsigned long long F, unsigned char* __restrict__ sel) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < R) sel[r] = counts[r] >= 2 && keys[r] != F * F - 1;
}
// 5e: components of the final adjacency ranked by (size desc, smallest frame asc)
__global__ void prn_rank_keys(int F, const int* __restrict__ size, unsigned long long* __restrict__ keys, int* __restrict__ nroots) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  if (size[f] > 0) {
    keys[f] = ((unsigned long long)(0x7fffffffu - (unsigned)size[f]) << 32) | (unsigned)f;
    atomicAdd(nroots, 1);
  } else {
    keys[f] = ~0ull;
  }
}
__global__ void prn_scatter_rank(int n, const unsigned long long* __restrict__ sorted, int* __restrict__ rank_of_root) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rank_of_root[(int)(sorted[i] & 0xffffffffull)] = i;
}
__global__ void prn_cluster_id(int F, const int* __restrict__ root, const unsigned char* __restrict__ in_adj,
                               const int* __restrict__ rank_of_root, int* __restrict__ cluster) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f < F) cluster[f] = in_adj[f] ? rank_of_root[root[f]] : -1;
}

inline int bit_width(unsigned long long v) {
  int b = 0;
  while (v) { ++b; v >>= 1; }
  return b;
}

struct PruneStats {
  long long covisible_pairs = 0, pairs_min5 = 0, visibility_edges = 0;
  double strong_threshold = 0;
  int clustering_iterations = 0, largest_component_frames = 0;
};

// Device scratch and the steps of one call; every host read-back is a count or a flag.
struct PruneRunner {
  b200sfm_ctx* ctx;
  cudaStream_t s;
  DevBuf<unsigned char> tmp;

  explicit PruneRunner(b200sfm_ctx* c) : ctx(c), s(c->stream) {}

  void ensure_tmp(size_t need) {
    if (need > tmp.n) tmp.alloc(need);
  }
  template <class T>
  T read(const T* d) {
    T h{};
    B200_CUDA_OK(cudaMemcpyAsync(&h, d, sizeof(T), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return h;
  }
  // keys [n] -> sorted unique keys + run lengths; returns the number of runs
  long long sort_rle(const unsigned long long* in, unsigned long long* sorted, long long n, int end_bit, unsigned long long* uniq,
                     int* counts, int* d_nruns) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, a, in, sorted, (int)n, 0, end_bit, s);
    cub::DeviceRunLengthEncode::Encode(nullptr, b, sorted, uniq, counts, d_nruns, (int)n, s);
    ensure_tmp(std::max(a, b));
    size_t nb = tmp.n;
    cub::DeviceRadixSort::SortKeys(tmp.p, nb, in, sorted, (int)n, 0, end_bit, s);
    nb = tmp.n;
    cub::DeviceRunLengthEncode::Encode(tmp.p, nb, sorted, uniq, counts, d_nruns, (int)n, s);
    return read(d_nruns);
  }
  template <class T>
  long long select(const T* in, const unsigned char* flags, T* out, long long n, int* d_n) {
    size_t a = 0;
    cub::DeviceSelect::Flagged(nullptr, a, in, flags, out, d_n, (int)n, s);
    ensure_tmp(a);
    size_t nb = tmp.n;
    cub::DeviceSelect::Flagged(tmp.p, nb, in, flags, out, d_n, (int)n, s);
    return read(d_n);
  }
  // union of the M endpoint pairs ends[e], ends[M + e] into parent (trk_hook sweeps until nothing changes), then flatten
  void unite(const int* ends, long long M, int* parent, int F, int* changed) {
    if (M > 0) {
      for (int sweep = 0; sweep < 64; ++sweep) {
        B200_CUDA_OK(cudaMemsetAsync(changed, 0, sizeof(int), s));
        B200_LAUNCH(ctx, trk_hook, cdiv(M, 256), 256, 0, M, ends, parent, changed);
        if (!read(changed)) break;
      }
    }
    B200_LAUNCH(ctx, trk_flatten, cdiv(F, 256), 256, 0, (long long)F, parent);
  }
  // the endpoint array [lo..., hi...] of the selected edges of ends [2E]
  long long compact_ends(const int* ends, long long E, const unsigned char* sel, int* out, int* d_n) {
    const long long k = select(ends, sel, out, E, d_n);
    select(ends + E, sel, out + k, E, d_n);
    return k;
  }

  // Returns false when a frame index is out of range.  cluster [F] and reg [F] (in/out) are host arrays.
  bool run(int F, int T, long long n, const long long* h_track_begin, const int* h_obs_frame, const unsigned char* h_self_loop,
           int min_obs, long long max_keys, int* h_cluster, unsigned char* h_reg, int* num_clusters, PruneStats& st) {
    const unsigned long long uF = (unsigned long long)F;
    DevBuf<long long> track_begin, slot_begin;
    DevBuf<int> obs_frame, obs_count, flag;
    DevBuf<unsigned char> self_loop;
    track_begin.alloc((size_t)T + 1); obs_frame.alloc(std::max(n, 1LL)); obs_count.alloc(F); flag.alloc(2); self_loop.alloc(F);
    if (h_self_loop) self_loop.upload(h_self_loop, F, s); else self_loop.zero(s);
    track_begin.upload(h_track_begin, (size_t)T + 1, s);
    obs_frame.upload(h_obs_frame, n, s);
    obs_count.zero(s);
    flag.zero(s);
    if (n > 0) B200_LAUNCH(ctx, prn_obs, cdiv(n, 256), 256, 0, n, T, track_begin.p, obs_frame.p, F, obs_count.p, flag.p);
    if (read(flag.p)) return false;
    *num_clusters = 0;
    for (int f = 0; f < F; ++f) h_cluster[f] = -1;
    if (F < 2 || T == 0) return true;                  // no frame pair: rule (iii)
    // ---- 2. covisibility counts
    slot_begin.alloc((size_t)T + 1);
    {
      DevBuf<long long> slots;
      slots.alloc((size_t)T + 1);
      B200_LAUNCH(ctx, prn_slot_count, cdiv(T + 1, 256), 256, 0, T, track_begin.p, slots.p);
      size_t a = 0;
      cub::DeviceScan::ExclusiveSum(nullptr, a, slots.p, slot_begin.p, T + 1, s);
      ensure_tmp(a);
      size_t nb = tmp.n;
      cub::DeviceScan::ExclusiveSum(tmp.p, nb, slots.p, slot_begin.p, T + 1, s);
    }
    const long long S = read(slot_begin.p + T);
    const int end_bit = bit_width(uF * uF - 1);
    const long long B = std::min<long long>(std::max<long long>(S, 1), max_keys);
    DevBuf<unsigned long long> keys, sorted, uniq;
    DevBuf<int> counts;
    keys.alloc(B); sorted.alloc(B); uniq.alloc(B); counts.alloc(B);
    struct Runs { DevBuf<unsigned long long> k; DevBuf<int> c; long long n = 0; };
    std::vector<Runs> passes((size_t)((S + B - 1) / B));
    long long R = 0;
    for (size_t p = 0; p < passes.size(); ++p) {
      const long long s0 = (long long)p * B, m = std::min(B, S - s0);
      B200_LAUNCH(ctx, prn_pair_keys, cdiv(m, 256), 256, 0, s0, m, T, slot_begin.p, track_begin.p, obs_frame.p, uF, keys.p);
      long long r = sort_rle(keys.p, sorted.p, m, end_bit, uniq.p, counts.p, flag.p);
      const unsigned long long last = read(uniq.p + r - 1);
      if (last == uF * uF - 1) --r;                    // the same-frame slots
      passes[p].n = r;
      if (passes.size() > 1 && r > 0) {
        passes[p].k.alloc(r); passes[p].c.alloc(r);
        B200_CUDA_OK(cudaMemcpyAsync(passes[p].k.p, uniq.p, r * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s));
        B200_CUDA_OK(cudaMemcpyAsync(passes[p].c.p, counts.p, r * sizeof(int), cudaMemcpyDeviceToDevice, s));
      }
      R += r;
      if (R > 0x7fffffffLL)                            // the merge sorts the runs of every pass with 32-bit counts
        throw InvalidInput{"more than 2^31 - 1 frame-pair runs over all passes: raise max_pair_keys_per_pass"};
    }
    keys.release(); sorted.release();
    const unsigned long long* pk = uniq.p;
    const int* pc = counts.p;
    DevBuf<unsigned long long> mk, mk_sorted;
    DevBuf<int> mc, mc_sorted;
    if (passes.size() > 1 && R > 0) {                  // merge the passes' runs: sort by key, sum the counts per key
      uniq.release(); counts.release();
      mk.alloc(R); mc.alloc(R); mk_sorted.alloc(R); mc_sorted.alloc(R);
      long long off = 0;
      for (auto& p : passes) {
        if (!p.n) continue;
        B200_CUDA_OK(cudaMemcpyAsync(mk.p + off, p.k.p, p.n * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, s));
        B200_CUDA_OK(cudaMemcpyAsync(mc.p + off, p.c.p, p.n * sizeof(int), cudaMemcpyDeviceToDevice, s));
        off += p.n;
        p.k.release(); p.c.release();
      }
      size_t a = 0, b = 0;
      cub::DeviceRadixSort::SortPairs(nullptr, a, mk.p, mk_sorted.p, mc.p, mc_sorted.p, (int)R, 0, end_bit, s);
      cub::DeviceReduce::ReduceByKey(nullptr, b, mk_sorted.p, mk.p, mc_sorted.p, mc.p, flag.p, cuda::std::plus<int>(), (int)R, s);
      ensure_tmp(std::max(a, b));
      size_t nb = tmp.n;
      cub::DeviceRadixSort::SortPairs(tmp.p, nb, mk.p, mk_sorted.p, mc.p, mc_sorted.p, (int)R, 0, end_bit, s);
      nb = tmp.n;
      cub::DeviceReduce::ReduceByKey(tmp.p, nb, mk_sorted.p, mk.p, mc_sorted.p, mc.p, flag.p, cuda::std::plus<int>(), (int)R, s);
      R = read(flag.p);
      pk = mk.p;
      pc = mc.p;
    }
    st.covisible_pairs = R;
    if (R == 0) return true;
    // ---- 3. visibility edges and the threshold
    DevBuf<unsigned char> eflag;
    DevBuf<int> min5;
    min5.alloc(R); eflag.alloc(R);
    B200_LAUNCH(ctx, prn_edge_flags, cdiv(R, 256), 256, 0, R, pk, pc, obs_count.p, min_obs, uF, min5.p, eflag.p);
    {
      size_t a = 0;
      DevBuf<int> n5;
      n5.alloc(1);
      cub::DeviceReduce::Sum(nullptr, a, min5.p, n5.p, (int)R, s);
      ensure_tmp(a);
      size_t nb = tmp.n;
      cub::DeviceReduce::Sum(tmp.p, nb, min5.p, n5.p, (int)R, s);
      st.pairs_min5 = read(n5.p);
    }
    DevBuf<unsigned long long> ekeys;
    DevBuf<int> w, ends;
    ekeys.alloc(R); w.alloc(R);
    const long long E = select(pk, eflag.p, ekeys.p, R, flag.p);
    select(pc, eflag.p, w.p, R, flag.p);
    st.visibility_edges = E;
    if (E == 0) return true;                           // rule (iii)
    mk.release(); mk_sorted.release(); mc.release(); mc_sorted.release(); uniq.release(); counts.release();
    ends.alloc(2 * E);
    B200_LAUNCH(ctx, prn_split_keys, cdiv(E, 256), 256, 0, E, ekeys.p, uF, ends.p);
    {
      DevBuf<int> ws, diff, ds;
      ws.alloc(E); diff.alloc(E); ds.alloc(E);
      size_t a = 0;
      cub::DeviceRadixSort::SortKeys(nullptr, a, w.p, ws.p, (int)E, 0, 32, s);
      ensure_tmp(a);
      size_t nb = tmp.n;
      cub::DeviceRadixSort::SortKeys(tmp.p, nb, w.p, ws.p, (int)E, 0, 32, s);
      const int median = read(ws.p + E / 2);
      B200_LAUNCH(ctx, prn_abs_diff, cdiv(E, 256), 256, 0, E, ws.p, median, diff.p);
      nb = tmp.n;
      cub::DeviceRadixSort::SortKeys(tmp.p, nb, diff.p, ds.p, (int)E, 0, 32, s);
      const int mad = read(ds.p + E / 2);
      st.strong_threshold = std::max((double)median - (double)mad, 20.);
    }
    const double thr = st.strong_threshold;
    // ---- 5a. largest connected component of the visibility graph (frame pairs + self-loops)
    DevBuf<unsigned char> in_adj, reg, sel;
    DevBuf<int> parent, size, cends;
    DevBuf<unsigned long long> best;
    in_adj.alloc(F); reg.alloc(F); sel.alloc(E); parent.alloc(F); size.alloc(F); cends.alloc(2 * E); best.alloc(1);
    B200_CUDA_OK(cudaMemcpyAsync(in_adj.p, self_loop.p, F, cudaMemcpyDeviceToDevice, s));
    B200_LAUNCH(ctx, prn_mark_ends, cdiv(E, 256), 256, 0, E, ends.p, in_adj.p);
    B200_LAUNCH(ctx, trk_iota, cdiv(F, 256), 256, 0, (long long)F, parent.p);
    unite(ends.p, E, parent.p, F, flag.p);
    size.zero(s);
    best.zero(s);
    B200_LAUNCH(ctx, prn_comp_size, cdiv(F, 256), 256, 0, F, parent.p, in_adj.p, size.p);
    B200_LAUNCH(ctx, prn_largest, cdiv(F, 256), 256, 0, F, size.p, best.p);
    B200_LAUNCH(ctx, prn_register, cdiv(F, 256), 256, 0, F, parent.p, in_adj.p, best.p, reg.p);
    st.largest_component_frames = (int)(read(best.p) >> 32);
    // ---- 5b. strong edges
    B200_LAUNCH(ctx, trk_iota, cdiv(F, 256), 256, 0, (long long)F, parent.p);
    B200_LAUNCH(ctx, prn_select_edges, cdiv(E, 256), 256, 0, E, ends.p, w.p, reg.p, parent.p, thr, 0, sel.p);
    long long M = compact_ends(ends.p, E, sel.p, cends.p, flag.p);
    unite(cends.p, M, parent.p, F, flag.p);
    // ---- 5c. merge sets joined by >= 2 slightly weaker edges, at most 10 passes
    {
      DevBuf<unsigned long long> rk, rsorted, runiq;
      DevBuf<int> rcount;
      rk.alloc(E); rsorted.alloc(E); runiq.alloc(E); rcount.alloc(E);
      int iteration = 0;
      bool status = true;
      while (status) {
        status = false;
        ++iteration;
        if (iteration > 10) break;
        B200_LAUNCH(ctx, prn_select_edges, cdiv(E, 256), 256, 0, E, ends.p, w.p, reg.p, parent.p, thr, 1, sel.p);
        B200_LAUNCH(ctx, prn_root_keys, cdiv(E, 256), 256, 0, E, ends.p, sel.p, parent.p, uF, rk.p);
        const long long r = sort_rle(rk.p, rsorted.p, E, end_bit, runiq.p, rcount.p, flag.p);
        B200_LAUNCH(ctx, prn_strong_pairs, cdiv(r, 256), 256, 0, r, runiq.p, rcount.p, uF, sel.p);
        DevBuf<unsigned long long> pk2;
        pk2.alloc(r);
        const long long k = select(runiq.p, sel.p, pk2.p, r, flag.p);
        if (k == 0) continue;
        status = true;
        B200_LAUNCH(ctx, prn_split_keys, cdiv(k, 256), 256, 0, k, pk2.p, uF, cends.p);
        unite(cends.p, k, parent.p, F, flag.p);
      }
      st.clustering_iterations = iteration;
    }
    // ---- 5d-e. components of the edges inside one set, ranked by (size desc, smallest frame asc)
    B200_LAUNCH(ctx, prn_select_edges, cdiv(E, 256), 256, 0, E, ends.p, w.p, reg.p, parent.p, thr, 2, sel.p);
    M = compact_ends(ends.p, E, sel.p, cends.p, flag.p);
    // adjacency after 5d: the registered self-loop frames and the endpoints of the surviving edges
    B200_LAUNCH(ctx, prn_registered_loops, cdiv(F, 256), 256, 0, F, self_loop.p, reg.p, in_adj.p);
    if (M > 0) B200_LAUNCH(ctx, prn_mark_ends, cdiv(M, 256), 256, 0, M, cends.p, in_adj.p);   // 5d may drop every edge
    B200_LAUNCH(ctx, trk_iota, cdiv(F, 256), 256, 0, (long long)F, parent.p);
    unite(cends.p, M, parent.p, F, flag.p);
    size.zero(s);
    B200_LAUNCH(ctx, prn_comp_size, cdiv(F, 256), 256, 0, F, parent.p, in_adj.p, size.p);
    DevBuf<unsigned long long> rkeys, rks;
    DevBuf<int> rank_of_root, cluster;
    rkeys.alloc(F); rks.alloc(F); rank_of_root.alloc(F); cluster.alloc(F);
    B200_CUDA_OK(cudaMemsetAsync(flag.p, 0, sizeof(int), s));
    B200_LAUNCH(ctx, prn_rank_keys, cdiv(F, 256), 256, 0, F, size.p, rkeys.p, flag.p);
    {
      size_t a = 0;
      cub::DeviceRadixSort::SortKeys(nullptr, a, rkeys.p, rks.p, F, 0, 64, s);
      ensure_tmp(a);
      size_t nb = tmp.n;
      cub::DeviceRadixSort::SortKeys(tmp.p, nb, rkeys.p, rks.p, F, 0, 64, s);
    }
    const int nc = read(flag.p);
    B200_LAUNCH(ctx, prn_scatter_rank, cdiv(std::max(nc, 1), 256), 256, 0, nc, rks.p, rank_of_root.p);
    B200_LAUNCH(ctx, prn_cluster_id, cdiv(F, 256), 256, 0, F, parent.p, in_adj.p, rank_of_root.p, cluster.p);
    cluster.download(h_cluster, F, s);
    reg.download(h_reg, F, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    *num_clusters = nc;
    return true;
  }
};

}  // namespace b200
