// track_select_kernels.cuh -- device side of TrackEngine::FindTracksForProblem (glomap/controllers/track_establishment.cc
// :153-227; SURVEY.md 8(f) item 4).  The reference walks the candidate tracks in descending (length, id) order and keeps a
// saturating per-image counter; that greedy loop has an exact data-parallel form:
//   * a counter runs 0, 1, ..., quota + 1 and then stays, so an observation increments its image's counter exactly when
//     its RANK -- the number of registered observations of that image in earlier-processed eligible tracks plus the
//     earlier ones of its own track -- is <= quota; a track is selected iff one of its observations does.  Without a
//     quota (min_num_tracks_per_view < 0, an unsigned comparison in the reference) that is "has a registered observation";
//   * the order of the observations inside a track is immaterial (repeats of one image belong to the same track);
//   * the "every camera saturated" stop changes nothing (no later track could increment a counter);
//   * the max_num_tracks stop is a prefix cut: keep a selected track while the inclusive count of selected tracks in
//     processing order is <= max_num_tracks + 1.
// Pipeline (index work only, exact):
//   1. registered ids: radix sort + unique; every observation's image -> index by binary search (-1: not registered)
//   2. observation -> track: the track index scattered at its first observation, inclusive max-scan
//   3. radix sort of the keys t * (R + 1) + image index (R: not registered): the observations of track t keep their CSR
//      range, and one exclusive scan of (registered, first of its (track, image)) packed in 64 bits gives the number of
//      registered observations and of distinct registered images of every track
//   4. eligibility: L >= min_views, L <= max_views, distinct >= min_views, all as unsigned 64-bit comparisons
//   5. track ids sorted descending (also the duplicate check); when the order matters, a stable descending sort by L of
//      that permutation gives the processing position of every track
//   6. quota: radix sort of the keys image index * T + position over the registered observations of eligible tracks, the
//      segment start of each image by a max-scan, rank = index - start; a rank <= quota flags the track's position
//   7. cut: inclusive scan of the flags in processing order
#pragma once
#include <cub/cub.cuh>

#include <algorithm>
#include <vector>

#include "context.cuh"
#include "track_kernels.cuh"   // trk_iota

namespace b200 {

struct TselMax {
  __host__ __device__ int operator()(int a, int b) const { return a > b ? a : b; }
};

inline int tsel_bits(unsigned long long v) {   // bit width of v (at least 1, a radix sort needs a non-empty range)
  int b = 1;
  while (b < 64 && (v >> b) != 0) ++b;
  return b;
}

// image -> index into the sorted unique registered ids, -1 when not registered
__global__ void tsel_lookup(long long n, const unsigned* __restrict__ obs_image, const unsigned* __restrict__ reg, int R,
                            int* __restrict__ ri) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned v = obs_image[i];
  int lo = 0, hi = R;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (reg[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  ri[i] = (lo < R && reg[lo] == v) ? lo : -1;
}
// head[begin[t]] = t for every non-empty track (distinct slots); the max-scan spreads it over the track's observations
__global__ void tsel_heads(int T, const long long* __restrict__ begin, int* __restrict__ head) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T && begin[t + 1] > begin[t]) head[begin[t]] = t;
}
__global__ void tsel_track_image_keys(long long n, const int* __restrict__ obs_track, const int* __restrict__ ri, int R,
                                      unsigned long long* __restrict__ key) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) key[i] = (unsigned long long)obs_track[i] * (unsigned long long)(R + 1) + (unsigned long long)(ri[i] < 0 ? R : ri[i]);
}
// low 32 bits: registered observation; high 32 bits: first observation of its (track, registered image)
__global__ void tsel_count_flags(long long n, const unsigned long long* __restrict__ key, int R, unsigned long long* __restrict__ v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { v[i] = 0; return; }
  const unsigned long long k = key[i];
  const bool reg = (k % (unsigned long long)(R + 1)) != (unsigned long long)R;
  const bool head = reg && (i == 0 || key[i - 1] != k);
  v[i] = (reg ? 1ull : 0ull) | (head ? (1ull << 32) : 0ull);
}
__global__ void tsel_eligible(int T, const long long* __restrict__ begin, const unsigned long long* __restrict__ scan,
                              unsigned long long min_views, unsigned long long max_views, unsigned char* __restrict__ eligible,
                              unsigned char* __restrict__ has_reg, long long* __restrict__ L_out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const unsigned long long L = (unsigned long long)(begin[t + 1] - begin[t]);
  const unsigned long long d = scan[begin[t + 1]] - scan[begin[t]];
  const unsigned long long nreg = d & 0xffffffffull, distinct = d >> 32;
  const bool e = L >= min_views && L <= max_views && distinct >= min_views;
  eligible[t] = e ? 1 : 0;
  has_reg[t] = (e && nreg > 0) ? 1 : 0;
  L_out[t] = (long long)L;
}
__global__ void tsel_dup(int T, const unsigned long long* __restrict__ ids_sorted, int* __restrict__ dup) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > 0 && i < T && ids_sorted[i] == ids_sorted[i - 1]) *dup = 1;
}
__global__ void tsel_gather_len(int T, const int* __restrict__ perm, const long long* __restrict__ L, unsigned* __restrict__ key) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < T) key[j] = (unsigned)L[perm[j]];
}
__global__ void tsel_positions(int T, const int* __restrict__ order, int* __restrict__ pos) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < T) pos[order[j]] = j;
}
// registered observation of an eligible track: image index * T + processing position; anything else: the sentinel R * T
__global__ void tsel_rank_keys(long long n, const int* __restrict__ obs_track, const int* __restrict__ ri,
                               const unsigned char* __restrict__ eligible, const int* __restrict__ pos, int T, int R,
                               unsigned long long* __restrict__ key) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = obs_track[i], r = ri[i];
  key[i] = (r >= 0 && eligible[t]) ? (unsigned long long)r * (unsigned long long)T + (unsigned long long)pos[t]
                                   : (unsigned long long)R * (unsigned long long)T;
}
__global__ void tsel_segment_heads(long long n, const unsigned long long* __restrict__ key, int T, int* __restrict__ start) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) start[i] = (i == 0 || key[i] / (unsigned long long)T != key[i - 1] / (unsigned long long)T) ? (int)i : 0;
}
// rank = index - start of the image's segment; a rank <= quota flags the position of the observation's track
__global__ void tsel_rank_flags(long long n, const unsigned long long* __restrict__ key, const int* __restrict__ seg_start,
                                int T, int R, long long quota, int* __restrict__ sel_pos) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = key[i];
  if (k >= (unsigned long long)R * (unsigned long long)T) return;
  if ((long long)(i - seg_start[i]) <= quota) sel_pos[k % (unsigned long long)T] = 1;
}
__global__ void tsel_scatter_pos(int T, const unsigned char* __restrict__ sel, const int* __restrict__ pos, int* __restrict__ sel_pos) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) sel_pos[pos[t]] = sel[t];
}
// keep[t] = selected at its position and (no cap or the inclusive count there <= cap)
__global__ void tsel_keep(int T, const int* __restrict__ pos, const int* __restrict__ sel_pos, const int* __restrict__ count_incl,
                          long long cap, unsigned char* __restrict__ keep) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int p = pos[t];
  keep[t] = (sel_pos[p] && (cap < 0 || (long long)count_incl[p] <= cap)) ? 1 : 0;
}

struct TrackSelectRunner {
  b200sfm_ctx* ctx;
  DevBuf<unsigned char> tmp;
  explicit TrackSelectRunner(b200sfm_ctx* c) : ctx(c) {}

  template <class F>
  void cub_call(F&& f) {   // size query, grow the scratch, run
    size_t need = 0;
    B200_CUDA_OK(f((void*)nullptr, need));
    if (need > tmp.n) tmp.alloc(need);
    size_t nb = tmp.n;
    B200_CUDA_OK(f((void*)tmp.p, nb));
  }

  // quota < 0: no per-image quota; cap < 0: no cap on the number of tracks (else max_num_tracks + 1).  Returns false when
  // two tracks share an id.
  bool run(int T, const unsigned long long* h_ids, const long long* h_begin, long long n, const unsigned* h_obs_image, int R_in,
           const unsigned* h_reg, long long quota, unsigned long long min_views, unsigned long long max_views, long long cap,
           unsigned char* h_keep, long long* h_num) {
    cudaStream_t s = ctx->stream;
    // 5a. track ids descending (duplicate check; first half of the processing order)
    DevBuf<unsigned long long> ids, ids_sorted;
    DevBuf<int> iota, perm;
    ids.alloc(T); ids_sorted.alloc(T); iota.alloc(T); perm.alloc(T);
    ids.upload(h_ids, T, s);
    B200_LAUNCH(ctx, trk_iota, cdiv(T, 256), 256, 0, (long long)T, iota.p);
    cub_call([&](void* p, size_t& nb) {
      return cub::DeviceRadixSort::SortPairsDescending(p, nb, ids.p, ids_sorted.p, iota.p, perm.p, T, 0, 64, s);
    });
    DevBuf<int> flag;
    flag.alloc(1);
    flag.zero(s);
    B200_LAUNCH(ctx, tsel_dup, cdiv(T, 256), 256, 0, T, ids_sorted.p, flag.p);
    int h_dup = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&h_dup, flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    // 1. registered ids, sorted and unique
    DevBuf<unsigned> reg, reg_sorted, reg_unique;
    DevBuf<int> d_R;
    d_R.alloc(1);
    d_R.zero(s);
    if (R_in > 0) {
      reg.alloc(R_in); reg_sorted.alloc(R_in); reg_unique.alloc(R_in);
      reg.upload(h_reg, R_in, s);
      cub_call([&](void* p, size_t& nb) { return cub::DeviceRadixSort::SortKeys(p, nb, reg.p, reg_sorted.p, R_in, 0, 32, s); });
      cub_call([&](void* p, size_t& nb) { return cub::DeviceSelect::Unique(p, nb, reg_sorted.p, reg_unique.p, d_R.p, R_in, s); });
    }
    int R = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&R, d_R.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    if (h_dup) return false;
    if (R == 0 || n == 0) {   // no registered observation anywhere: nothing is selected
      std::fill(h_keep, h_keep + T, (unsigned char)0);
      *h_num = 0;
      return true;
    }
    // 1b-2. observations: registered index and track
    DevBuf<long long> begin;
    DevBuf<unsigned> obs_image;
    DevBuf<int> ri, head, obs_track;
    begin.alloc((size_t)T + 1); obs_image.alloc(n); ri.alloc(n); head.alloc(n); obs_track.alloc(n);
    begin.upload(h_begin, (size_t)T + 1, s);
    obs_image.upload(h_obs_image, n, s);
    B200_LAUNCH(ctx, tsel_lookup, cdiv(n, 256), 256, 0, n, obs_image.p, reg_unique.p, R, ri.p);
    obs_image.release();
    head.zero(s);
    B200_LAUNCH(ctx, tsel_heads, cdiv(T, 256), 256, 0, T, begin.p, head.p);
    cub_call([&](void* p, size_t& nb) { return cub::DeviceScan::InclusiveScan(p, nb, head.p, obs_track.p, TselMax(), (int)n, s); });
    // 3. per track: registered observations and distinct registered images
    DevBuf<unsigned long long> key, key_sorted, cnt, cnt_scan;
    key.alloc(n); key_sorted.alloc(n);
    B200_LAUNCH(ctx, tsel_track_image_keys, cdiv(n, 256), 256, 0, n, obs_track.p, ri.p, R, key.p);
    const int bits_ti = tsel_bits((unsigned long long)T * (unsigned long long)(R + 1) - 1);
    cub_call([&](void* p, size_t& nb) { return cub::DeviceRadixSort::SortKeys(p, nb, key.p, key_sorted.p, (int)n, 0, bits_ti, s); });
    cnt.alloc(n + 1); cnt_scan.alloc(n + 1);
    B200_LAUNCH(ctx, tsel_count_flags, cdiv(n + 1, 256), 256, 0, n, key_sorted.p, R, cnt.p);
    cub_call([&](void* p, size_t& nb) { return cub::DeviceScan::ExclusiveSum(p, nb, cnt.p, cnt_scan.p, (int)(n + 1), s); });
    // 4. eligibility
    DevBuf<unsigned char> eligible, has_reg, keep;
    DevBuf<long long> L;
    eligible.alloc(T); has_reg.alloc(T); keep.alloc(T); L.alloc(T);
    B200_LAUNCH(ctx, tsel_eligible, cdiv(T, 256), 256, 0, T, begin.p, cnt_scan.p, min_views, max_views, eligible.p, has_reg.p, L.p);
    cnt.release(); cnt_scan.release();
    if (quota < 0) {
      // no quota: selected = eligible with a registered observation; the cut only matters when it bites
      std::vector<unsigned char> sel(T);
      has_reg.download(sel.data(), T, s);
      B200_CUDA_OK(cudaStreamSynchronize(s));
      long long count = 0;
      for (unsigned char c : sel) count += c;
      if (cap < 0 || count <= cap) {
        std::copy(sel.begin(), sel.end(), h_keep);
        *h_num = count;
        return true;
      }
    }
    // 5b. processing position: stable descending sort of the id-sorted permutation by length
    DevBuf<unsigned> lkey, lkey_sorted;
    DevBuf<int> order, pos;
    lkey.alloc(T); lkey_sorted.alloc(T); order.alloc(T); pos.alloc(T);
    B200_LAUNCH(ctx, tsel_gather_len, cdiv(T, 256), 256, 0, T, perm.p, L.p, lkey.p);
    const int bits_l = tsel_bits((unsigned long long)n);
    cub_call([&](void* p, size_t& nb) {
      return cub::DeviceRadixSort::SortPairsDescending(p, nb, lkey.p, lkey_sorted.p, perm.p, order.p, T, 0, bits_l, s);
    });
    B200_LAUNCH(ctx, tsel_positions, cdiv(T, 256), 256, 0, T, order.p, pos.p);
    DevBuf<int> sel_pos;
    sel_pos.alloc(T);
    if (quota < 0) {
      B200_LAUNCH(ctx, tsel_scatter_pos, cdiv(T, 256), 256, 0, T, has_reg.p, pos.p, sel_pos.p);
    } else {
      // 6. ranks per registered image in processing order
      B200_LAUNCH(ctx, tsel_rank_keys, cdiv(n, 256), 256, 0, n, obs_track.p, ri.p, eligible.p, pos.p, T, R, key.p);
      const int bits_r = tsel_bits((unsigned long long)R * (unsigned long long)T);
      cub_call([&](void* p, size_t& nb) { return cub::DeviceRadixSort::SortKeys(p, nb, key.p, key_sorted.p, (int)n, 0, bits_r, s); });
      obs_track.release(); ri.release();
      DevBuf<int> seg_start;
      seg_start.alloc(n);
      B200_LAUNCH(ctx, tsel_segment_heads, cdiv(n, 256), 256, 0, n, key_sorted.p, T, head.p);
      cub_call([&](void* p, size_t& nb) { return cub::DeviceScan::InclusiveScan(p, nb, head.p, seg_start.p, TselMax(), (int)n, s); });
      sel_pos.zero(s);
      B200_LAUNCH(ctx, tsel_rank_flags, cdiv(n, 256), 256, 0, n, key_sorted.p, seg_start.p, T, R, quota, sel_pos.p);
    }
    // 7. the max_num_tracks cut
    DevBuf<int> count_incl;
    count_incl.alloc(T);
    if (cap >= 0)
      cub_call([&](void* p, size_t& nb) { return cub::DeviceScan::InclusiveSum(p, nb, sel_pos.p, count_incl.p, T, s); });
    B200_LAUNCH(ctx, tsel_keep, cdiv(T, 256), 256, 0, T, pos.p, sel_pos.p, count_incl.p, cap, keep.p);
    keep.download(h_keep, T, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    long long num = 0;
    for (int t = 0; t < T; ++t) num += h_keep[t];
    *h_num = num;
    return true;
  }
};

}  // namespace b200
