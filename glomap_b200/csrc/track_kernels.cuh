// track_kernels.cuh -- device side of TrackEngine::EstablishFullTracks (glomap/controllers/track_establishment.cc:5-150;
// SURVEY.md 8(f) item 4): the union-find over all inlier matches (BlindConcatenation, :19-63) and the collection of the
// components into tracks with the inconsistency test (TrackCollection, :65-150).  Byte / index work, HBM-bound:
//   1. nodes = sorted unique global feature ids (image_id << 32 | feature_id, :48-53) of both endpoints  (radix sort)
//   2. endpoints -> node indices (binary search), pixel of every node from any match that touches it
//   3. connected components: lock-free union-find (compare-and-swap hooking of roots, path halving), swept until a pass
//      changes nothing; the
//      nodes are sorted by id, so the root of a component is its SMALLEST global id -- the reference's rule (:56-60)
//   4. stable sort of the nodes by root -> tracks in ascending track id, observations of a track in ascending global id
//   5. a track is discarded (observations cleared, id kept, :118-131) when two of its features inside ONE image are
//      further apart than thres_inconsistency pixels
// The selection FindTracksForProblem (:153-227) is track_select_kernels.cuh.
#pragma once
#include <cub/cub.cuh>

#include <vector>

#include "context.cuh"

namespace b200 {

__global__ void trk_iota(long long n, int* __restrict__ a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = (int)i;
}
// flags[i] = 1 where sorted[i] starts a new value
__global__ void trk_head_flags(long long n, const unsigned long long* __restrict__ sorted, int* __restrict__ flags) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = (i == 0 || sorted[i] != sorted[i - 1]) ? 1 : 0;
}
// node table from the sorted endpoint list: rank = inclusive scan of the head flags - 1
__global__ void trk_fill_nodes(long long n2, const unsigned long long* __restrict__ sorted, const int* __restrict__ src,
                               const int* __restrict__ flags, const int* __restrict__ rank_incl, const double2* __restrict__ xy_ep,
                               unsigned long long* __restrict__ node_gid, double2* __restrict__ node_xy, int* __restrict__ ep_node) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n2) return;
  const int r = rank_incl[i] - 1;
  ep_node[src[i]] = r;                 // endpoint src[i] (0..M-1: first, M..2M-1: second feature of a match) is node r
  if (flags[i]) {
    node_gid[r] = sorted[i];
    node_xy[r] = xy_ep[src[i]];
  }
}
__device__ __forceinline__ int trk_find(int* __restrict__ parent, int i) {
  int p = parent[i];
  while (p != i) {                     // path halving
    const int g = parent[p];
    if (g != p) parent[i] = g;
    i = p;
    p = parent[i];
  }
  return i;
}
__global__ void trk_hook(long long M, const int* __restrict__ ep_node, int* __restrict__ parent, int* __restrict__ changed) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M) return;
  int ra = trk_find(parent, ep_node[e]), rb = trk_find(parent, ep_node[M + e]);
  while (ra != rb) {                   // link the larger ROOT under the smaller one (the smallest id ends up as the root)
    if (ra < rb) { const int t = ra; ra = rb; rb = t; }
    const int old = atomicCAS(&parent[ra], ra, rb);   // only a node that still is a root may be re-parented
    *changed = 1;
    if (old == ra) break;
    ra = trk_find(parent, ra);         // somebody else hooked ra meanwhile: retry from the current roots
    rb = trk_find(parent, rb);
  }
}
__global__ void trk_flatten(long long n, int* __restrict__ parent) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) parent[i] = trk_find(parent, (int)i);
}
// nodes sorted by (root, id): head flags of the tracks
__global__ void trk_track_heads(long long n, const int* __restrict__ root_sorted, int* __restrict__ flags) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = (i == 0 || root_sorted[i] != root_sorted[i - 1]) ? 1 : 0;
}
// inconsistency: node i against the following nodes of the same track AND image (adjacent: sorted by global id)
__global__ void trk_inconsistent(long long n, const int* __restrict__ root_sorted, const int* __restrict__ node_sorted,
                                 const int* __restrict__ track_of, const unsigned long long* __restrict__ node_gid,
                                 const double2* __restrict__ node_xy, double thres2, int* __restrict__ bad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int ni = node_sorted[i];
  const unsigned img = (unsigned)(node_gid[ni] >> 32);
  const double2 a = node_xy[ni];
  for (long long j = i + 1; j < n && root_sorted[j] == root_sorted[i]; ++j) {
    const int nj = node_sorted[j];
    if ((unsigned)(node_gid[nj] >> 32) != img) break;
    const double dx = node_xy[nj].x - a.x, dy = node_xy[nj].y - a.y;
    if (dx * dx + dy * dy > thres2) { bad[track_of[i] - 1] = 1; break; }
  }
}
// per track: id = smallest global id, kept length
__global__ void trk_track_table(long long n, int T, const int* __restrict__ flags, const int* __restrict__ track_of,
                                const int* __restrict__ node_sorted, const unsigned long long* __restrict__ node_gid,
                                unsigned long long* __restrict__ track_id, int* __restrict__ track_start) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (flags[i]) {
    const int t = track_of[i] - 1;
    track_id[t] = node_gid[node_sorted[i]];
    track_start[t] = (int)i;
  }
  if (i == n - 1) track_start[T] = (int)n;
}
__global__ void trk_kept_len(int T, const int* __restrict__ track_start, const int* __restrict__ bad, long long* __restrict__ len) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) len[t] = bad[t] ? 0 : (long long)(track_start[t + 1] - track_start[t]);
  if (t == T) len[t] = 0;
}
__global__ void trk_emit(long long n, const int* __restrict__ track_of, const int* __restrict__ track_start,
                         const long long* __restrict__ begin, const int* __restrict__ bad, const int* __restrict__ node_sorted,
                         const unsigned long long* __restrict__ node_gid, unsigned* __restrict__ obs_image,
                         unsigned* __restrict__ obs_feature) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = track_of[i] - 1;
  if (bad[t]) return;
  const long long dst = begin[t] + (i - track_start[t]);
  const unsigned long long g = node_gid[node_sorted[i]];
  obs_image[dst] = (unsigned)(g >> 32);
  obs_feature[dst] = (unsigned)(g & 0xffffffffull);
}

}  // namespace b200

// Result of one establishment, resident until read out and freed
struct b200sfm_tracks {
  b200sfm_ctx* ctx = nullptr;
  long long n_nodes = 0, n_obs = 0;
  int T = 0, discarded = 0, sweeps = 0;
  b200::DevBuf<unsigned long long> track_id;
  b200::DevBuf<long long> begin;
  b200::DevBuf<unsigned> obs_image, obs_feature;

  void build(long long M, const unsigned long long* h_g1, const unsigned long long* h_g2, const double* h_xy1, const double* h_xy2,
             double thres) {
    using namespace b200;
    cudaStream_t s = ctx->stream;
    if (M <= 0) return;
    if (2 * M >= 2147483647LL) throw InvalidInput{"too many matches for 32-bit node indices"};
    const long long n2 = 2 * M;
    DevBuf<unsigned long long> ep, ep_sorted, node_gid;
    DevBuf<double2> xy_ep, node_xy;
    DevBuf<int> src, src_sorted, flags, rank, ep_node;
    ep.alloc(n2); ep_sorted.alloc(n2); xy_ep.alloc(n2); src.alloc(n2); src_sorted.alloc(n2); flags.alloc(n2); rank.alloc(n2);
    ep_node.alloc(n2);
    ep.upload(h_g1, M, s);
    B200_CUDA_OK(cudaMemcpyAsync(ep.p + M, h_g2, M * sizeof(unsigned long long), cudaMemcpyHostToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(xy_ep.p, h_xy1, M * sizeof(double2), cudaMemcpyHostToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(xy_ep.p + M, h_xy2, M * sizeof(double2), cudaMemcpyHostToDevice, s));
    B200_LAUNCH(ctx, trk_iota, cdiv(n2, 256), 256, 0, n2, src.p);
    size_t need = 0, need2 = 0, need3 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, need, ep.p, ep_sorted.p, src.p, src_sorted.p, (int)n2, 0, 64, s);
    cub::DeviceScan::InclusiveSum(nullptr, need2, flags.p, rank.p, (int)n2, s);
    cub::DeviceRadixSort::SortPairs(nullptr, need3, src.p, src_sorted.p, src.p, src_sorted.p, (int)n2, 0, 32, s);
    DevBuf<unsigned char> tmp;
    tmp.alloc(std::max(need, std::max(need2, need3)));
    size_t nb = tmp.n;
    cub::DeviceRadixSort::SortPairs(tmp.p, nb, ep.p, ep_sorted.p, src.p, src_sorted.p, (int)n2, 0, 64, s);
    B200_LAUNCH(ctx, trk_head_flags, cdiv(n2, 256), 256, 0, n2, ep_sorted.p, flags.p);
    nb = tmp.n;
    cub::DeviceScan::InclusiveSum(tmp.p, nb, flags.p, rank.p, (int)n2, s);
    int h_n = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&h_n, rank.p + n2 - 1, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    n_nodes = h_n;
    node_gid.alloc(n_nodes); node_xy.alloc(n_nodes);
    B200_LAUNCH(ctx, trk_fill_nodes, cdiv(n2, 256), 256, 0, n2, ep_sorted.p, src_sorted.p, flags.p, rank.p, xy_ep.p, node_gid.p, node_xy.p,
                ep_node.p);
    // connected components
    DevBuf<int> parent, changed;
    parent.alloc(n_nodes); changed.alloc(1);
    B200_LAUNCH(ctx, trk_iota, cdiv(n_nodes, 256), 256, 0, n_nodes, parent.p);
    for (sweeps = 0; sweeps < 64; ++sweeps) {
      changed.zero(s);
      B200_LAUNCH(ctx, trk_hook, cdiv(M, 256), 256, 0, M, ep_node.p, parent.p, changed.p);
      int h_changed = 0;
      B200_CUDA_OK(cudaMemcpyAsync(&h_changed, changed.p, sizeof(int), cudaMemcpyDeviceToHost, s));
      B200_CUDA_OK(cudaStreamSynchronize(s));
      if (!h_changed) break;
    }
    B200_LAUNCH(ctx, trk_flatten, cdiv(n_nodes, 256), 256, 0, n_nodes, parent.p);
    // tracks: stable sort of the (id-sorted) nodes by root
    DevBuf<int> node_idx, root_sorted, node_sorted, tflags, track_of;
    node_idx.alloc(n_nodes); root_sorted.alloc(n_nodes); node_sorted.alloc(n_nodes); tflags.alloc(n_nodes); track_of.alloc(n_nodes);
    B200_LAUNCH(ctx, trk_iota, cdiv(n_nodes, 256), 256, 0, n_nodes, node_idx.p);
    nb = tmp.n;
    cub::DeviceRadixSort::SortPairs(tmp.p, nb, parent.p, root_sorted.p, node_idx.p, node_sorted.p, (int)n_nodes, 0, 32, s);
    B200_LAUNCH(ctx, trk_track_heads, cdiv(n_nodes, 256), 256, 0, n_nodes, root_sorted.p, tflags.p);
    nb = tmp.n;
    cub::DeviceScan::InclusiveSum(tmp.p, nb, tflags.p, track_of.p, (int)n_nodes, s);
    int h_T = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&h_T, track_of.p + n_nodes - 1, sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    T = h_T;
    DevBuf<int> bad, track_start;
    DevBuf<long long> len;
    bad.alloc(T); track_start.alloc((size_t)T + 1); len.alloc((size_t)T + 1);
    track_id.alloc(T); begin.alloc((size_t)T + 1);
    bad.zero(s);
    B200_LAUNCH(ctx, trk_inconsistent, cdiv(n_nodes, 256), 256, 0, n_nodes, root_sorted.p, node_sorted.p, track_of.p, node_gid.p, node_xy.p,
                thres * thres, bad.p);
    B200_LAUNCH(ctx, trk_track_table, cdiv(n_nodes, 256), 256, 0, n_nodes, T, tflags.p, track_of.p, node_sorted.p, node_gid.p, track_id.p,
                track_start.p);
    B200_LAUNCH(ctx, trk_kept_len, cdiv(T + 1, 256), 256, 0, T, track_start.p, bad.p, len.p);
    size_t need4 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, need4, len.p, begin.p, T + 1, s);
    if (need4 > tmp.n) tmp.alloc(need4);
    nb = tmp.n;
    cub::DeviceScan::ExclusiveSum(tmp.p, nb, len.p, begin.p, T + 1, s);
    long long h_obs = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&h_obs, begin.p + T, sizeof(long long), cudaMemcpyDeviceToHost, s));
    std::vector<int> h_bad(T);
    B200_CUDA_OK(cudaMemcpyAsync(h_bad.data(), bad.p, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost, s));
    B200_CUDA_OK(cudaStreamSynchronize(s));
    n_obs = h_obs;
    discarded = 0;
    for (int b : h_bad) discarded += b != 0;
    obs_image.alloc(std::max<long long>(n_obs, 1)); obs_feature.alloc(std::max<long long>(n_obs, 1));
    B200_LAUNCH(ctx, trk_emit, cdiv(n_nodes, 256), 256, 0, n_nodes, track_of.p, track_start.p, begin.p, bad.p, node_sorted.p, node_gid.p,
                obs_image.p, obs_feature.p);
    B200_CUDA_OK(cudaStreamSynchronize(s));   // the scratch buffers go out of scope
  }
};
