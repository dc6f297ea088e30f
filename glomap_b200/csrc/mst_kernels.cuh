// mst_kernels.cuh -- device side of RotationEstimator::InitializeFromMaximumSpanningTree (glomap/estimators/
// global_rotation_averaging.cc:87-138 + math/tree.cc:78-153).  The reference runs Kruskal on max_w - w and composes the
// relative rotations along a BFS of the tree; the same result in O(log n) data-parallel rounds:
//   1. order: one stable radix sort of the FP64 keys max_w - w (-0 folded into +0) carrying the edge index, so an edge's
//      RANK encodes (key, index) -- a total order, hence one minimum spanning forest, the one a stable Kruskal gives
//   2. Boruvka by rank: every component takes its outgoing edge of minimum rank (atomicMin on the rank), roots hook across
//      it (of a mutual pair -- both chose the same edge -- the lower component id stays a root), pointer jumping flattens
//      the components, and the edges inside one component are dropped before the next round (self loops in the first)
//   3. rooting by an Euler tour of the tree: arcs sorted by source give every node a cyclic list; the successor of u->v
//      is the arc after v->u in v's list; the tour is cut before the root's first arc and ranked by pointer jumping
//      (Wyllie).  u->v points down iff it precedes v->u; then parent[v] = u -- the parents any BFS from the root gives
//   4. composition: A_v = R_rel of v's tree edge when v is its ej, R_rel^T when v is its ei (.cc:125-134), and
//      R_v = A_v A_parent ... R_root by synchronous pointer jumping over the ancestors (3x3 FP64 products, double-buffered,
//      so the association of every product is fixed and repeated calls are bit-identical)
// Only the rows of R_rel of tree edges are uploaded (gathered on the host once the tree is known).
#pragma once
#include <cub/cub.cuh>

#include <algorithm>
#include <utility>
#include <vector>

#include "context.cuh"
#include "track_kernels.cuh"   // trk_iota

namespace b200 {

constexpr int kMstNone = 0x7fffffff;

__global__ void mst_keys(int E, const double* __restrict__ w, double wmax, double* __restrict__ key) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= E) return;
  const double k = wmax - w[i];
  key[i] = k == 0.0 ? 0.0 : k;   // the radix sort orders -0 before +0; the comparison Kruskal makes does not
}
// endpoints in rank order
__global__ void mst_gather_ends(int E, const int* __restrict__ order, const int* __restrict__ ei, const int* __restrict__ ej,
                                int* __restrict__ eu, int* __restrict__ ev) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= E) return;
  eu[r] = ei[order[r]];
  ev[r] = ej[order[r]];
}
__global__ void mst_fill(int n, int v, int* __restrict__ a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}
// the components are flat (comp[x] is x's root): each end's component records the minimum rank leaving it
__global__ void mst_min_edge(int m, const int* __restrict__ act, const int* __restrict__ eu, const int* __restrict__ ev,
                             const int* __restrict__ comp, int* __restrict__ best) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int r = act[i], a = comp[eu[r]], b = comp[ev[r]];
  if (a == b) return;
  atomicMin(&best[a], r);
  atomicMin(&best[b], r);
}
// hook[v]: a non-root keeps its root; a root with an outgoing edge points across it, except the lower id of a mutual pair
__global__ void mst_hook(int n, const int* __restrict__ comp, const int* __restrict__ best, const int* __restrict__ eu,
                         const int* __restrict__ ev, int* __restrict__ hook, unsigned char* __restrict__ in_tree) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int c = comp[v];
  const int r = c == v ? best[v] : kMstNone;
  if (r == kMstNone) {
    hook[v] = c;
    return;
  }
  const int a = comp[eu[r]], b = comp[ev[r]];
  const int other = a == v ? b : a;
  in_tree[r] = 1;
  hook[v] = (best[other] == r && v < other) ? v : other;
}
// one pointer-jumping step in place: a pointer only ever moves to an ancestor, and a pass without a change leaves every
// node pointing at a root
__global__ void mst_jump(int n, int* __restrict__ p, int* __restrict__ changed) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int a = p[v], b = p[a];
  if (a != b) {
    p[v] = b;
    *changed = 1;
  }
}
struct MstCross {   // an edge between two components (the components flat)
  const int *eu, *ev, *comp;
  __device__ bool operator()(int r) const { return comp[eu[r]] != comp[ev[r]]; }
};
// arc a = 2k: eu -> ev of tree edge k, a = 2k + 1 the reverse
__global__ void mst_arcs(int A, const int* __restrict__ te, const int* __restrict__ eu, const int* __restrict__ ev,
                         int* __restrict__ src, int* __restrict__ arc) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A) return;
  const int r = te[a >> 1];
  src[a] = (a & 1) ? ev[r] : eu[r];
  arc[a] = a;
}
// with the arcs sorted by source: position of every arc and the segment [lo, hi) of every node with an arc
__global__ void mst_segments(int A, const int* __restrict__ ssrc, const int* __restrict__ sarc, int* __restrict__ pos,
                             int* __restrict__ lo, int* __restrict__ hi) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A) return;
  const int v = ssrc[p];
  pos[sarc[p]] = p;
  if (p == 0 || ssrc[p - 1] != v) lo[v] = p;
  if (p == A - 1 || ssrc[p + 1] != v) hi[v] = p + 1;
}
// successor in the tour (-1: the last arc, the one before the root's first arc); arcs outside the root's component are
// not ranked (-2)
__global__ void mst_succ(int A, const int* __restrict__ src, const int* __restrict__ sarc, const int* __restrict__ pos,
                         const int* __restrict__ lo, const int* __restrict__ hi, const int* __restrict__ comp, int root,
                         int* __restrict__ succ, int* __restrict__ dist) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A) return;
  if (comp[src[a]] != comp[root]) {
    succ[a] = -2;
    dist[a] = 0;
    return;
  }
  const int t = a ^ 1, v = src[t];
  int p = pos[t] + 1;
  if (p == hi[v]) p = lo[v];
  const int s = sarc[p] == sarc[lo[root]] ? -1 : sarc[p];
  succ[a] = s;
  dist[a] = s >= 0 ? 1 : 0;
}
// Wyllie list ranking: dist = number of arcs after this one in the tour
__global__ void mst_rank_step(int A, const int* __restrict__ nx, const int* __restrict__ dist, int* __restrict__ nx2,
                              int* __restrict__ dist2) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= A) return;
  const int s = nx[a];
  if (s < 0) {
    nx2[a] = s;
    dist2[a] = dist[a];
    return;
  }
  dist2[a] = dist[a] + dist[s];
  nx2[a] = nx[s];
}
// edge ids of the tree edges, for the host gather of their R_rel rows
__global__ void mst_tree_edge_ids(int m, const int* __restrict__ te, const int* __restrict__ order, int* __restrict__ eid) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) eid[k] = order[te[k]];
}
// tree edge k of the root's component: the arc that comes first in the tour points down; the child gets its parent and
// A_child (R_rel when the child is ej, R_rel^T when it is ei)
__global__ void mst_orient(int m, const int* __restrict__ te, const int* __restrict__ eu, const int* __restrict__ ev,
                           const int* __restrict__ dist, const int* __restrict__ comp, int root, const double* __restrict__ Rt,
                           int* __restrict__ parent, int* __restrict__ anc, int* __restrict__ depth, double* __restrict__ M) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const int r = te[k], x = eu[r], y = ev[r];
  if (comp[x] != comp[root]) return;
  const bool xy_down = dist[2 * k] > dist[2 * k + 1];
  const int child = xy_down ? y : x, par = xy_down ? x : y;
  parent[child] = par;
  anc[child] = par;
  depth[child] = 1;
  const double* a = Rt + 9 * (size_t)k;
  double* c = M + 9 * (size_t)child;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c[3 * i + j] = child == y ? a[3 * i + j] : a[3 * j + i];
}
__device__ __forceinline__ void mst_mul3(const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ c) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
}
// M_v = A_v ... A_w over the path from v up to (excluding) anc[v]: one synchronous jump M_v <- M_v M_anc, anc <- anc[anc]
__global__ void mst_compose_step(int n, int root, const int* __restrict__ anc, const int* __restrict__ depth,
                                 const double* __restrict__ M, int* __restrict__ anc2, int* __restrict__ depth2,
                                 double* __restrict__ M2, int* __restrict__ more) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int a = anc[v];
  if (a < 0 || a == root) {   // unreached, the root, or done
    anc2[v] = a;
    depth2[v] = depth[v];
    for (int i = 0; i < 9; ++i) M2[9 * (size_t)v + i] = M[9 * (size_t)v + i];
    return;
  }
  mst_mul3(M + 9 * (size_t)v, M + 9 * (size_t)a, M2 + 9 * (size_t)v);
  const int aa = anc[a];
  anc2[v] = aa;
  depth2[v] = depth[v] + depth[a];
  if (aa != root) *more = 1;
}
__global__ void mst_apply(int n, int root, const int* __restrict__ parent, const double* __restrict__ M,
                          const double* __restrict__ Rroot, double* __restrict__ R) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n || parent[v] < 0) return;
  if (v == root) {
    for (int i = 0; i < 9; ++i) R[9 * (size_t)v + i] = Rroot[i];
  } else {
    mst_mul3(M + 9 * (size_t)v, Rroot, R + 9 * (size_t)v);
  }
}

struct MstStats {
  int num_reached = 0, num_tree_edges = 0, boruvka_rounds = 0, max_depth = 0;
};

struct MstRunner {
  b200sfm_ctx* ctx;
  DevBuf<unsigned char> tmp;
  explicit MstRunner(b200sfm_ctx* c) : ctx(c) {}

  template <class F>
  void cub_call(F&& f) {   // size query, grow the scratch, run
    size_t need = 0;
    B200_CUDA_OK(f((void*)nullptr, need));
    if (need > tmp.n) tmp.alloc(need);
    size_t nb = tmp.n;
    B200_CUDA_OK(f((void*)tmp.p, nb));
  }
  int read_int(const int* d) {
    int h = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&h, d, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return h;
  }
  // pointer jumping on p until every node points at a root
  void flatten(int n, int* p, int* flag) {
    do {
      B200_CUDA_OK(cudaMemsetAsync(flag, 0, sizeof(int), ctx->stream));
      B200_LAUNCH(ctx, mst_jump, cdiv(n, 256), 256, 0, n, p, flag);
    } while (read_int(flag));
  }

  // Arguments validated by the caller: E >= 1, endpoints in [0, n), finite weights with maximum wmax.  R [n][9] in/out
  // (rows of unreached nodes untouched), parent [n] out.
  void run(int n, int E, const int* h_ei, const int* h_ej, const double* h_Rrel, const double* h_w, double wmax, int root,
           double* h_R, int* h_parent, MstStats& st) {
    cudaStream_t s = ctx->stream;
    // 1. ranks
    DevBuf<int> eu, ev, order;
    DevBuf<double> key_sorted;
    eu.alloc(E); ev.alloc(E); order.alloc(E); key_sorted.alloc(E);
    {
      DevBuf<int> ei, ej, iota;
      DevBuf<double> w, key;
      ei.alloc(E); ej.alloc(E); iota.alloc(E); w.alloc(E); key.alloc(E);
      ei.upload(h_ei, E, s); ej.upload(h_ej, E, s); w.upload(h_w, E, s);
      B200_LAUNCH(ctx, mst_keys, cdiv(E, 256), 256, 0, E, w.p, wmax, key.p);
      B200_LAUNCH(ctx, trk_iota, cdiv(E, 256), 256, 0, (long long)E, iota.p);
      cub_call([&](void* p, size_t& nb) { return cub::DeviceRadixSort::SortPairs(p, nb, key.p, key_sorted.p, iota.p, order.p, E, 0, 64, s); });
      B200_LAUNCH(ctx, mst_gather_ends, cdiv(E, 256), 256, 0, E, order.p, ei.p, ej.p, eu.p, ev.p);
    }
    key_sorted.release();
    // 2. Boruvka rounds over the edges that still join two components
    DevBuf<int> comp, hook, best, act, act2, d_num, flag;
    DevBuf<unsigned char> in_tree;
    comp.alloc(n); hook.alloc(n); best.alloc(n); act.alloc(E); act2.alloc(E); d_num.alloc(1); flag.alloc(1);
    in_tree.alloc(E);
    in_tree.zero(s);
    B200_LAUNCH(ctx, trk_iota, cdiv(n, 256), 256, 0, (long long)n, comp.p);
    B200_LAUNCH(ctx, trk_iota, cdiv(E, 256), 256, 0, (long long)E, act.p);
    int m_act = E;
    for (;;) {
      cub_call([&](void* p, size_t& nb) {
        return cub::DeviceSelect::If(p, nb, act.p, act2.p, d_num.p, m_act, MstCross{eu.p, ev.p, comp.p}, s);
      });
      std::swap(act.p, act2.p);
      m_act = read_int(d_num.p);
      if (m_act == 0) break;
      ++st.boruvka_rounds;
      B200_LAUNCH(ctx, mst_fill, cdiv(n, 256), 256, 0, n, kMstNone, best.p);
      B200_LAUNCH(ctx, mst_min_edge, cdiv(m_act, 256), 256, 0, m_act, act.p, eu.p, ev.p, comp.p, best.p);
      B200_LAUNCH(ctx, mst_hook, cdiv(n, 256), 256, 0, n, comp.p, best.p, eu.p, ev.p, hook.p, in_tree.p);
      flatten(n, hook.p, flag.p);
      std::swap(comp.p, hook.p);
    }
    act2.release(); best.release(); hook.release();
    DevBuf<int> te;
    te.alloc(std::max(n - 1, 1));
    B200_LAUNCH(ctx, trk_iota, cdiv(E, 256), 256, 0, (long long)E, act.p);
    cub_call([&](void* p, size_t& nb) { return cub::DeviceSelect::Flagged(p, nb, act.p, in_tree.p, te.p, d_num.p, E, s); });
    const int m = read_int(d_num.p);
    st.num_tree_edges = m;
    act.release(); in_tree.release();

    // 3-4. parents and rotations of the root's component
    DevBuf<int> parent, anc, anc2, depth, depth2;
    DevBuf<double> M, M2, Rroot, Rout;
    parent.alloc(n); anc.alloc(n); anc2.alloc(n); depth.alloc(n); depth2.alloc(n);
    M.alloc(9 * (size_t)n); M2.alloc(9 * (size_t)n); Rroot.alloc(9); Rout.alloc(9 * (size_t)n);
    B200_LAUNCH(ctx, mst_fill, cdiv(n, 256), 256, 0, n, -1, parent.p);
    B200_LAUNCH(ctx, mst_fill, cdiv(n, 256), 256, 0, n, -1, anc.p);
    depth.zero(s);
    M.zero(s);
    B200_CUDA_OK(cudaMemcpyAsync(parent.p + root, &root, sizeof(int), cudaMemcpyHostToDevice, s));
    B200_CUDA_OK(cudaMemcpyAsync(anc.p + root, &root, sizeof(int), cudaMemcpyHostToDevice, s));
    Rroot.upload(h_R + 9 * (size_t)root, 9, s);
    if (m > 0) {
      // R_rel rows of the tree edges only
      DevBuf<int> eid;
      eid.alloc(m);
      B200_LAUNCH(ctx, mst_tree_edge_ids, cdiv(m, 256), 256, 0, m, te.p, order.p, eid.p);
      std::vector<int> h_eid(m);
      eid.download(h_eid.data(), m, s);
      const int A = 2 * m;
      DevBuf<int> src, arc, ssrc, sarc, pos, lo, hi, succ, dist, nx2, dist2;
      src.alloc(A); arc.alloc(A); ssrc.alloc(A); sarc.alloc(A); pos.alloc(A); lo.alloc(n); hi.alloc(n);
      succ.alloc(A); dist.alloc(A); nx2.alloc(A); dist2.alloc(A);
      B200_LAUNCH(ctx, mst_arcs, cdiv(A, 256), 256, 0, A, te.p, eu.p, ev.p, src.p, arc.p);
      const int bits = std::max(1, 32 - __builtin_clz((unsigned)n));
      cub_call([&](void* p, size_t& nb) { return cub::DeviceRadixSort::SortPairs(p, nb, src.p, ssrc.p, arc.p, sarc.p, A, 0, bits, s); });
      B200_LAUNCH(ctx, mst_segments, cdiv(A, 256), 256, 0, A, ssrc.p, sarc.p, pos.p, lo.p, hi.p);
      B200_LAUNCH(ctx, mst_succ, cdiv(A, 256), 256, 0, A, src.p, sarc.p, pos.p, lo.p, hi.p, comp.p, root, succ.p, dist.p);
      for (int span = 1; span < A; span *= 2) {
        B200_LAUNCH(ctx, mst_rank_step, cdiv(A, 256), 256, 0, A, succ.p, dist.p, nx2.p, dist2.p);
        std::swap(succ.p, nx2.p);
        std::swap(dist.p, dist2.p);
      }
      B200_CUDA_OK(cudaStreamSynchronize(s));   // h_eid
      std::vector<double> h_Rt(9 * (size_t)m);
      for (int k = 0; k < m; ++k) std::copy(h_Rrel + 9 * (size_t)h_eid[k], h_Rrel + 9 * (size_t)h_eid[k] + 9, h_Rt.data() + 9 * (size_t)k);
      DevBuf<double> Rt;
      Rt.alloc(9 * (size_t)m);
      Rt.upload(h_Rt.data(), 9 * (size_t)m, s);
      B200_LAUNCH(ctx, mst_orient, cdiv(m, 256), 256, 0, m, te.p, eu.p, ev.p, dist.p, comp.p, root, Rt.p, parent.p, anc.p,
                  depth.p, M.p);
      do {
        B200_CUDA_OK(cudaMemsetAsync(flag.p, 0, sizeof(int), s));
        B200_LAUNCH(ctx, mst_compose_step, cdiv(n, 256), 256, 0, n, root, anc.p, depth.p, M.p, anc2.p, depth2.p, M2.p, flag.p);
        std::swap(anc.p, anc2.p);
        std::swap(depth.p, depth2.p);
        std::swap(M.p, M2.p);
      } while (read_int(flag.p));
    }
    B200_LAUNCH(ctx, mst_apply, cdiv(n, 256), 256, 0, n, root, parent.p, M.p, Rroot.p, Rout.p);
    std::vector<int> h_par(n), h_depth(n);
    std::vector<double> h_Rout(9 * (size_t)n);
    parent.download(h_par.data(), n, s);
    depth.download(h_depth.data(), n, s);
    Rout.download(h_Rout.data(), 9 * (size_t)n, s);
    B200_CUDA_OK(cudaStreamSynchronize(s));
    for (int v = 0; v < n; ++v) {
      if (h_par[v] < 0) continue;
      ++st.num_reached;
      st.max_depth = std::max(st.max_depth, h_depth[v]);
      std::copy(h_Rout.data() + 9 * (size_t)v, h_Rout.data() + 9 * (size_t)v + 9, h_R + 9 * (size_t)v);
    }
    if (h_parent) std::copy(h_par.begin(), h_par.end(), h_parent);
  }
};

}  // namespace b200
