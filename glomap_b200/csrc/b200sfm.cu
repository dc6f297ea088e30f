// b200sfm.cu -- C ABI (include/b200sfm.h) over the device solvers.
#include "../../include/b200sfm.h"

#include <new>

#include "ba_solver.cuh"
#include "context.cuh"
#include "gp_solver.cuh"
#include "gravity_kernels.cuh"
#include "mst_kernels.cuh"
#include "pair_kernels.cuh"
#include "prune_kernels.cuh"
#include "ra_solver.cuh"
#include "rig_init_kernels.cuh"
#include "track_kernels.cuh"
#include "track_select_kernels.cuh"
#include "vgc_solver.cuh"
#include "view_graph_kernels.cuh"
#include "pair_config_kernels.cuh"

namespace {

cudaStream_t pool_stream(const b200sfm_ctx* ctx) {
  static const bool dist_pool = !(getenv("B200SFM_ASYNC_ALLOC_DIST") && atoi(getenv("B200SFM_ASYNC_ALLOC_DIST")) == 0);
  return ctx && (ctx->world == 1 || dist_pool) ? ctx->stream : nullptr;
}

template <class F>
int guarded(b200sfm_ctx* ctx, F&& f) {
  // device buffers come from the stream-ordered pool of the context's stream (cudaMallocAsync): a repeated one-shot call
  // re-uses its ~30 buffers instead of paying cudaMalloc / cudaFree (a device-wide synchronisation each), which at 8 GPUs
  // dominated the end-to-end call.  NCCL takes pool memory as ordinary send / receive buffers.
  // B200SFM_ASYNC_ALLOC_DIST=0 restores plain cudaMalloc for multi-rank contexts.
  b200::AllocScope alloc_scope(pool_stream(ctx));
  try {
    return f();
  } catch (const b200::CudaError& e) {
    if (ctx) ctx->err = "CUDA error: " + e.msg + " (line " + std::to_string(e.line) + ")";
    return B200SFM_ERR_CUDA;
  } catch (const NcclError& e) {
    if (ctx) ctx->err = "NCCL error: " + e.msg;
    return B200SFM_ERR_NCCL;
  } catch (const std::bad_alloc&) {
    if (ctx) ctx->err = "host allocation failed";
    return B200SFM_ERR_CUDA;
  } catch (const b200::InvalidInput& e) {
    if (ctx) ctx->err = e.msg;
    return B200SFM_ERR_INVALID_ARG;
  } catch (const std::exception& e) {   // nothing may escape through the extern "C" boundary
    if (ctx) ctx->err = std::string("internal error: ") + e.what();
    return B200SFM_ERR_CUDA;
  } catch (...) {
    if (ctx) ctx->err = "internal error (unknown exception)";
    return B200SFM_ERR_CUDA;
  }
}

// A rank that fails while its peers are inside a collective must not leave them blocked for ever: abort the
// communicator (the peers' pending collectives then fail instead of waiting) before the status is returned.
int finish(b200sfm_ctx* ctx, int rc) {
  // a peer-memory all-reduce that gave up waiting for a rank (p2p_allreduce.cuh) leaves an error word behind
  if (ctx && ctx->world > 1 && ctx->p2p.ready && rc == B200SFM_OK && ctx->p2p.timed_out(ctx->stream)) {
    ctx->err = "peer-memory all-reduce timed out waiting for a rank";
    rc = B200SFM_ERR_NCCL;
  }
  if (ctx && ctx->world > 1 && ctx->comm && (rc == B200SFM_ERR_CUDA || rc == B200SFM_ERR_NCCL)) {
    if (nccl_api().CommAbort) nccl_api().CommAbort(ctx->comm);
    ctx->comm = nullptr;
    ctx->err += " [communicator aborted]";
  }
  return rc;
}

// SPMD guard for the sharded create calls: every rank learns whether ANY rank holds an empty or invalid shard, so
// all of them return the same status instead of one returning early and the others blocking in the next all-reduce.
int agree_status(b200sfm_ctx* ctx, int local_rc) {
  if (!ctx || ctx->world == 1 || !ctx->comm) return local_rc;
  int agreed = local_rc;
  int rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200::DevBuf<double> flag;
    flag.alloc(1);
    const double v = (double)local_rc;
    B200_CUDA_OK(cudaMemcpyAsync(flag.p, &v, sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    ctx->allreduce_max(flag.p, 1);
    double out = 0;
    B200_CUDA_OK(cudaMemcpyAsync(&out, flag.p, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    agreed = (int)out;
    return (int)B200SFM_OK;
  });
  if (rc != B200SFM_OK) return finish(ctx, rc);
  if (agreed != B200SFM_OK && local_rc == B200SFM_OK) ctx->err = "another rank reported an empty or invalid shard";
  return agreed;
}

int create_common(int device, b200sfm_ctx** out) {
  if (!out) return B200SFM_ERR_INVALID_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return B200SFM_ERR_CUDA;   // no CPU fallback
  if (device < 0) device = 0;
  if (device >= ndev) return B200SFM_ERR_INVALID_ARG;
  if (cudaSetDevice(device) != cudaSuccess) return B200SFM_ERR_CUDA;
  b200sfm_ctx* c = new b200sfm_ctx();
  c->device = device;
  if (cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMallocHost(&c->h_scal, b200sfm_ctx::kHScal * sizeof(double)) != cudaSuccess) {
    delete c;
    return B200SFM_ERR_CUDA;
  }
  if (b200::async_alloc_enabled()) {   // keep freed device memory in the pool between solves (best effort)
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      uint64_t thr = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    cudaGetLastError();
  }
  *out = c;
  return B200SFM_OK;
}

}  // namespace

namespace {
struct DevBufRaw {
  void* p = nullptr;
  size_t n = 0;
  bool ensure(size_t bytes) {
    if (bytes <= n) return true;
    if (p) cudaFree(p);
    p = nullptr; n = 0;
    if (cudaMalloc(&p, bytes) != cudaSuccess) return false;
    n = bytes;
    return true;
  }
  ~DevBufRaw() { if (p) cudaFree(p); }
};
}  // namespace

extern "C" {

int b200sfm_version(void) { return B200SFM_VERSION; }

int b200sfm_create(int device, b200sfm_ctx** out) { return create_common(device, out); }

int b200sfm_nccl_unique_id(void* out_id) {
  if (!out_id) return B200SFM_ERR_INVALID_ARG;
  std::string err;
  if (!nccl_api().load(err)) return B200SFM_ERR_NCCL;
  ncclUniqueId id;
  if (nccl_api().GetUniqueId(&id) != ncclSuccess) return B200SFM_ERR_NCCL;
  static_assert(sizeof(ncclUniqueId) == B200SFM_NCCL_ID_BYTES, "ncclUniqueId size");
  std::memcpy(out_id, &id, sizeof(id));
  return B200SFM_OK;
}

int b200sfm_create_dist(int device, int rank, int world_size, const void* nccl_id, b200sfm_ctx** out) {
  if (world_size < 1 || rank < 0 || rank >= world_size || (world_size > 1 && !nccl_id)) return B200SFM_ERR_INVALID_ARG;
  int rc = create_common(device, out);
  if (rc != B200SFM_OK) return rc;
  b200sfm_ctx* c = *out;
  c->rank = rank;
  c->world = world_size;
  if (world_size > 1) {
    if (!nccl_api().load(c->err)) { b200sfm_destroy(c); *out = nullptr; return B200SFM_ERR_NCCL; }
    ncclUniqueId id;
    std::memcpy(&id, nccl_id, sizeof(id));
    if (nccl_api().CommInitRank(&c->comm, world_size, id, rank) != ncclSuccess) {
      b200sfm_destroy(c);
      *out = nullptr;
      return B200SFM_ERR_NCCL;
    }
    // Peer-memory all-reduce for the per-iteration vectors (p2p_allreduce.cuh).  B200SFM_P2P_AR=0 keeps NCCL; a rank
    // without peer access to the others makes every rank fall back (the verdict is exchanged inside setup()).
    // OPT-IN (B200SFM_P2P_AR=1): NCCL's all-reduce of this size was faster than this kernel at 2 and 8 GPUs where it was
    // measured (not on H100), so NCCL stays the default.
    const char* pe = getenv("B200SFM_P2P_AR");
    const bool want_p2p = pe && atoi(pe) == 1;
    if (want_p2p) {
      DevBufRaw stage;   // gather over NCCL: every rank fills its slot of a zeroed buffer, the sum is the concatenation
      auto gather = [&](void* host, size_t bytes_per_rank) -> bool {
        const size_t words = (bytes_per_rank + 7) / 8, total = words * (size_t)world_size;
        if (!stage.ensure(total * 8)) return false;
        std::vector<unsigned long long> h(total, 0ull);
        std::memcpy(h.data() + words * rank, reinterpret_cast<char*>(host) + bytes_per_rank * rank, bytes_per_rank);
        if (cudaMemcpyAsync(stage.p, h.data(), total * 8, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) return false;
        if (nccl_api().AllReduce(stage.p, stage.p, total, ncclUint64, ncclSum, c->comm, c->stream) != ncclSuccess) return false;
        if (cudaMemcpyAsync(h.data(), stage.p, total * 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess) return false;
        if (cudaStreamSynchronize(c->stream) != cudaSuccess) return false;
        for (int r = 0; r < world_size; ++r)
          std::memcpy(reinterpret_cast<char*>(host) + bytes_per_rank * r, h.data() + words * r, bytes_per_rank);
        return true;
      };
      c->p2p.setup(device, rank, world_size, /*cap doubles*/ (size_t)1 << 19, gather);
      cudaGetLastError();
    }
  }
  return B200SFM_OK;
}

void b200sfm_destroy(b200sfm_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->comm) nccl_api().CommDestroy(ctx->comm);
  if (ctx->p2p.ready) {   // the peers have this rank's buffer mapped: everybody stops using it before anybody frees
    cudaStreamSynchronize(ctx->stream);
    if (ctx->comm) {
      double* d = nullptr;
      if (cudaMalloc(&d, sizeof(double)) == cudaSuccess) {
        cudaMemsetAsync(d, 0, sizeof(double), ctx->stream);
        nccl_api().AllReduce(d, d, 1, ncclFloat64, ncclSum, ctx->comm, ctx->stream);
        cudaStreamSynchronize(ctx->stream);
        cudaFree(d);
      }
    }
    ctx->p2p.release();
  }
  if (ctx->comm_stream) {
    cudaStreamSynchronize(ctx->comm_stream);
    cudaStreamDestroy(ctx->comm_stream);
    cudaEventDestroy(ctx->ev_half);
    cudaEventDestroy(ctx->ev_comm);
  }
  if (ctx->stream) {
    cudaStreamSynchronize(ctx->stream);
    cudaStreamDestroy(ctx->stream);
  }
  if (b200::async_alloc_enabled()) {   // give the cached device memory back
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, ctx->device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
    cudaGetLastError();
  }
  if (ctx->h_scal) cudaFreeHost(ctx->h_scal);
  delete ctx;
}

const char* b200sfm_last_error(const b200sfm_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int b200sfm_rank(const b200sfm_ctx* ctx) { return ctx ? ctx->rank : -1; }
int b200sfm_world_size(const b200sfm_ctx* ctx) { return ctx ? ctx->world : -1; }
void* b200sfm_cuda_stream(const b200sfm_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int64_t b200sfm_kernel_launches(const b200sfm_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ---- BA ----------------------------------------------------------------------
void b200sfm_ba_default_opts(b200sfm_ba_opts* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  // bundle_adjustment.h:14-32
  o->optimize_rig_poses = 0;
  o->optimize_rotations = 1;
  o->optimize_translation = 1;
  o->optimize_intrinsics = 1;
  o->optimize_principal_point = 0;
  o->optimize_points = 1;
  o->min_num_view_per_track = 3;
  o->max_num_iterations = 200;
  o->thres_loss_function = 1.0;
  o->function_tolerance = 1e-5;   // optimization_base.h:22
  o->gradient_tolerance = 1e-10;
  o->parameter_tolerance = 1e-8;
  o->pcg_max_iterations = 500;
  o->pcg_min_iterations = 0;
  o->pcg_rel_tolerance = 1e-2;
  o->preconditioner = 1;
  o->profile_kernels = 0;
  o->fixed_num_iterations = 0;
}

int b200sfm_ba_problem_create(b200sfm_ctx* ctx, int32_t C, int32_t P, int64_t N, int32_t K, const int64_t* pt_obs_begin,
                              const int32_t* obs_cam, const double* obs_xy, const int32_t* cam_intr,
                              const int32_t* intr_model, const uint8_t* cam_const_mask, int32_t min_num_view_per_track,
                              b200sfm_ba_problem** out) {
  if (!ctx || !out) return B200SFM_ERR_INVALID_ARG;
  *out = nullptr;
  auto precheck = [&]() -> int {
    if (C <= 0 || P <= 0 || N <= 0 || K <= 0) { ctx->err = "empty problem (no images / tracks / observations)"; return B200SFM_ERR_EMPTY; }
    if (!pt_obs_begin || !obs_cam || !obs_xy || !cam_intr || !intr_model) { ctx->err = "null input array"; return B200SFM_ERR_INVALID_ARG; }
    if (N >= (1ll << 31)) { ctx->err = "N must be < 2^31 per rank"; return B200SFM_ERR_INVALID_ARG; }
    if (pt_obs_begin[0] != 0 || pt_obs_begin[P] != N) { ctx->err = "pt_obs_begin must start at 0 and end at N"; return B200SFM_ERR_INVALID_ARG; }
    for (int k = 0; k < K; ++k)
      if (intr_model[k] < 0 || intr_model[k] > 3) { ctx->err = "unsupported camera model id " + std::to_string(intr_model[k]); return B200SFM_ERR_UNSUPPORTED; }
    return B200SFM_OK;
  };
  int rc = agree_status(ctx, precheck());
  if (rc != B200SFM_OK) return rc;
  b200sfm_ba_problem* p = nullptr;
  rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    p = new b200sfm_ba_problem();
    p->create(ctx, C, P, N, K, pt_obs_begin, obs_cam, obs_xy, cam_intr, intr_model, cam_const_mask,
              min_num_view_per_track, nullptr);
    return (int)B200SFM_OK;
  });
  rc = agree_status(ctx, finish(ctx, rc));
  if (rc != B200SFM_OK) {
    if (p) b200sfm_ba_problem_free(p);
    return rc;
  }
  *out = p;
  return B200SFM_OK;
}

int b200sfm_ba_problem_create_rig(b200sfm_ctx* ctx, int32_t F, int32_t P, int64_t N, int32_t K, int32_t S,
                                  const int64_t* pt_obs_begin, const int32_t* obs_frame, const uint16_t* obs_sensor,
                                  const double* obs_xy, const double* sensor_quat_xyzw, const double* sensor_trans,
                                  const int32_t* sensor_intr, const int32_t* intr_model, const uint8_t* frame_const_mask,
                                  int32_t min_num_view_per_track, b200sfm_ba_problem** out) {
  if (!ctx || !out) return B200SFM_ERR_INVALID_ARG;
  *out = nullptr;
  auto precheck = [&]() -> int {
    if (F <= 0 || P <= 0 || N <= 0 || K <= 0 || S <= 0) { ctx->err = "empty problem (no frames / tracks / observations / sensors)"; return B200SFM_ERR_EMPTY; }
    if (!pt_obs_begin || !obs_frame || !obs_sensor || !obs_xy || !sensor_quat_xyzw || !sensor_trans || !sensor_intr || !intr_model) {
      ctx->err = "null input array";
      return B200SFM_ERR_INVALID_ARG;
    }
    if (N >= (1ll << 31)) { ctx->err = "N must be < 2^31 per rank"; return B200SFM_ERR_INVALID_ARG; }
    if (S > 65535 || (long long)F * S >= (1ll << 31) - 1) { ctx->err = "too many sensors (S <= 65535, F * S < 2^31)"; return B200SFM_ERR_INVALID_ARG; }
    if (pt_obs_begin[0] != 0 || pt_obs_begin[P] != N) { ctx->err = "pt_obs_begin must start at 0 and end at N"; return B200SFM_ERR_INVALID_ARG; }
    for (int k = 0; k < K; ++k)
      if (intr_model[k] < 0 || intr_model[k] > 3) { ctx->err = "unsupported camera model id " + std::to_string(intr_model[k]); return B200SFM_ERR_UNSUPPORTED; }
    for (int i = 0; i < S; ++i)
      if (sensor_intr[i] < 0 || sensor_intr[i] >= K) { ctx->err = "sensor_intr out of range"; return B200SFM_ERR_INVALID_ARG; }
    for (int64_t o = 0; o < N; ++o)
      if (obs_sensor[o] >= S || obs_frame[o] < 0 || obs_frame[o] >= F) { ctx->err = "obs_frame / obs_sensor out of range"; return B200SFM_ERR_INVALID_ARG; }
    return B200SFM_OK;
  };
  int rc = agree_status(ctx, precheck());
  if (rc != B200SFM_OK) return rc;
  b200sfm_ba_problem* p = nullptr;
  rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    p = new b200sfm_ba_problem();
    p->create(ctx, F, P, N, K, pt_obs_begin, obs_frame, obs_xy, nullptr, intr_model, frame_const_mask,
              min_num_view_per_track, nullptr, S, obs_sensor, sensor_quat_xyzw, sensor_trans, sensor_intr);
    return (int)B200SFM_OK;
  });
  rc = agree_status(ctx, finish(ctx, rc));
  if (rc != B200SFM_OK) {
    if (p) b200sfm_ba_problem_free(p);
    return rc;
  }
  *out = p;
  return B200SFM_OK;
}

int b200sfm_ba_problem_set_images(b200sfm_ba_problem* p, int32_t I, const int32_t* image_frame, const int32_t* image_sensor) {
  if (!p || I <= 0 || !image_frame || !image_sensor) return B200SFM_ERR_INVALID_ARG;
  if (p->S <= 0) { p->ctx->err = "the problem has no rig sensors (b200sfm_ba_problem_create_rig)"; return B200SFM_ERR_INVALID_ARG; }
  for (int32_t i = 0; i < I; ++i)
    if (image_frame[i] < 0 || image_frame[i] >= p->C || image_sensor[i] < 0 || image_sensor[i] >= p->S) {
      p->ctx->err = "image_frame / image_sensor out of range";
      return B200SFM_ERR_INVALID_ARG;
    }
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->set_images(I, image_frame, image_sensor);
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_set_sensor_variable(b200sfm_ba_problem* p, const uint8_t* sensor_variable) {
  if (!p || !sensor_variable) return B200SFM_ERR_INVALID_ARG;
  if (p->S <= 0) { p->ctx->err = "the problem has no rig sensors (b200sfm_ba_problem_create_rig)"; return B200SFM_ERR_INVALID_ARG; }
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->set_sensor_variable(sensor_variable);
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_get_sensor_poses(b200sfm_ba_problem* p, double* sensor_quat_xyzw, double* sensor_trans) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  if (p->S <= 0) { p->ctx->err = "the problem has no rig sensors (b200sfm_ba_problem_create_rig)"; return B200SFM_ERR_INVALID_ARG; }
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->get_sensor_poses(sensor_quat_xyzw, sensor_trans);
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_set_state(b200sfm_ba_problem* p, const double* intr_params, const double* quat_xyzw,
                                 const double* trans, const double* points) {
  if (!p || !intr_params || !quat_xyzw || !trans || !points) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->set_state(intr_params, quat_xyzw, trans, points, nullptr);
    B200_CUDA_OK(cudaStreamSynchronize(p->ctx->stream));
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_get_state(b200sfm_ba_problem* p, double* intr_params, double* quat_xyzw, double* trans,
                                 double* points) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->get_state(intr_params, quat_xyzw, trans, points, nullptr);
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_save_state(b200sfm_ba_problem* p) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->save_state();
    B200_CUDA_OK(cudaStreamSynchronize(p->ctx->stream));
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_restore_state(b200sfm_ba_problem* p) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    if (!p->restore_state()) { p->ctx->err = "no saved state"; return (int)B200SFM_ERR_INVALID_ARG; }
    B200_CUDA_OK(cudaStreamSynchronize(p->ctx->stream));
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_solve(b200sfm_ba_problem* p, const b200sfm_ba_opts* opts, b200sfm_lm_stats* stats) {
  if (!p || !opts) return B200SFM_ERR_INVALID_ARG;
  return finish(p->ctx, guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    if (opts->min_num_view_per_track != p->min_views) {
      p->ctx->err = "min_num_view_per_track differs from the value the problem was created with";
      return (int)B200SFM_ERR_INVALID_ARG;
    }
    if (stats) std::memset(stats, 0, sizeof(*stats));
    return p->solve(*opts, stats);
  }));
}

int b200sfm_ba_problem_cost(b200sfm_ba_problem* p, const b200sfm_ba_opts* opts, double* cost) {
  if (!p || !opts || !cost) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    B200_LAUNCH(p->ctx, b200::k_eff_mask, b200::cdiv(p->C, 256), 256, 0, p->C, p->cam_mask_base.p, 0, 0, p->cam_mask.p);
    *cost = p->eval_cost(p->cur, opts->thres_loss_function);
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_normalize(b200sfm_ba_problem* p, int32_t fixed_scale, double extent, double p0, double p1,
                                 double* scale_out, double* translation_out) {
  if (!p || !(extent > 0.0) || !(p0 >= 0.0) || !(p1 <= 1.0) || !(p0 <= p1)) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->normalize(fixed_scale != 0, extent, p0, p1, scale_out, translation_out);
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_undistort(b200sfm_ba_problem* p, double* bearings_out) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->undistort(bearings_out);
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_filter_reprojection(b200sfm_ba_problem* p, double max_reprojection_error, uint8_t* keep,
                                           int64_t* num_tracks_changed) {
  if (!p || !keep) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    const long long n = p->run_filter(0, max_reprojection_error, nullptr, nullptr, keep);
    if (num_tracks_changed) *num_tracks_changed = n;
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_filter_angle(b200sfm_ba_problem* p, const double* bearings, const uint8_t* cam_calibrated,
                                    double max_angle_error_deg, uint8_t* keep, int64_t* num_tracks_changed) {
  if (!p || !keep) return B200SFM_ERR_INVALID_ARG;   // bearings == NULL: the resident ones (b200sfm_ba_problem_undistort)
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    const long long n = p->run_filter(1, max_angle_error_deg, bearings, cam_calibrated, keep);
    if (num_tracks_changed) *num_tracks_changed = n;
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_filter_reprojection_normalized(b200sfm_ba_problem* p, const double* bearings,
                                                      double max_reprojection_error, uint8_t* keep,
                                                      int64_t* num_tracks_changed) {
  if (!p || !keep) return B200SFM_ERR_INVALID_ARG;   // bearings == NULL: the resident ones (b200sfm_ba_problem_undistort)
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    const long long n = p->run_filter(3, max_reprojection_error, bearings, nullptr, keep);
    if (num_tracks_changed) *num_tracks_changed = n;
    return (int)B200SFM_OK;
  });
}

int b200sfm_ba_problem_filter_triangulation_angle(b200sfm_ba_problem* p, double min_angle_deg, uint8_t* keep_track,
                                                  int64_t* num_tracks_removed) {
  if (!p || !keep_track) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    const long long n = p->run_filter(2, min_angle_deg, nullptr, nullptr, keep_track);
    if (num_tracks_removed) *num_tracks_removed = n;
    return (int)B200SFM_OK;
  });
}

// ---- test probe (include/b200sfm_testing.h) ----------------------------------------------------------------------
int b200sfm_test_ba_step(b200sfm_ba_problem* p, const b200sfm_ba_opts* opts, double first_radius, double radius,
                         b200sfm_test_ba_step_out* out) {
  if (!p || !opts || !out || !(radius > 0.0) || first_radius < 0.0) return B200SFM_ERR_INVALID_ARG;
  if (p->ctx->world > 1) { p->ctx->err = "the test probe is single-rank only"; return B200SFM_ERR_INVALID_ARG; }
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    if (opts->min_num_view_per_track != p->min_views) {
      p->ctx->err = "min_num_view_per_track differs from the value the problem was created with";
      return (int)B200SFM_ERR_INVALID_ARG;
    }
    p->test_step(*opts, first_radius, radius, out);
    return (int)B200SFM_OK;
  });
}

int b200sfm_test_ba_apply(b200sfm_ba_problem* p, const double* x, double* y) {
  if (!p || !x || !y) return B200SFM_ERR_INVALID_ARG;
  if (p->ctx->world > 1) { p->ctx->err = "the test probe is single-rank only"; return B200SFM_ERR_INVALID_ARG; }
  if (!p->probe_ready) { p->ctx->err = "b200sfm_test_ba_apply needs a preceding b200sfm_test_ba_step"; return B200SFM_ERR_INVALID_ARG; }
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->test_apply(x, y);
    return (int)B200SFM_OK;
  });
}

void b200sfm_ba_problem_free(b200sfm_ba_problem* p) {
  if (!p) return;
  cudaSetDevice(p->ctx->device);
  cudaStreamSynchronize(p->ctx->stream);
  b200::AllocScope alloc_scope(pool_stream(p->ctx));   // back to the stream-ordered pool
  delete p;
}

int b200sfm_ba_solve(b200sfm_ctx* ctx, const b200sfm_ba_opts* opts, int32_t C, int32_t P, int64_t N, int32_t K,
                     const int64_t* pt_obs_begin, const int32_t* obs_cam, const double* obs_xy, const int32_t* cam_intr,
                     const int32_t* intr_model, double* intr_params, double* quat_xyzw, double* trans,
                     const uint8_t* cam_const_mask, double* points, b200sfm_lm_stats* stats) {
  if (!ctx || !opts || !intr_params || !quat_xyzw || !trans || !points) return B200SFM_ERR_INVALID_ARG;
  b200sfm_lm_stats st{};
  cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr, e3 = nullptr;
  b200sfm_ba_problem* p = nullptr;
  const long long launches0 = ctx->launches;
  int rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    B200_CUDA_OK(cudaEventCreate(&e0)); B200_CUDA_OK(cudaEventCreate(&e1));
    B200_CUDA_OK(cudaEventCreate(&e2)); B200_CUDA_OK(cudaEventCreate(&e3));
    B200_CUDA_OK(cudaEventRecord(e0, ctx->stream));
    return (int)B200SFM_OK;
  });
  if (rc != B200SFM_OK) return rc;
  rc = b200sfm_ba_problem_create(ctx, C, P, N, K, pt_obs_begin, obs_cam, obs_xy, cam_intr, intr_model, cam_const_mask,
                                 opts->min_num_view_per_track, &p);
  if (rc == B200SFM_OK) {
    rc = guarded(ctx, [&]() {
      st.h2d_bytes = N * 20 + ((long long)P + 1) * 4 + (long long)C * 5 + K * 4;
      p->set_state(intr_params, quat_xyzw, trans, points, &st);
      B200_CUDA_OK(cudaEventRecord(e1, ctx->stream));
      const long long upload_launches = ctx->launches - launches0;
      b200sfm_lm_stats solve_st = st;
      solve_st.kernel_launches = upload_launches;
      int r = p->solve(*opts, &solve_st);
      if (r != B200SFM_OK) return r;
      B200_CUDA_OK(cudaEventRecord(e2, ctx->stream));
      p->get_state(intr_params, quat_xyzw, trans, points, &solve_st);
      B200_CUDA_OK(cudaEventRecord(e3, ctx->stream));
      B200_CUDA_OK(cudaEventSynchronize(e3));
      float a, b, c;
      B200_CUDA_OK(cudaEventElapsedTime(&a, e0, e1));
      B200_CUDA_OK(cudaEventElapsedTime(&b, e2, e3));
      B200_CUDA_OK(cudaEventElapsedTime(&c, e0, e3));
      solve_st.ms_h2d = a;
      solve_st.ms_d2h = b;
      solve_st.ms_total = c;
      st = solve_st;
      return (int)B200SFM_OK;
    });
  }
  if (p) b200sfm_ba_problem_free(p);
  for (cudaEvent_t e : {e0, e1, e2, e3})
    if (e) cudaEventDestroy(e);
  if (stats) *stats = st;
  return rc;
}

// ---- image pair inliers ----------------------------------------------------------
int b200sfm_image_pairs_inlier_count(b200sfm_ctx* ctx, int32_t num_images, const int64_t* feature_begin, const double* features,
                                     const int32_t* image_intr, int32_t K, const int32_t* intr_model, const double* intr_params,
                                     int64_t num_pairs, const int32_t* pair_image1, const int32_t* pair_image2,
                                     const int32_t* pair_config, const double* pair_quat_xyzw, const double* pair_trans,
                                     const double* pair_F, const double* pair_H, const int64_t* match_begin, const int32_t* matches,
                                     double max_epipolar_error_E, double max_epipolar_error_F, double max_epipolar_error_H,
                                     uint8_t* is_inlier, int32_t* num_inliers, double* score) {
  if (!ctx || num_images < 0 || K < 0 || num_pairs < 0) return B200SFM_ERR_INVALID_ARG;
  if (num_pairs == 0) return B200SFM_OK;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if (!feature_begin || (num_images > 0 && !image_intr) || (K > 0 && (!intr_model || !intr_params)) || !pair_image1 ||
      !pair_image2 || !pair_config || !pair_quat_xyzw || !pair_trans || !pair_F || !pair_H || !match_begin || !num_inliers || !score)
    return invalid("null argument");
  if (feature_begin[0] != 0) return invalid("feature_begin[0] must be 0");
  for (int32_t i = 0; i < num_images; ++i)
    if (feature_begin[i + 1] < feature_begin[i]) return invalid("feature_begin must be non-decreasing");
  const long long nf = feature_begin[num_images];
  if (nf > 0 && !features) return invalid("null features");
  if (match_begin[0] != 0) return invalid("match_begin[0] must be 0");
  std::vector<unsigned char> need(num_images, 0);   // images with features_undist: the images of a CALIBRATED pair
  for (int64_t e = 0; e < num_pairs; ++e) {
    if (match_begin[e + 1] < match_begin[e]) return invalid("match_begin must be non-decreasing");
    const int32_t a = pair_image1[e], b = pair_image2[e];
    if (a < 0 || a >= num_images || b < 0 || b >= num_images) return invalid("pair image index out of range");
    if (pair_config[e] != B200SFM_TWO_VIEW_CALIBRATED) continue;
    for (int32_t i : {a, b}) {
      if (image_intr[i] < 0 || image_intr[i] >= K) return invalid("image_intr index out of range");
      const int32_t m = intr_model[image_intr[i]];
      if (m < B200SFM_SIMPLE_PINHOLE || m > B200SFM_RADIAL) {
        ctx->err = "camera model " + std::to_string(m) + " of a CALIBRATED pair is not supported";
        return B200SFM_ERR_UNSUPPORTED;
      }
      need[i] = 1;
    }
  }
  const long long M = match_begin[num_pairs];
  if (M > 0 && (!matches || !is_inlier)) return invalid("null matches / is_inlier");
  return guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    if (!b200::image_pairs_inlier_count(ctx, num_images, nf, feature_begin, features, image_intr, K, intr_model, intr_params, num_pairs,
                                        pair_image1, pair_image2, pair_config, pair_quat_xyzw, pair_trans, pair_F, pair_H, match_begin,
                                        matches, max_epipolar_error_E, max_epipolar_error_F, max_epipolar_error_H, need.data(), is_inlier,
                                        num_inliers, score))
      throw b200::InvalidInput{"match feature index out of range of its image"};
    return (int)B200SFM_OK;
  });
}

// ---- view-graph passes of stage 3 -------------------------------------------------
int b200sfm_view_graph_filter_rotations(b200sfm_ctx* ctx, int32_t num_images, const double* cam_from_world_quat_xyzw,
                                        const uint8_t* image_registered, int64_t num_pairs, const int32_t* pair_image1,
                                        const int32_t* pair_image2, const double* pair_quat_xyzw, double max_angle_deg,
                                        uint8_t* pair_valid, int64_t* num_invalidated) {
  if (!ctx || num_images < 0 || num_pairs < 0 || !num_invalidated) return B200SFM_ERR_INVALID_ARG;
  *num_invalidated = 0;
  if (num_pairs == 0) return B200SFM_OK;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if ((num_images > 0 && !cam_from_world_quat_xyzw) || !pair_image1 || !pair_image2 || !pair_quat_xyzw || !pair_valid)
    return invalid("null argument");
  return guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200::ViewGraphRunner r(ctx);
    long long n = 0;
    if (!r.filter_rotations(num_images, cam_from_world_quat_xyzw, image_registered, num_pairs, pair_image1, pair_image2,
                            pair_quat_xyzw, max_angle_deg, pair_valid, &n))
      throw b200::InvalidInput{"pair image index outside [0, num_images)"};
    B200_CUDA_OK(cudaGetLastError());
    *num_invalidated = n;
    return (int)B200SFM_OK;
  });
}

int b200sfm_view_graph_keep_largest_component(b200sfm_ctx* ctx, int32_t num_frames, int32_t num_images, const int32_t* image_frame,
                                              int64_t num_pairs, const int32_t* pair_image1, const int32_t* pair_image2,
                                              uint8_t* pair_valid, uint8_t* frame_registered, int32_t* num_registered_images) {
  if (!ctx || num_frames < 0 || num_images < 0 || num_pairs < 0 || !num_registered_images) return B200SFM_ERR_INVALID_ARG;
  *num_registered_images = 0;
  if (num_pairs == 0) return B200SFM_OK;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if ((num_images > 0 && !image_frame) || (num_frames > 0 && !frame_registered) || !pair_image1 || !pair_image2 || !pair_valid)
    return invalid("null argument");
  return guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200::ViewGraphRunner r(ctx);
    int n = 0;
    if (!r.keep_largest_component(num_frames, num_images, image_frame, num_pairs, pair_image1, pair_image2, pair_valid,
                                  frame_registered, &n))
      throw b200::InvalidInput{"pair image index outside [0, num_images) or image_frame outside [0, num_frames)"};
    B200_CUDA_OK(cudaGetLastError());
    *num_registered_images = n;
    return (int)B200SFM_OK;
  });
}

// ---- stage 0: UpdateImagePairsConfig -----------------------------------------------
int b200sfm_view_graph_update_pairs_config(b200sfm_ctx* ctx, int32_t K, const int32_t* intr_model, const double* intr_params,
                                           const uint8_t* has_prior_focal, int64_t num_pairs, const int32_t* pair_cam1,
                                           const int32_t* pair_cam2, const uint8_t* pair_valid, const double* pair_quat_xyzw,
                                           const double* pair_trans, int32_t* pair_config, double* pair_F, int64_t* num_promoted) {
  if (!ctx || K < 0 || num_pairs < 0 || !num_promoted) return B200SFM_ERR_INVALID_ARG;
  *num_promoted = 0;
  if (num_pairs == 0) return B200SFM_OK;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if ((K > 0 && (!intr_model || !intr_params || !has_prior_focal)) || !pair_cam1 || !pair_cam2 || !pair_valid ||
      !pair_quat_xyzw || !pair_trans || !pair_config || !pair_F)
    return invalid("null argument");
  if (K == 0) return invalid("pair camera index outside [0, K)");
  return guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    long long n = 0;
    const int r = b200::update_image_pairs_config(ctx, K, intr_model, intr_params, has_prior_focal, num_pairs, pair_cam1, pair_cam2,
                                                  pair_valid, pair_quat_xyzw, pair_trans, pair_config, pair_F, &n);
    if (r == 1) throw b200::InvalidInput{"pair camera index outside [0, K)"};
    if (r == 2) {
      ctx->err = "camera model outside 0-3 in a pair to be promoted to CALIBRATED";
      return (int)B200SFM_ERR_UNSUPPORTED;
    }
    B200_CUDA_OK(cudaGetLastError());
    *num_promoted = n;
    return (int)B200SFM_OK;
  });
}

// ---- view-graph calibration -------------------------------------------------------
void b200sfm_vgc_default_opts(b200sfm_vgc_opts* o) {
  if (!o) return;
  *o = b200sfm_vgc_opts{};
  o->max_num_iterations = 100;
  o->max_num_line_search_step_size_iterations = 20;
  o->thres_loss_function = 1e-2;
  o->function_tolerance = 1e-5;
  o->gradient_tolerance = 1e-10;
  o->parameter_tolerance = 1e-8;
  o->thres_lower_ratio = 0.1;
  o->thres_higher_ratio = 10.0;
  o->thres_two_view_error = 2.0;
  o->pcg_max_iterations = 1000;
  o->pcg_min_iterations = 0;
  o->pcg_rel_tolerance = 1e-12;
}

int b200sfm_view_graph_calibrate(b200sfm_ctx* ctx, const b200sfm_vgc_opts* opts, int32_t K, const double* principal_point,
                                 double* focal, const uint8_t* focal_constant, int64_t E, const int32_t* cam1,
                                 const int32_t* cam2, const double* F, uint8_t* pair_valid, uint8_t* cam_accepted,
                                 double* pair_residual, b200sfm_lm_stats* stats) {
  if (!ctx || !opts || K < 0 || E < 0) return B200SFM_ERR_INVALID_ARG;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if (E > 0 && (!principal_point || !focal || !cam1 || !cam2 || !F || !pair_valid || !cam_accepted))
    return invalid("null argument");
  if (E > 0x7fffffffLL) return invalid("more than 2^31 - 1 pairs");
  if (ctx->world > 1) {
    ctx->err = "view-graph calibration runs on a single-rank context";
    return B200SFM_ERR_UNSUPPORTED;
  }
  b200sfm_lm_stats st{};
  st.usable = 1;
  st.num_observations = E;
  // cameras with a parameter block (used by a pair) and the variable ones among them (.cc:105-120)
  std::vector<uint8_t> has_block(K, 0), var(K, 0);
  for (int64_t e = 0; e < E; ++e) {
    const int32_t a = cam1[e], b = cam2[e];
    if (a < 0 || a >= K || b < 0 || b >= K) return invalid("pair camera index out of range [0, K)");
    has_block[a] = has_block[b] = 1;
  }
  int n_var = 0;
  for (int32_t k = 0; k < K; ++k) {
    var[k] = has_block[k] && !(focal_constant && focal_constant[k]);
    n_var += var[k];
  }
  if (n_var == 0) {   // E == 0 included: "No cameras to optimize", return true (.cc:30-35)
    if (stats) *stats = st;
    return B200SFM_OK;
  }
  const int rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200::VgcSolver sv;
    std::vector<double> f0(focal, focal + K);
    double ms_h2d = 0, ms_d2h = 0;
    sv.create(ctx, K, E, principal_point, focal, var.data(), cam1, cam2, F, &ms_h2d);
    sv.solve(*opts, st);
    sv.finish(opts->thres_two_view_error, focal, pair_valid, pair_residual, &ms_d2h);
    st.ms_h2d = ms_h2d;
    st.ms_d2h = ms_d2h;
    st.h2d_bytes = E * (9 * 8 + 2 * 4) + (int64_t)K * (3 * 8 + 1);
    st.d2h_bytes = E * (1 + (pair_residual ? 16 : 0)) + (int64_t)K * 8;
    // CopyBackResults (.cc:122-148): a camera whose estimate is out of [lower, higher] x its focal keeps its parameters
    for (int32_t k = 0; k < K; ++k) {
      if (!has_block[k]) {
        focal[k] = f0[k];
        cam_accepted[k] = 0;
        continue;
      }
      const double ratio = focal[k] / f0[k];
      cam_accepted[k] = (ratio > opts->thres_higher_ratio || ratio < opts->thres_lower_ratio) ? 0 : 1;
    }
    return (int)B200SFM_OK;
  });
  if (stats) *stats = st;
  return rc;
}

// ---- reconstruction pruning -------------------------------------------------------
int b200sfm_prune_weakly_connected(b200sfm_ctx* ctx, int32_t num_frames, int64_t num_tracks, const int64_t* track_begin,
                                   const int32_t* obs_frame, const uint8_t* frame_self_loop, int32_t min_num_observations,
                                   int64_t max_pair_keys_per_pass, int32_t* cluster_id, uint8_t* is_registered,
                                   int32_t* num_clusters, b200sfm_prune_stats* stats) {
  if (!ctx || num_frames < 0 || num_tracks < 0 || !track_begin || !num_clusters || (num_frames > 0 && (!cluster_id || !is_registered)))
    return B200SFM_ERR_INVALID_ARG;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if (num_tracks > 0x7ffffffeLL) return invalid("more than 2^31 - 2 tracks");
  if (track_begin[0] != 0) return invalid("track_begin[0] must be 0");
  for (int64_t t = 0; t < num_tracks; ++t)
    if (track_begin[t + 1] < track_begin[t]) return invalid("track_begin must be non-decreasing");
  const long long n = track_begin[num_tracks];
  if (n > 0 && !obs_frame) return invalid("null obs_frame");
  if (ctx->world > 1) {
    ctx->err = "reconstruction pruning runs on a single-rank context";
    return B200SFM_ERR_UNSUPPORTED;
  }
  const long long max_keys = max_pair_keys_per_pass <= 0 ? (1LL << 27) : std::min<long long>(max_pair_keys_per_pass, 1LL << 30);
  b200::PruneStats st;
  const int rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200::PruneRunner r(ctx);
    static_assert(sizeof(long long) == sizeof(int64_t), "track_begin is 64-bit");
    if (!r.run(num_frames, (int)num_tracks, n, reinterpret_cast<const long long*>(track_begin), obs_frame, frame_self_loop,
               min_num_observations, max_keys, cluster_id, is_registered, num_clusters, st))
      throw b200::InvalidInput{"obs_frame outside [0, num_frames)"};
    B200_CUDA_OK(cudaGetLastError());   // a failed launch of this call is reported here, not left pending for the next caller
    return (int)B200SFM_OK;
  });
  if (stats) {
    stats->covisible_pairs = st.covisible_pairs;
    stats->pairs_min5 = st.pairs_min5;
    stats->visibility_edges = st.visibility_edges;
    stats->strong_threshold = st.strong_threshold;
    stats->clustering_iterations = st.clustering_iterations;
    stats->largest_component_frames = st.largest_component_frames;
  }
  return rc;
}

// ---- gravity refinement -----------------------------------------------------------
void b200sfm_gravity_default_opts(b200sfm_gravity_opts* o) {
  if (!o) return;
  *o = b200sfm_gravity_opts{};
  o->max_outlier_ratio = 0.5;
  o->max_gravity_error = 1.0;
  o->min_num_neighbors = 7;
  o->max_num_iterations = 100;
  o->function_tolerance = 1e-5;
  o->gradient_tolerance = 1e-10;
  o->parameter_tolerance = 1e-8;
}

int b200sfm_gravity_refine(b200sfm_ctx* ctx, const b200sfm_gravity_opts* opts, int32_t F, const double* R_align,
                           const uint8_t* has_gravity, int64_t E, const int32_t* frame1, const int32_t* frame2,
                           const double* M, double* gravity, uint8_t* status, b200sfm_gravity_stats* stats) {
  if (!ctx || !opts || F < 0 || E < 0) return B200SFM_ERR_INVALID_ARG;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if (E > 0 && (!R_align || !has_gravity || !frame1 || !frame2 || !M || !gravity || !status)) return invalid("null argument");
  if (E >= (1LL << 30)) return invalid("2^30 or more pairs");
  if (ctx->world > 1) {
    ctx->err = "gravity refinement runs on a single-rank context";
    return B200SFM_ERR_UNSUPPORTED;
  }
  const auto t0 = std::chrono::steady_clock::now();
  b200::GravityStats st;
  int rc = B200SFM_OK;
  if (E > 0 && F > 0) {
    rc = guarded(ctx, [&]() {
      B200_CUDA_OK(cudaSetDevice(ctx->device));
      const b200::GravityParams prm{opts->max_outlier_ratio,  opts->max_gravity_error,  opts->min_num_neighbors,
                                    opts->max_num_iterations, opts->function_tolerance, opts->gradient_tolerance,
                                    opts->parameter_tolerance};
      b200::GravityRunner r(ctx);
      const int bad = r.run(prm, F, R_align, has_gravity, E, frame1, frame2, M, gravity, status, st);
      B200_CUDA_OK(cudaGetLastError());   // a failed launch of this call is reported here, not left pending for the next caller
      if (bad & 1) throw b200::InvalidInput{"frame index outside [0, F)"};
      if (bad & 2) throw b200::InvalidInput{"a frame with gravity has a non-finite or zero gravity"};
      if (bad & 4) throw b200::InvalidInput{"a pair has a non-finite M"};
      return (int)B200SFM_OK;
    });
  } else if (E > 0) {
    rc = invalid("frame index outside [0, F)");   // F == 0: every index is out of range
  }
  if (stats) {
    *stats = b200sfm_gravity_stats{};
    stats->error_prone_frames = st.error_prone;
    stats->rectified_frames = st.rectified;
    stats->too_few_terms = st.too_few;
    stats->max_lm_iterations = st.max_lm_iterations;
    stats->lm_iterations = st.lm_iterations;
    stats->ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    stats->ms_h2d = st.ms_h2d;
    stats->ms_error_test = st.ms_error_test;
    stats->ms_csr = st.ms_csr;
    stats->ms_refine = st.ms_refine;
  }
  return rc;
}

// ---- track establishment ----------------------------------------------------------
int b200sfm_tracks_establish(b200sfm_ctx* ctx, int64_t num_matches, const uint64_t* gid1, const uint64_t* gid2, const double* xy1,
                             const double* xy2, double thres_inconsistency, b200sfm_tracks** out, int64_t* num_tracks,
                             int64_t* num_observations, int64_t* num_discarded) {
  if (!ctx || !out || num_matches < 0 || (num_matches > 0 && (!gid1 || !gid2 || !xy1 || !xy2)) || !(thres_inconsistency >= 0.0))
    return B200SFM_ERR_INVALID_ARG;
  *out = nullptr;
  b200sfm_tracks* t = nullptr;
  int rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    t = new b200sfm_tracks();
    t->ctx = ctx;
    static_assert(sizeof(unsigned long long) == sizeof(uint64_t), "global feature ids are 64-bit");
    t->build(num_matches, reinterpret_cast<const unsigned long long*>(gid1), reinterpret_cast<const unsigned long long*>(gid2), xy1, xy2,
             thres_inconsistency);
    return (int)B200SFM_OK;
  });
  if (rc != B200SFM_OK) {
    if (t) {
      guarded(ctx, [&]() { delete t; return (int)B200SFM_OK; });
    }
    return rc;
  }
  *out = t;
  if (num_tracks) *num_tracks = t->T;
  if (num_observations) *num_observations = t->n_obs;
  if (num_discarded) *num_discarded = t->discarded;
  return B200SFM_OK;
}

int b200sfm_tracks_get(b200sfm_tracks* t, uint64_t* track_ids, int64_t* begin, uint32_t* obs_image, uint32_t* obs_feature) {
  if (!t) return B200SFM_ERR_INVALID_ARG;
  return guarded(t->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(t->ctx->device));
    cudaStream_t s = t->ctx->stream;
    if (t->T > 0) {
      if (track_ids) B200_CUDA_OK(cudaMemcpyAsync(track_ids, t->track_id.p, (size_t)t->T * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
      if (begin) B200_CUDA_OK(cudaMemcpyAsync(begin, t->begin.p, ((size_t)t->T + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
      if (obs_image && t->n_obs > 0) B200_CUDA_OK(cudaMemcpyAsync(obs_image, t->obs_image.p, (size_t)t->n_obs * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      if (obs_feature && t->n_obs > 0)
        B200_CUDA_OK(cudaMemcpyAsync(obs_feature, t->obs_feature.p, (size_t)t->n_obs * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    } else if (begin) {
      begin[0] = 0;
    }
    B200_CUDA_OK(cudaStreamSynchronize(s));
    return (int)B200SFM_OK;
  });
}

void b200sfm_tracks_free(b200sfm_tracks* t) {
  if (!t) return;
  guarded(t->ctx, [&]() {
    cudaSetDevice(t->ctx->device);
    delete t;
    return (int)B200SFM_OK;
  });
}

int b200sfm_tracks_select(b200sfm_ctx* ctx, int64_t num_tracks, const uint64_t* track_ids, const int64_t* begin,
                          const uint32_t* obs_image, int32_t num_registered, const uint32_t* registered_image_ids,
                          int32_t min_num_tracks_per_view, int32_t min_num_view_per_track, int32_t max_num_view_per_track,
                          int32_t max_num_tracks, uint8_t* keep, int64_t* num_selected) {
  if (!ctx || !begin || !num_selected || num_tracks < 0 || num_registered < 0) return B200SFM_ERR_INVALID_ARG;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if (num_tracks > 0 && (!track_ids || !keep)) return invalid("null track_ids or keep");
  if (num_registered > 0 && !registered_image_ids) return invalid("null registered_image_ids");
  if (num_tracks > 0x7ffffffeLL) return invalid("more than 2^31 - 2 tracks");
  if (begin[0] != 0) return invalid("begin[0] must be 0");
  for (int64_t t = 0; t < num_tracks; ++t)
    if (begin[t + 1] < begin[t]) return invalid("begin must be non-decreasing");
  const long long n = begin[num_tracks];
  if (n > 0x7ffffffeLL) return invalid("more than 2^31 - 2 observations");
  if (n > 0 && !obs_image) return invalid("null obs_image");
  *num_selected = 0;
  if (num_tracks == 0) return B200SFM_OK;
  // the reference compares these int options with size_t / track_t values: a negative one converts to a huge unsigned
  const long long quota = min_num_tracks_per_view < 0 ? -1 : (long long)min_num_tracks_per_view;
  const unsigned long long min_views = (unsigned long long)(long long)min_num_view_per_track;
  const unsigned long long max_views = (unsigned long long)(long long)max_num_view_per_track;
  const long long cap = max_num_tracks < 0 ? -1 : (long long)max_num_tracks + 1;
  return guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200::TrackSelectRunner r(ctx);
    static_assert(sizeof(unsigned long long) == sizeof(uint64_t) && sizeof(long long) == sizeof(int64_t), "64-bit ids and offsets");
    long long num = 0;
    if (!r.run((int)num_tracks, reinterpret_cast<const unsigned long long*>(track_ids), reinterpret_cast<const long long*>(begin), n,
               obs_image, num_registered, registered_image_ids, quota, min_views, max_views, cap, keep, &num))
      throw b200::InvalidInput{"two tracks share a track id"};
    B200_CUDA_OK(cudaGetLastError());   // a failed launch of this call is reported here, not left pending for the next caller
    *num_selected = num;
    return (int)B200SFM_OK;
  });
}

// ---- GP ----------------------------------------------------------------------
void b200sfm_gp_default_opts(b200sfm_gp_opts* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  // global_positioning.h:22-49, optimization_base.h:18-23
  o->optimize_positions = 1;
  o->optimize_points = 1;
  o->optimize_scales = 1;
  o->min_num_view_per_track = 3;
  o->max_num_iterations = 100;
  o->max_num_line_search_step_size_iterations = 20;
  o->thres_loss_function = 0.1;
  o->function_tolerance = 1e-5;
  o->gradient_tolerance = 1e-10;
  o->parameter_tolerance = 1e-8;
  o->pcg_max_iterations = 1000;
  o->pcg_min_iterations = 0;
  o->pcg_rel_tolerance = 1e-2;
  o->preconditioner = 1;
}

int b200sfm_gp_problem_create(b200sfm_ctx* ctx, int32_t C, int32_t P, int64_t N, const int64_t* pt_obs_begin,
                              const int32_t* obs_cam, const double* obs_dir, const uint8_t* cam_calibrated,
                              const uint8_t* cam_const_mask, int32_t min_num_view_per_track, b200sfm_gp_problem** out) {
  if (!ctx || !out) return B200SFM_ERR_INVALID_ARG;
  *out = nullptr;
  auto precheck = [&]() -> int {
    if (C <= 0 || P <= 0 || N <= 0) { ctx->err = "empty problem (no images / tracks / observations)"; return B200SFM_ERR_EMPTY; }
    if (!pt_obs_begin || !obs_cam || !obs_dir) { ctx->err = "null input array"; return B200SFM_ERR_INVALID_ARG; }
    if (N >= (1ll << 31)) { ctx->err = "N must be < 2^31 per rank"; return B200SFM_ERR_INVALID_ARG; }
    if (pt_obs_begin[0] != 0 || pt_obs_begin[P] != N) { ctx->err = "pt_obs_begin must start at 0 and end at N"; return B200SFM_ERR_INVALID_ARG; }
    return B200SFM_OK;
  };
  int rc = agree_status(ctx, precheck());
  if (rc != B200SFM_OK) return rc;
  b200sfm_gp_problem* p = nullptr;
  rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    p = new b200sfm_gp_problem();
    p->create(ctx, C, P, N, pt_obs_begin, obs_cam, obs_dir, cam_calibrated, cam_const_mask, min_num_view_per_track);
    return (int)B200SFM_OK;
  });
  rc = agree_status(ctx, finish(ctx, rc));
  if (rc != B200SFM_OK) {
    if (p) b200sfm_gp_problem_free(p);
    return rc;
  }
  *out = p;
  return B200SFM_OK;
}

int b200sfm_gp_problem_set_rig_terms(b200sfm_gp_problem* p, const double* obs_offset, const uint8_t* obs_calibrated) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->set_rig_terms(obs_offset, obs_calibrated);
    return (int)B200SFM_OK;
  });
}

int b200sfm_gp_problem_set_rig_unknown(b200sfm_gp_problem* p, int32_t num_unknown_sensors, const int32_t* obs_unknown_sensor,
                                       const double* frame_rot, const double* centers) {
  if (!p || num_unknown_sensors <= 0 || !obs_unknown_sensor || !frame_rot || !centers) return B200SFM_ERR_INVALID_ARG;
  for (long long o = 0; o < p->N; ++o)
    if (obs_unknown_sensor[o] < -1 || obs_unknown_sensor[o] >= num_unknown_sensors) {
      p->ctx->err = "obs_unknown_sensor out of range";
      return B200SFM_ERR_INVALID_ARG;
    }
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->set_rig_unknown(num_unknown_sensors, obs_unknown_sensor, frame_rot, centers);
    return (int)B200SFM_OK;
  });
}

int b200sfm_gp_problem_get_rig_unknown(b200sfm_gp_problem* p, double* centers) {
  if (!p || !centers || p->n_us <= 0) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->get_rig_unknown(centers);
    return (int)B200SFM_OK;
  });
}

int b200sfm_gp_problem_set_state(b200sfm_gp_problem* p, const double* centers, const double* points, const double* scales) {
  if (!p || !centers || !points || !scales) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->set_state(centers, points, scales);
    B200_CUDA_OK(cudaStreamSynchronize(p->ctx->stream));
    return (int)B200SFM_OK;
  });
}

int b200sfm_gp_problem_get_state(b200sfm_gp_problem* p, double* centers, double* points, double* scales) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->get_state(centers, points, scales);
    return (int)B200SFM_OK;
  });
}

int b200sfm_gp_problem_save_state(b200sfm_gp_problem* p) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->save_state();
    B200_CUDA_OK(cudaStreamSynchronize(p->ctx->stream));
    return (int)B200SFM_OK;
  });
}

int b200sfm_gp_problem_restore_state(b200sfm_gp_problem* p) {
  if (!p) return B200SFM_ERR_INVALID_ARG;
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    if (!p->restore_state()) { p->ctx->err = "no saved state"; return (int)B200SFM_ERR_INVALID_ARG; }
    B200_CUDA_OK(cudaStreamSynchronize(p->ctx->stream));
    return (int)B200SFM_OK;
  });
}

int b200sfm_gp_problem_solve(b200sfm_gp_problem* p, const b200sfm_gp_opts* opts, b200sfm_lm_stats* stats) {
  if (!p || !opts) return B200SFM_ERR_INVALID_ARG;
  return finish(p->ctx, guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    if (opts->min_num_view_per_track != p->min_views) {
      p->ctx->err = "min_num_view_per_track differs from the value the problem was created with";
      return (int)B200SFM_ERR_INVALID_ARG;
    }
    if (stats) std::memset(stats, 0, sizeof(*stats));
    return p->solve(*opts, stats);
  }));
}

// ---- GP test probe (include/b200sfm_testing.h) -------------------------------------------------------------------
int b200sfm_test_gp_step(b200sfm_gp_problem* p, const b200sfm_gp_opts* opts, double first_radius, double radius,
                         double alpha, b200sfm_test_gp_step_out* out) {
  if (!p || !opts || !out || !(radius > 0.0) || first_radius < 0.0 || !(alpha > 0.0)) return B200SFM_ERR_INVALID_ARG;
  if (p->ctx->world > 1) { p->ctx->err = "the test probe is single-rank only"; return B200SFM_ERR_INVALID_ARG; }
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    if (opts->min_num_view_per_track != p->min_views) {
      p->ctx->err = "min_num_view_per_track differs from the value the problem was created with";
      return (int)B200SFM_ERR_INVALID_ARG;
    }
    p->test_step(*opts, first_radius, radius, alpha, out);
    return (int)B200SFM_OK;
  });
}

int b200sfm_test_gp_apply(b200sfm_gp_problem* p, const double* x, double* y) {
  if (!p || !x || !y) return B200SFM_ERR_INVALID_ARG;
  if (p->ctx->world > 1) { p->ctx->err = "the test probe is single-rank only"; return B200SFM_ERR_INVALID_ARG; }
  if (!p->probe_ready) { p->ctx->err = "b200sfm_test_gp_apply needs a preceding b200sfm_test_gp_step"; return B200SFM_ERR_INVALID_ARG; }
  return guarded(p->ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(p->ctx->device));
    p->test_apply(x, y);
    return (int)B200SFM_OK;
  });
}

void b200sfm_gp_problem_free(b200sfm_gp_problem* p) {
  if (!p) return;
  cudaSetDevice(p->ctx->device);
  cudaStreamSynchronize(p->ctx->stream);
  b200::AllocScope alloc_scope(pool_stream(p->ctx));   // back to the stream-ordered pool
  delete p;
}

int b200sfm_gp_solve(b200sfm_ctx* ctx, const b200sfm_gp_opts* opts, int32_t C, int32_t P, int64_t N,
                     const int64_t* pt_obs_begin, const int32_t* obs_cam, const double* obs_dir,
                     const uint8_t* cam_calibrated, const uint8_t* cam_const_mask, double* centers, double* points,
                     double* scales, b200sfm_lm_stats* stats) {
  if (!ctx || !opts || !centers || !points || !scales) return B200SFM_ERR_INVALID_ARG;
  b200sfm_gp_problem* p = nullptr;
  b200sfm_lm_stats st{};
  const long long launches0 = ctx->launches;
  int rc = b200sfm_gp_problem_create(ctx, C, P, N, pt_obs_begin, obs_cam, obs_dir, cam_calibrated, cam_const_mask,
                                     opts->min_num_view_per_track, &p);
  if (rc == B200SFM_OK) {
    rc = guarded(ctx, [&]() {
      p->set_state(centers, points, scales);
      int r = p->solve(*opts, &st);
      if (r != B200SFM_OK) return r;
      p->get_state(centers, points, scales);
      st.kernel_launches = ctx->launches - launches0;
      st.h2d_bytes = N * 36 + ((long long)P + 1) * 4 + ((long long)C + P) * 24;
      st.d2h_bytes = N * 8 + ((long long)C + P) * 24;
      return (int)B200SFM_OK;
    });
  }
  if (p) b200sfm_gp_problem_free(p);
  if (stats) *stats = st;
  return rc;
}

// ---- RA ----------------------------------------------------------------------
void b200sfm_ra_default_opts(b200sfm_ra_opts* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  // global_rotation_averaging.h:41-71
  o->max_num_l1_iterations = 5;
  o->max_num_irls_iterations = 100;
  o->weight_type = 0;
  o->use_weight = 0;
  o->l1_step_convergence_threshold = 1e-3;
  o->irls_step_convergence_threshold = 1e-3;
  o->irls_loss_parameter_sigma = 5.0;
  o->l1_max_admm_iterations = 10;   // .cc:484
  o->l1_rho = 1.0;
  o->l1_absolute_tolerance = 1e-4;
  o->l1_relative_tolerance = 1e-2;
  o->pcg_max_iterations = 5000;
  o->pcg_rel_tolerance = 1e-8;
}

int b200sfm_ra_solve(b200sfm_ctx* ctx, const b200sfm_ra_opts* opts, int32_t n_frames, int64_t n_edges,
                     const int32_t* ei, const int32_t* ej, const double* R_rel, const double* edge_w,
                     int32_t fixed_frame, double* theta, b200sfm_ra_stats* stats) {
  return b200sfm_ra_solve_gravity(ctx, opts, n_frames, n_edges, ei, ej, R_rel, edge_w, nullptr, fixed_frame, theta, stats);
}

int b200sfm_ra_solve_gravity(b200sfm_ctx* ctx, const b200sfm_ra_opts* opts, int32_t n_frames, int64_t n_edges,
                             const int32_t* ei, const int32_t* ej, const double* R_rel, const double* edge_w,
                             const uint8_t* frame_has_gravity, int32_t fixed_frame, double* theta,
                             b200sfm_ra_stats* stats) {
  if (!ctx || !opts || !theta) return B200SFM_ERR_INVALID_ARG;
  if (n_frames <= 0) { ctx->err = "no frames"; return B200SFM_ERR_EMPTY; }
  if (n_edges < 0 || (n_edges > 0 && (!ei || !ej || !R_rel))) { ctx->err = "null edge array"; return B200SFM_ERR_INVALID_ARG; }
  if (fixed_frame < 0 || fixed_frame >= n_frames) { ctx->err = "fixed_frame out of range"; return B200SFM_ERR_INVALID_ARG; }
  for (int64_t e = 0; e < n_edges; ++e)
    if (ei[e] < 0 || ei[e] >= n_frames || ej[e] < 0 || ej[e] >= n_frames) { ctx->err = "edge index out of range"; return B200SFM_ERR_INVALID_ARG; }
  b200sfm_ra_stats st{};
  int rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200sfm_ra_problem p;
    p.create(ctx, n_frames, n_edges, ei, ej, R_rel, edge_w, opts->use_weight, fixed_frame, theta, frame_has_gravity);
    int r = p.solve(*opts, &st);
    if (r != B200SFM_OK) return r;
    p.theta.download(theta, (size_t)n_frames * 3, ctx->stream);
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return (int)B200SFM_OK;
  });
  if (stats) *stats = st;
  return finish(ctx, rc);
}

int b200sfm_ra_solve_rig(b200sfm_ctx* ctx, const b200sfm_ra_opts* opts, int32_t n_frames, int32_t n_cams, int64_t n_edges,
                         const int32_t* ei, const int32_t* ej, const int32_t* eci, const int32_t* ecj, const double* R_rel,
                         const double* edge_w, const int32_t* cam_frames_begin, const int32_t* cam_frames,
                         int32_t fixed_frame, double* theta, b200sfm_ra_stats* stats) {
  if (!ctx || !opts || !theta) return B200SFM_ERR_INVALID_ARG;
  if (n_frames <= 0) { ctx->err = "no frames"; return B200SFM_ERR_EMPTY; }
  if (n_cams <= 0 || !eci || !ecj || !cam_frames_begin || !cam_frames) { ctx->err = "no unknown cameras (use b200sfm_ra_solve)"; return B200SFM_ERR_INVALID_ARG; }
  if (n_edges < 0 || (n_edges > 0 && (!ei || !ej || !R_rel))) { ctx->err = "null edge array"; return B200SFM_ERR_INVALID_ARG; }
  if (fixed_frame < 0 || fixed_frame >= n_frames) { ctx->err = "fixed_frame out of range"; return B200SFM_ERR_INVALID_ARG; }
  const int n = n_frames + n_cams;
  for (int64_t e = 0; e < n_edges; ++e) {
    if (ei[e] < 0 || ei[e] >= n_frames || ej[e] < 0 || ej[e] >= n_frames) { ctx->err = "edge index out of range"; return B200SFM_ERR_INVALID_ARG; }
    if ((eci[e] != -1 && (eci[e] < n_frames || eci[e] >= n)) || (ecj[e] != -1 && (ecj[e] < n_frames || ecj[e] >= n))) {
      ctx->err = "camera node out of range (must be -1 or in [n_frames, n_frames + n_cams))";
      return B200SFM_ERR_INVALID_ARG;
    }
  }
  if (cam_frames_begin[0] != 0) { ctx->err = "cam_frames_begin must start at 0"; return B200SFM_ERR_INVALID_ARG; }
  for (int c = 0; c < n_cams; ++c)
    if (cam_frames_begin[c + 1] < cam_frames_begin[c]) { ctx->err = "cam_frames_begin must be non-decreasing"; return B200SFM_ERR_INVALID_ARG; }
  for (int k = 0; k < cam_frames_begin[n_cams]; ++k)
    if (cam_frames[k] < 0 || cam_frames[k] >= n_frames) { ctx->err = "cam_frames out of range"; return B200SFM_ERR_INVALID_ARG; }
  if (ctx->world > 1) { ctx->err = "unknown cam_from_rig rotations: single-process contexts only"; return B200SFM_ERR_UNSUPPORTED; }
  b200sfm_ra_stats st{};
  int rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200sfm_ra_problem p;
    p.create(ctx, n, n_edges, ei, ej, R_rel, edge_w, opts->use_weight, fixed_frame, theta, nullptr, n_cams, eci, ecj,
             cam_frames_begin, cam_frames);
    int r = p.solve(*opts, &st);
    if (r != B200SFM_OK) return r;
    p.theta.download(theta, (size_t)n * 3, ctx->stream);
    B200_CUDA_OK(cudaStreamSynchronize(ctx->stream));
    return (int)B200SFM_OK;
  });
  if (stats) *stats = st;
  return finish(ctx, rc);
}

// ---- RA test probe (include/b200sfm_testing.h) -------------------------------------------------------------------
struct b200sfm_test_ra_problem {
  b200sfm_ra_problem p;
  int square = -1;   // the system b200sfm_test_ra_system prepared last (-1: none yet)
};

int b200sfm_test_ra_problem_create(b200sfm_ctx* ctx, const b200sfm_ra_opts* opts, int32_t n_frames, int32_t n_cams,
                                   int64_t n_edges, const int32_t* ei, const int32_t* ej, const int32_t* eci,
                                   const int32_t* ecj, const double* R_rel, const double* edge_w,
                                   const uint8_t* frame_has_gravity, const int32_t* cam_frames_begin,
                                   const int32_t* cam_frames, int32_t fixed_frame, const double* theta,
                                   b200sfm_test_ra_problem** out) {
  if (!ctx || !opts || !theta || !out) return B200SFM_ERR_INVALID_ARG;
  *out = nullptr;
  if (ctx->world > 1) { ctx->err = "the test probe is single-rank only"; return B200SFM_ERR_INVALID_ARG; }
  if (n_frames <= 0 || n_cams < 0) { ctx->err = "no frames"; return B200SFM_ERR_INVALID_ARG; }
  if (n_cams > 0 && (!eci || !ecj || !cam_frames_begin || !cam_frames)) { ctx->err = "null camera array"; return B200SFM_ERR_INVALID_ARG; }
  if (n_edges < 0 || (n_edges > 0 && (!ei || !ej || !R_rel))) { ctx->err = "null edge array"; return B200SFM_ERR_INVALID_ARG; }
  if (fixed_frame < 0 || fixed_frame >= n_frames) { ctx->err = "fixed_frame out of range"; return B200SFM_ERR_INVALID_ARG; }
  const int n = n_frames + n_cams;
  for (int64_t e = 0; e < n_edges; ++e) {
    if (ei[e] < 0 || ei[e] >= n_frames || ej[e] < 0 || ej[e] >= n_frames) { ctx->err = "edge index out of range"; return B200SFM_ERR_INVALID_ARG; }
    if (n_cams > 0 && ((eci[e] != -1 && (eci[e] < n_frames || eci[e] >= n)) || (ecj[e] != -1 && (ecj[e] < n_frames || ecj[e] >= n)))) {
      ctx->err = "camera node out of range (must be -1 or in [n_frames, n_frames + n_cams))";
      return B200SFM_ERR_INVALID_ARG;
    }
  }
  if (n_cams > 0) {
    if (cam_frames_begin[0] != 0) { ctx->err = "cam_frames_begin must start at 0"; return B200SFM_ERR_INVALID_ARG; }
    for (int c = 0; c < n_cams; ++c)
      if (cam_frames_begin[c + 1] < cam_frames_begin[c]) { ctx->err = "cam_frames_begin must be non-decreasing"; return B200SFM_ERR_INVALID_ARG; }
    for (int k = 0; k < cam_frames_begin[n_cams]; ++k)
      if (cam_frames[k] < 0 || cam_frames[k] >= n_frames) { ctx->err = "cam_frames out of range"; return B200SFM_ERR_INVALID_ARG; }
  }
  return guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    auto* h = new b200sfm_test_ra_problem;
    try {
      h->p.create(ctx, n, n_edges, ei, ej, R_rel, edge_w, opts->use_weight, fixed_frame, theta, frame_has_gravity, n_cams,
                  eci, ecj, cam_frames_begin, cam_frames);
    } catch (...) {
      delete h;
      throw;
    }
    *out = h;
    return (int)B200SFM_OK;
  });
}

void b200sfm_test_ra_problem_free(b200sfm_test_ra_problem* h) {
  if (!h) return;
  cudaSetDevice(h->p.ctx->device);
  cudaStreamSynchronize(h->p.ctx->stream);
  b200::AllocScope alloc_scope(pool_stream(h->p.ctx));   // back to the stream-ordered pool
  delete h;
}

int b200sfm_test_ra_problem_info(b200sfm_test_ra_problem* h, b200sfm_test_ra_info* info, int32_t* agg_of) {
  if (!h || !info) return B200SFM_ERR_INVALID_ARG;
  return guarded(h->p.ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(h->p.ctx->device));
    h->p.test_info(info, agg_of);
    return (int)B200SFM_OK;
  });
}

int b200sfm_test_ra_system(b200sfm_test_ra_problem* h, int32_t mode, double sigma2, int32_t square,
                           b200sfm_test_ra_system_out* out) {
  if (!h || !out || mode < 0 || mode > 2 || (square != 0 && square != 1) || (mode == 1 && !(sigma2 > 0.0)))
    return B200SFM_ERR_INVALID_ARG;
  return guarded(h->p.ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(h->p.ctx->device));
    h->p.test_system(mode, sigma2, square, out);
    h->square = square;
    return (int)B200SFM_OK;
  });
}

static int ra_probe_ready(b200sfm_test_ra_problem* h) {
  if (h->square >= 0) return B200SFM_OK;
  h->p.ctx->err = "the RA probe needs a preceding b200sfm_test_ra_system";
  return B200SFM_ERR_INVALID_ARG;
}

int b200sfm_test_ra_apply(b200sfm_test_ra_problem* h, const double* x, double* y) {
  if (!h || !x || !y) return B200SFM_ERR_INVALID_ARG;
  if (ra_probe_ready(h) != B200SFM_OK) return B200SFM_ERR_INVALID_ARG;
  return guarded(h->p.ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(h->p.ctx->device));
    h->p.test_apply(h->square, x, y);
    return (int)B200SFM_OK;
  });
}

int b200sfm_test_ra_precond(b200sfm_test_ra_problem* h, const double* r, double* z) {
  if (!h || !r || !z) return B200SFM_ERR_INVALID_ARG;
  if (ra_probe_ready(h) != B200SFM_OK) return B200SFM_ERR_INVALID_ARG;
  return guarded(h->p.ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(h->p.ctx->device));
    h->p.test_precond(r, z);
    return (int)B200SFM_OK;
  });
}

int b200sfm_test_ra_pcg(b200sfm_test_ra_problem* h, int32_t k, const double* warm_x, double* x_out, int32_t* iterations) {
  if (!h || !x_out || k < 1) return B200SFM_ERR_INVALID_ARG;
  if (ra_probe_ready(h) != B200SFM_OK) return B200SFM_ERR_INVALID_ARG;
  return guarded(h->p.ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(h->p.ctx->device));
    const int it = h->p.test_pcg(h->square, k, warm_x, x_out);
    if (iterations) *iterations = it;
    return (int)B200SFM_OK;
  });
}

int b200sfm_test_ra_admm_step(b200sfm_test_ra_problem* h, double rho, const double* x, const double* b, double* z,
                              double* u, double* rsu, double* norms) {
  if (!h || !x || !b || !z || !u || !rsu || !norms || !(rho > 0.0)) return B200SFM_ERR_INVALID_ARG;
  if (ra_probe_ready(h) != B200SFM_OK) return B200SFM_ERR_INVALID_ARG;
  return guarded(h->p.ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(h->p.ctx->device));
    h->p.test_admm_step(rho, x, b, z, u, rsu, norms);
    return (int)B200SFM_OK;
  });
}

int b200sfm_test_ra_update(b200sfm_test_ra_problem* h, const double* step, double* theta_out, double* sums) {
  if (!h || !step || !theta_out || !sums) return B200SFM_ERR_INVALID_ARG;
  return guarded(h->p.ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(h->p.ctx->device));
    h->p.test_update(step, theta_out, sums);
    return (int)B200SFM_OK;
  });
}

int b200sfm_ra_mst_init(b200sfm_ctx* ctx, int32_t n_nodes, int64_t n_edges, const int32_t* ei, const int32_t* ej,
                        const double* R_rel, const double* weight, int32_t root, double* R, int32_t* parent,
                        b200sfm_mst_stats* stats) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!ctx || !R || n_nodes < 1 || n_edges < 0) return B200SFM_ERR_INVALID_ARG;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if (n_edges > 0 && (!ei || !ej || !R_rel || !weight)) return invalid("null edge array");
  if (n_edges > INT32_MAX) return invalid("more than 2^31 - 1 edges");
  if (root < 0 || root >= n_nodes) return invalid("root out of range");
  double wmax = -INFINITY;
  for (int64_t e = 0; e < n_edges; ++e) {
    if (ei[e] < 0 || ei[e] >= n_nodes || ej[e] < 0 || ej[e] >= n_nodes) return invalid("edge index out of range");
    if (!std::isfinite(weight[e])) return invalid("non-finite edge weight");
    wmax = std::max(wmax, weight[e]);
  }
  if (ctx->world > 1) {
    ctx->err = "the spanning tree needs every edge: single-rank contexts only";
    return B200SFM_ERR_UNSUPPORTED;
  }
  const long long launches0 = ctx->launches;
  b200::MstStats st;
  int rc = B200SFM_OK;
  if (n_edges == 0) {   // the root alone
    if (parent) {
      std::fill(parent, parent + n_nodes, -1);
      parent[root] = root;
    }
    st.num_reached = 1;
  } else {
    rc = guarded(ctx, [&]() {
      B200_CUDA_OK(cudaSetDevice(ctx->device));
      b200::MstRunner r(ctx);
      r.run(n_nodes, (int)n_edges, ei, ej, R_rel, weight, wmax, root, R, parent, st);
      B200_CUDA_OK(cudaGetLastError());   // a failed launch of this call is reported here, not left pending for the next caller
      return (int)B200SFM_OK;
    });
  }
  if (stats) {
    *stats = b200sfm_mst_stats{};
    stats->num_reached = st.num_reached;
    stats->num_tree_edges = st.num_tree_edges;
    stats->boruvka_rounds = st.boruvka_rounds;
    stats->max_depth = st.max_depth;
    stats->kernel_launches = ctx->launches - launches0;
    stats->ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  }
  return rc;
}

int b200sfm_rig_rotations_from_images(b200sfm_ctx* ctx, int64_t n_images, int32_t n_frames, int32_t n_cameras,
                                      const int32_t* image_frame, const int32_t* image_camera,
                                      const uint8_t* image_estimated, const double* cam_from_world,
                                      const int32_t* frame_ref_camera, const uint8_t* camera_known, double* cam_from_rig,
                                      int32_t* cam_samples, double* rig_from_world, int32_t* frame_samples,
                                      b200sfm_rig_init_stats* stats) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!ctx) return B200SFM_ERR_INVALID_ARG;
  auto invalid = [&](const char* msg) { ctx->err = msg; return (int)B200SFM_ERR_INVALID_ARG; };
  if (!image_frame || !image_camera || !cam_from_world || !frame_ref_camera || !camera_known || !cam_from_rig || !rig_from_world)
    return invalid("null array");
  if (n_images < 1 || n_images > INT32_MAX) return invalid("n_images must be in [1, 2^31 - 1]");
  if (n_frames < 1 || n_cameras < 1) return invalid("n_frames and n_cameras must be at least 1");
  for (int64_t i = 0; i < n_images; ++i) {
    if (image_frame[i] < -1 || image_frame[i] >= n_frames) return invalid("image frame index out of range");
    if (image_camera[i] < 0 || image_camera[i] >= n_cameras) return invalid("image camera index out of range");
  }
  for (int32_t f = 0; f < n_frames; ++f)
    if (frame_ref_camera[f] < 0 || frame_ref_camera[f] >= n_cameras) return invalid("frame reference camera out of range");
  if (ctx->world > 1) {
    ctx->err = "the frames' samples span every image: single-rank contexts only";
    return B200SFM_ERR_UNSUPPORTED;
  }
  const long long launches0 = ctx->launches;
  b200::RigInitStats st;
  const int rc = guarded(ctx, [&]() {
    B200_CUDA_OK(cudaSetDevice(ctx->device));
    b200::RigInitRunner r(ctx);
    r.run((int)n_images, n_frames, n_cameras, image_frame, image_camera, image_estimated, cam_from_world, frame_ref_camera,
          camera_known, cam_from_rig, cam_samples, rig_from_world, frame_samples, st);
    B200_CUDA_OK(cudaGetLastError());   // a failed launch of this call is reported here, not left pending for the next caller
    return (int)B200SFM_OK;
  });
  if (stats) {
    *stats = b200sfm_rig_init_stats{};
    stats->num_ref_frames = st.num_ref_frames;
    stats->num_cam_samples = st.num_cam_samples;
    stats->num_cams_averaged = st.num_cams_averaged;
    stats->num_frame_samples = st.num_frame_samples;
    stats->num_frames_averaged = st.num_frames_averaged;
    stats->kernel_launches = ctx->launches - launches0;
    stats->ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  }
  return rc;
}

}  // extern "C"
