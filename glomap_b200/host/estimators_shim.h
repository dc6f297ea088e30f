// estimators_shim.h -- C++ drop-in for glomap's three estimator classes over
// the C ABI (include/b200sfm.h).  Same class names, constructor / method
// signatures, option fields and bool-return error behaviour as
//   glomap::RotationEstimator   glomap/estimators/global_rotation_averaging.h:39-87
//   glomap::GlobalPositioner    glomap/estimators/global_positioning.h:9-70
//   glomap::BundleAdjuster      glomap/estimators/bundle_adjustment.h:12-51
// Each Solve flattens the unordered_map world into SoA in SORTED-ID order
// (deterministic, unlike the reference's hash-map order), calls the GPU solver
// and scatters the results back in place.  Known (constant) camera rigs are
// supported in BundleAdjuster and GlobalPositioner (frames = pose blocks, every
// image carries its sensor's cam_from_rig); optimize_rig_poses (BA) marks the non-reference sensors as unknowns
// and writes the optimised cam_from_rig back.  Rigs with a not-yet-calibrated sensor: RA and GP estimate the unknown
// cam_from_rig blocks, and SolveRotationAveraging starts them with the trivial-rig pre-pass.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <array>
#include <map>
#include <limits>
#include <queue>
#include <set>
#include <random>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "../../include/b200sfm.h"
#include "scene_min.h"

namespace b200sfm_shim {
using namespace b200host;

// One context per CUDA device, created on first use.  `gpu_index` is the reference's option string
// (bundle_adjustment.h:24, global_positioning.h:42: "-1" = the default device, otherwise the first index of a
// comma-separated list -- the reference hands the list to Ceres/cuDSS, which uses one device as well).
inline b200sfm_ctx* DefaultContext(const std::string& gpu_index = "-1") {
  static std::map<int, b200sfm_ctx*> ctxs;
  int device = 0;
  try {
    device = std::stoi(gpu_index);
  } catch (...) {
    device = -1;
  }
  if (device < 0) device = 0;
  auto it = ctxs.find(device);
  if (it != ctxs.end()) return it->second;
  b200sfm_ctx* ctx = nullptr;
  if (b200sfm_create(device, &ctx) != B200SFM_OK) {
    std::fprintf(stderr, "b200sfm: no CUDA device %d / context creation failed (there is no CPU fallback)\n", device);
    return nullptr;   // not cached: a later call may name a valid device
  }
  ctxs[device] = ctx;
  return ctx;
}

// How every entry point turns the scene into flat arrays: the sorted-id order, the camera blocks, an image's
// cam_from_rig and the rotation algebra.  Which entities become blocks, how they are numbered and what an entry point
// does with a missing entity stay with each entry point.
namespace detail {

// The entries of an id-keyed map as (id, pointer) in ascending id, only those `keep` accepts.
template <class Map, class Keep>
auto SortedEntries(Map& m, Keep keep) {
  std::vector<std::pair<typename Map::key_type, decltype(&m.begin()->second)>> out;
  for (auto& [id, v] : m)
    if (keep(v)) out.emplace_back(id, &v);
  std::sort(out.begin(), out.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  return out;
}
template <class Map>
auto SortedEntries(Map& m) {
  return SortedEntries(m, [](const auto&) { return true; });
}
// id -> position in a vector of SortedEntries
template <class Id, class T>
std::unordered_map<Id, int32_t> PositionOf(const std::vector<std::pair<Id, T>>& sorted) {
  std::unordered_map<Id, int32_t> pos;
  for (size_t i = 0; i < sorted.size(); ++i) pos.emplace(sorted[i].first, (int32_t)i);
  return pos;
}

// Camera blocks: model_id and params zero-padded to B200SFM_INTR_STRIDE (params beyond the stride are not passed),
// one block per camera of `cams` ((id, Camera*) pairs) in their order.
template <class CameraPtrs>
void PackCameras(const CameraPtrs& cams, std::vector<int32_t>& model, std::vector<double>& intr) {
  model.clear();
  intr.assign(cams.size() * B200SFM_INTR_STRIDE, 0.0);
  for (size_t k = 0; k < cams.size(); ++k) {
    const auto& c = *cams[k].second;
    model.push_back(static_cast<int32_t>(c.model_id));   // colmap::CameraModelId is an enum class
    for (size_t j = 0; j < c.params.size() && j < (size_t)B200SFM_INTR_STRIDE; ++j) intr[k * B200SFM_INTR_STRIDE + j] = c.params[j];
  }
}
// the inverse of PackCameras: the blocks' params back into the cameras
template <class CameraPtrs>
void UnpackCameras(const std::vector<double>& intr, const CameraPtrs& cams) {
  for (size_t k = 0; k < cams.size(); ++k) {
    auto& c = *cams[k].second;
    for (size_t j = 0; j < c.params.size() && j < (size_t)B200SFM_INTR_STRIDE; ++j) c.params[j] = intr[k * B200SFM_INTR_STRIDE + j];
  }
}
// one SIMPLE_PINHOLE block with f = 1, for a device problem whose intrinsics are never read, so that a camera model the
// call does not read cannot refuse it
inline void PlaceholderCamera(std::vector<int32_t>& model, std::vector<double>& intr) {
  model.assign(1, B200SFM_SIMPLE_PINHOLE);
  intr.assign(B200SFM_INTR_STRIDE, 0.0);
  intr[0] = 1.0;
}

// An image's cam_from_rig through the rig the caller holds (null: none): the identity for a trivial frame or the rig's
// reference sensor, the rig's stored pose when it has one, otherwise missing (`pose` is then the identity).
enum class CamFromRigStatus { kIdentity, kKnown, kMissing };
template <class RigT, class ImageT>
CamFromRigStatus ResolveCamFromRig(RigT* rig, const ImageT& im, Rigid3d& pose) {
  pose = Rigid3d();
  if (im.HasTrivialFrame() || (rig && b200host_adapt::IsRefSensor(*rig, im.camera_id))) return CamFromRigStatus::kIdentity;
  if (!rig || !b200host_adapt::HasCamFromRig(*rig, im.camera_id)) return CamFromRigStatus::kMissing;
  pose = b200host_adapt::CamFromRig(*rig, im.camera_id);
  return CamFromRigStatus::kKnown;
}

// Rotation algebra: quaternions xyzw (Eigen's coeffs() order), matrices row-major.
inline void QuatMul(const double* a, const double* b, double* o) {   // o = a (x) b
  const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  const double y = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
  const double z = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
  const double w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  o[0] = x; o[1] = y; o[2] = z; o[3] = w;
}
inline void QuatConj(const double* a, double* o) { o[0] = -a[0]; o[1] = -a[1]; o[2] = -a[2]; o[3] = a[3]; }
inline void QuatToR(const double* q, double R[9]) {
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double x = q[0] / n, y = q[1] / n, z = q[2] / n, w = q[3] / n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
}
// rotation matrix -> unit quaternion, w >= 0 (Shepperd's branches, as Eigen's conversion)
inline void RToQuat(const double* R, double* q) {
  const double tr = R[0] + R[4] + R[8];
  if (tr > 0) {
    const double s = std::sqrt(tr + 1.0) * 2;
    q[3] = 0.25 * s; q[0] = (R[7] - R[5]) / s; q[1] = (R[2] - R[6]) / s; q[2] = (R[3] - R[1]) / s;
  } else if (R[0] > R[4] && R[0] > R[8]) {
    const double s = std::sqrt(1.0 + R[0] - R[4] - R[8]) * 2;
    q[3] = (R[7] - R[5]) / s; q[0] = 0.25 * s; q[1] = (R[1] + R[3]) / s; q[2] = (R[2] + R[6]) / s;
  } else if (R[4] > R[8]) {
    const double s = std::sqrt(1.0 + R[4] - R[0] - R[8]) * 2;
    q[3] = (R[2] - R[6]) / s; q[0] = (R[1] + R[3]) / s; q[1] = 0.25 * s; q[2] = (R[5] + R[7]) / s;
  } else {
    const double s = std::sqrt(1.0 + R[8] - R[0] - R[4]) * 2;
    q[3] = (R[3] - R[1]) / s; q[0] = (R[2] + R[6]) / s; q[1] = (R[5] + R[7]) / s; q[2] = 0.25 * s;
  }
  if (q[3] < 0) for (int k = 0; k < 4; ++k) q[k] = -q[k];
}
inline void QuatToAngleAxis(const double* q, double* v) {
  double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  if (n > 0) {
    const double ang = 2 * std::atan2(n, std::fabs(q[3]));
    const double f = (q[3] < 0 ? -ang : ang) / n;
    v[0] = q[0] * f; v[1] = q[1] * f; v[2] = q[2] * f;
  } else {
    v[0] = v[1] = v[2] = 0;
  }
}
inline void AngleAxisToQuat(const double* v, double* q) {
  const double n = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (n > 0) {
    const double s = std::sin(n / 2) / n;
    q[0] = v[0] * s; q[1] = v[1] * s; q[2] = v[2] * s; q[3] = std::cos(n / 2);
  } else {
    q[0] = q[1] = q[2] = 0; q[3] = 1;
  }
}
// C = A B and C = A^T B for a 3x3 A and a 3xN B (N = 1: a vector); every element is summed left to right,
// a[r][0] b[0][c] + a[r][1] b[1][c] + a[r][2] b[2][c].  C may be A or B.
template <int N = 3>
inline void MulAB(const double* A, const double* B, double* C) {
  double T[3 * N];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < N; ++c) T[N * r + c] = A[3 * r] * B[c] + A[3 * r + 1] * B[N + c] + A[3 * r + 2] * B[2 * N + c];
  std::copy(T, T + 3 * N, C);
}
template <int N = 3>
inline void MulAtB(const double* A, const double* B, double* C) {
  double T[3 * N];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < N; ++c) T[N * r + c] = A[r] * B[c] + A[3 + r] * B[N + c] + A[6 + r] * B[2 * N + c];
  std::copy(T, T + 3 * N, C);
}

}  // namespace detail

// colmap::AverageQuaternions with unit weights: dominant eigenvector of sum q q^T (sign-invariant), by power iteration
inline void AverageQuaternions(const std::vector<std::array<double, 4>>& qs, double* out) {
  double M[4][4] = {};
  for (const auto& q : qs)
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) M[r][c] += q[r] * q[c];
  double v[4] = {qs[0][0], qs[0][1], qs[0][2], qs[0][3]};
  for (int it = 0; it < 200; ++it) {
    double u[4] = {0, 0, 0, 0};
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) u[r] += M[r][c] * v[c];
    const double n = std::sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2] + u[3] * u[3]);
    if (!(n > 0)) break;
    for (int k = 0; k < 4; ++k) v[k] = u[k] / n;
  }
  for (int k = 0; k < 4; ++k) out[k] = v[k];
}

// ---------------------------------------------------------------------------
struct OptimizationBaseOptions {                 // optimization_base.h:10-24
  double thres_loss_function = 1e-1;
  struct SolverOptions {
    int max_num_iterations = 100;
    double function_tolerance = 1e-5;
    double gradient_tolerance = 1e-10;
    double parameter_tolerance = 1e-8;
  } solver_options;
};

struct BundleAdjusterOptions : public OptimizationBaseOptions {   // bundle_adjustment.h:12-37
  bool optimize_rig_poses = false;
  bool optimize_rotations = true;
  bool optimize_translation = true;
  bool optimize_intrinsics = true;
  bool optimize_principal_point = false;
  bool optimize_points = true;
  bool use_gpu = true;
  std::string gpu_index = "-1";
  int min_num_images_gpu_solver = 50;
  int min_num_view_per_track = 3;
  // PCG knobs of this implementation
  double pcg_rel_tolerance = 1e-2;
  int pcg_max_iterations = 500;
  BundleAdjusterOptions() {
    thres_loss_function = 1.;
    solver_options.max_num_iterations = 200;
  }
};

class BundleAdjuster {
 public:
  BundleAdjuster(const BundleAdjusterOptions& options) : options_(options) {}
  BundleAdjusterOptions& GetOptions() { return options_; }
  b200sfm_lm_stats summary{};

  // bundle_adjustment.cc:11-106
  bool Solve(std::unordered_map<rig_t, Rig>& rigs, std::unordered_map<camera_t, Camera>& cameras,
             std::unordered_map<frame_t, Frame>& frames, std::unordered_map<image_t, Image>& images,
             std::unordered_map<track_t, Track>& tracks) {
    if (images.empty()) { std::fprintf(stderr, "Number of images = 0\n"); return false; }     // .cc:17-20
    if (tracks.empty()) { std::fprintf(stderr, "Number of tracks = 0\n"); return false; }     // .cc:21-24
    b200sfm_ctx* ctx = DefaultContext(options_.gpu_index);
    if (!ctx) return false;
    // every frame and every camera is a block, in sorted-id order; the gauge frame is chosen below, once it is known
    // which frames carry observations (.cc:252-266)
    const auto fsorted = detail::SortedEntries(frames);
    auto fidx = detail::PositionOf(fsorted);
    const auto csorted = detail::SortedEntries(cameras);
    auto cidx = detail::PositionOf(csorted);
    const int C = (int)fsorted.size(), K = (int)csorted.size();
    std::vector<double> quat(4 * (size_t)C), trans(3 * (size_t)C), intr;
    std::vector<int32_t> cam_intr(C, 0), intr_model;
    std::vector<uint8_t> mask(C, 0);
    for (int i = 0; i < C; ++i) {
      const Rigid3d& pose = fsorted[i].second->RigFromWorld();
      for (int k = 0; k < 4; ++k) quat[4 * i + k] = pose.rotation.coeffs().data()[k];
      for (int k = 0; k < 3; ++k) trans[3 * i + k] = pose.translation[k];
    }
    detail::PackCameras(csorted, intr_model, intr);
    // sensors = the (rig, camera) pairs of all images in sorted order, each resolved from the first of its images met
    bool any_rig = false;
    for (auto& [id, im] : images) any_rig = any_rig || !im.HasTrivialFrame();
    struct ImageBlocks { const Image* im; int32_t frame, sensor; };
    std::unordered_map<image_t, ImageBlocks> blocks_of;
    std::map<std::pair<rig_t, camera_t>, std::pair<int32_t, Rigid3d>> sensors;   // (index, cam_from_rig)
    std::vector<double> sensor_q, sensor_t;
    std::vector<int32_t> sensor_intr;
    std::vector<uint8_t> sensor_var;   // optimize_rig_poses: every non-reference sensor is an unknown (.cc:162-180,296-308)
    if (any_rig) {
      for (auto& [id, im] : images) {
        const auto key = std::make_pair(frames[im.frame_id].RigId(), im.camera_id);
        auto s = sensors.find(key);
        if (s != sensors.end()) continue;
        s = sensors.emplace(key, std::make_pair(0, Rigid3d())).first;
        detail::ResolveCamFromRig(im.HasTrivialFrame() ? nullptr : &rigs[key.first], im, s->second.second);   // missing: identity
      }
      int32_t n = 0;
      for (auto& [key, s] : sensors) {
        s.first = n++;
        for (int k = 0; k < 4; ++k) sensor_q.push_back(s.second.rotation.coeffs().data()[k]);
        for (int k = 0; k < 3; ++k) sensor_t.push_back(s.second.translation[k]);
        sensor_intr.push_back(cidx[key.second]);
        // NonRefSensors() of the rig (.cc:299); Image::HasTrivialFrame() is exactly IsRefSensor (scene/image.h:73-76)
        sensor_var.push_back((options_.optimize_rig_poses && !b200host_adapt::IsRefSensor(rigs[key.first], key.second)) ? 1 : 0);
      }
      if (n > 65535) { std::fprintf(stderr, "b200sfm: too many rig sensors\n"); return false; }
      for (auto& [id, im] : images)
        blocks_of[id] = {&im, fidx[im.frame_id], sensors[{frames[im.frame_id].RigId(), im.camera_id}].first};
    } else {
      for (auto& [id, im] : images) {
        blocks_of[id] = {&im, fidx[im.frame_id], 0};
        cam_intr[fidx[im.frame_id]] = cidx[im.camera_id];
      }
    }
    const auto tsorted = detail::SortedEntries(tracks);
    const int P = (int)tsorted.size();
    std::vector<int64_t> ptb(1, 0);
    std::vector<int32_t> obs_cam;
    std::vector<uint16_t> obs_sensor;
    std::vector<double> obs_xy, points(3 * (size_t)P);
    for (int p = 0; p < P; ++p) {
      const Track& t = *tsorted[p].second;
      // .cc:122: the track is skipped on ITS observation count; observations of missing images are dropped afterwards
      // (.cc:125), so the device gets min_num_view_per_track = 1 and a skipped track simply carries no observation
      const bool keep = (int)t.observations.size() >= options_.min_num_view_per_track;
      for (const auto& ob : t.observations) {
        if (!keep) break;
        auto it = blocks_of.find(ob.first);
        if (it == blocks_of.end()) continue;                                                  // .cc:125
        obs_cam.push_back(it->second.frame);
        if (any_rig) obs_sensor.push_back((uint16_t)it->second.sensor);
        obs_xy.push_back(it->second.im->features[ob.second][0]);
        obs_xy.push_back(it->second.im->features[ob.second][1]);
      }
      ptb.push_back((int64_t)obs_cam.size());
      for (int k = 0; k < 3; ++k) points[3 * (size_t)p + k] = t.xyz[k];
    }
    {   // .cc:252-266: the first frame (map order; here sorted-id order) that HAS a parameter block is held constant
      std::vector<uint8_t> used(C, 0);
      for (int32_t f : obs_cam) used[f] = 1;
      for (int i = 0; i < C; ++i)
        if (used[i]) { mask[i] = 3; break; }
    }
    b200sfm_ba_opts o;
    b200sfm_ba_default_opts(&o);
    o.optimize_rig_poses = options_.optimize_rig_poses; o.optimize_rotations = options_.optimize_rotations;
    o.optimize_translation = options_.optimize_translation; o.optimize_intrinsics = options_.optimize_intrinsics;
    o.optimize_principal_point = options_.optimize_principal_point; o.optimize_points = options_.optimize_points;
    o.min_num_view_per_track = 1;   // the track-length rule was applied above, on track.observations.size()
    o.max_num_iterations = options_.solver_options.max_num_iterations;
    o.thres_loss_function = options_.thres_loss_function;
    o.function_tolerance = options_.solver_options.function_tolerance;
    o.gradient_tolerance = options_.solver_options.gradient_tolerance;
    o.parameter_tolerance = options_.solver_options.parameter_tolerance;
    o.pcg_rel_tolerance = options_.pcg_rel_tolerance; o.pcg_max_iterations = options_.pcg_max_iterations;
    int rc;
    if (any_rig) {   // known rigs: resident-problem path (bundle_adjustment.cc:147-161)
      b200sfm_ba_problem* prob = nullptr;
      rc = b200sfm_ba_problem_create_rig(ctx, C, P, (int64_t)obs_cam.size(), K, (int32_t)sensor_intr.size(), ptb.data(),
                                         obs_cam.data(), obs_sensor.data(), obs_xy.data(), sensor_q.data(), sensor_t.data(),
                                         sensor_intr.data(), intr_model.data(), mask.data(), o.min_num_view_per_track, &prob);
      if (rc == B200SFM_OK) rc = b200sfm_ba_problem_set_state(prob, intr.data(), quat.data(), trans.data(), points.data());
      if (rc == B200SFM_OK && options_.optimize_rig_poses) rc = b200sfm_ba_problem_set_sensor_variable(prob, sensor_var.data());
      if (rc == B200SFM_OK) rc = b200sfm_ba_problem_solve(prob, &o, &summary);
      if (rc == B200SFM_OK) rc = b200sfm_ba_problem_get_state(prob, intr.data(), quat.data(), trans.data(), points.data());
      if (rc == B200SFM_OK && options_.optimize_rig_poses) {   // the optimised cam_from_rig back into the rigs, in place
        rc = b200sfm_ba_problem_get_sensor_poses(prob, sensor_q.data(), sensor_t.data());
        if (rc == B200SFM_OK)
          for (auto& [key, s] : sensors) {
            const int32_t idx = s.first;
            if (!sensor_var[idx]) continue;
            Rigid3d cfr;
            for (int k = 0; k < 4; ++k) cfr.rotation.coeffs().data()[k] = sensor_q[4 * (size_t)idx + k];
            for (int k = 0; k < 3; ++k) cfr.translation[k] = sensor_t[3 * (size_t)idx + k];
            b200host_adapt::SetCamFromRig(rigs[key.first], key.second, cfr);
          }
      }
      b200sfm_ba_problem_free(prob);
    } else {
      rc = b200sfm_ba_solve(ctx, &o, C, P, (int64_t)obs_cam.size(), K, ptb.data(), obs_cam.data(), obs_xy.data(),
                            cam_intr.data(), intr_model.data(), intr.data(), quat.data(), trans.data(), mask.data(),
                            points.data(), &summary);
    }
    if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm_ba_solve: %s\n", b200sfm_last_error(ctx)); return false; }
    for (int i = 0; i < C; ++i) {                                                             // results in place (.cc:140-146)
      Rigid3d& pose = fsorted[i].second->RigFromWorld();
      for (int k = 0; k < 4; ++k) pose.rotation.coeffs().data()[k] = quat[4 * i + k];
      for (int k = 0; k < 3; ++k) pose.translation[k] = trans[3 * i + k];
    }
    for (int p = 0; p < P; ++p)
      for (int k = 0; k < 3; ++k) tsorted[p].second->xyz[k] = points[3 * (size_t)p + k];
    detail::UnpackCameras(intr, csorted);
    return summary.usable != 0;                                                               // .cc:105
  }

 private:
  BundleAdjusterOptions options_;
};

// ---------------------------------------------------------------------------
struct GlobalPositionerOptions : public OptimizationBaseOptions {   // global_positioning.h:9-54
  enum ConstraintType { ONLY_POINTS, ONLY_CAMERAS, POINTS_AND_CAMERAS_BALANCED, POINTS_AND_CAMERAS };
  bool generate_random_positions = true, generate_random_points = true, generate_scales = true;
  bool optimize_positions = true, optimize_points = true, optimize_scales = true;
  bool use_gpu = true;
  std::string gpu_index = "-1";
  int min_num_images_gpu_solver = 50;
  int min_num_view_per_track = 3;
  unsigned seed = 1;
  ConstraintType constraint_type = ONLY_POINTS;
  double constraint_reweight_scale = 1.0;
  double pcg_rel_tolerance = 1e-2;
  int pcg_max_iterations = 1000;
  GlobalPositionerOptions() { thres_loss_function = 1e-1; }
};

class GlobalPositioner {
 public:
  GlobalPositioner(const GlobalPositionerOptions& options) : options_(options) { random_generator_.seed(options_.seed); }
  GlobalPositionerOptions& GetOptions() { return options_; }
  b200sfm_lm_stats summary{};

  // global_positioning.cc:28-93 (ONLY_POINTS, trivial rigs)
  bool Solve(const ViewGraph& view_graph, std::unordered_map<rig_t, Rig>& rigs,
             std::unordered_map<camera_t, Camera>& cameras, std::unordered_map<frame_t, Frame>& frames,
             std::unordered_map<image_t, Image>& images, std::unordered_map<track_t, Track>& tracks) {
    (void)view_graph;
    if (images.empty()) { std::fprintf(stderr, "Number of images = 0\n"); return false; }     // .cc:37-40
    if (tracks.empty()) { std::fprintf(stderr, "Number of tracks = 0\n"); return false; }     // .cc:46-50
    if (options_.constraint_type != GlobalPositionerOptions::ONLY_POINTS) {
      std::fprintf(stderr, "b200sfm: only ONLY_POINTS is implemented\n");
      return false;
    }
    b200sfm_ctx* ctx = DefaultContext(options_.gpu_index);
    if (!ctx) return false;
    const auto fsorted = detail::SortedEntries(frames);   // every frame is a block
    auto fidx = detail::PositionOf(fsorted);
    const int C = (int)fsorted.size();
    std::uniform_real_distribution<double> U(-1, 1);
    std::vector<double> centers(3 * (size_t)C), Rm(9 * (size_t)C);
    std::vector<uint8_t> calibrated(C, 1);
    for (int i = 0; i < C; ++i) {
      const Rigid3d& pose = fsorted[i].second->RigFromWorld();
      double* R = &Rm[9 * (size_t)i];
      detail::QuatToR(pose.rotation.coeffs().data(), R);
      if (options_.generate_random_positions && options_.optimize_positions) {
        for (int k = 0; k < 3; ++k) centers[3 * i + k] = 100.0 * U(random_generator_);        // .cc:158-159
      } else {                                                                                // CenterFromPose: -R^T t
        const double t[3] = {pose.translation[0], pose.translation[1], pose.translation[2]};
        detail::MulAtB<1>(R, t, &centers[3 * i]);
        for (int k = 0; k < 3; ++k) centers[3 * i + k] = -centers[3 * i + k];
      }
    }
    bool any_rig = false;
    for (auto& [id, im] : images) {
      calibrated[fidx[im.frame_id]] = cameras[im.camera_id].has_prior_focal_length ? 1 : 0;
      any_rig = any_rig || !im.HasTrivialFrame();
    }
    std::vector<double> obs_off;      // known rigs: R_cw^T t_cam_from_rig per observation (.cc:339-345)
    std::vector<uint8_t> obs_cal;     // the loss is chosen per CAMERA (.cc:313-316)
    // sensors whose cam_from_rig translation is still NaN (rotation averaging estimated their rotation only): their
    // centre in the rig frame is an unknown of this solve, RigUnknownBATAPairwiseDirectionError (.cc:355-372)
    // (numbered in order of first appearance; `urot` holds their cam_from_rig for the write-back)
    std::map<std::pair<rig_t, camera_t>, int> usens;
    std::vector<Rigid3d> urot;
    std::vector<int32_t> obs_usens;
    const auto tsorted = detail::SortedEntries(tracks);
    const int P = (int)tsorted.size();
    std::vector<int64_t> ptb(1, 0);
    std::vector<int32_t> obs_cam;
    std::vector<double> obs_dir, points(3 * (size_t)P);
    for (int p = 0; p < P; ++p) {
      Track& t = *tsorted[p].second;
      const bool keep = (int)t.observations.size() >= options_.min_num_view_per_track;         // .cc:257-258
      for (const auto& ob : t.observations) {
        if (!keep) break;
        auto it = images.find(ob.first);
        if (it == images.end() || !it->second.IsRegistered()) continue;                      // .cc:279-282
        const Image& im = it->second;
        const double b[3] = {im.features_undist[ob.second][0], im.features_undist[ob.second][1], im.features_undist[ob.second][2]};
        if (std::isnan(b[0]) || std::isnan(b[1]) || std::isnan(b[2])) continue;               // .cc:286-292
        const int ci = fidx[im.frame_id];
        const double* R = &Rm[9 * (size_t)ci];
        double dir[3];
        if (any_rig) {
          // cam_from_world = cam_from_rig * rig_from_world;  t_obs = R_cw^T b,  t_rig = R_cw^T t_cam_from_rig
          Rigid3d cfr;   // a missing cam_from_rig stays the identity
          detail::ResolveCamFromRig(im.HasTrivialFrame() ? nullptr : &rigs[frames[im.frame_id].RigId()], im, cfr);
          int us = -1;
          if (std::isnan(cfr.translation[0]) || std::isnan(cfr.translation[1]) || std::isnan(cfr.translation[2])) {
            const auto key = std::make_pair(frames[im.frame_id].RigId(), im.camera_id);
            auto u = usens.find(key);
            if (u == usens.end()) {
              u = usens.emplace(key, (int)usens.size()).first;
              urot.push_back(cfr);
            }
            us = u->second;
            cfr.translation[0] = cfr.translation[1] = cfr.translation[2] = 0.0;   // no known offset: the centre is the unknown
          }
          obs_usens.push_back(us);
          double Rs[9], off[3];
          detail::QuatToR(cfr.rotation.coeffs().data(), Rs);
          const double t_cr[3] = {cfr.translation[0], cfr.translation[1], cfr.translation[2]};
          detail::MulAtB<1>(Rs, b, dir);          // R_cr^T b
          detail::MulAtB<1>(Rs, t_cr, off);       // R_cr^T t_cr
          detail::MulAtB<1>(R, dir, dir);
          detail::MulAtB<1>(R, off, off);
          obs_off.insert(obs_off.end(), off, off + 3);
          obs_cal.push_back(cameras[im.camera_id].has_prior_focal_length ? 1 : 0);
        } else {
          detail::MulAtB<1>(R, b, dir);           // R^T b (.cc:294-296)
        }
        obs_dir.insert(obs_dir.end(), dir, dir + 3);
        obs_cam.push_back(ci);
      }
      ptb.push_back((int64_t)obs_cam.size());
      const bool rnd = options_.optimize_points && options_.generate_random_points &&
                       (int)t.observations.size() >= options_.min_num_view_per_track;
      for (int k = 0; k < 3; ++k) points[3 * (size_t)p + k] = rnd ? 100.0 * U(random_generator_) : t.xyz[k];   // .cc:261-264
      if (rnd) t.is_initialized = true;
    }
    std::vector<double> scales(obs_cam.size(), 1.0);                                          // .cc:298
    b200sfm_gp_opts o;
    b200sfm_gp_default_opts(&o);
    o.optimize_positions = options_.optimize_positions; o.optimize_points = options_.optimize_points;
    o.optimize_scales = options_.optimize_scales;
    o.min_num_view_per_track = 1;   // the track-length rule was applied above, on track.observations.size()
    o.max_num_iterations = options_.solver_options.max_num_iterations;
    o.thres_loss_function = options_.thres_loss_function;
    o.function_tolerance = options_.solver_options.function_tolerance;
    o.pcg_rel_tolerance = options_.pcg_rel_tolerance; o.pcg_max_iterations = options_.pcg_max_iterations;
    int rc;
    if (any_rig) {   // RigBATA with the rig scales held constant (.cc:325-346,493-497)
      b200sfm_gp_problem* prob = nullptr;
      rc = b200sfm_gp_problem_create(ctx, C, P, (int64_t)obs_cam.size(), ptb.data(), obs_cam.data(), obs_dir.data(),
                                     calibrated.data(), nullptr, o.min_num_view_per_track, &prob);
      if (rc == B200SFM_OK) rc = b200sfm_gp_problem_set_rig_terms(prob, obs_off.data(), obs_cal.data());
      // unknown sensor centres: U(-1, 1)^3 when the positions are optimised (.cc:440-453), in order of first appearance
      std::vector<double> ucen(3 * usens.size(), 0.0);
      if (!usens.empty()) {
        if (options_.optimize_positions)
          for (double& v : ucen) v = U(random_generator_);
        if (rc == B200SFM_OK)
          rc = b200sfm_gp_problem_set_rig_unknown(prob, (int32_t)usens.size(), obs_usens.data(), Rm.data(), ucen.data());
      }
      if (rc == B200SFM_OK) rc = b200sfm_gp_problem_set_state(prob, centers.data(), points.data(), scales.data());
      if (rc == B200SFM_OK) rc = b200sfm_gp_problem_solve(prob, &o, &summary);
      if (rc == B200SFM_OK) rc = b200sfm_gp_problem_get_state(prob, centers.data(), points.data(), scales.data());
      if (rc == B200SFM_OK && !usens.empty()) {
        rc = b200sfm_gp_problem_get_rig_unknown(prob, ucen.data());
        if (rc == B200SFM_OK)
          for (auto& [key, idx] : usens) {   // ConvertResults: centre -> translation = -(R_cr u)  (.cc:578-582)
            Rigid3d cfr = urot[idx];
            double Rs[9], t[3];
            detail::QuatToR(cfr.rotation.coeffs().data(), Rs);
            detail::MulAB<1>(Rs, &ucen[3 * (size_t)idx], t);
            for (int k = 0; k < 3; ++k) cfr.translation[k] = -t[k];
            b200host_adapt::SetCamFromRig(rigs[key.first], key.second, cfr);
          }
      }
      b200sfm_gp_problem_free(prob);
    } else {
      rc = b200sfm_gp_solve(ctx, &o, C, P, (int64_t)obs_cam.size(), ptb.data(), obs_cam.data(), obs_dir.data(),
                            calibrated.data(), nullptr, centers.data(), points.data(), scales.data(), &summary);
    }
    if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm_gp_solve: %s\n", b200sfm_last_error(ctx)); return false; }
    for (int i = 0; i < C; ++i) {                                                             // ConvertResults: t = -R c (.cc:566-568)
      double t[3];
      detail::MulAB<1>(&Rm[9 * (size_t)i], &centers[3 * (size_t)i], t);
      for (int k = 0; k < 3; ++k) fsorted[i].second->RigFromWorld().translation[k] = -t[k];
    }
    for (int p = 0; p < P; ++p)
      for (int k = 0; k < 3; ++k) tsorted[p].second->xyz[k] = points[3 * (size_t)p + k];
    return summary.usable != 0;
  }

 private:
  GlobalPositionerOptions options_;
  std::mt19937 random_generator_;
};

// ---------------------------------------------------------------------------
struct RotationEstimatorOptions {   // global_rotation_averaging.h:39-75
  int max_num_l1_iterations = 5;
  double l1_step_convergence_threshold = 0.001;
  int max_num_irls_iterations = 100;
  double irls_step_convergence_threshold = 0.001;
  double irls_loss_parameter_sigma = 5.0;
  enum WeightType { GEMAN_MCCLURE, HALF_NORM } weight_type = GEMAN_MCCLURE;
  bool skip_initialization = false;
  bool use_weight = false;
  bool use_gravity = false;
  double pcg_rel_tolerance = 1e-8;
};

namespace detail {
inline b200sfm_ra_opts RaOpts(const RotationEstimatorOptions& options) {
  b200sfm_ra_opts o;
  b200sfm_ra_default_opts(&o);
  o.max_num_l1_iterations = options.max_num_l1_iterations; o.max_num_irls_iterations = options.max_num_irls_iterations;
  o.l1_step_convergence_threshold = options.l1_step_convergence_threshold;
  o.irls_step_convergence_threshold = options.irls_step_convergence_threshold;
  o.irls_loss_parameter_sigma = options.irls_loss_parameter_sigma;
  o.weight_type = options.weight_type == RotationEstimatorOptions::HALF_NORM ? 1 : 0;
  o.use_weight = options.use_weight; o.pcg_rel_tolerance = options.pcg_rel_tolerance;
  return o;
}
}  // namespace detail

class RotationEstimator {
 public:
  explicit RotationEstimator(const RotationEstimatorOptions& options) : options_(options) {}
  b200sfm_ra_stats summary{};

  // InitializeFromMaximumSpanningTree (global_rotation_averaging.cc:87-138 + math/tree.cc:78-153): Kruskal on
  // (max #inliers - #inliers), BFS from the first registered image, composition of the relative rotations along the
  // tree, then ConvertRotationsFromImageToRig (rotation_initializer.cc:7-120) for trivial frames and calibrated rigs:
  // rig_from_world = average over the frame's images of cam_from_rig^-1 * cam_from_world.  Images are enumerated in
  // sorted-id order (the reference: unordered_map order), so the root is the smallest registered image id.
  void InitializeFromMaximumSpanningTree(const ViewGraph& view_graph, std::unordered_map<rig_t, Rig>& rigs,
                                         std::unordered_map<frame_t, Frame>& frames,
                                         std::unordered_map<image_t, Image>& images) {
    auto registered = [&](const Image& im) {
      auto f = frames.find(im.frame_id);
      return f != frames.end() && f->second.is_registered;
    };
    const auto isorted = detail::SortedEntries(images, registered);
    const auto idx = detail::PositionOf(isorted);
    const int n = (int)isorted.size();
    if (n == 0) return;
    struct Edge { double w; int a, b; const ImagePair* pr; };
    const auto psorted = detail::SortedEntries(view_graph.image_pairs, [](const ImagePair& pr) { return pr.is_valid; });
    double max_w = 0;
    for (const auto& [id, pr] : psorted) max_w = std::max(max_w, (double)pr->inliers.size());   // tree.cc:93-100 (INLIER_NUM)
    std::vector<Edge> edges;
    for (const auto& [id, pr] : psorted) {
      auto a = idx.find(pr->image_id1), b = idx.find(pr->image_id2);
      if (a == idx.end() || b == idx.end()) continue;                                         // tree.cc:113-116
      edges.push_back({max_w - (double)pr->inliers.size(), a->second, b->second, pr});
    }
    std::stable_sort(edges.begin(), edges.end(), [](const Edge& x, const Edge& y) { return x.w < y.w; });
    std::vector<int> uf(n);
    for (int i = 0; i < n; ++i) uf[i] = i;
    auto find = [&](int x) { while (uf[x] != x) { uf[x] = uf[uf[x]]; x = uf[x]; } return x; };
    std::vector<std::vector<std::pair<int, const ImagePair*>>> adj(n);
    for (const Edge& e : edges) {
      const int ra = find(e.a), rb = find(e.b);
      if (ra == rb) continue;
      uf[ra] = rb;
      adj[e.a].push_back({e.b, e.pr});
      adj[e.b].push_back({e.a, e.pr});
    }
    // BFS from index 0; cam_from_world rotation of the root = identity (default-constructed, .cc:112)
    std::vector<std::array<double, 4>> q(n, {{0, 0, 0, 1}});
    std::vector<char> seen(n, 0);
    std::queue<int> bfs;
    bfs.push(0);
    seen[0] = 1;
    while (!bfs.empty()) {
      const int cur = bfs.front();
      bfs.pop();
      for (const auto& [nb, pr] : adj[cur]) {
        if (seen[nb]) continue;
        seen[nb] = 1;
        const double* r21 = pr->cam2_from_cam1.rotation.coeffs().data();
        if (pr->image_id1 == isorted[nb].first) {   // 1_R_w = 2_R_1^T * 2_R_w   (.cc:125-129)
          double inv[4];
          detail::QuatConj(r21, inv);
          detail::QuatMul(inv, q[cur].data(), q[nb].data());
        } else {                                    // 2_R_w = 2_R_1 * 1_R_w     (.cc:130-134)
          detail::QuatMul(r21, q[cur].data(), q[nb].data());
        }
        bfs.push(nb);
      }
    }
    // ConvertRotationsFromImageToRig: per frame, average cam_from_rig^-1 * cam_from_world over its estimated images
    std::map<frame_t, std::vector<std::array<double, 4>>> per_frame;
    for (int i = 0; i < n; ++i) {
      if (!seen[i]) continue;                    // not reached by the tree: not estimated (rotation_initializer.cc:101-102)
      const Image& im = *isorted[i].second;
      std::array<double, 4> r = q[i];
      Rigid3d c;
      const auto s = detail::ResolveCamFromRig(im.HasTrivialFrame() ? nullptr : &rigs[frames[im.frame_id].RigId()], im, c);
      if (s == detail::CamFromRigStatus::kMissing) continue;                                  // .cc:108-111
      if (s == detail::CamFromRigStatus::kKnown) {
        double inv[4];
        detail::QuatConj(c.rotation.coeffs().data(), inv);
        detail::QuatMul(inv, q[i].data(), r.data());
      }
      per_frame[im.frame_id].push_back(r);
    }
    for (auto& [fid, qs] : per_frame) {
      double avg[4];
      AverageQuaternions(qs, avg);
      double* out = frames[fid].RigFromWorld().rotation.coeffs().data();
      for (int k = 0; k < 4; ++k) out[k] = avg[k];
    }
  }

  // global_rotation_averaging.cc:40-85 (3-DoF frames and, with use_gravity, 1-DoF frames that carry a gravity
  // prior; trivial frames, known rigs and rigs with sensors whose cam_from_rig rotation is estimated alongside).
  bool EstimateRotations(const ViewGraph& view_graph, std::unordered_map<rig_t, Rig>& rigs,
                         std::unordered_map<frame_t, Frame>& frames, std::unordered_map<image_t, Image>& images) {
    if (options_.use_gravity) {   // .cc:47-59: gravity-aligned averaging needs every rig calibrated
      for (auto& [rig_id, rig] : rigs)
        if (!b200host_adapt::AllSensorsCalibrated(rig)) {
          std::fprintf(stderr, "Rig %u has an uncalibrated sensor, but the gravity aligned rotation is requested. "
                               "Please add the rig calibration.\n", (unsigned)rig_id);
          return false;
        }
    }
    b200sfm_ctx* ctx = DefaultContext();
    if (!ctx) return false;
    if (!options_.skip_initialization && !options_.use_gravity)                               // .cc:60-63
      InitializeFromMaximumSpanningTree(view_graph, rigs, frames, images);
    const auto fsorted = detail::SortedEntries(frames, [](const Frame& f) { return f.is_registered; });
    const auto fidx = detail::PositionOf(fsorted);
    const int n = (int)fsorted.size();
    if (n == 0) return false;
    std::vector<double> theta(3 * (size_t)n);
    for (int i = 0; i < n; ++i) detail::QuatToAngleAxis(fsorted[i].second->RigFromWorld().rotation.coeffs().data(), &theta[3 * (size_t)i]);   // .cc:223-224
    // Cameras whose cam_from_rig rotation has to be estimated (.cc:162-194): non-reference sensors of the rigs of the
    // registered images without a cam_from_rig, or with one whose translation is still NaN (its rotation is then the
    // initial value, .cc:186-190; else zero, .cc:239-241).  They become nodes n, n + 1, ... in ascending camera id.
    std::map<camera_t, std::pair<rig_t, const Image*>> cam_rig;   // the rig and an image of the camera
    for (auto& [id, im] : images) {
      const auto fit = frames.find(im.frame_id);
      if (fit == frames.end() || !fit->second.is_registered) continue;
      if (im.HasTrivialFrame()) continue;   // == IsRefSensor of its rig (scene/image.h:73-76): never estimated
      cam_rig[im.camera_id] = {fit->second.RigId(), &im};
    }
    std::map<camera_t, int> ucam;
    for (auto& [cam, rig_im] : cam_rig) {
      Rigid3d c;
      const auto s = detail::ResolveCamFromRig(&rigs[rig_im.first], *rig_im.second, c);
      if (s == detail::CamFromRigStatus::kIdentity) continue;
      const bool has = s == detail::CamFromRigStatus::kKnown;
      if (!has || std::isnan(c.translation[0]) || std::isnan(c.translation[1]) || std::isnan(c.translation[2])) {
        const int node = n + (int)ucam.size();
        ucam[cam] = node;
        double aa[3] = {0, 0, 0};
        if (has) detail::QuatToAngleAxis(c.rotation.coeffs().data(), aa);
        theta.insert(theta.end(), aa, aa + 3);
      }
    }
    const int n_cams = (int)ucam.size();
    // use_gravity (.cc:207-217): a frame with a gravity prior keeps theta = (0, phi, 0), phi = RotUpToAngle(R_align^T R);
    // the first such frame (sorted-id order) is the fixed one
    std::vector<uint8_t> has_gravity(n, 0);
    std::vector<double> R_align(9 * (size_t)n, 0.0);
    int fixed_frame = 0;
    bool any_gravity = false;
    if (options_.use_gravity) {
      for (int i = 0; i < n; ++i) {
        const Frame& f = *fsorted[i].second;
        if (!f.HasGravity()) continue;
        double* Ra = &R_align[9 * (size_t)i];
        b200host_adapt::RAlignRowMajor(f, Ra);
        double R0[9], M[9], q[4], aa[3];
        detail::QuatToR(f.RigFromWorld().rotation.coeffs().data(), R0);
        detail::MulAtB(Ra, R0, M);   // R_align^T R
        detail::RToQuat(M, q);
        detail::QuatToAngleAxis(q, aa);
        theta[3 * (size_t)i] = 0.0; theta[3 * (size_t)i + 1] = aa[1]; theta[3 * (size_t)i + 2] = 0.0;
        has_gravity[i] = 1;
        if (!any_gravity) fixed_frame = i;
        any_gravity = true;
      }
    }
    // cam_from_rig of an image of a known rig as a matrix (a missing one counts as the identity)
    auto Rc = [&](const Image& im, double out[9]) {
      Rigid3d c;
      detail::ResolveCamFromRig(&rigs[frames[im.frame_id].RigId()], im, c);
      detail::QuatToR(c.rotation.coeffs().data(), out);
    };
    const auto psorted = detail::SortedEntries(view_graph.image_pairs, [](const ImagePair& pr) { return pr.is_valid; });
    std::vector<int32_t> ei, ej, eci, ecj;
    std::vector<double> Rrel, w;
    for (const auto& [id, pr] : psorted) {
      const auto i1 = images.find(pr->image_id1), i2 = images.find(pr->image_id2);
      if (i1 == images.end() || i2 == images.end()) continue;
      const auto f1 = fidx.find(i1->second.frame_id), f2 = fidx.find(i2->second.frame_id);
      if (f1 == fidx.end() || f2 == fidx.end()) continue;                                     // .cc:365-368
      double R[9];
      detail::QuatToR(pr->cam2_from_cam1.rotation.coeffs().data(), R);
      // known rigs: the unknowns are the frame rotations, R_rel = R_c2r2^T R_21 R_c1r1 (.cc:274-309); an image
      // pair inside one frame is a self loop and is skipped (.cc:300-303)
      // (has_sensor_from_rig of the reference: a non-reference sensor with a KNOWN cam_from_rig; an unknown one
      //  contributes the identity here and its own -I / +I block, .cc:281-296,425-440)
      const auto u1 = ucam.find(i1->second.camera_id), u2 = ucam.find(i2->second.camera_id);
      const bool rig1 = !i1->second.HasTrivialFrame() && u1 == ucam.end();
      const bool rig2 = !i2->second.HasTrivialFrame() && u2 == ucam.end();
      if (rig1 && rig2 && f1->second == f2->second) continue;
      double T[9];
      if (rig1) { Rc(i1->second, T); detail::MulAB(R, T, R); }
      if (rig2) { Rc(i2->second, T); detail::MulAtB(T, R, R); }                               // Rc^T R
      if (any_gravity) {   // align the relative rotation with the gravity frames (.cc:311-326)
        if (has_gravity[f1->second]) detail::MulAB(R, &R_align[9 * (size_t)f1->second], R);
        if (has_gravity[f2->second]) detail::MulAtB(&R_align[9 * (size_t)f2->second], R, R);   // R_align^T R
      }
      ei.push_back(f1->second);
      ej.push_back(f2->second);
      eci.push_back(u1 == ucam.end() || i1->second.HasTrivialFrame() ? -1 : u1->second);
      ecj.push_back(u2 == ucam.end() || i2->second.HasTrivialFrame() ? -1 : u2->second);
      Rrel.insert(Rrel.end(), R, R + 9);
      w.push_back(pr->weight);
    }
    const b200sfm_ra_opts o = detail::RaOpts(options_);
    int rc;
    if (n_cams > 0) {   // frames that hold an image of each unknown camera (the quaternion average of .cc:675-693 runs over them)
      std::map<camera_t, std::set<int>> cam_frames_of;
      for (auto& [id, im] : images) {
        const auto u = ucam.find(im.camera_id);
        const auto f = fidx.find(im.frame_id);
        if (u != ucam.end() && f != fidx.end() && !im.HasTrivialFrame()) cam_frames_of[im.camera_id].insert(f->second);
      }
      std::vector<int32_t> cfb(1, 0), cf;
      for (auto& [cam, node] : ucam) {
        for (int f : cam_frames_of[cam]) cf.push_back(f);
        cfb.push_back((int32_t)cf.size());
      }
      rc = b200sfm_ra_solve_rig(ctx, &o, n, n_cams, (int64_t)ei.size(), ei.data(), ej.data(), eci.data(), ecj.data(), Rrel.data(),
                                w.data(), cfb.data(), cf.data(), 0, theta.data(), &summary);
    } else if (any_gravity) {
      rc = b200sfm_ra_solve_gravity(ctx, &o, n, (int64_t)ei.size(), ei.data(), ej.data(), Rrel.data(), w.data(), has_gravity.data(),
                                    fixed_frame, theta.data(), &summary);
    } else {
      rc = b200sfm_ra_solve(ctx, &o, n, (int64_t)ei.size(), ei.data(), ej.data(), Rrel.data(), w.data(), 0, theta.data(), &summary);
    }
    if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm_ra_solve: %s\n", b200sfm_last_error(ctx)); return false; }
    if (!summary.usable) return false;                                                        // NaN (.cc:508-512,590-593)
    for (int i = 0; i < n; ++i) {                                                             // ConvertResults (.cc:787-798)
      Rigid3d& pose = fsorted[i].second->RigFromWorld();
      double* qout = pose.rotation.coeffs().data();
      if (has_gravity[i]) {   // R = R_align * AngleToRotUp(phi)
        double qa[4], M[9];
        detail::AngleAxisToQuat(&theta[3 * (size_t)i], qa);
        detail::QuatToR(qa, M);
        detail::MulAB(&R_align[9 * (size_t)i], M, M);
        detail::RToQuat(M, qout);
      } else {
        detail::AngleAxisToQuat(&theta[3 * (size_t)i], qout);
      }
      for (int k = 0; k < 3; ++k) pose.translation[k] = 0.0;                                  // Vector3d::Zero() (.cc:795)
    }
    for (auto& [cam, node] : ucam) {   // the estimated cam_from_rig rotations, translation not known yet (.cc:800-813)
      Rigid3d c;
      detail::AngleAxisToQuat(&theta[3 * (size_t)node], c.rotation.coeffs().data());
      for (int k = 0; k < 3; ++k) c.translation[k] = std::numeric_limits<double>::quiet_NaN();
      b200host_adapt::SetCamFromRig(rigs[cam_rig[cam].first], cam, c);
    }
    return true;
  }

 private:
  const RotationEstimatorOptions& options_;   // the reference stores a const& too (.h:140)
};

// ---------------------------------------------------------------------------
struct InlierThresholdOptions {   // glomap/types.h:18-32
  double max_angle_error = 1.;
  double max_reprojection_error = 1e-2;
  double min_triangulation_angle = 1.;
  double max_epipolar_error_E = 1.;
  double max_epipolar_error_F = 4.;
  double max_epipolar_error_H = 4.;
  double min_inlier_num = 30;
  double min_inlier_ratio = 0.25;
  double max_rotation_error = 10.;
};

// ImagePairsInlierCount (processors/image_pair_inliers.cc:200-213) on the device: the pairs whose inliers are cleared
// (all, or with clean_inliers = false only those without inliers) and of those the valid ones are scored.  Images,
// cameras and pairs are flattened in sorted-id order; ImagePair::inliers is rewritten in ascending row order.
// A template over the view graph and the options so that, inside a glomap build, the caller's own
// glomap::InlierThresholdOptions (glomap/types.h, not an estimator header the shim replaces) is accepted as it is.
template <class ViewGraphT, class InlierOptions>
void ImagePairsInlierCount(ViewGraphT& view_graph, const std::unordered_map<camera_t, Camera>& cameras,
                           const std::unordered_map<image_t, Image>& images, const InlierOptions& options, bool clean_inliers) {
  using Pair = typename std::remove_reference<decltype(view_graph.image_pairs.begin()->second)>::type;
  std::vector<Pair*> scored;
  for (auto& [id, pr] : detail::SortedEntries(view_graph.image_pairs)) {
    if (!clean_inliers && pr->inliers.size() > 0) continue;
    pr->inliers.clear();
    if (pr->is_valid) scored.push_back(pr);
  }
  if (scored.empty()) return;
  b200sfm_ctx* ctx = DefaultContext();
  if (!ctx) return;
  const auto csorted = detail::SortedEntries(cameras);
  const auto cidx = detail::PositionOf(csorted);
  std::vector<int32_t> intr_model;
  std::vector<double> intr;
  detail::PackCameras(csorted, intr_model, intr);
  const auto isorted = detail::SortedEntries(images);
  const auto iidx = detail::PositionOf(isorted);
  std::vector<int64_t> feature_begin(1, 0);
  std::vector<double> features;
  std::vector<int32_t> image_intr;
  for (auto& [id, im] : isorted) {
    auto c = cidx.find(im->camera_id);
    image_intr.push_back(c == cidx.end() ? -1 : c->second);
    for (const auto& f : im->features) { features.push_back(f[0]); features.push_back(f[1]); }
    feature_begin.push_back((int64_t)features.size() / 2);
  }
  const int64_t E = (int64_t)scored.size();
  std::vector<int32_t> img1, img2, config, matches;
  std::vector<double> quat, trans, F, H;
  std::vector<int64_t> match_begin(1, 0);
  for (Pair* pr : scored) {
    auto a = iidx.find(pr->image_id1), b = iidx.find(pr->image_id2);
    if (a == iidx.end() || b == iidx.end()) { std::fprintf(stderr, "b200sfm: image pair with an unknown image\n"); return; }
    img1.push_back(a->second); img2.push_back(b->second); config.push_back(pr->config);
    for (int k = 0; k < 4; ++k) quat.push_back(pr->cam2_from_cam1.rotation.coeffs().data()[k]);
    for (int k = 0; k < 3; ++k) trans.push_back(pr->cam2_from_cam1.translation[k]);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) { F.push_back(pr->F(r, c)); H.push_back(pr->H(r, c)); }
    for (long k = 0; k < (long)pr->matches.rows(); ++k) { matches.push_back(pr->matches(k, 0)); matches.push_back(pr->matches(k, 1)); }
    match_begin.push_back((int64_t)matches.size() / 2);
  }
  std::vector<uint8_t> is_inlier(match_begin.back());
  std::vector<int32_t> num_inliers(E);
  std::vector<double> score(E);
  const int rc = b200sfm_image_pairs_inlier_count(
      ctx, (int32_t)image_intr.size(), feature_begin.data(), features.data(), image_intr.data(), (int32_t)intr_model.size(),
      intr_model.data(), intr.data(), E, img1.data(), img2.data(), config.data(), quat.data(), trans.data(), F.data(), H.data(),
      match_begin.data(), matches.data(), options.max_epipolar_error_E, options.max_epipolar_error_F, options.max_epipolar_error_H,
      is_inlier.data(), num_inliers.data(), score.data());
  if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm: ImagePairsInlierCount failed: %s\n", b200sfm_last_error(ctx)); return; }
  for (int64_t e = 0; e < E; ++e)
    for (int64_t k = match_begin[e]; k < match_begin[e + 1]; ++k)
      if (is_inlier[k]) scored[e]->inliers.push_back((int)(k - match_begin[e]));
}

// processors/relpose_filter.{h,cc}: the two inlier filters the mapper runs after ImagePairsInlierCount (global_mapper.cc:67-70)
struct RelPoseFilter {
  template <class ViewGraphT>
  static void FilterInlierNum(ViewGraphT& view_graph, int min_inlier_num) {   // relpose_filter.cc:35-48
    for (auto& [id, pr] : view_graph.image_pairs)
      if (pr.is_valid && pr.inliers.size() < (size_t)min_inlier_num) pr.is_valid = false;   // size_t comparison as in the reference
  }
  template <class ViewGraphT>
  static void FilterInlierRatio(ViewGraphT& view_graph, double min_inlier_ratio) {   // relpose_filter.cc:50-65
    for (auto& [id, pr] : view_graph.image_pairs)   // 0 matches: NaN, not below the threshold -- the pair stays valid
      if (pr.is_valid && pr.inliers.size() / double(pr.matches.rows()) < min_inlier_ratio) pr.is_valid = false;
  }
  // relpose_filter.cc:7-33 on the device (b200sfm_view_graph_filter_rotations): images are flattened in sorted-id order
  // with their cam_from_world rotation (cam_from_rig * rig_from_world for a non-reference camera of a rig) and their
  // registration, the valid pairs in sorted pair-id order.  A registered image whose frame has no pose, or whose
  // cam_from_rig is unknown, gets a NaN rotation, so its pairs are kept.  Returns the number of pairs invalidated; -1 and
  // nothing changed when a pair names an unknown image or the device call fails (message on stderr).
  template <class ViewGraphT, class ImageMap>
  static int64_t FilterRotations(ViewGraphT& view_graph, const ImageMap& images, double max_angle) {
    using Pair = typename std::remove_reference<decltype(view_graph.image_pairs.begin()->second)>::type;
    const auto isorted = detail::SortedEntries(images);
    const auto iidx = detail::PositionOf(isorted);
    std::vector<double> quat;
    std::vector<uint8_t> reg;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    for (auto& [id, im] : isorted) {
      reg.push_back(im->IsRegistered() ? 1 : 0);
      double q[4] = {nan, nan, nan, nan};
      if (reg.back() && im->frame_ptr->HasPose()) {
        const double* r = im->frame_ptr->RigFromWorld().rotation.coeffs().data();
        auto* rig = im->frame_ptr->RigPtr();
        Rigid3d c;   // an image of a frame without a rig: the identity
        const auto s = rig ? detail::ResolveCamFromRig(rig, *im, c) : detail::CamFromRigStatus::kIdentity;
        if (s == detail::CamFromRigStatus::kIdentity) std::copy(r, r + 4, q);
        if (s == detail::CamFromRigStatus::kKnown) detail::QuatMul(c.rotation.coeffs().data(), r, q);
      }
      quat.insert(quat.end(), q, q + 4);
    }
    std::vector<Pair*> pairs;
    std::vector<int32_t> img1, img2;
    std::vector<double> rel;
    for (auto& [id, pr] : detail::SortedEntries(view_graph.image_pairs, [](const Pair& p) { return p.is_valid; })) {
      auto a = iidx.find(pr->image_id1), b = iidx.find(pr->image_id2);
      if (a == iidx.end() || b == iidx.end()) { std::fprintf(stderr, "b200sfm: image pair with an unknown image\n"); return -1; }
      pairs.push_back(pr);
      img1.push_back(a->second);
      img2.push_back(b->second);
      const double* q = pr->cam2_from_cam1.rotation.coeffs().data();
      rel.insert(rel.end(), q, q + 4);
    }
    if (pairs.empty()) return 0;
    b200sfm_ctx* ctx = DefaultContext();
    if (!ctx) return -1;
    std::vector<uint8_t> valid(pairs.size(), 1);
    int64_t n = 0;
    const int rc = b200sfm_view_graph_filter_rotations(ctx, (int32_t)reg.size(), quat.data(), reg.data(), (int64_t)pairs.size(),
                                                       img1.data(), img2.data(), rel.data(), max_angle, valid.data(), &n);
    if (rc != B200SFM_OK) {
      std::fprintf(stderr, "b200sfm: FilterRotations failed: %s\n", b200sfm_last_error(ctx));
      return -1;
    }
    for (size_t e = 0; e < pairs.size(); ++e)
      if (!valid[e]) pairs[e]->is_valid = false;
    return n;
  }
};

// ViewGraph::KeepLargestConnectedComponents (scene/view_graph.cc:56-97) on the device
// (b200sfm_view_graph_keep_largest_component): frames, images and pairs are flattened in sorted-id order; is_registered of
// every frame and is_valid of every pair are written back.  Equally large components: the one holding the smallest frame
// id.  Returns the number of registered images; 0 and nothing changed without a valid pair, and also when a pair names an
// unknown image, an image an unknown frame, or the device call fails (message on stderr).  The host version
// KeepLargestConnectedComponents below computes the same and is what SolveRotationAveraging and the CLI call.
template <class ViewGraphT, class FrameMap, class ImageMap>
int KeepLargestConnectedComponentsDevice(ViewGraphT& view_graph, FrameMap& frames, ImageMap& images) {
  using Pair = typename std::remove_reference<decltype(view_graph.image_pairs.begin()->second)>::type;
  const auto fr = detail::SortedEntries(frames);
  const auto fidx = detail::PositionOf(fr);
  std::vector<uint8_t> reg;
  for (auto& [id, f] : fr) reg.push_back(f->is_registered ? 1 : 0);
  const auto isorted = detail::SortedEntries(images);
  const auto iidx = detail::PositionOf(isorted);
  std::vector<int32_t> image_frame;
  for (auto& [id, im] : isorted) {
    auto f = fidx.find(im->frame_id);
    if (f == fidx.end()) { std::fprintf(stderr, "b200sfm: image of an unknown frame\n"); return 0; }
    image_frame.push_back(f->second);
  }
  std::vector<Pair*> pairs;
  std::vector<int32_t> img1, img2;
  std::vector<uint8_t> valid;
  for (auto& [id, pr] : detail::SortedEntries(view_graph.image_pairs)) {
    auto a = iidx.find(pr->image_id1), b = iidx.find(pr->image_id2);
    if (a == iidx.end() || b == iidx.end()) { std::fprintf(stderr, "b200sfm: image pair with an unknown image\n"); return 0; }
    pairs.push_back(pr);
    img1.push_back(a->second);
    img2.push_back(b->second);
    valid.push_back(pr->is_valid ? 1 : 0);
  }
  if (pairs.empty()) return 0;
  b200sfm_ctx* ctx = DefaultContext();
  if (!ctx) return 0;
  int32_t n = 0;
  const int rc = b200sfm_view_graph_keep_largest_component(ctx, (int32_t)fr.size(), (int32_t)image_frame.size(), image_frame.data(),
                                                           (int64_t)pairs.size(), img1.data(), img2.data(), valid.data(), reg.data(), &n);
  if (rc != B200SFM_OK) {
    std::fprintf(stderr, "b200sfm: KeepLargestConnectedComponents failed: %s\n", b200sfm_last_error(ctx));
    return 0;
  }
  if (n == 0) return 0;
  for (size_t f = 0; f < fr.size(); ++f) fr[f].second->is_registered = reg[f] != 0;
  for (size_t e = 0; e < pairs.size(); ++e) pairs[e]->is_valid = valid[e] != 0;
  return n;
}


// ---------------------------------------------------------------------------
struct ViewGraphCalibratorOptions : public OptimizationBaseOptions {   // view_graph_calibration.h:10-29
  double thres_lower_ratio = 0.1;
  double thres_higher_ratio = 10;
  double thres_two_view_error = 2.;
  int max_num_line_search_step_size_iterations = 20;   // Ceres default
  // PCG knobs of the device solver (the reference factors the normal matrix exactly, view_graph_calibration.cc:21-24)
  int pcg_max_iterations = 1000;
  double pcg_rel_tolerance = 1e-12;
  ViewGraphCalibratorOptions() { thres_loss_function = 1e-2; }
};

// The camera accessors the calibrator needs: glomap::Camera's own inside a glomap build (scene/camera.h:22-33 and
// colmap::Camera::FocalLengthIdxs), the COLMAP parameter layout of models 0-3 over scene_min.h otherwise.  Templates, so
// that a glomap build which never calls the calibrator does not need these members.
#ifdef B200SFM_WITH_GLOMAP
template <class CameraT>
double VgcFocal(const CameraT& c) { return c.Focal(); }
template <class CameraT>
void VgcPrincipalPoint(const CameraT& c, double* pp) {
  const auto p = c.PrincipalPoint();
  pp[0] = p(0);
  pp[1] = p(1);
}
template <class CameraT>
std::vector<size_t> VgcFocalLengthIdxs(const CameraT& c) {
  std::vector<size_t> out;
  for (const size_t idx : c.FocalLengthIdxs()) out.push_back(idx);
  return out;
}
#else
template <class CameraT>
bool VgcIsPinhole(const CameraT& c) { return static_cast<int>(c.model_id) == B200SFM_PINHOLE; }
template <class CameraT>
double VgcFocal(const CameraT& c) { return VgcIsPinhole(c) ? (c.params[0] + c.params[1]) / 2.0 : c.params[0]; }
template <class CameraT>
void VgcPrincipalPoint(const CameraT& c, double* pp) {
  const size_t o = VgcIsPinhole(c) ? 2 : 1;
  pp[0] = c.params[o];
  pp[1] = c.params[o + 1];
}
template <class CameraT>
std::vector<size_t> VgcFocalLengthIdxs(const CameraT& c) {
  return VgcIsPinhole(c) ? std::vector<size_t>{0, 1} : std::vector<size_t>{0};
}
#endif

// ViewGraphCalibrator (view_graph_calibration.{h,cc}) on the device: the valid CALIBRATED / UNCALIBRATED pairs are
// flattened in sorted pair-id order and the cameras in sorted camera-id order; CopyBackResults sets every
// FocalLengthIdxs() entry and has_refined_focal_length of the cameras the ratio test accepts, FilterImagePairs
// invalidates the pairs above thres_two_view_error.  Returns summary.IsSolutionUsable(); false also when the device call
// fails (message on stderr).  A template over the view graph and the scene maps so that it takes glomap's own ImagePair
// and Camera.
class ViewGraphCalibrator {
 public:
  explicit ViewGraphCalibrator(const ViewGraphCalibratorOptions& options) : options_(options) {}

  template <class ViewGraphT, class CameraMap, class ImageMap>
  bool Solve(ViewGraphT& view_graph, CameraMap& cameras, ImageMap& images) {
    using Pair = typename std::remove_reference<decltype(view_graph.image_pairs.begin()->second)>::type;
    const auto cams = detail::SortedEntries(cameras);
    const auto cidx = detail::PositionOf(cams);
    std::vector<double> pp, focal;
    std::vector<uint8_t> prior;
    for (auto& [id, c] : cams) {
      double p[2];
      VgcPrincipalPoint(*c, p);
      pp.push_back(p[0]); pp.push_back(p[1]);
      focal.push_back(VgcFocal(*c));
      prior.push_back(c->has_prior_focal_length ? 1 : 0);
    }
    std::vector<Pair*> qual;
    std::vector<int32_t> cam1, cam2;
    std::vector<double> F;
    for (auto& [id, pr] : detail::SortedEntries(view_graph.image_pairs)) {
      if (pr->config != B200SFM_TWO_VIEW_CALIBRATED && pr->config != B200SFM_TWO_VIEW_UNCALIBRATED) continue;
      if (!pr->is_valid) continue;
      auto a = images.find(pr->image_id1), b = images.find(pr->image_id2);
      if (a == images.end() || b == images.end()) { std::fprintf(stderr, "b200sfm: image pair with an unknown image\n"); return false; }
      auto ca = cidx.find(a->second.camera_id), cb = cidx.find(b->second.camera_id);
      if (ca == cidx.end() || cb == cidx.end()) { std::fprintf(stderr, "b200sfm: image with an unknown camera\n"); return false; }
      qual.push_back(pr);
      cam1.push_back(ca->second);
      cam2.push_back(cb->second);
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) F.push_back(pr->F(r, c));
    }
    const int32_t K = (int32_t)cams.size();
    const int64_t E = (int64_t)qual.size();
    b200sfm_vgc_opts o;
    b200sfm_vgc_default_opts(&o);
    o.max_num_iterations = options_.solver_options.max_num_iterations;
    o.max_num_line_search_step_size_iterations = options_.max_num_line_search_step_size_iterations;
    o.thres_loss_function = options_.thres_loss_function;
    o.function_tolerance = options_.solver_options.function_tolerance;
    o.gradient_tolerance = options_.solver_options.gradient_tolerance;
    o.parameter_tolerance = options_.solver_options.parameter_tolerance;
    o.thres_lower_ratio = options_.thres_lower_ratio;
    o.thres_higher_ratio = options_.thres_higher_ratio;
    o.thres_two_view_error = options_.thres_two_view_error;
    o.pcg_max_iterations = options_.pcg_max_iterations;
    o.pcg_rel_tolerance = options_.pcg_rel_tolerance;
    b200sfm_ctx* ctx = DefaultContext();
    if (!ctx) return false;
    std::vector<uint8_t> valid(E, 1), accepted(K, 0);
    b200sfm_lm_stats st{};
    const int rc = b200sfm_view_graph_calibrate(ctx, &o, K, pp.data(), focal.data(), prior.data(), E, cam1.data(), cam2.data(),
                                                F.data(), valid.data(), accepted.data(), nullptr, &st);
    if (rc != B200SFM_OK) {
      std::fprintf(stderr, "b200sfm: ViewGraphCalibrator failed: %s\n", b200sfm_last_error(ctx));
      return false;
    }
    for (int32_t k = 0; k < K; ++k) {
      if (!accepted[k]) continue;
      cams[k].second->has_refined_focal_length = true;
      for (const size_t idx : VgcFocalLengthIdxs(*cams[k].second)) cams[k].second->params[idx] = focal[k];
    }
    for (int64_t e = 0; e < E; ++e)
      if (!valid[e]) qual[e]->is_valid = false;
    return st.usable != 0;
  }

 private:
  ViewGraphCalibratorOptions options_;
};

// ---------------------------------------------------------------------------
// ViewGraphManipulater::UpdateImagePairsConfig (processors/view_graph_manipulation.cc:178-237), the first half of stage 0
// of GlobalMapper::Solve, on the device (b200sfm_view_graph_update_pairs_config): the cameras are flattened in sorted
// camera-id order (model_id and params), every pair in sorted pair-id order with its validity.  The promoted pairs get
// config CALIBRATED and F = K2^-T [t]x R K1^-1 of the cam2_from_cam1 they carry; nothing else changes.  Returns the
// number of pairs promoted; -1 and nothing changed when a pair names an unknown image, an image an unknown camera, or the
// device call fails (message on stderr; a promoted pair whose camera model is outside 0-3 fails it).  DecomposeRelPose,
// the second half of stage 0, is COLMAP code and not part of the shim.
struct ViewGraphManipulater {
  template <class ViewGraphT, class CameraMap, class ImageMap>
  static int64_t UpdateImagePairsConfig(ViewGraphT& view_graph, const CameraMap& cameras, const ImageMap& images) {
    using Pair = typename std::remove_reference<decltype(view_graph.image_pairs.begin()->second)>::type;
    const auto csorted = detail::SortedEntries(cameras);
    const auto cidx = detail::PositionOf(csorted);
    std::vector<int32_t> model;
    std::vector<double> params;
    detail::PackCameras(csorted, model, params);
    std::vector<uint8_t> prior;
    for (auto& [id, c] : csorted) prior.push_back(c->has_prior_focal_length ? 1 : 0);
    std::vector<Pair*> pairs;
    std::vector<int32_t> cam1, cam2, config;
    std::vector<uint8_t> valid;
    std::vector<double> quat, trans, F;
    for (auto& [id, pr] : detail::SortedEntries(view_graph.image_pairs)) {
      auto a = images.find(pr->image_id1), b = images.find(pr->image_id2);
      if (a == images.end() || b == images.end()) { std::fprintf(stderr, "b200sfm: image pair with an unknown image\n"); return -1; }
      auto ca = cidx.find(a->second.camera_id), cb = cidx.find(b->second.camera_id);
      if (ca == cidx.end() || cb == cidx.end()) { std::fprintf(stderr, "b200sfm: image with an unknown camera\n"); return -1; }
      pairs.push_back(pr);
      cam1.push_back(ca->second);
      cam2.push_back(cb->second);
      valid.push_back(pr->is_valid ? 1 : 0);
      config.push_back((int32_t)pr->config);
      const double* q = pr->cam2_from_cam1.rotation.coeffs().data();
      quat.insert(quat.end(), q, q + 4);
      for (int k = 0; k < 3; ++k) trans.push_back(pr->cam2_from_cam1.translation[k]);
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) F.push_back(pr->F(r, c));
    }
    if (pairs.empty()) return 0;
    b200sfm_ctx* ctx = DefaultContext();
    if (!ctx) return -1;
    int64_t n = 0;
    const int rc = b200sfm_view_graph_update_pairs_config(ctx, (int32_t)model.size(), model.data(), params.data(), prior.data(),
                                                          (int64_t)pairs.size(), cam1.data(), cam2.data(), valid.data(), quat.data(),
                                                          trans.data(), config.data(), F.data(), &n);
    if (rc != B200SFM_OK) {
      std::fprintf(stderr, "b200sfm: UpdateImagePairsConfig failed: %s\n", b200sfm_last_error(ctx));
      return -1;
    }
    for (size_t e = 0; e < pairs.size(); ++e) {
      if (config[e] == (int32_t)pairs[e]->config) continue;
      pairs[e]->config = config[e];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) pairs[e]->F(r, c) = F[9 * e + 3 * r + c];
    }
    return n;
  }
};

// ---------------------------------------------------------------------------
// PruneWeaklyConnectedImages (processors/reconstruction_pruning.{h,cc}), stage 8 of GlobalMapper::Solve, on the device:
// frames are flattened in sorted frame-id order and tracks in sorted track-id order, each observation becomes the frame
// index of its image; a frame with >= 2 images present gets a self-loop (its intra-frame edges, :63-104).  Writes
// is_registered and cluster_id of every frame back and returns the number of clusters.  min_num_images has no effect,
// as in the reference (EstablishStrongClusters calls MarkConnectedComponents with its default -1).  Returns 0 and
// changes nothing when the device call fails or an observation names an unknown image or frame (message on stderr).
template <class FrameMap, class ImageMap, class TrackMap>
image_t PruneWeaklyConnectedImages(FrameMap& frames, ImageMap& images, TrackMap& tracks, int min_num_images = 2,
                                   int min_num_observations = 0) {
  (void)min_num_images;
  const auto fr = detail::SortedEntries(frames);
  const auto fidx = detail::PositionOf(fr);
  const int32_t F = (int32_t)fr.size();
  std::vector<int32_t> images_of(F, 0);
  for (auto& [id, im] : images) {
    auto it = fidx.find(im.frame_id);
    if (it != fidx.end()) ++images_of[it->second];
  }
  std::vector<uint8_t> self_loop(F), reg(F);
  for (int32_t f = 0; f < F; ++f) {
    self_loop[f] = images_of[f] >= 2 ? 1 : 0;
    reg[f] = fr[f].second->is_registered ? 1 : 0;
  }
  const auto tsorted = detail::SortedEntries(tracks);
  std::vector<int64_t> begin{0};
  std::vector<int32_t> obs_frame;
  for (auto& [id, t] : tsorted) {
    for (const auto& ob : t->observations) {
      auto im = images.find(ob.first);
      if (im == images.end()) { std::fprintf(stderr, "b200sfm: track observation of an unknown image\n"); return 0; }
      auto f = fidx.find(im->second.frame_id);
      if (f == fidx.end()) { std::fprintf(stderr, "b200sfm: image of an unknown frame\n"); return 0; }
      obs_frame.push_back(f->second);
    }
    begin.push_back((int64_t)obs_frame.size());
  }
  b200sfm_ctx* ctx = DefaultContext();
  if (!ctx) return 0;
  std::vector<int32_t> cluster(F, -1);
  int32_t num_clusters = 0;
  const int rc = b200sfm_prune_weakly_connected(ctx, F, (int64_t)tsorted.size(), begin.data(), obs_frame.data(), self_loop.data(),
                                                min_num_observations, 0, cluster.data(), reg.data(), &num_clusters, nullptr);
  if (rc != B200SFM_OK) {
    std::fprintf(stderr, "b200sfm: PruneWeaklyConnectedImages failed: %s\n", b200sfm_last_error(ctx));
    return 0;
  }
  for (int32_t f = 0; f < F; ++f) {
    fr[f].second->is_registered = reg[f] != 0;
    fr[f].second->cluster_id = cluster[f];
  }
  return (image_t)num_clusters;
}

// ---------------------------------------------------------------------------
struct TrackEstablishmentOptions {   // track_establishment.h:10-25 (field for field)
  double thres_inconsistency = 10.;
  int min_num_tracks_per_view = -1;
  int min_num_view_per_track = 3;
  int max_num_view_per_track = 100;
  int max_num_tracks = 10000000;
};

// TrackEngine (controllers/track_establishment.{h,cc}), stage 4 of GlobalMapper::Solve, on the device.  The constructor
// takes any options type with the reference's five fields (glomap's own TrackEstablishmentOptions inside a glomap
// build) and copies them.
//   EstablishFullTracks: the inlier matches of the valid pairs (sorted pair-id order) as image_id << 32 | feature_id with
//     their pixels from Image::features -> b200sfm_tracks_establish; every track, the discarded ones with no observations,
//     goes into `tracks` (cleared first, :7).  Returns the number of tracks.
//   FindTracksForProblem: tracks in sorted track-id order, registered = the images whose frame is registered ->
//     b200sfm_tracks_select; the selected tracks are copied with their observations restricted to the registered images.
//     Returns the number selected.
// Both return 0 and leave their output unchanged when the device call fails or a pair or observation names an unknown
// image (message on stderr).
// A class template (deduced from the constructor's arguments) so that it is compiled only where it is used.
template <class ViewGraphT = ViewGraph, class ImageMap = std::unordered_map<image_t, Image>>
class TrackEngine {
 public:
  template <class Options>
  TrackEngine(const ViewGraphT& view_graph, const ImageMap& images, const Options& options)
      : view_graph_(view_graph), images_(images) {
    options_.thres_inconsistency = options.thres_inconsistency;
    options_.min_num_tracks_per_view = options.min_num_tracks_per_view;
    options_.min_num_view_per_track = options.min_num_view_per_track;
    options_.max_num_view_per_track = options.max_num_view_per_track;
    options_.max_num_tracks = options.max_num_tracks;
  }

  size_t EstablishFullTracks(std::unordered_map<track_t, Track>& tracks) {
    std::vector<uint64_t> g1, g2;
    std::vector<double> xy1, xy2;
    for (const auto& [id, pr] : detail::SortedEntries(view_graph_.image_pairs)) {
      if (!pr->is_valid) continue;
      auto a = images_.find(pr->image_id1), b = images_.find(pr->image_id2);
      if (a == images_.end() || b == images_.end()) { std::fprintf(stderr, "b200sfm: image pair with an unknown image\n"); return 0; }
      for (const int k : pr->inliers) {
        const long f1 = pr->matches(k, 0), f2 = pr->matches(k, 1);
        if (f1 < 0 || f2 < 0 || f1 >= (long)a->second.features.size() || f2 >= (long)b->second.features.size()) {
          std::fprintf(stderr, "b200sfm: inlier match with a feature outside its image\n");
          return 0;
        }
        g1.push_back((uint64_t)pr->image_id1 << 32 | (uint64_t)f1);
        g2.push_back((uint64_t)pr->image_id2 << 32 | (uint64_t)f2);
        xy1.push_back(a->second.features[f1][0]); xy1.push_back(a->second.features[f1][1]);
        xy2.push_back(b->second.features[f2][0]); xy2.push_back(b->second.features[f2][1]);
      }
    }
    b200sfm_ctx* ctx = DefaultContext();
    if (!ctx) return 0;
    b200sfm_tracks* h = nullptr;
    int64_t T = 0, n = 0, discarded = 0;
    int rc = b200sfm_tracks_establish(ctx, (int64_t)g1.size(), g1.data(), g2.data(), xy1.data(), xy2.data(), options_.thres_inconsistency,
                                      &h, &T, &n, &discarded);
    std::vector<uint64_t> ids(T);
    std::vector<int64_t> begin(T + 1, 0);
    std::vector<uint32_t> img(n), feat(n);
    if (rc == B200SFM_OK) rc = b200sfm_tracks_get(h, ids.data(), begin.data(), img.data(), feat.data());
    b200sfm_tracks_free(h);
    if (rc != B200SFM_OK) {
      std::fprintf(stderr, "b200sfm: TrackEngine::EstablishFullTracks failed: %s\n", b200sfm_last_error(ctx));
      return 0;
    }
    tracks.clear();
    for (int64_t t = 0; t < T; ++t) {
      Track& tr = tracks[(track_t)ids[t]];
      tr.track_id = (track_t)ids[t];
      for (int64_t k = begin[t]; k < begin[t + 1]; ++k) tr.observations.emplace_back((image_t)img[k], (feature_t)feat[k]);
    }
    return tracks.size();
  }

  size_t FindTracksForProblem(const std::unordered_map<track_t, Track>& tracks_full,
                              std::unordered_map<track_t, Track>& tracks_selected) {
    const auto tsorted = detail::SortedEntries(tracks_full);
    std::vector<uint64_t> ids;
    std::vector<int64_t> begin{0};
    std::vector<uint32_t> obs_image;
    for (const auto& [id, t] : tsorted) {
      ids.push_back((uint64_t)id);
      for (const auto& ob : t->observations) obs_image.push_back((uint32_t)ob.first);
      begin.push_back((int64_t)obs_image.size());
    }
    std::set<image_t> registered;
    for (const auto& [id, im] : images_)
      if (im.IsRegistered()) registered.insert(id);
    const std::vector<uint32_t> reg(registered.begin(), registered.end());
    b200sfm_ctx* ctx = DefaultContext();
    if (!ctx) return 0;
    std::vector<uint8_t> keep(ids.size(), 0);
    int64_t num = 0;
    const int rc = b200sfm_tracks_select(ctx, (int64_t)ids.size(), ids.data(), begin.data(), obs_image.data(), (int32_t)reg.size(),
                                         reg.data(), options_.min_num_tracks_per_view, options_.min_num_view_per_track,
                                         options_.max_num_view_per_track, options_.max_num_tracks, keep.data(), &num);
    if (rc != B200SFM_OK) {
      std::fprintf(stderr, "b200sfm: TrackEngine::FindTracksForProblem failed: %s\n", b200sfm_last_error(ctx));
      return 0;
    }
    std::unordered_map<track_t, Track> out;
    size_t t = 0;
    for (const auto& [id, tr] : tsorted) {
      if (keep[t++]) {
        Track& o = out[id];
        o.track_id = id;
        for (const auto& ob : tr->observations)
          if (registered.count(ob.first)) o.observations.push_back(ob);
      }
    }
    tracks_selected = out;
    return tracks_selected.size();
  }

 private:
  TrackEstablishmentOptions options_;
  const ViewGraphT& view_graph_;
  const ImageMap& images_;
};

// ---------------------------------------------------------------------------
// GravityRefiner (estimators/gravity_refinement.{h,cc}), run by `rotation_averager --refine_gravity 1`, on the device
// (b200sfm_gravity_refine): frames in sorted frame-id order, valid pairs in sorted pair-id order whose two images have
// gravity (a frame prior and, off the rig's reference sensor, a known cam_from_rig), M = R_c2^T R_rel R_c1.  Accepted
// frames get gravity_info.SetGravity(g); their rig_from_world is left alone, as in the reference.  Every error-prone
// frame is refined against the priors as they were on entry (include/b200sfm.h states the rules).
// Weak, so that a host linked against a libb200sfm without these entries (an older build, a test double) still links;
// RefineGravity then reports the missing entry and changes nothing.
extern "C" {
void b200sfm_gravity_default_opts(b200sfm_gravity_opts* opts) __attribute__((weak));
int b200sfm_gravity_refine(b200sfm_ctx* ctx, const b200sfm_gravity_opts* opts, int32_t F, const double* R_align,
                           const uint8_t* has_gravity, int64_t E, const int32_t* frame1, const int32_t* frame2,
                           const double* M, double* gravity, uint8_t* status, b200sfm_gravity_stats* stats) __attribute__((weak));
}

struct GravityRefinerOptions : public OptimizationBaseOptions {   // gravity_refinement.h:12-26
  double max_outlier_ratio = 0.5;
  double max_gravity_error = 1.;
  int min_num_neighbors = 7;
};

class GravityRefiner {
 public:
  explicit GravityRefiner(const GravityRefinerOptions& options) : options_(options) {}
  b200sfm_gravity_stats summary{};

  template <class ViewGraphT, class FrameMap, class ImageMap>
  void RefineGravity(const ViewGraphT& view_graph, FrameMap& frames, ImageMap& images) {
    using Pair = std::remove_reference_t<decltype(view_graph.image_pairs.begin()->second)>;
    const auto fr = detail::SortedEntries(frames);
    const auto fidx = detail::PositionOf(fr);
    const int32_t F = (int32_t)fr.size();
    std::vector<double> R_align(9 * (size_t)F, 0.0);
    std::vector<uint8_t> has(F, 0);
    for (int32_t f = 0; f < F; ++f) {
      has[f] = fr[f].second->HasGravity() ? 1 : 0;
      if (has[f]) b200host_adapt::RAlignRowMajor(*fr[f].second, &R_align[9 * (size_t)f]);
    }
    // an image's cam_from_rig rotation; false: the image has no gravity (image.h:78-84)
    auto cam_rot = [&](const auto& im, int32_t f, double R[9]) {
      Rigid3d c;
      if (!has[f] || detail::ResolveCamFromRig(fr[f].second->RigPtr(), im, c) == detail::CamFromRigStatus::kMissing) return false;
      detail::QuatToR(c.rotation.coeffs().data(), R);
      return true;
    };
    std::vector<int32_t> f1, f2;
    std::vector<double> M;
    for (const auto& [id, pp] : detail::SortedEntries(view_graph.image_pairs, [](const Pair& pr) { return pr.is_valid; })) {
      const Pair& pr = *pp;
      const auto i1 = images.find(pr.image_id1), i2 = images.find(pr.image_id2);
      if (i1 == images.end() || i2 == images.end()) continue;
      const auto a = fidx.find(i1->second.frame_id), b = fidx.find(i2->second.frame_id);
      if (a == fidx.end() || b == fidx.end()) continue;
      double Rc1[9], Rc2[9], Me[9];
      if (!cam_rot(i1->second, a->second, Rc1) || !cam_rot(i2->second, b->second, Rc2)) continue;   // .cc:62-64,149
      detail::QuatToR(pr.cam2_from_cam1.rotation.coeffs().data(), Me);
      detail::MulAB(Me, Rc1, Me);    // R Rc1
      detail::MulAtB(Rc2, Me, Me);   // Rc2^T (R Rc1)
      f1.push_back(a->second);
      f2.push_back(b->second);
      M.insert(M.end(), Me, Me + 9);
    }
    if (f1.empty()) { std::fprintf(stderr, "Adjacency list not established\n"); return; }   // .cc:14-17
    if (!b200sfm_gravity_refine || !b200sfm_gravity_default_opts) {
      std::fprintf(stderr, "b200sfm: this libb200sfm has no b200sfm_gravity_refine\n");
      return;
    }
    b200sfm_ctx* ctx = DefaultContext();
    if (!ctx) return;
    b200sfm_gravity_opts o;
    b200sfm_gravity_default_opts(&o);
    o.max_outlier_ratio = options_.max_outlier_ratio;
    o.max_gravity_error = options_.max_gravity_error;
    o.min_num_neighbors = options_.min_num_neighbors;
    o.max_num_iterations = options_.solver_options.max_num_iterations;
    o.function_tolerance = options_.solver_options.function_tolerance;
    o.gradient_tolerance = options_.solver_options.gradient_tolerance;
    o.parameter_tolerance = options_.solver_options.parameter_tolerance;
    std::vector<double> g(3 * (size_t)F, 0.0);
    std::vector<uint8_t> status(F, 0);
    const int rc = b200sfm_gravity_refine(ctx, &o, F, R_align.data(), has.data(), (int64_t)f1.size(), f1.data(), f2.data(),
                                          M.data(), g.data(), status.data(), &summary);
    if (rc != B200SFM_OK) {
      std::fprintf(stderr, "b200sfm: RefineGravity failed: %s\n", b200sfm_last_error(ctx));
      return;
    }
    for (int32_t f = 0; f < F; ++f)
      if (status[f] == 2) b200host_adapt::SetFrameGravity(*fr[f].second, &g[3 * (size_t)f]);   // .cc:119-123
    std::fprintf(stderr, "Number of rectified frames: %d / %d\n", summary.rectified_frames, summary.error_prone_frames);
  }

 private:
  GravityRefinerOptions options_;
};

// ViewGraph::KeepLargestConnectedComponents (scene/view_graph.cc:56-97) over frames: the frames of the largest component
// of the valid pairs stay registered, every other frame is deregistered and the pairs that leave the component become
// invalid.  Equally large components: the one with the smallest frame id.  Returns the number of images registered.
template <class ViewGraphT, class FrameMap, class ImageMap>
int KeepLargestConnectedComponents(ViewGraphT& view_graph, FrameMap& frames, ImageMap& images) {
  std::map<frame_t, std::vector<frame_t>> adj;
  for (auto& [id, pr] : view_graph.image_pairs) {
    if (!pr.is_valid) continue;
    const auto i1 = images.find(pr.image_id1), i2 = images.find(pr.image_id2);
    if (i1 == images.end() || i2 == images.end()) continue;
    adj[i1->second.frame_id].push_back(i2->second.frame_id);
    adj[i2->second.frame_id].push_back(i1->second.frame_id);
  }
  std::map<frame_t, int> comp;
  std::vector<size_t> size;
  for (auto& [s, _] : adj) {
    if (comp.count(s)) continue;
    const int c = (int)size.size();
    size.push_back(0);
    std::queue<frame_t> q;
    q.push(s);
    comp[s] = c;
    while (!q.empty()) {
      const frame_t u = q.front();
      q.pop();
      ++size[c];
      for (frame_t v : adj[u])
        if (!comp.count(v)) { comp[v] = c; q.push(v); }
    }
  }
  int best = -1;
  for (int c = 0; c < (int)size.size(); ++c)
    if (best < 0 || size[c] > size[best]) best = c;
  for (auto& [id, f] : frames) {
    const auto it = comp.find(id);
    f.is_registered = it != comp.end() && it->second == best;
  }
  for (auto& [id, pr] : view_graph.image_pairs) {
    const auto i1 = images.find(pr.image_id1), i2 = images.find(pr.image_id2);
    if (i1 == images.end() || i2 == images.end()) { pr.is_valid = false; continue; }
    const auto a = comp.find(i1->second.frame_id), b = comp.find(i2->second.frame_id);
    if (a == comp.end() || b == comp.end() || a->second != best || b->second != best) pr.is_valid = false;
  }
  int n = 0;
  for (auto& [id, im] : images) {
    const auto it = comp.find(im.frame_id);
    n += it != comp.end() && it->second == best;
  }
  return n;
}

// SolveRotationAveraging (controllers/rotation_averager.{h,cc}:8-197): with use_gravity and use_stratified, the
// pairs whose two images have gravity are solved first as a 1-DoF problem on their largest component, unless there is
// none or they are more than 95 % of the pairs; then the whole graph.  With a rig whose sensor is not calibrated and
// !skip_initialization, RigRotationPrePass (below) first estimates the cam_from_rig and rig_from_world rotations with
// trivial rigs (.cc:81-175); the solve then starts from them (skip_initialization, .cc:177-182).
struct RotationAveragerOptions : public RotationEstimatorOptions {   // rotation_averager.h:7-12
  RotationAveragerOptions() = default;
  RotationAveragerOptions(const RotationEstimatorOptions& o) : RotationEstimatorOptions(o) {}
  bool use_stratified = true;
};

// The trivial-rig pre-pass of SolveRotationAveraging (.cc:81-175) on flat arrays in sorted-id order (glomap's Rig / Frame
// objects cannot be constructed here):
//   1. the registered images; a camera is known when it is its rig's reference sensor (identity) or has a cam_from_rig
//   2. trivial layout: frame f keeps its images of known cameras, every image of an unknown camera is a frame of its own
//      (.cc:84-158); the valid pairs are folded onto those frames with the known cam_from_rig (R_c2^T R_21 R_c1), pairs
//      inside one trivial frame dropped (global_rotation_averaging.cc:300-303)
//   3. the largest component of the trivial frames (.cc:160): pairs with an image outside it become invalid
//   4. b200sfm_ra_mst_init on the images of that component (InitializeFromMaximumSpanningTree at image level, root = the
//      smallest id) and b200sfm_rig_rotations_from_images for the trivial rigs
//   5. b200sfm_ra_solve on the trivial frames (.cc:162-166), the image rotations composed from it (.cc:169-173), and
//      b200sfm_rig_rotations_from_images for the real rigs (.cc:175)
//   6. write-back: averaged cam_from_rig with a NaN translation through SetCamFromRig, averaged rig_from_world with a NaN
//      translation (rotation_initializer.cc:75-76,85-87,120)
// Weak, so that a host linked against a libb200sfm without these entries (an older build, a test double) still links;
// the pre-pass then reports the missing entry and SolveRotationAveraging returns false.
extern "C" {
int b200sfm_ra_mst_init(b200sfm_ctx* ctx, int32_t n_nodes, int64_t n_edges, const int32_t* ei, const int32_t* ej,
                        const double* R_rel, const double* weight, int32_t root, double* R, int32_t* parent,
                        b200sfm_mst_stats* stats) __attribute__((weak));
int b200sfm_rig_rotations_from_images(b200sfm_ctx* ctx, int64_t n_images, int32_t n_frames, int32_t n_cameras,
                                      const int32_t* image_frame, const int32_t* image_camera,
                                      const uint8_t* image_estimated, const double* cam_from_world,
                                      const int32_t* frame_ref_camera, const uint8_t* camera_known, double* cam_from_rig,
                                      int32_t* cam_samples, double* rig_from_world, int32_t* frame_samples,
                                      b200sfm_rig_init_stats* stats) __attribute__((weak));
}
inline bool RigRotationPrePass(ViewGraph& view_graph, std::unordered_map<rig_t, Rig>& rigs,
                               std::unordered_map<frame_t, Frame>& frames, std::unordered_map<image_t, Image>& images,
                               const RotationEstimatorOptions& options) {
  if (!b200sfm_ra_mst_init || !b200sfm_rig_rotations_from_images) {
    std::fprintf(stderr, "b200sfm: this libb200sfm has no b200sfm_ra_mst_init / b200sfm_rig_rotations_from_images\n");
    return false;
  }
  b200sfm_ctx* ctx = DefaultContext();
  if (!ctx) return false;
  // 1. registered frames, images and cameras in sorted-id order
  const auto fsorted = detail::SortedEntries(frames, [](const Frame& f) { return f.is_registered; });
  const auto fidx = detail::PositionOf(fsorted);
  const auto isorted = detail::SortedEntries(images, [&](const Image& im) { return fidx.count(im.frame_id) != 0; });
  const auto iidx = detail::PositionOf(isorted);
  const int F = (int)fsorted.size(), I = (int)isorted.size();
  if (F == 0 || I == 0) return false;
  auto rig_of = [&](const Frame& f) -> Rig* {
    const auto it = rigs.find(f.RigId());
    return it == rigs.end() ? nullptr : &it->second;
  };
  std::map<camera_t, int> cidx;
  std::map<camera_t, std::pair<rig_t, const Image*>> cam_rig;   // the rig and an image of the camera
  for (auto& [id, im] : isorted) {
    cidx[im->camera_id] = 0;
    cam_rig[im->camera_id] = {frames[im->frame_id].RigId(), im};
  }
  for (auto& [id, f] : fsorted)
    if (Rig* r = rig_of(*f)) cidx[b200host_adapt::RefCameraId(*r)] = 0;
  std::vector<camera_t> cids;
  for (auto& [c, k] : cidx) { k = (int)cids.size(); cids.push_back(c); }
  const int K = (int)cids.size();
  std::vector<uint8_t> known(K, 1);
  std::vector<double> cq(4 * (size_t)K, 0.0), cq_triv;
  for (int c = 0; c < K; ++c) cq[4 * (size_t)c + 3] = 1.0;
  for (auto& [cam, rig_im] : cam_rig) {
    const auto it = rigs.find(rig_im.first);
    if (it == rigs.end()) continue;
    Rigid3d c;
    const auto s = detail::ResolveCamFromRig(&it->second, *rig_im.second, c);
    if (s == detail::CamFromRigStatus::kMissing) known[cidx[cam]] = 0;
    if (s == detail::CamFromRigStatus::kKnown)
      std::copy(c.rotation.coeffs().data(), c.rotation.coeffs().data() + 4, &cq[4 * (size_t)cidx[cam]]);
  }
  cq_triv = cq;   // the trivial rigs: an unknown camera is the reference sensor of its own rig (identity)
  std::vector<int32_t> ref_cam(F), img_frame(I), img_cam(I), tf(I);
  for (int f = 0; f < F; ++f) {
    Rig* r = rig_of(*fsorted[f].second);
    ref_cam[f] = r ? cidx[b200host_adapt::RefCameraId(*r)] : -1;
  }
  std::vector<int32_t> tref(ref_cam);
  for (int i = 0; i < I; ++i) {
    const Image& im = *isorted[i].second;
    img_frame[i] = fidx.at(im.frame_id);
    img_cam[i] = cidx[im.camera_id];
    if (ref_cam[img_frame[i]] < 0) ref_cam[img_frame[i]] = tref[img_frame[i]] = img_cam[i];   // no rig: the first image
    if (known[img_cam[i]]) {
      tf[i] = img_frame[i];
    } else {
      tf[i] = (int)tref.size();
      tref.push_back(img_cam[i]);
    }
  }
  for (int c = 0; c < K; ++c)
    if (!known[c]) { cq_triv[4 * (size_t)c] = cq_triv[4 * (size_t)c + 1] = cq_triv[4 * (size_t)c + 2] = 0; cq_triv[4 * (size_t)c + 3] = 1; }
  const int T = (int)tref.size();
  // 2. valid pairs between registered images, folded onto the trivial frames
  struct P { ImagePair* pr; int a, b; };
  std::vector<P> pairs;
  for (auto& [id, pr] : detail::SortedEntries(view_graph.image_pairs, [](const ImagePair& p) { return p.is_valid; })) {
    const auto a = iidx.find(pr->image_id1), b = iidx.find(pr->image_id2);
    if (a != iidx.end() && b != iidx.end()) pairs.push_back({pr, a->second, b->second});
  }
  // 3. largest component of the trivial frames (equally large: the one with the smallest frame)
  std::vector<int> comp(T, -1), size;
  {
    std::vector<std::vector<int>> adj(T);
    for (const P& p : pairs)
      if (tf[p.a] != tf[p.b]) { adj[tf[p.a]].push_back(tf[p.b]); adj[tf[p.b]].push_back(tf[p.a]); }
    for (int s0 = 0; s0 < T; ++s0) {
      if (comp[s0] >= 0 || adj[s0].empty()) continue;
      const int c = (int)size.size();
      size.push_back(0);
      std::queue<int> q;
      q.push(s0);
      comp[s0] = c;
      while (!q.empty()) {
        const int u = q.front();
        q.pop();
        ++size[c];
        for (int v : adj[u])
          if (comp[v] < 0) { comp[v] = c; q.push(v); }
      }
    }
  }
  if (size.empty()) return false;
  const int best = (int)(std::max_element(size.begin(), size.end()) - size.begin());
  std::vector<uint8_t> in_t(I);
  for (int i = 0; i < I; ++i) in_t[i] = comp[tf[i]] == best;
  std::vector<P> kept;
  for (const P& p : pairs) {
    if (in_t[p.a] && in_t[p.b]) kept.push_back(p);
    else p.pr->is_valid = false;                                                              // .cc:160
  }
  // 4. image-level maximum spanning tree over the images of the component, then the trivial rigs
  std::vector<int> inode(I, -1);
  int n_t = 0;
  for (int i = 0; i < I; ++i)
    if (in_t[i]) inode[i] = n_t++;
  std::vector<int32_t> mi, mj;
  std::vector<double> mR, mw;
  for (const P& p : kept) {
    double R[9];
    detail::QuatToR(p.pr->cam2_from_cam1.rotation.coeffs().data(), R);
    mi.push_back(inode[p.a]); mj.push_back(inode[p.b]);
    mR.insert(mR.end(), R, R + 9);
    mw.push_back((double)p.pr->inliers.size());                                               // tree.cc:93-100 (INLIER_NUM)
  }
  std::vector<double> Rimg(9 * (size_t)n_t, 0.0);
  for (int v = 0; v < n_t; ++v) Rimg[9 * (size_t)v] = Rimg[9 * (size_t)v + 4] = Rimg[9 * (size_t)v + 8] = 1.0;
  std::vector<int32_t> parent(n_t);
  int rc = b200sfm_ra_mst_init(ctx, n_t, (int64_t)mi.size(), mi.data(), mj.data(), mR.data(), mw.data(), 0, Rimg.data(),
                               parent.data(), nullptr);
  if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm_ra_mst_init: %s\n", b200sfm_last_error(ctx)); return false; }
  std::vector<double> qimg(4 * (size_t)I, 0.0), tq(4 * (size_t)T, 0.0), fq(4 * (size_t)F);
  std::vector<int32_t> t_frame(I), cam_n(K), frame_n(F), t_frame_n(T);
  std::vector<uint8_t> est(I, 0), all_known(K, 1);
  for (int i = 0; i < I; ++i) {
    t_frame[i] = in_t[i] ? tf[i] : -1;
    if (in_t[i] && parent[inode[i]] >= 0) {
      est[i] = 1;
      detail::RToQuat(&Rimg[9 * (size_t)inode[i]], &qimg[4 * (size_t)i]);
    } else {
      qimg[4 * (size_t)i + 3] = 1.0;
    }
  }
  for (int t = 0; t < T; ++t) tq[4 * (size_t)t + 3] = 1.0;
  std::vector<double> cq_out(cq_triv);
  rc = b200sfm_rig_rotations_from_images(ctx, I, T, K, t_frame.data(), img_cam.data(), est.data(), qimg.data(), tref.data(),
                                         all_known.data(), cq_out.data(), cam_n.data(), tq.data(), t_frame_n.data(), nullptr);
  if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm_rig_rotations_from_images: %s\n", b200sfm_last_error(ctx)); return false; }
  // 5. rotation averaging of the trivial frames of the component (result status ignored, as in the reference)
  std::vector<int> tnode(T, -1);
  int nT = 0;
  for (int t = 0; t < T; ++t)
    if (comp[t] == best) tnode[t] = nT++;
  std::vector<int32_t> ti, tj;
  std::vector<double> tR, tw, theta(3 * (size_t)nT);
  for (const P& p : kept) {
    if (tf[p.a] == tf[p.b]) continue;
    double Rc1[9], Rc2[9], B[9];
    detail::QuatToR(p.pr->cam2_from_cam1.rotation.coeffs().data(), B);
    detail::QuatToR(&cq_triv[4 * (size_t)img_cam[p.a]], Rc1);
    detail::QuatToR(&cq_triv[4 * (size_t)img_cam[p.b]], Rc2);
    detail::MulAB(B, Rc1, B);    // R21 Rc1
    detail::MulAtB(Rc2, B, B);   // Rc2^T R21 Rc1
    ti.push_back(tnode[tf[p.a]]); tj.push_back(tnode[tf[p.b]]);
    tR.insert(tR.end(), B, B + 9);
    tw.push_back(p.pr->weight);
  }
  for (int t = 0; t < T; ++t)
    if (tnode[t] >= 0) detail::QuatToAngleAxis(&tq[4 * (size_t)t], &theta[3 * (size_t)tnode[t]]);
  const b200sfm_ra_opts o = detail::RaOpts(options);
  b200sfm_ra_stats st{};
  rc = b200sfm_ra_solve(ctx, &o, nT, (int64_t)ti.size(), ti.data(), tj.data(), tR.data(), tw.data(), 0, theta.data(), &st);
  if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm_ra_solve: %s\n", b200sfm_last_error(ctx)); return false; }
  for (int i = 0; i < I; ++i) {   // cam_from_world = cam_from_rig (trivial) * rig_from_world (trivial frame)
    est[i] = in_t[i];
    if (!in_t[i]) continue;
    double qf[4];
    detail::AngleAxisToQuat(&theta[3 * (size_t)tnode[tf[i]]], qf);
    detail::QuatMul(&cq_triv[4 * (size_t)img_cam[i]], qf, &qimg[4 * (size_t)i]);
  }
  // the real rigs
  for (int f = 0; f < F; ++f) {
    const double* c = fsorted[f].second->RigFromWorld().rotation.coeffs().data();
    std::copy(c, c + 4, &fq[4 * (size_t)f]);
  }
  rc = b200sfm_rig_rotations_from_images(ctx, I, F, K, img_frame.data(), img_cam.data(), est.data(), qimg.data(), ref_cam.data(),
                                         known.data(), cq.data(), cam_n.data(), fq.data(), frame_n.data(), nullptr);
  if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm_rig_rotations_from_images: %s\n", b200sfm_last_error(ctx)); return false; }
  // 6. write-back
  const double nan = std::numeric_limits<double>::quiet_NaN();
  for (int c = 0; c < K; ++c) {
    if (known[c] || cam_n[c] == 0) continue;
    Rigid3d pose;
    std::copy(&cq[4 * (size_t)c], &cq[4 * (size_t)c] + 4, pose.rotation.coeffs().data());
    for (int k = 0; k < 3; ++k) pose.translation[k] = nan;
    b200host_adapt::SetCamFromRig(rigs[cam_rig[cids[c]].first], cids[c], pose);
  }
  for (int f = 0; f < F; ++f) {
    if (frame_n[f] == 0) continue;
    Rigid3d& p = fsorted[f].second->RigFromWorld();
    std::copy(&fq[4 * (size_t)f], &fq[4 * (size_t)f] + 4, p.rotation.coeffs().data());
    for (int k = 0; k < 3; ++k) p.translation[k] = nan;
  }
  return true;
}

inline bool SolveRotationAveraging(ViewGraph& view_graph, std::unordered_map<rig_t, Rig>& rigs,
                                   std::unordered_map<frame_t, Frame>& frames, std::unordered_map<image_t, Image>& images,
                                   const RotationAveragerOptions& options) {
  KeepLargestConnectedComponents(view_graph, frames, images);                                 // .cc:13
  auto image_has_gravity = [&](const Image& im) {
    const auto f = frames.find(im.frame_id);
    Rigid3d c;
    return f != frames.end() && f->second.HasGravity() &&
           detail::ResolveCamFromRig(f->second.RigPtr(), im, c) != detail::CamFromRigStatus::kMissing;
  };
  auto registered = [&](const Image& im) {
    const auto f = frames.find(im.frame_id);
    return f != frames.end() && f->second.is_registered;
  };
  bool solve_1dof = options.use_gravity && options.use_stratified;
  ViewGraph view_graph_grav;
  size_t total_pairs = 0;
  if (solve_1dof) {
    for (const auto& [pair_id, pr] : view_graph.image_pairs) {                                 // .cc:22-39
      if (!pr.is_valid) continue;
      const auto i1 = images.find(pr.image_id1), i2 = images.find(pr.image_id2);
      if (i1 == images.end() || i2 == images.end() || !registered(i1->second) || !registered(i2->second)) continue;
      ++total_pairs;
      if (image_has_gravity(i1->second) && image_has_gravity(i2->second)) {
        ImagePair p = pr;
        p.is_valid = true;
        view_graph_grav.image_pairs.emplace(pair_id, p);
      }
    }
  }
  const size_t grav_pairs = view_graph_grav.image_pairs.size();
  std::fprintf(stderr, "Total image pairs: %zu, gravity image pairs: %zu\n", total_pairs, grav_pairs);
  solve_1dof = solve_1dof && !(grav_pairs == 0 || grav_pairs > total_pairs * 0.95);          // .cc:49-50
  if (solve_1dof) {
    KeepLargestConnectedComponents(view_graph_grav, frames, images);                          // .cc:56
    RotationEstimatorOptions o1 = options;
    RotationEstimator est_grav(o1);
    if (!est_grav.EstimateRotations(view_graph_grav, rigs, frames, images)) return false;
    KeepLargestConnectedComponents(view_graph, frames, images);                               // .cc:62
  }
  bool unknown_cams = false;
  for (auto& [rig_id, rig] : rigs) unknown_cams = unknown_cams || !b200host_adapt::AllSensorsCalibrated(rig);
  if (unknown_cams && !options.skip_initialization) {
    if (!RigRotationPrePass(view_graph, rigs, frames, images, options)) return false;
    KeepLargestConnectedComponents(view_graph, frames, images);   // frames whose pairs all left with the trivial component
    RotationEstimatorOptions o = options;
    o.skip_initialization = true;                                                             // .cc:177-181
    RotationEstimator est(o);
    const bool ok = est.EstimateRotations(view_graph, rigs, frames, images);
    KeepLargestConnectedComponents(view_graph, frames, images);                               // .cc:182
    return ok;
  }
  RotationEstimatorOptions o = options;
  if (unknown_cams) o.skip_initialization = false;                                            // .cc:188-190
  RotationEstimator est(o);
  const bool ok = est.EstimateRotations(view_graph, rigs, frames, images);
  KeepLargestConnectedComponents(view_graph, frames, images);                                 // .cc:195
  return ok;
}

// ---------------------------------------------------------------------------
// The processors GlobalMapper::Solve runs between its solvers (controllers/global_mapper.cc:62,155-186,231-337) on the
// device.  Each call stands alone: it flattens the maps in sorted-id order, runs the device and writes back only what the
// reference writes.  A call that fails -- a failed device call, an observation of an unknown image, an image of an unknown
// camera or without a posed frame, a feature outside its image, a rig sensor without cam_from_rig, a camera model outside
// 0-3 where the intrinsics are read -- prints a message on stderr and changes nothing.
namespace detail {

// The tracks' observations as a device problem: trivial frames -> one pose block per image (b200sfm_ba_problem_create),
// otherwise frames plus (rig, camera) sensors (b200sfm_ba_problem_create_rig).  Only the pixel filter reads intrinsics
// (`pixels`); the other filters get one placeholder SIMPLE_PINHOLE block, so that a camera model they never read cannot
// refuse them.  `cameras` null: the filter reads no camera at all (no calibration flag either).
struct FlatTracks {
  bool rig = false;
  int32_t F = 0, S = 0, K = 0, P = 0;
  std::vector<int64_t> ptb{0};
  std::vector<int32_t> obs_frame, cam_intr, sensor_intr, intr_model;
  std::vector<uint16_t> obs_sensor;
  std::vector<double> obs_xy, bearings, quat, trans, sensor_q, sensor_t, intr, points;
  std::vector<uint8_t> calibrated;   // has_prior_focal_length per pose block (trivial frames) or per sensor (rigs)
  int64_t N() const { return (int64_t)obs_frame.size(); }
};

template <class CameraMap, class ImageMap, class TrackPtrs>
bool Flatten(const CameraMap* cameras, const ImageMap& images, const TrackPtrs& tsorted, bool pixels, bool bearings,
             FlatTracks& out) {
  using Img = typename ImageMap::mapped_type;
  auto fail = [](const char* msg) { std::fprintf(stderr, "b200sfm: %s\n", msg); return false; };
  // pass 1: every observation is resolved to a record of its image with one hash lookup; an image is looked up in
  // `images` and checked once, when it is first seen
  struct Rec { image_t id; const Img* im; int32_t block = 0, sensor = 0; };
  std::vector<Rec> recs;
  std::unordered_map<image_t, int32_t> rec_of;
  size_t n_obs = 0;
  for (const auto& [id, t] : tsorted) n_obs += t->observations.size();
  std::vector<int32_t> obs_rec;
  obs_rec.reserve(n_obs);
  for (const auto& [id, t] : tsorted)
    for (const auto& ob : t->observations) {
      auto r = rec_of.find(ob.first);
      if (r == rec_of.end()) {
        auto it = images.find(ob.first);
        if (it == images.end()) return fail("track observation of an unknown image");
        const Img& im = it->second;
        if (!im.frame_ptr || !im.frame_ptr->HasPose()) return fail("image without a posed frame");
        r = rec_of.emplace(ob.first, (int32_t)recs.size()).first;
        recs.push_back(Rec{ob.first, &im});
        out.rig = out.rig || !im.HasTrivialFrame();
      }
      const Img& im = *recs[r->second].im;
      const size_t nf = bearings ? im.features_undist.size() : im.features.size();
      if ((pixels || bearings) && (size_t)ob.second >= nf) return fail("track observation of a feature outside its image");
      obs_rec.push_back(r->second);
    }
  // cameras of the observed images, in sorted camera-id order
  std::set<camera_t> observed;
  if (cameras)
    for (const Rec& r : recs) {
      if (cameras->find(r.im->camera_id) == cameras->end()) return fail("image of an unknown camera");
      observed.insert(r.im->camera_id);
    }
  std::vector<std::pair<camera_t, const typename CameraMap::mapped_type*>> csorted;
  for (camera_t id : observed) csorted.emplace_back(id, &cameras->at(id));
  auto cidx = PositionOf(csorted);
  if (pixels) PackCameras(csorted, out.intr_model, out.intr);
  else PlaceholderCamera(out.intr_model, out.intr);
  out.K = (int32_t)out.intr_model.size();
  auto block = [&](camera_t c) { return pixels ? cidx[c] : 0; };
  auto prior = [&](camera_t c) -> uint8_t { return cameras && cameras->at(c).has_prior_focal_length ? 1 : 0; };
  // pose blocks: the images (trivial frames) or their frames, in sorted id order
  std::map<uint64_t, std::vector<Rec*>> by_block;
  for (Rec& r : recs) by_block[out.rig ? (uint64_t)r.im->frame_id : (uint64_t)r.id].push_back(&r);
  for (auto& [key, rs] : by_block) {
    for (Rec* r : rs) r->block = out.F;
    ++out.F;
    const Img* im = rs.front()->im;
    const auto& pose = im->frame_ptr->RigFromWorld();
    for (int k = 0; k < 4; ++k) out.quat.push_back(pose.rotation.coeffs().data()[k]);
    for (int k = 0; k < 3; ++k) out.trans.push_back(pose.translation[k]);
    if (!out.rig) {
      out.cam_intr.push_back(block(im->camera_id));
      out.calibrated.push_back(prior(im->camera_id));
    }
  }
  // rigs: the (rig, camera) sensors in sorted order; a reference sensor carries the identity
  if (out.rig) {
    std::map<std::pair<rig_t, camera_t>, std::vector<Rec*>> by_sensor;
    for (Rec& r : recs) by_sensor[{r.im->frame_ptr->RigId(), r.im->camera_id}].push_back(&r);
    for (auto& [key, rs] : by_sensor) {
      for (Rec* r : rs) r->sensor = out.S;
      ++out.S;
      const Img* im = rs.front()->im;
      Rigid3d cfr;
      if (ResolveCamFromRig(im->frame_ptr->RigPtr(), *im, cfr) == CamFromRigStatus::kMissing)
        return fail("image of a rig sensor without cam_from_rig");
      for (int k = 0; k < 4; ++k) out.sensor_q.push_back(cfr.rotation.coeffs().data()[k]);
      for (int k = 0; k < 3; ++k) out.sensor_t.push_back(cfr.translation[k]);
      out.sensor_intr.push_back(block(key.second));
      out.calibrated.push_back(prior(key.second));
    }
    if (out.S > 65535) return fail("too many rig sensors");
  }
  // pass 2: observations in track order from their records, points
  out.obs_frame.resize(n_obs);
  if (out.rig) out.obs_sensor.resize(n_obs);
  out.obs_xy.assign(2 * n_obs, 0.0);
  if (bearings) out.bearings.resize(3 * n_obs);
  out.ptb.reserve(tsorted.size() + 1);
  out.points.reserve(3 * tsorted.size());
  size_t o = 0;
  for (const auto& [id, t] : tsorted) {
    for (const auto& ob : t->observations) {
      const Rec& r = recs[obs_rec[o]];
      out.obs_frame[o] = r.block;
      if (out.rig) out.obs_sensor[o] = (uint16_t)r.sensor;
      if (pixels) {
        const auto& xy = r.im->features[ob.second];
        out.obs_xy[2 * o] = xy[0];
        out.obs_xy[2 * o + 1] = xy[1];
      }
      if (bearings) {
        const auto& u = r.im->features_undist[ob.second];
        for (int k = 0; k < 3; ++k) out.bearings[3 * o + k] = u[k];
      }
      ++o;
    }
    out.ptb.push_back((int64_t)o);
    for (int k = 0; k < 3; ++k) out.points.push_back(t->xyz[k]);
    ++out.P;
  }
  return true;
}

// Creates the problem of `f` and loads its state; min_num_view_per_track = 1 keeps every non-empty track in the problem
// (the filters read every observation of every track, whatever its length).
inline int CreateProblem(b200sfm_ctx* ctx, FlatTracks& f, b200sfm_ba_problem** prob) {
  int rc;
  if (f.rig)
    rc = b200sfm_ba_problem_create_rig(ctx, f.F, f.P, f.N(), f.K, f.S, f.ptb.data(), f.obs_frame.data(), f.obs_sensor.data(),
                                       f.obs_xy.data(), f.sensor_q.data(), f.sensor_t.data(), f.sensor_intr.data(),
                                       f.intr_model.data(), nullptr, 1, prob);
  else
    rc = b200sfm_ba_problem_create(ctx, f.F, f.P, f.N(), f.K, f.ptb.data(), f.obs_frame.data(), f.obs_xy.data(), f.cam_intr.data(),
                                   f.intr_model.data(), nullptr, 1, prob);
  if (rc == B200SFM_OK) rc = b200sfm_ba_problem_set_state(*prob, f.intr.data(), f.quat.data(), f.trans.data(), f.points.data());
  return rc;
}

// mode 0: pixel reprojection, 1: angle, 2: triangulation angle, 3: reprojection in the normalised image plane
template <class CameraMap, class ImageMap, class TrackMap>
int RunTrackFilter(int mode, const CameraMap* cameras, const ImageMap& images, TrackMap& tracks, double threshold, const char* name) {
  const auto tsorted = SortedEntries(tracks);
  if (tsorted.empty()) return 0;
  FlatTracks f;
  if (!Flatten(cameras, images, tsorted, mode == 0, mode == 1 || mode == 3, f)) return 0;
  if (f.N() == 0) {   // no observation: nothing changes, except that every track fails the triangulation angle
    if (mode != 2) return 0;
    for (auto& [id, t] : tsorted) t->observations.clear();
    return (int)tsorted.size();
  }
  b200sfm_ctx* ctx = DefaultContext();
  if (!ctx) return 0;
  b200sfm_ba_problem* prob = nullptr;
  int rc = CreateProblem(ctx, f, &prob);
  std::vector<uint8_t> keep(mode == 2 ? (size_t)f.P : (size_t)f.N());
  int64_t n = 0;
  if (rc == B200SFM_OK) {
    if (mode == 0) rc = b200sfm_ba_problem_filter_reprojection(prob, threshold, keep.data(), &n);
    if (mode == 1) rc = b200sfm_ba_problem_filter_angle(prob, f.bearings.data(), f.calibrated.data(), threshold, keep.data(), &n);
    if (mode == 2) rc = b200sfm_ba_problem_filter_triangulation_angle(prob, threshold, keep.data(), &n);
    if (mode == 3) rc = b200sfm_ba_problem_filter_reprojection_normalized(prob, f.bearings.data(), threshold, keep.data(), &n);
  }
  b200sfm_ba_problem_free(prob);
  if (rc != B200SFM_OK) {
    std::fprintf(stderr, "b200sfm: TrackFilter::%s failed: %s\n", name, b200sfm_last_error(ctx));
    return 0;
  }
  int64_t p = 0;
  for (auto& [id, t] : tsorted) {
    if (mode == 2) {
      if (!keep[p]) t->observations.clear();                                                  // track_filter.cc:118-121
    } else {
      const int64_t b = f.ptb[p], e = f.ptb[p + 1];
      if (std::find(keep.begin() + b, keep.begin() + e, 0) != keep.begin() + e) {            // .cc:44-47
        std::vector<std::pair<image_t, feature_t>> kept;
        for (int64_t o = b; o < e; ++o)
          if (keep[o]) kept.emplace_back(t->observations[o - b].first, t->observations[o - b].second);
        t->observations.assign(kept.begin(), kept.end());
      }
    }
    ++p;
  }
  return (int)n;
}

}  // namespace detail

// TrackFilter (processors/track_filter.{h,cc}) on the device: the tracks in sorted track-id order over
// b200sfm_ba_problem_create / _create_rig, then b200sfm_ba_problem_filter_*.  Track::observations are rewritten as the
// reference rewrites them and the number of tracks changed (removed, for the triangulation angle) is returned; 0 and
// nothing changed on failure.
//   FilterTracksByReprojection: in_normalized_image (the mapper's default) reads Image::features_undist
//     (_filter_reprojection_normalized), otherwise the pixels of Image::features and the cameras' intrinsics.
//   FilterTracksByAngle: features_undist, the threshold doubled for a camera without has_prior_focal_length (.cc:61-76).
//   FilterTrackTriangulationAngle: a track without a pair of rays wider than min_angle loses all its observations.
struct TrackFilter {
  template <class ViewGraphT, class CameraMap, class ImageMap, class TrackMap>
  static int FilterTracksByReprojection(const ViewGraphT& view_graph, const CameraMap& cameras, const ImageMap& images,
                                        TrackMap& tracks, double max_reprojection_error = 1e-2, bool in_normalized_image = true) {
    (void)view_graph;
    // the normalised-plane variant reads no camera (track_filter.cc:23-31)
    return detail::RunTrackFilter(in_normalized_image ? 3 : 0, in_normalized_image ? nullptr : &cameras, images, tracks,
                                             max_reprojection_error, "FilterTracksByReprojection");
  }
  template <class ViewGraphT, class CameraMap, class ImageMap, class TrackMap>
  static int FilterTracksByAngle(const ViewGraphT& view_graph, const CameraMap& cameras, const ImageMap& images, TrackMap& tracks,
                                 double max_angle_error = 1.) {
    (void)view_graph;
    return detail::RunTrackFilter(1, &cameras, images, tracks, max_angle_error, "FilterTracksByAngle");
  }
  template <class ViewGraphT, class ImageMap, class TrackMap>
  static int FilterTrackTriangulationAngle(const ViewGraphT& view_graph, const ImageMap& images, TrackMap& tracks,
                                           double min_angle = 1.) {
    (void)view_graph;
    using Cam = std::unordered_map<camera_t, Camera>;
    return detail::RunTrackFilter(2, static_cast<const Cam*>(nullptr), images, tracks, min_angle,
                                             "FilterTrackTriangulationAngle");
  }
};

// UndistortImages (processors/image_undistorter.{h,cc}) on the device (b200sfm_undistort_features): the images in sorted
// id order whose features_undist does not hold one bearing per feature, or all of them with clean_points, have their
// features undistorted through the camera blocks of their cameras (sorted camera-id order) and features_undist replaced.
template <class CameraMap, class ImageMap>
void UndistortImages(CameraMap& cameras, ImageMap& images, bool clean_points) {
  using Img = typename ImageMap::mapped_type;
  const auto todo = detail::SortedEntries(images, [&](const Img& im) {
    return clean_points || im.features_undist.size() != im.features.size();               // image_undistorter.cc:11-16
  });
  if (todo.empty()) return;
  std::set<camera_t> used;
  for (auto& [id, im] : todo) {
    if (cameras.find(im->camera_id) == cameras.end()) { std::fprintf(stderr, "b200sfm: image of an unknown camera\n"); return; }
    used.insert(im->camera_id);
  }
  std::vector<std::pair<camera_t, const typename CameraMap::mapped_type*>> csorted;
  for (camera_t id : used) csorted.emplace_back(id, &cameras.at(id));
  auto cidx = detail::PositionOf(csorted);
  std::vector<int32_t> model, feat_intr;
  std::vector<double> params, xy;
  detail::PackCameras(csorted, model, params);
  for (auto& [id, im] : todo)
    for (const auto& f : im->features) {
      feat_intr.push_back(cidx[im->camera_id]);
      xy.push_back(f[0]);
      xy.push_back(f[1]);
    }
  const int64_t n = (int64_t)feat_intr.size();
  std::vector<double> b(3 * (size_t)n);
  if (n > 0) {
    b200sfm_ctx* ctx = DefaultContext();
    if (!ctx) return;
    const int rc = b200sfm_undistort_features(ctx, (int32_t)model.size(), model.data(), params.data(), n, feat_intr.data(), xy.data(),
                                              b.data());
    if (rc != B200SFM_OK) { std::fprintf(stderr, "b200sfm: UndistortImages failed: %s\n", b200sfm_last_error(ctx)); return; }
  }
  size_t o = 0;
  for (auto& [id, im] : todo) {
    im->features_undist.resize(im->features.size());
    for (auto& u : im->features_undist) {
      for (int k = 0; k < 3; ++k) u[k] = b[3 * o + k];
      ++o;
    }
  }
}

#ifdef B200SFM_SHIM_HAS_SIM3D
// NormalizeReconstruction (processors/reconstruction_normalizer.{h,cc}) on the device (b200sfm_ba_problem_normalize): the
// posed frames in sorted frame-id order as a rig problem -- (rig, camera) sensors, a trivial frame's camera with the
// identity -- whose image table (b200sfm_ba_problem_set_images) is the registered images, so that the robust box and mean
// run over their centres as in the reference.  The similarity moves the frames' translations and the tracks' points;
// every non-reference cam_from_rig translation of every rig is scaled on the host (.cc:70-78).  Returns the similarity;
// the identity and nothing changed on failure, and also without a registered image (the reference indexes an empty
// vector there).  The problem carries the points and one placeholder observation: the normalisation reads no observation.
template <class RigMap, class CameraMap, class FrameMap, class ImageMap, class TrackMap>
b200host_adapt::Sim3d NormalizeReconstruction(RigMap& rigs, CameraMap& cameras, FrameMap& frames, ImageMap& images, TrackMap& tracks,
                                              bool fixed_scale = false, double extent = 10., double p0 = 0.1, double p1 = 0.9) {
  (void)cameras;
  using Frm = typename FrameMap::mapped_type;
  using Img = typename ImageMap::mapped_type;
  const double zero[3] = {0, 0, 0};
  const b200host_adapt::Sim3d identity = b200host_adapt::MakeSim3d(1.0, zero);
  const auto fr = detail::SortedEntries(frames, [](const Frm& f) { return f.HasPose(); });
  const auto fidx = detail::PositionOf(fr);
  std::vector<double> quat, trans;
  for (auto& [id, f] : fr) {
    for (int k = 0; k < 4; ++k) quat.push_back(f->RigFromWorld().rotation.coeffs().data()[k]);
    for (int k = 0; k < 3; ++k) trans.push_back(f->RigFromWorld().translation[k]);
  }
  const auto reg = detail::SortedEntries(images, [](const Img& im) { return im.IsRegistered(); });
  if (reg.empty()) { std::fprintf(stderr, "b200sfm: NormalizeReconstruction without a registered image\n"); return identity; }
  std::map<std::pair<rig_t, camera_t>, int32_t> sidx;
  std::vector<int32_t> image_frame, image_sensor;
  std::vector<double> sensor_q, sensor_t;
  for (auto& [id, im] : reg) {
    const auto f = fidx.find(im->frame_id);
    if (f == fidx.end()) { std::fprintf(stderr, "b200sfm: registered image without a posed frame\n"); return identity; }
    Frm& frame = *fr[f->second].second;
    const auto key = std::make_pair(frame.RigId(), im->camera_id);
    auto s = sidx.find(key);
    if (s == sidx.end()) {
      s = sidx.emplace(key, (int32_t)sidx.size()).first;
      Rigid3d cfr;
      if (detail::ResolveCamFromRig(frame.RigPtr(), *im, cfr) == detail::CamFromRigStatus::kMissing) {
        std::fprintf(stderr, "b200sfm: image of a rig sensor without cam_from_rig\n");
        return identity;
      }
      for (int k = 0; k < 4; ++k) sensor_q.push_back(cfr.rotation.coeffs().data()[k]);
      for (int k = 0; k < 3; ++k) sensor_t.push_back(cfr.translation[k]);
    }
    image_frame.push_back(f->second);
    image_sensor.push_back(s->second);
  }
  const int32_t S = (int32_t)sidx.size();
  if (S > 65535) { std::fprintf(stderr, "b200sfm: too many rig sensors\n"); return identity; }
  const auto tsorted = detail::SortedEntries(tracks);
  const int32_t P = std::max<int32_t>((int32_t)tsorted.size(), 1);
  std::vector<double> points(3 * (size_t)P, 0.0);
  {
    size_t p = 0;
    for (auto& [id, t] : tsorted) { for (int k = 0; k < 3; ++k) points[3 * p + k] = t->xyz[k]; ++p; }
  }
  std::vector<int64_t> ptb(P + 1, 1);
  ptb[0] = 0;   // the placeholder observation belongs to point 0
  const int32_t obs_frame = 0;
  const uint16_t obs_sensor = 0;
  const double obs_xy[2] = {0, 0};
  std::vector<int32_t> intr_model, sensor_intr(S, 0);
  std::vector<double> intr;
  detail::PlaceholderCamera(intr_model, intr);
  b200sfm_ctx* ctx = DefaultContext();
  if (!ctx) return identity;
  b200sfm_ba_problem* prob = nullptr;
  double scale = 1.0, t[3] = {0, 0, 0};
  int rc = b200sfm_ba_problem_create_rig(ctx, (int32_t)fr.size(), P, 1, 1, S, ptb.data(), &obs_frame, &obs_sensor, obs_xy, sensor_q.data(),
                                         sensor_t.data(), sensor_intr.data(), intr_model.data(), nullptr, 1, &prob);
  if (rc == B200SFM_OK) rc = b200sfm_ba_problem_set_state(prob, intr.data(), quat.data(), trans.data(), points.data());
  if (rc == B200SFM_OK) rc = b200sfm_ba_problem_set_images(prob, (int32_t)image_frame.size(), image_frame.data(), image_sensor.data());
  if (rc == B200SFM_OK) rc = b200sfm_ba_problem_normalize(prob, fixed_scale ? 1 : 0, extent, p0, p1, &scale, t);
  if (rc == B200SFM_OK) rc = b200sfm_ba_problem_get_state(prob, nullptr, nullptr, trans.data(), points.data());
  b200sfm_ba_problem_free(prob);
  if (rc != B200SFM_OK) {
    std::fprintf(stderr, "b200sfm: NormalizeReconstruction failed: %s\n", b200sfm_last_error(ctx));
    return identity;
  }
  for (size_t f = 0; f < fr.size(); ++f)                                                       // .cc:64-68
    for (int k = 0; k < 3; ++k) fr[f].second->RigFromWorld().translation[k] = trans[3 * f + k];
  for (auto& [id, rig] : rigs) b200host_adapt::ScaleCamFromRigTranslations(rig, scale);        // .cc:70-78
  size_t p = 0;
  for (auto& [id, tr] : tsorted) { for (int k = 0; k < 3; ++k) tr->xyz[k] = points[3 * p + k]; ++p; }   // .cc:80-82
  return b200host_adapt::MakeSim3d(scale, t);
}
#else
// A glomap build without <colmap/geometry/sim3.h> on its include path: NormalizeReconstruction cannot return
// colmap::Sim3d, and a call says so instead of the function going missing.
template <class RigMap, class... Rest>
void NormalizeReconstruction(RigMap&, Rest&&...) {
  static_assert(sizeof(RigMap) == 0, "b200sfm_shim::NormalizeReconstruction needs <colmap/geometry/sim3.h> on the include path");
}
#endif

}  // namespace b200sfm_shim
