// scene_min.h -- minimal stand-ins for the glomap / COLMAP scene types the
// estimator shim touches (the real ones need COLMAP + Eigen, absent here).
// Field and accessor names follow the reference so that estimators_shim.h
// compiles unchanged against either:
//   glomap/scene/image.h:10-45, frame.h:11-27, track.h:12-24, camera.h:12,
//   image_pair.h:13-40, view_graph.h:12, types.h:32-40; colmap Rigid3d and Sim3d.
// Define B200SFM_WITH_GLOMAP to use the real headers instead.
#pragma once
#ifdef B200SFM_WITH_GLOMAP
#include "glomap/scene/types_sfm.h"
namespace b200host = glomap;
namespace b200host_adapt {
// cam_from_rig of a camera of a rig (colmap::Rig::SensorFromRig)
inline glomap::Rigid3d CamFromRig(glomap::Rig& rig, glomap::camera_t camera_id) {
  return rig.SensorFromRig(glomap::sensor_t(glomap::SensorType::CAMERA, camera_id));
}
// optimised cam_from_rig back into the rig (bundle_adjustment.cc:162-166 takes the same mutable reference)
inline void SetCamFromRig(glomap::Rig& rig, glomap::camera_t camera_id, const glomap::Rigid3d& pose) {
  rig.SensorFromRig(glomap::sensor_t(glomap::SensorType::CAMERA, camera_id)) = pose;
}
inline bool AllSensorsCalibrated(const glomap::Rig& rig) {
  for (const auto& [sensor_id, sensor] : rig.NonRefSensors())
    if (!sensor.has_value()) return false;
  return true;
}
inline bool IsRefSensor(const glomap::Rig& rig, glomap::camera_t camera_id) { return rig.RefSensorId().id == camera_id; }
inline glomap::camera_t RefCameraId(const glomap::Rig& rig) { return rig.RefSensorId().id; }
inline bool HasCamFromRig(const glomap::Rig& rig, glomap::camera_t camera_id) {
  return rig.MaybeSensorFromRig(glomap::sensor_t(glomap::SensorType::CAMERA, camera_id)).has_value();
}
// GravityInfo::GetRAlign() (scene/frame.h:16) as row-major doubles
inline void RAlignRowMajor(const glomap::Frame& f, double out[9]) {
  const Eigen::Matrix3d& R = f.gravity_info.GetRAlign();
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) out[3 * r + c] = R(r, c);
}
// cam_from_rig rotation (quaternion xyzw) of a non-reference camera through the frame's rig pointer; false when unknown
inline bool FrameCamFromRig(const glomap::Frame& f, glomap::camera_t camera_id, double q[4]) {
  if (!f.RigPtr()) return false;
  const auto& c = f.RigPtr()->MaybeSensorFromRig(glomap::sensor_t(glomap::SensorType::CAMERA, camera_id));
  if (!c.has_value()) return false;
  for (int k = 0; k < 4; ++k) q[k] = c->rotation.coeffs().data()[k];
  return true;
}
// GravityInfo::SetGravity (scene/frame.h:46-50): gravity and R_align = GetAlignRot(g).  A template, so that it is
// compiled only where a refiner writes gravity back.
template <class FrameT>
inline void SetFrameGravity(FrameT& f, const double g[3]) {
  Eigen::Vector3d v;
  for (int k = 0; k < 3; ++k) v[k] = g[k];
  f.gravity_info.SetGravity(v);
}
// NormalizeReconstruction (reconstruction_normalizer.cc:70-78): every non-reference sensor_from_rig translation of the rig
// times `scale`.  A template, so that it is compiled only where the normaliser is.
template <class RigT>
inline void ScaleCamFromRigTranslations(RigT& rig, double scale) {
  for (auto& [sensor_id, sensor_from_rig_opt] : rig.NonRefSensors()) {
    if (!sensor_from_rig_opt.has_value()) continue;
    auto sensor_from_rig = sensor_from_rig_opt.value();
    for (int k = 0; k < 3; ++k) sensor_from_rig.translation[k] *= scale;
    rig.SetSensorFromRig(sensor_id, sensor_from_rig);
  }
}
}  // namespace b200host_adapt
// colmap::Sim3d, the return type of NormalizeReconstruction, where the COLMAP build provides it
#if __has_include(<colmap/geometry/sim3.h>)
#include <colmap/geometry/sim3.h>
#define B200SFM_SHIM_HAS_SIM3D 1
namespace b200host_adapt {
using Sim3d = colmap::Sim3d;
// the similarity X' = scale X + t with the identity rotation
inline Sim3d MakeSim3d(double scale, const double t[3]) {
  Eigen::Quaterniond q;
  double* c = q.coeffs().data();
  c[0] = c[1] = c[2] = 0.0;
  c[3] = 1.0;
  Eigen::Vector3d v;
  for (int k = 0; k < 3; ++k) v[k] = t[k];
  return Sim3d(scale, q, v);
}
}  // namespace b200host_adapt
#endif
#else
#include <map>
#include <array>
#include <cmath>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace b200host {

using image_t = uint32_t;
using camera_t = uint32_t;
using frame_t = uint32_t;
using rig_t = uint32_t;
using track_t = uint64_t;
using image_pair_t = uint64_t;
using feature_t = uint32_t;

struct Quaternion {   // Eigen::Quaterniond: coeffs() is (x, y, z, w); the shim only uses coeffs().data()
  double c[4] = {0, 0, 0, 1};
  struct Coeffs { double* p; double* data() const { return p; } };
  struct ConstCoeffs { const double* p; const double* data() const { return p; } };
  Coeffs coeffs() { return Coeffs{c}; }
  ConstCoeffs coeffs() const { return ConstCoeffs{c}; }
};
struct Rigid3d {
  Quaternion rotation;
  std::array<double, 3> translation{{0, 0, 0}};
};
struct Sim3d {   // colmap::Sim3d: X' = scale * rotation * X + translation (NormalizeReconstruction's return value)
  double scale = 1;
  Quaternion rotation;
  std::array<double, 3> translation{{0, 0, 0}};
};
struct Camera {
  camera_t camera_id = 0;
  int model_id = 0;                  // colmap::CameraModelId
  std::vector<double> params;
  bool has_prior_focal_length = true;
  bool has_refined_focal_length = false;   // set by ViewGraphCalibrator
};
struct Rig {   // colmap::Rig: one reference sensor (identity) + non-reference sensors, calibrated (cam_from_rig) or not yet
  rig_t rig_id = 0;
  camera_t ref_camera_id = 0;                    // RefSensorId().id
  std::map<camera_t, Rigid3d> cam_from_rig;      // calibrated non-reference sensors (MaybeSensorFromRig has a value)
  std::vector<camera_t> uncalibrated;            // non-reference sensors without a cam_from_rig yet
  Rigid3d SensorFromRig(camera_t camera_id) const {
    auto it = cam_from_rig.find(camera_id);
    return it == cam_from_rig.end() ? Rigid3d{} : it->second;
  }
};
struct GravityInfo {   // scene/frame.h:11-27
  bool has_gravity = false;
  double R_align[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};   // row-major; second COLUMN = gravity direction
  std::array<double, 3> gravity_in_rig{{0, 0, 0}};
  // GetAlignRot (math/gravity.cc:11-24): any right-handed orthonormal completion of the gravity direction (the
  // reference takes the Householder one; the 1-DoF angle about gravity absorbs the choice)
  void SetGravity(const std::array<double, 3>& g) {
    gravity_in_rig = g;
    const double n = std::sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
    const double v[3] = {g[0] / n, g[1] / n, g[2] / n};
    const double a[3] = {std::fabs(v[0]) < 0.9 ? 1.0 : 0.0, 0.0, std::fabs(v[0]) < 0.9 ? 0.0 : 1.0};
    double x[3] = {v[1] * a[2] - v[2] * a[1], v[2] * a[0] - v[0] * a[2], v[0] * a[1] - v[1] * a[0]};
    const double xn = std::sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    for (double& e : x) e /= xn;
    const double z[3] = {x[1] * v[2] - x[2] * v[1], x[2] * v[0] - x[0] * v[2], x[0] * v[1] - x[1] * v[0]};
    for (int r = 0; r < 3; ++r) { R_align[3 * r] = x[r]; R_align[3 * r + 1] = v[r]; R_align[3 * r + 2] = z[r]; }
    has_gravity = true;
  }
};
struct Frame {
  frame_t frame_id = 0;
  GravityInfo gravity_info;
  bool HasGravity() const { return gravity_info.has_gravity; }
  rig_t rig_id = 0;
  rig_t RigId() const { return rig_id; }
  bool is_registered = true;
  int cluster_id = -1;                 // set by PruneWeaklyConnectedImages
  struct Rig* rig_ptr = nullptr;       // colmap::Frame::RigPtr()
  struct Rig* RigPtr() const { return rig_ptr; }
  Rigid3d rig_from_world;
  Rigid3d& RigFromWorld() { return rig_from_world; }
  const Rigid3d& RigFromWorld() const { return rig_from_world; }
  bool HasPose() const { return true; }
};
struct Image {
  image_t image_id = 0;
  camera_t camera_id = 0;
  frame_t frame_id = 0;
  std::string file_name;
  Frame* frame_ptr = nullptr;
  std::vector<std::array<double, 2>> features;          // distorted pixels (scene/image.h:29)
  std::vector<std::array<double, 3>> features_undist;   // unit bearings (scene/image.h:31)
  bool trivial_frame = true;                            // false: the frame holds several images of a rig
  bool IsRegistered() const { return frame_ptr && frame_ptr->is_registered; }
  bool HasTrivialFrame() const { return trivial_frame; }
};
struct Track {
  track_t track_id = 0;
  std::array<double, 3> xyz{{0, 0, 0}};
  std::vector<std::pair<image_t, feature_t>> observations;
  bool is_initialized = false;
};
struct Matrix3 {   // Eigen::Matrix3d: the shim reads and writes M(r, c)
  double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  double operator()(int r, int c) const { return m[3 * r + c]; }
  double& operator()(int r, int c) { return m[3 * r + c]; }
};
struct MatchMatrix {   // Eigen::MatrixXi with two columns: (k, 0) feature in image 1, (k, 1) feature in image 2
  std::vector<std::array<int, 2>> rows_;
  long rows() const { return (long)rows_.size(); }
  int operator()(long r, int c) const { return rows_[r][c]; }
};
struct ImagePair {
  image_t image_id1 = 0, image_id2 = 0;
  bool is_valid = true;
  double weight = -1;
  std::vector<int> inliers;                      // scene/image_pair.h: indices of the inlier matches
  Rigid3d cam2_from_cam1;
  int config = 0;                                // colmap::TwoViewGeometry::ConfigurationType
  Matrix3 F, H;
  MatchMatrix matches;
};
struct ViewGraph {
  std::unordered_map<image_pair_t, ImagePair> image_pairs;
};
inline image_pair_t ImagePairToPairId(image_t a, image_t b) {   // colmap::ImagePairToPairId
  if (a > b) std::swap(a, b);
  return (image_pair_t)a * 2147483647ull + b;
}

}  // namespace b200host
namespace b200host_adapt {
inline b200host::Rigid3d CamFromRig(b200host::Rig& rig, b200host::camera_t camera_id) { return rig.SensorFromRig(camera_id); }
inline void SetCamFromRig(b200host::Rig& rig, b200host::camera_t camera_id, const b200host::Rigid3d& pose) {
  rig.cam_from_rig[camera_id] = pose;
}
// every non-reference sensor of the rig has a cam_from_rig (global_rotation_averaging.cc:47-59)
inline bool AllSensorsCalibrated(const b200host::Rig& rig) { return rig.uncalibrated.empty(); }
inline bool IsRefSensor(const b200host::Rig& rig, b200host::camera_t camera_id) { return camera_id == rig.ref_camera_id; }
inline b200host::camera_t RefCameraId(const b200host::Rig& rig) { return rig.ref_camera_id; }
inline bool HasCamFromRig(const b200host::Rig& rig, b200host::camera_t camera_id) { return rig.cam_from_rig.count(camera_id) != 0; }
inline void RAlignRowMajor(const b200host::Frame& f, double out[9]) {
  for (int k = 0; k < 9; ++k) out[k] = f.gravity_info.R_align[k];
}
inline bool FrameCamFromRig(const b200host::Frame& f, b200host::camera_t camera_id, double q[4]) {
  if (!f.RigPtr() || !HasCamFromRig(*f.RigPtr(), camera_id)) return false;
  const b200host::Rigid3d c = f.RigPtr()->SensorFromRig(camera_id);
  for (int k = 0; k < 4; ++k) q[k] = c.rotation.c[k];
  return true;
}
inline void SetFrameGravity(b200host::Frame& f, const double g[3]) { f.gravity_info.SetGravity({{g[0], g[1], g[2]}}); }
inline void ScaleCamFromRigTranslations(b200host::Rig& rig, double scale) {
  for (auto& [camera_id, pose] : rig.cam_from_rig)
    for (double& v : pose.translation) v *= scale;
}
#define B200SFM_SHIM_HAS_SIM3D 1
using Sim3d = b200host::Sim3d;
inline Sim3d MakeSim3d(double scale, const double t[3]) {
  Sim3d s;
  s.scale = scale;
  s.translation = {{t[0], t[1], t[2]}};
  return s;
}
}  // namespace b200host_adapt
#endif
