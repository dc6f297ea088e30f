// TEST STUB (tests only, never shipped): colmap::Sim3d as colmap/geometry/sim3.h declares it (scale, rotation,
// translation and the (scale, rotation, translation) constructor), the return type of glomap's NormalizeReconstruction.
#pragma once
#include "../../glomap/scene/types_sfm.h"

namespace colmap {
struct Sim3d {
  double scale = 1;
  Eigen::Quaterniond rotation;
  Eigen::Vector3d translation;
  Sim3d() = default;
  Sim3d(double s, const Eigen::Quaterniond& q, const Eigen::Vector3d& t) : scale(s), rotation(q), translation(t) {}
};
}  // namespace colmap
