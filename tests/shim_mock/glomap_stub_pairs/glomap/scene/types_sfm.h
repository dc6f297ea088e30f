// TEST STUB (tests only, never shipped): the glomap stub of tests/shim_mock/glomap_stub with ImagePair as the reference
// declares it (glomap/scene/image_pair.h:13-57: config, E / F / H, cam2_from_cam1, Eigen::MatrixXi matches,
// std::vector<int> inliers) and glomap::InlierThresholdOptions (glomap/types.h:18-32), for type-checking the shim's
// ImagePairsInlierCount / RelPoseFilter branch that is compiled inside a glomap build.
#pragma once
#define ImagePair ImagePairOfTheEstimatorStub_
#define ViewGraph ViewGraphOfTheEstimatorStub_
#include "../../../glomap_stub/glomap/scene/types_sfm.h"
#undef ImagePair
#undef ViewGraph

namespace Eigen {
struct MatrixXi {   // column-major storage, as Eigen's default
  std::vector<int> v;
  long r = 0;
  long rows() const { return r; }
  int operator()(long i, long j) const { return v[j * r + i]; }
};
}  // namespace Eigen

namespace glomap {
struct ImagePair {
  image_t image_id1 = 0, image_id2 = 0;
  bool is_valid = true;
  double weight = -1;
  int config = 0;   // colmap::TwoViewGeometry::ConfigurationType
  Eigen::Matrix3d E, F, H;
  Rigid3d cam2_from_cam1;
  Eigen::MatrixXi matches;
  std::vector<int> inliers;
};
struct ViewGraph {
  std::unordered_map<image_pair_t, ImagePair> image_pairs;
};
struct InlierThresholdOptions {
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
}  // namespace glomap
