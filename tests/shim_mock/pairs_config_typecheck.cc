// TEST (tests only): the shim's ViewGraphManipulater::UpdateImagePairsConfig in its -DB200SFM_WITH_GLOMAP form,
// instantiated with the glomap Camera and Image of tests/shim_mock/glomap_stub_vgc and an ImagePair whose F is written
// through F(r, c) as Eigen::Matrix3d allows (glomap/scene/image_pair.h:13-57: int config, Eigen::Matrix3d F, Rigid3d
// cam2_from_cam1) -- compiled with -fsyntax-only by tests/test_view_graph_manipulation_cpu.py.
#include "estimators_shim.h"

namespace pairs_config_stub {
struct Matrix3d {   // Eigen::Matrix3d: M(r, c) reads and writes
  double m[9] = {};
  double operator()(int r, int c) const { return m[3 * r + c]; }
  double& operator()(int r, int c) { return m[3 * r + c]; }
};
struct ImagePair {
  glomap::image_t image_id1 = 0, image_id2 = 0;
  bool is_valid = true;
  int config = 0;
  Matrix3d F;
  glomap::Rigid3d cam2_from_cam1;
};
struct ViewGraph {
  std::unordered_map<glomap::image_pair_t, ImagePair> image_pairs;
};
}  // namespace pairs_config_stub

int64_t Run(pairs_config_stub::ViewGraph& vg, const std::unordered_map<glomap::camera_t, glomap::Camera>& cameras,
            const std::unordered_map<glomap::image_t, glomap::Image>& images) {
  return b200sfm_shim::ViewGraphManipulater::UpdateImagePairsConfig(vg, cameras, images);
}
