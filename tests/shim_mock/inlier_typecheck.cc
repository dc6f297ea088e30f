// TEST (tests only): the image-pair functions of the shim in their -DB200SFM_WITH_GLOMAP form, instantiated with the
// glomap types of tests/shim_mock/glomap_stub_pairs and glomap's own InlierThresholdOptions -- compiled with -fsyntax-only
// by tests/test_image_pair_inliers_cpu.py.
#include "estimators_shim.h"

void Run(glomap::ViewGraph& vg, const std::unordered_map<glomap::camera_t, glomap::Camera>& cameras,
         const std::unordered_map<glomap::image_t, glomap::Image>& images) {
  const glomap::InlierThresholdOptions options;
  b200sfm_shim::ImagePairsInlierCount(vg, cameras, images, options, true);
  b200sfm_shim::RelPoseFilter::FilterInlierNum(vg, (int)options.min_inlier_num);
  b200sfm_shim::RelPoseFilter::FilterInlierRatio(vg, options.min_inlier_ratio);
}
