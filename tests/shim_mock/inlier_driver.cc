// TEST DRIVER (tests only): ImagePairsInlierCount and the two RelPoseFilter filters of the shim against the recording test
// double (mock_image_pair_inliers.c, which marks every match row k of the call with k % 3 != 1 as an inlier).  The expectations are
// in tests/test_image_pair_inliers_cpu.py.
#include <cstdio>

#include "estimators_shim.h"

using namespace b200sfm_shim;

int main() {
  std::unordered_map<camera_t, Camera> cameras;
  std::unordered_map<image_t, Image> images;
  ViewGraph vg;
  for (camera_t c : {7u, 3u}) {
    Camera cam; cam.camera_id = c; cam.model_id = c == 7 ? 1 : 0;
    cam.params = c == 7 ? std::vector<double>{500.0, 510.0, 320.0, 240.0} : std::vector<double>{600.0, 300.0, 200.0};
    cameras[c] = cam;
  }
  // images 30, 10, 20 with 2, 3, 4 features; image 20 uses camera 7, the others camera 3
  for (image_t i : {30u, 10u, 20u}) {
    Image im; im.image_id = i; im.camera_id = i == 20 ? 7 : 3;
    for (int f = 0; f < (int)(i / 10 + 1); ++f) im.features.push_back({{1.0 * i + f, 2.0 * i - f}});
    images[i] = im;
  }
  // pairs (10,20) CALIBRATED, 5 matches; (30,10) UNCALIBRATED, 3 matches with old inliers; (20,30) PLANAR, 4 matches, invalid
  auto add = [&](image_t a, image_t b, int config, int m, bool valid, std::vector<int> old) {
    ImagePair p; p.image_id1 = a; p.image_id2 = b; p.config = config; p.is_valid = valid; p.inliers = old;
    for (int k = 0; k < 4; ++k) p.cam2_from_cam1.rotation.c[k] = 0.1 * (a + k) + 0.01 * b;
    p.cam2_from_cam1.translation = {{1.0 * a, 1.0 * b, -1.0}};
    for (int k = 0; k < 9; ++k) { p.F.m[k] = a + 0.5 * k; p.H.m[k] = b - 0.25 * k; }
    for (int k = 0; k < m; ++k) p.matches.rows_.push_back({{k % 2, (k + 1) % 2}});
    vg.image_pairs[ImagePairToPairId(a, b)] = p;
  };
  add(10, 20, 2, 5, true, {4});
  add(30, 10, 3, 3, true, {0, 2});
  add(20, 30, 4, 4, false, {1});
  InlierThresholdOptions opt;
  opt.max_epipolar_error_E = 2.0;
  ImagePairsInlierCount(vg, cameras, images, opt, false);   // (30,10) keeps its inliers, (20,30) is cleared, not scored
  ImagePairsInlierCount(vg, cameras, images, opt, true);    // all cleared, the two valid pairs scored
  for (auto key : {ImagePairToPairId(10, 20), ImagePairToPairId(30, 10), ImagePairToPairId(20, 30)}) {
    const ImagePair& p = vg.image_pairs[key];
    std::printf("inliers %u %u", p.image_id1, p.image_id2);
    for (int k : p.inliers) std::printf(" %d", k);
    std::printf("\n");
  }
  RelPoseFilter::FilterInlierNum(vg, 3);       // (10,20): 3 inliers stays, (30,10): 2 inliers -> invalid
  ImagePair empty; empty.image_id1 = 40; empty.image_id2 = 50;
  vg.image_pairs[ImagePairToPairId(40, 50)] = empty;
  RelPoseFilter::FilterInlierRatio(vg, 0.65);  // (10,20): 3/5 -> invalid; (40,50): 0/0 stays valid
  for (auto key : {ImagePairToPairId(10, 20), ImagePairToPairId(30, 10), ImagePairToPairId(20, 30), ImagePairToPairId(40, 50)})
    std::printf("valid %d\n", (int)vg.image_pairs[key].is_valid);
  std::printf("inlier driver ok\n");
  return 0;
}
