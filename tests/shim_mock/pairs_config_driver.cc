// TEST DRIVER (tests only): the shim's ViewGraphManipulater::UpdateImagePairsConfig against the recording test double
// (mock_pairs_config.c: every UNCALIBRATED pair e promoted, F[e][k] = 100 * e + k).  The expectations are in
// tests/test_view_graph_manipulation_cpu.py.
#include <cstdio>

#include "estimators_shim.h"

using namespace b200sfm_shim;

int main() {
  std::unordered_map<camera_t, Camera> cameras;
  std::unordered_map<image_t, Image> images;
  ViewGraph vg;
  // camera 7 PINHOLE and camera 3 SIMPLE_PINHOLE with a prior focal, camera 9 SIMPLE_RADIAL without
  auto cam = [&](camera_t id, int model, std::vector<double> params, bool prior) {
    Camera c; c.camera_id = id; c.model_id = model; c.params = params; c.has_prior_focal_length = prior;
    cameras[id] = c;
  };
  cam(7, 1, {500.0, 510.0, 320.0, 240.0}, true);
  cam(3, 0, {600.0, 300.0, 200.0}, true);
  cam(9, 2, {700.0, 350.0, 250.0, 0.01}, false);
  // images 10, 30 -> camera 3; 20 -> camera 7; 40 -> camera 9
  for (auto [i, c] : std::vector<std::pair<image_t, camera_t>>{{10, 3}, {30, 3}, {20, 7}, {40, 9}}) {
    Image im; im.image_id = i; im.camera_id = c;
    images[i] = im;
  }
  auto add = [&](image_t a, image_t b, int config, bool valid) {
    ImagePair p; p.image_id1 = a; p.image_id2 = b; p.config = config; p.is_valid = valid;
    for (int k = 0; k < 9; ++k) p.F.m[k] = a + 0.5 * k + 0.01 * b;
    double q[4] = {0.1, 0.2, 0.3, 0.9};
    for (int k = 0; k < 4; ++k) p.cam2_from_cam1.rotation.coeffs().data()[k] = q[k];
    p.cam2_from_cam1.translation = {{(double)a, (double)b, 0.5}};
    vg.image_pairs[ImagePairToPairId(a, b)] = p;
  };
  add(10, 20, 2, true);    // CALIBRATED: cameras 3, 7
  add(30, 10, 3, true);    // UNCALIBRATED, same camera 3
  add(20, 30, 3, true);    // UNCALIBRATED: cameras 7, 3
  add(40, 20, 2, false);   // invalid CALIBRATED: passed with its validity
  const int64_t n = ViewGraphManipulater::UpdateImagePairsConfig(vg, cameras, images);
  std::printf("promoted %lld\n", (long long)n);
  const image_pair_t keys[4] = {ImagePairToPairId(10, 20), ImagePairToPairId(30, 10), ImagePairToPairId(20, 30),
                                ImagePairToPairId(40, 20)};
  for (auto key : keys) std::printf("config %d\n", vg.image_pairs[key].config);
  for (int e = 0; e < 3; ++e) {
    std::printf("F");
    for (int k = 0; k < 9; ++k) std::printf(" %.17g", vg.image_pairs[keys[e]].F(k / 3, k % 3));
    std::printf("\n");
  }
  std::printf("pairs config driver ok\n");
  return 0;
}
