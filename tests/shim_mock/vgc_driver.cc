// TEST DRIVER (tests only): the shim's ViewGraphCalibrator against the recording test double
// (mock_view_graph_calibration.c: focal[k] = 1000 + k, camera k accepted when k is even, pair e invalidated when e is
// even).  The expectations are in tests/test_view_graph_calibration_cpu.py.
#include <cstdio>

#include "estimators_shim.h"

using namespace b200sfm_shim;

int main() {
  std::unordered_map<camera_t, Camera> cameras;
  std::unordered_map<image_t, Image> images;
  ViewGraph vg;
  // camera 7 PINHOLE, camera 3 SIMPLE_PINHOLE with a prior focal, camera 9 SIMPLE_RADIAL
  auto cam = [&](camera_t id, int model, std::vector<double> params, bool prior) {
    Camera c; c.camera_id = id; c.model_id = model; c.params = params; c.has_prior_focal_length = prior;
    cameras[id] = c;
  };
  cam(7, 1, {500.0, 510.0, 320.0, 240.0}, false);
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
    vg.image_pairs[ImagePairToPairId(a, b)] = p;
  };
  add(10, 20, 2, true);    // CALIBRATED: cameras 3, 7
  add(30, 10, 3, true);    // UNCALIBRATED, same camera 3
  add(20, 30, 4, true);    // PLANAR: skipped
  add(40, 20, 2, false);   // invalid: skipped (camera 9 has no qualifying pair)
  ViewGraphCalibratorOptions opt;
  opt.thres_two_view_error = 3.0;
  ViewGraphCalibrator calibrator(opt);
  const bool ok = calibrator.Solve(vg, cameras, images);
  std::printf("usable %d\n", (int)ok);
  for (camera_t c : {3u, 7u, 9u}) {
    std::printf("camera %u refined %d params", c, (int)cameras[c].has_refined_focal_length);
    for (double v : cameras[c].params) std::printf(" %.17g", v);
    std::printf("\n");
  }
  for (auto key : {ImagePairToPairId(10, 20), ImagePairToPairId(30, 10), ImagePairToPairId(20, 30), ImagePairToPairId(40, 20)})
    std::printf("valid %d\n", (int)vg.image_pairs[key].is_valid);
  std::printf("vgc driver ok\n");
  return 0;
}
