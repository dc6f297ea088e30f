// TEST DRIVER (tests only): the shim's GravityRefiner and KeepLargestConnectedComponents against the recording test
// double (mock_gravity.c: frame index f with gravity gets status 2 and gravity (0, 1, f) when f is even).  The
// expectations are in tests/test_rotation_averager_cpu.py.
#include <cstdio>

#include "estimators_shim.h"

using namespace b200sfm_shim;

int main() {
  std::unordered_map<rig_t, Rig> rigs;
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  ViewGraph vg;
  // rig 1: reference camera 1, camera 2 at a known cam_from_rig (90 deg about z), camera 3 not calibrated
  Rig& rig = rigs[1];
  rig.rig_id = 1; rig.ref_camera_id = 1;
  rig.cam_from_rig[2].rotation.c[2] = std::sqrt(0.5); rig.cam_from_rig[2].rotation.c[3] = std::sqrt(0.5);
  rig.uncalibrated.push_back(3);
  // frames 30, 10, 20, 40 (sorted: 10 -> 0, 20 -> 1, 30 -> 2, 40 -> 3); 40 has no gravity
  for (frame_t f : {30u, 10u, 20u, 40u}) {
    Frame fr; fr.frame_id = f; fr.rig_id = 1; fr.rig_ptr = &rigs[1];
    if (f != 40) fr.gravity_info.SetGravity({{0.1 * f, 1.0, -0.02 * f}});
    frames[f] = fr;
  }
  // images: 101 (frame 10), 201 / 202 / 203 (frame 20: cameras 1, 2, 3), 301 (frame 30), 401 (frame 40)
  for (auto [i, f, c] : std::vector<std::array<uint32_t, 3>>{{101, 10, 1}, {201, 20, 1}, {202, 20, 2}, {203, 20, 3},
                                                             {301, 30, 1}, {401, 40, 1}}) {
    Image im; im.image_id = i; im.frame_id = f; im.camera_id = c; im.trivial_frame = c == 1;
    images[i] = im;
  }
  auto pair = [&](image_t a, image_t b, double qz, bool valid) {
    ImagePair p; p.image_id1 = a; p.image_id2 = b; p.is_valid = valid;
    p.cam2_from_cam1.rotation.c[2] = qz; p.cam2_from_cam1.rotation.c[3] = std::sqrt(1 - qz * qz);
    vg.image_pairs[ImagePairToPairId(a, b)] = p;
  };
  pair(301, 101, 0.1, true);    // trivial - trivial
  pair(101, 202, 0.2, true);    // into the rig camera 2
  pair(201, 202, 0.3, true);    // inside frame 20
  pair(203, 101, 0.4, true);    // uncalibrated camera 3: no gravity, skipped
  pair(101, 401, 0.5, true);    // frame 40 has no gravity: skipped
  pair(202, 301, 0.6, false);   // invalid: skipped
  GravityRefinerOptions o;
  o.max_gravity_error = 2.5;
  GravityRefiner(o).RefineGravity(vg, frames, images);
  for (frame_t f : {10u, 20u, 30u, 40u}) {
    const auto& gi = frames[f].gravity_info;
    std::printf("frame %u gravity %d %.17g %.17g %.17g\n", f, (int)gi.has_gravity, gi.gravity_in_rig[0], gi.gravity_in_rig[1],
                gi.gravity_in_rig[2]);
  }
  // frames 10, 30 joined; 20 joined to 10 through a valid pair; 40 too -> one component; drop pair 101-401
  vg.image_pairs[ImagePairToPairId(101, 401)].is_valid = false;
  vg.image_pairs[ImagePairToPairId(203, 101)].is_valid = false;
  const int n = KeepLargestConnectedComponents(vg, frames, images);
  std::printf("lcc images %d registered", n);
  for (frame_t f : {10u, 20u, 30u, 40u}) std::printf(" %d", (int)frames[f].is_registered);
  std::printf("\ngravity driver ok\n");
  return 0;
}
