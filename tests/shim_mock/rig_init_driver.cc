// TEST DRIVER (tests only): the shim's SolveRotationAveraging with a rig whose camera 3 has no cam_from_rig yet, over the
// recording test doubles (mock_b200sfm.c, mock_rig_init.c).  The expectations are in tests/test_rig_rotation_init_cpu.py.
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
  for (frame_t f : {30u, 10u, 20u}) {
    Frame fr; fr.frame_id = f; fr.rig_id = 1; fr.rig_ptr = &rigs[1];
    frames[f] = fr;
  }
  // images 11 12 13 / 21 22 23 / 31 32: frame 10 * (id / 10), camera id % 10
  for (image_t i : {11u, 12u, 13u, 21u, 22u, 23u, 31u, 32u}) {
    Image im; im.image_id = i; im.frame_id = 10 * (i / 10); im.camera_id = i % 10; im.trivial_frame = im.camera_id == 1;
    im.frame_ptr = &frames[im.frame_id];
    images[i] = im;
  }
  int k = 0;
  for (auto [a, b] : std::vector<std::array<image_t, 2>>{{11, 12}, {11, 13}, {11, 21}, {21, 22}, {21, 23}, {21, 31}, {31, 32}}) {
    ImagePair p; p.image_id1 = a; p.image_id2 = b; p.weight = 1.0 + k;
    p.inliers.resize(10 + k);
    const double qz = 0.05 * (k + 1);
    p.cam2_from_cam1.rotation.c[2] = qz; p.cam2_from_cam1.rotation.c[3] = std::sqrt(1 - qz * qz);
    vg.image_pairs[ImagePairToPairId(a, b)] = p;
    ++k;
  }
  RotationAveragerOptions o;
  const bool ok = SolveRotationAveraging(vg, rigs, frames, images, o);
  const Rigid3d c3 = rigs[1].cam_from_rig[3];
  std::printf("ok %d\ncam3 %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", (int)ok, c3.rotation.c[0], c3.rotation.c[1],
              c3.rotation.c[2], c3.rotation.c[3], c3.translation[0], c3.translation[1], c3.translation[2]);
  std::printf("registered %d %d %d\n", (int)frames[10].is_registered, (int)frames[20].is_registered, (int)frames[30].is_registered);
  std::printf("rig init driver %s\n", ok ? "ok" : "failed");
  return ok ? 0 : 1;
}
