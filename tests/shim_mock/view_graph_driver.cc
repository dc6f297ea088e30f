// TEST DRIVER (tests only): the shim's RelPoseFilter::FilterRotations and KeepLargestConnectedComponentsDevice against the
// recording test double (mock_view_graph.c: the filter invalidates the pairs at odd indices; the component pass keeps
// every frame but the last, invalidates the pair at index 0 and returns 100 + num_images).  The expectations are in
// tests/test_view_graph_cpu.py.
#include <cstdio>

#include "estimators_shim.h"

using namespace b200sfm_shim;

int main() {
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  ViewGraph vg;
  Rig rig;
  rig.ref_camera_id = 1;
  rig.cam_from_rig[2].rotation.c[2] = 0.6;   // camera 2: (0, 0, 0.6, 0.8) from the rig
  rig.cam_from_rig[2].rotation.c[3] = 0.8;
  // frames 30, 10, 20 (sorted: 10 -> 0, 20 -> 1, 30 -> 2); frame 20 holds the rig's images 201 (reference) and 202
  for (frame_t f : {30u, 10u, 20u}) {
    Frame fr;
    fr.frame_id = f;
    fr.is_registered = f != 30;
    frames[f] = fr;
  }
  frames[10].rig_from_world.rotation.c[0] = 0.6;
  frames[10].rig_from_world.rotation.c[3] = 0.8;
  frames[20].rig_from_world.rotation.c[1] = 0.6;
  frames[20].rig_from_world.rotation.c[3] = 0.8;
  frames[20].rig_ptr = &rig;
  struct Spec { image_t id; camera_t cam; frame_t frame; bool trivial; };
  for (const Spec& s : std::vector<Spec>{{301, 7, 30, true}, {202, 2, 20, false}, {101, 5, 10, true}, {201, 1, 20, false}}) {
    Image im;
    im.image_id = s.id;
    im.camera_id = s.cam;
    im.frame_id = s.frame;
    im.trivial_frame = s.trivial;
    images[s.id] = im;
  }
  for (auto& [id, im] : images) im.frame_ptr = &frames[im.frame_id];
  auto pair = [&](image_t a, image_t b, double marker, bool valid) {
    ImagePair p;
    p.image_id1 = a;
    p.image_id2 = b;
    p.is_valid = valid;
    p.cam2_from_cam1.rotation.c[0] = marker;
    vg.image_pairs[ImagePairToPairId(a, b)] = p;
  };
  pair(201, 202, 0.4, true);
  pair(201, 301, 0.5, false);
  pair(101, 301, 0.3, true);
  pair(202, 101, 0.2, true);
  pair(101, 201, 0.1, true);
  const int64_t cut = RelPoseFilter::FilterRotations(vg, images, 5.0);
  std::printf("filtered %lld\n", (long long)cut);
  const int n = KeepLargestConnectedComponentsDevice(vg, frames, images);
  std::printf("registered images %d\n", n);
  for (frame_t f : {10u, 20u, 30u}) std::printf("frame %u registered %d\n", f, (int)frames[f].is_registered);
  for (auto [a, b] : std::vector<std::pair<image_t, image_t>>{{101, 201}, {101, 202}, {101, 301}, {201, 202}, {201, 301}})
    std::printf("pair %u %u valid %d\n", a, b, (int)vg.image_pairs[ImagePairToPairId(a, b)].is_valid);
  std::printf("view graph driver ok\n");
  return 0;
}
