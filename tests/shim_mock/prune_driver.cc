// TEST DRIVER (tests only): the shim's PruneWeaklyConnectedImages against the recording test double (mock_prune.c:
// frame index f gets cluster f % 3 and stays registered, except f % 3 == 2: -1, deregistered).  The expectations are in
// tests/test_reconstruction_pruning_cpu.py.
#include <cstdio>

#include "estimators_shim.h"

using namespace b200sfm_shim;

int main() {
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  std::unordered_map<track_t, Track> tracks;
  // frames 30, 10, 20 (sorted: 10 -> 0, 20 -> 1, 30 -> 2); frame 20 is a rig frame with images 201 and 202
  for (frame_t f : {30u, 10u, 20u}) {
    Frame fr; fr.frame_id = f; fr.is_registered = f != 30;
    frames[f] = fr;
  }
  for (auto [i, f] : std::vector<std::pair<image_t, frame_t>>{{101, 10}, {201, 20}, {202, 20}, {301, 30}}) {
    Image im; im.image_id = i; im.frame_id = f;
    images[i] = im;
  }
  auto track = [&](track_t id, std::vector<image_t> ims) {
    Track t; t.track_id = id;
    for (image_t i : ims) t.observations.push_back({i, 0});
    tracks[id] = t;
  };
  track(7, {301, 101, 202});
  track(3, {201, 202});
  track(5, {101, 301, 201, 101});
  const image_t n = PruneWeaklyConnectedImages(frames, images, tracks, 2, 4);
  std::printf("clusters %u\n", n);
  for (frame_t f : {10u, 20u, 30u}) std::printf("frame %u registered %d cluster %d\n", f, (int)frames[f].is_registered, frames[f].cluster_id);
  std::printf("prune driver ok\n");
  return 0;
}
