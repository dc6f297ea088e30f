// TEST (tests only): a glomap build whose include path lacks <colmap/geometry/sim3.h> (the stub of
// tests/shim_mock/glomap_stub has none).  The shim still declares NormalizeReconstruction, and calling it fails with the
// shim's static_assert naming the missing header -- tests/test_shim_processors_cpu.py expects that compile error.
#include "estimators_shim.h"

void Run(std::unordered_map<glomap::rig_t, glomap::Rig>& rigs, std::unordered_map<glomap::camera_t, glomap::Camera>& cameras,
         std::unordered_map<glomap::frame_t, glomap::Frame>& frames, std::unordered_map<glomap::image_t, glomap::Image>& images,
         std::unordered_map<glomap::track_t, glomap::Track>& tracks) {
  using b200sfm_shim::NormalizeReconstruction;
  NormalizeReconstruction(rigs, cameras, frames, images, tracks);
}
