// TEST (tests only): the shim's TrackFilter, UndistortImages and NormalizeReconstruction in their -DB200SFM_WITH_GLOMAP
// form, instantiated with the glomap types of tests/shim_mock/glomap_stub_processors and returning colmap::Sim3d --
// compiled with -fsyntax-only by tests/test_shim_processors_cpu.py.
#include "estimators_shim.h"

colmap::Sim3d Run(glomap::ViewGraph& vg, std::unordered_map<glomap::rig_t, glomap::Rig>& rigs,
                  std::unordered_map<glomap::camera_t, glomap::Camera>& cameras,
                  std::unordered_map<glomap::frame_t, glomap::Frame>& frames, std::unordered_map<glomap::image_t, glomap::Image>& images,
                  std::unordered_map<glomap::track_t, glomap::Track>& tracks) {
  using b200sfm_shim::TrackFilter;
  b200sfm_shim::UndistortImages(cameras, images, true);
  int n = TrackFilter::FilterTracksByAngle(vg, cameras, images, tracks, 1.0);
  n += TrackFilter::FilterTrackTriangulationAngle(vg, images, tracks, 1.0);
  n += TrackFilter::FilterTracksByReprojection(vg, cameras, images, tracks, 1e-2, true);
  n += TrackFilter::FilterTracksByReprojection(vg, cameras, images, tracks);
  (void)n;
  return b200sfm_shim::NormalizeReconstruction(rigs, cameras, frames, images, tracks);
}
