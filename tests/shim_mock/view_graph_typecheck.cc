// TEST (tests only): the shim's RelPoseFilter::FilterRotations and KeepLargestConnectedComponentsDevice in their
// -DB200SFM_WITH_GLOMAP form, instantiated with the glomap stub types of tests/shim_mock/glomap_stub (ImagePair::is_valid
// and cam2_from_cam1, Frame::is_registered / RigFromWorld / RigPtr, Image::frame_ptr / camera_id / IsRegistered) --
// compiled with -fsyntax-only by tests/test_view_graph_cpu.py.
#include "estimators_shim.h"

int Run(glomap::ViewGraph& vg, std::unordered_map<glomap::frame_t, glomap::Frame>& frames,
        std::unordered_map<glomap::image_t, glomap::Image>& images) {
  b200sfm_shim::RelPoseFilter::FilterRotations(vg, images, 10.0);
  return b200sfm_shim::KeepLargestConnectedComponentsDevice(vg, frames, images);
}
