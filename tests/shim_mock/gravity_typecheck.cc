// TEST (tests only): the shim's GravityRefiner, KeepLargestConnectedComponents and the gravity adapters in their
// -DB200SFM_WITH_GLOMAP form, instantiated with glomap stub types (the prune stub with GravityInfo::SetGravity, as
// glomap/scene/frame.h:18 declares it) -- compiled with -fsyntax-only by tests/test_rotation_averager_cpu.py.
#include "estimators_shim.h"

void Run(const glomap::ViewGraph& vg, glomap::ViewGraph& vg2, std::unordered_map<glomap::frame_t, glomap::Frame>& frames,
         std::unordered_map<glomap::image_t, glomap::Image>& images) {
  b200sfm_shim::GravityRefinerOptions o;
  b200sfm_shim::GravityRefiner(o).RefineGravity(vg, frames, images);
  b200sfm_shim::KeepLargestConnectedComponents(vg2, frames, images);
}
