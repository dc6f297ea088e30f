// TEST (tests only): the shim's PruneWeaklyConnectedImages in its -DB200SFM_WITH_GLOMAP form, instantiated with the glomap
// types of tests/shim_mock/glomap_stub_prune -- compiled with -fsyntax-only by tests/test_reconstruction_pruning_cpu.py.
#include "estimators_shim.h"

glomap::image_t Run(std::unordered_map<glomap::frame_t, glomap::Frame>& frames,
                    std::unordered_map<glomap::image_t, glomap::Image>& images,
                    std::unordered_map<glomap::track_t, glomap::Track>& tracks) {
  return b200sfm_shim::PruneWeaklyConnectedImages(frames, images, tracks);
}
