// TEST (tests only): the shim's TrackEngine in its -DB200SFM_WITH_GLOMAP form, constructed from glomap's own
// TrackEstablishmentOptions and instantiated with the glomap types of tests/shim_mock/glomap_stub_tracks -- compiled with
// -fsyntax-only by tests/test_track_selection_cpu.py.
#include "estimators_shim.h"

size_t Run(const glomap::ViewGraph& vg, const std::unordered_map<glomap::image_t, glomap::Image>& images,
           std::unordered_map<glomap::track_t, glomap::Track>& full, std::unordered_map<glomap::track_t, glomap::Track>& selected) {
  const glomap::TrackEstablishmentOptions options;
  b200sfm_shim::TrackEngine engine(vg, images, options);
  engine.EstablishFullTracks(full);
  return engine.FindTracksForProblem(full, selected);
}
