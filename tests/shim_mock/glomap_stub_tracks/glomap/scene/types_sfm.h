// TEST STUB (tests only, never shipped): the glomap stub of tests/shim_mock/glomap_stub_pairs (ImagePair with
// Eigen::MatrixXi matches and std::vector<int> inliers; Image with features and IsRegistered(); Track) plus
// glomap::TrackEstablishmentOptions as glomap/controllers/track_establishment.h:10-25 declares it, for type-checking the
// shim's TrackEngine in the form compiled inside a glomap build.
#pragma once
#include "../../../glomap_stub_pairs/glomap/scene/types_sfm.h"

namespace glomap {
struct TrackEstablishmentOptions {
  double thres_inconsistency = 10.;
  int min_num_tracks_per_view = -1;
  int min_num_view_per_track = 3;
  int max_num_view_per_track = 100;
  int max_num_tracks = 10000000;
};
}  // namespace glomap
