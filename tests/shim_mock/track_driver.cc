// TEST DRIVER (tests only): the shim's TrackEngine against the recording test double (mock_track_select.c) or, built
// against libb200sfm.so, against the device.  Reads nothing; prints the tracks of both methods in sorted id order.
//   track_driver mock : a hand world; the expectations are in tests/test_track_selection_cpu.py
//   track_driver FILE : the world in FILE (tests/test_track_selection_gpu.py writes it), with the options
//     "images I" then I lines "image_id registered num_features x0 y0 x1 y1 ...",
//     "pairs E" then E lines "image_id1 image_id2 is_valid num_matches f1 f2 ... num_inliers k ...",
//     "options min_num_tracks_per_view min_num_view_per_track max_num_view_per_track max_num_tracks thres_inconsistency"
#include <cstdio>
#include <fstream>
#include <string>

#include "estimators_shim.h"

using namespace b200sfm_shim;

static void print_tracks(const char* what, size_t n, const std::unordered_map<track_t, Track>& tracks) {
  std::printf("%s %zu\n", what, n);
  std::map<track_t, const Track*> sorted;
  for (const auto& [id, t] : tracks) sorted[id] = &t;
  for (const auto& [id, t] : sorted) {
    std::printf("track %llu %llu", (unsigned long long)id, (unsigned long long)t->track_id);
    for (const auto& ob : t->observations) std::printf(" %u:%u", ob.first, ob.second);
    std::printf("\n");
  }
}

int main(int argc, char** argv) {
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  ViewGraph vg;
  TrackEstablishmentOptions opt;
  const bool mock = argc < 2 || std::string(argv[1]) == "mock";
  if (mock) {
    // images 30, 10, 20 (frames of the same id); image 30's frame is not registered
    for (image_t i : {30u, 10u, 20u}) {
      Frame fr; fr.frame_id = i; fr.is_registered = i != 30;
      frames[i] = fr;
    }
    for (image_t i : {30u, 10u, 20u}) {
      Image im; im.image_id = i; im.frame_id = i; im.frame_ptr = &frames[i];
      for (int f = 0; f < 3; ++f) im.features.push_back({{1.0 * i + f, -1.0 * f}});
      images[i] = im;
    }
    auto add = [&](image_t a, image_t b, bool valid, std::vector<std::array<int, 2>> m, std::vector<int> inl) {
      ImagePair p; p.image_id1 = a; p.image_id2 = b; p.is_valid = valid; p.inliers = inl;
      p.matches.rows_ = m;
      vg.image_pairs[ImagePairToPairId(a, b)] = p;
    };
    add(20, 30, true, {{{0, 1}}, {{2, 2}}}, {1});           // pair id of (20, 30) sorts after (10, 20)
    add(10, 20, true, {{{1, 0}}, {{2, 1}}, {{0, 2}}}, {2, 0});
    add(10, 30, false, {{{0, 0}}}, {0});                    // invalid: ignored
    opt.thres_inconsistency = 2.5;
    opt.min_num_tracks_per_view = 4;
    opt.min_num_view_per_track = 1;
    opt.max_num_view_per_track = -7;
    opt.max_num_tracks = 9;
  } else {
    std::ifstream in(argv[1]);
    std::string word;
    size_t I = 0, E = 0;
    in >> word >> I;
    std::vector<std::pair<image_t, bool>> reg;
    for (size_t k = 0; k < I; ++k) {
      image_t id; int r; size_t nf;
      in >> id >> r >> nf;
      Image im; im.image_id = id; im.frame_id = id;
      for (size_t f = 0; f < nf; ++f) { double x, y; in >> x >> y; im.features.push_back({{x, y}}); }
      images[id] = im;
      Frame fr; fr.frame_id = id; fr.is_registered = r != 0;
      frames[id] = fr;
    }
    for (auto& [id, im] : images) im.frame_ptr = &frames[id];
    in >> word >> E;
    for (size_t e = 0; e < E; ++e) {
      ImagePair p; int valid; size_t nm, ni;
      in >> p.image_id1 >> p.image_id2 >> valid >> nm;
      p.is_valid = valid != 0;
      for (size_t k = 0; k < nm; ++k) { int a, b; in >> a >> b; p.matches.rows_.push_back({{a, b}}); }
      in >> ni;
      for (size_t k = 0; k < ni; ++k) { int r; in >> r; p.inliers.push_back(r); }
      vg.image_pairs[ImagePairToPairId(p.image_id1, p.image_id2)] = p;
    }
    in >> word >> opt.min_num_tracks_per_view >> opt.min_num_view_per_track >> opt.max_num_view_per_track >> opt.max_num_tracks
       >> opt.thres_inconsistency;
  }
  TrackEngine engine(vg, images, opt);
  std::unordered_map<track_t, Track> full, selected;
  Track stale; stale.track_id = 99;
  full[99] = stale;                                   // cleared by EstablishFullTracks
  const size_t n_full = engine.EstablishFullTracks(full);
  print_tracks("full", n_full, full);
  if (mock) {   // a hand map for the selection: ids out of order, unregistered image 30, repeated image 10
    full.clear();
    auto track = [&](track_t id, std::vector<image_t> ims) {
      Track t; t.track_id = id;
      for (image_t i : ims) t.observations.push_back({i, (feature_t)(i + id)});
      full[id] = t;
    };
    track(50, {10, 30, 20});
    track(20, {30, 10, 10});
    track(40, {20});
  }
  const size_t n_sel = engine.FindTracksForProblem(full, selected);
  print_tracks("selected", n_sel, selected);
  std::printf("track driver ok\n");
  return 0;
}
