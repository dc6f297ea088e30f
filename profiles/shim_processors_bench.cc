// Host-to-host timing of the shim's TrackFilter, UndistortImages and NormalizeReconstruction, built against
// libb200sfm.so by profiles/shim_processors_bench.py, which writes the scene this reads.
//   shim_processors_bench DIR REPS
// DIR holds dims.txt ("C P N K") and the raw little-endian arrays of a trivial-frame scene: quat.bin [C][4],
// trans.bin [C][3], points.bin [P][3], ptb.bin [P+1] int64, obs_cam.bin [N] int32, obs_xy.bin [N][2], cam_intr.bin [C]
// int32, intr_model.bin [K] int32, intr_params.bin [K][12], bearings.bin [N][3], prior.bin [K] uint8.  Image c + 1 is
// camera c's image on frame c + 1 through camera cam_intr[c] + 1; every observation is a feature of its image; track p
// has id p + 1.  Each call runs REPS times on a fresh copy of the maps it changes (the copy is not timed); prints one
// JSON line per call with the median, minimum and maximum in ms and the call's return value.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <fstream>
#include <string>

#include "estimators_shim.h"

using namespace b200sfm_shim;

template <class T>
static std::vector<T> load(const std::string& dir, const char* name, size_t n) {
  std::vector<T> v(n);
  std::ifstream in(dir + "/" + name, std::ios::binary);
  in.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * sizeof(T)));
  if (!in) { std::fprintf(stderr, "cannot read %s\n", name); std::exit(2); }
  return v;
}

template <class F>
static void timed(const char* name, int reps, F&& call) {
  std::vector<double> ms;
  double result = 0;
  for (int r = 0; r < reps; ++r) {
    double t = 0;
    result = call(t);
    ms.push_back(t);
  }
  std::sort(ms.begin(), ms.end());
  std::printf("{\"call\": \"%s\", \"ms_median\": %.3f, \"ms_min\": %.3f, \"ms_max\": %.3f, \"reps\": %d, \"result\": %.17g}\n", name,
              ms[ms.size() / 2], ms.front(), ms.back(), reps, result);
  std::fflush(stdout);
}

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: shim_processors_bench DIR REPS\n"); return 2; }
  const std::string dir = argv[1];
  const int reps = std::stoi(argv[2]);
  size_t C, P, N, K;
  std::ifstream(dir + "/dims.txt") >> C >> P >> N >> K;
  const auto quat = load<double>(dir, "quat.bin", 4 * C), trans = load<double>(dir, "trans.bin", 3 * C);
  const auto points = load<double>(dir, "points.bin", 3 * P), xy = load<double>(dir, "obs_xy.bin", 2 * N);
  const auto bear = load<double>(dir, "bearings.bin", 3 * N), params = load<double>(dir, "intr_params.bin", 12 * K);
  const auto ptb = load<int64_t>(dir, "ptb.bin", P + 1);
  const auto obs_cam = load<int32_t>(dir, "obs_cam.bin", N), cam_intr = load<int32_t>(dir, "cam_intr.bin", C);
  const auto model = load<int32_t>(dir, "intr_model.bin", K);
  const auto prior = load<uint8_t>(dir, "prior.bin", K);

  std::unordered_map<camera_t, Camera> cameras;
  for (size_t k = 0; k < K; ++k) {
    Camera& c = cameras[(camera_t)k + 1];
    c.camera_id = (camera_t)k + 1;
    c.model_id = model[k];
    c.params.assign(&params[12 * k], &params[12 * k] + 12);
    c.has_prior_focal_length = prior[k] != 0;
  }
  std::unordered_map<rig_t, Rig> rigs;
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  for (size_t c = 0; c < C; ++c) {
    Frame& f = frames[(frame_t)c + 1];
    f.frame_id = (frame_t)c + 1;
    for (int k = 0; k < 4; ++k) f.rig_from_world.rotation.c[k] = quat[4 * c + k];
    for (int k = 0; k < 3; ++k) f.rig_from_world.translation[k] = trans[3 * c + k];
  }
  for (size_t c = 0; c < C; ++c) {
    Image& im = images[(image_t)c + 1];
    im.image_id = (image_t)c + 1;
    im.camera_id = (camera_t)cam_intr[c] + 1;
    im.frame_id = (frame_t)c + 1;
    im.frame_ptr = &frames[(frame_t)c + 1];
  }
  std::unordered_map<track_t, Track> tracks;
  tracks.reserve(P);
  for (size_t p = 0; p < P; ++p) {
    Track& t = tracks[(track_t)p + 1];
    t.track_id = (track_t)p + 1;
    for (int k = 0; k < 3; ++k) t.xyz[k] = points[3 * p + k];
    for (int64_t o = ptb[p]; o < ptb[p + 1]; ++o) {
      Image& im = images[(image_t)obs_cam[o] + 1];
      t.observations.emplace_back(im.image_id, (feature_t)im.features.size());
      im.features.push_back({{xy[2 * o], xy[2 * o + 1]}});
      im.features_undist.push_back({{bear[3 * o], bear[3 * o + 1], bear[3 * o + 2]}});
    }
  }
  std::fprintf(stderr, "scene: %zu images, %zu tracks, %zu observations\n", C, P, N);

  using clock = std::chrono::steady_clock;
  auto ms_since = [](clock::time_point t0) { return std::chrono::duration<double, std::milli>(clock::now() - t0).count(); };
  const ViewGraph vg;
  auto filter = [&](const char* name, auto&& call) {
    timed(name, reps, [&](double& t) {
      std::unordered_map<track_t, Track> work = tracks;
      const auto t0 = clock::now();
      const int n = call(work);
      t = ms_since(t0);
      return (double)n;
    });
  };
  filter("FilterTracksByReprojection(in_normalized_image, 1e-2)",
         [&](auto& w) { return TrackFilter::FilterTracksByReprojection(vg, cameras, images, w, 1e-2, true); });
  filter("FilterTracksByReprojection(pixels, 3)",
         [&](auto& w) { return TrackFilter::FilterTracksByReprojection(vg, cameras, images, w, 3.0, false); });
  filter("FilterTracksByAngle(1)", [&](auto& w) { return TrackFilter::FilterTracksByAngle(vg, cameras, images, w, 1.0); });
  filter("FilterTrackTriangulationAngle(1)", [&](auto& w) { return TrackFilter::FilterTrackTriangulationAngle(vg, images, w, 1.0); });
  timed("UndistortImages(clean_points)", reps, [&](double& t) {
    const auto t0 = clock::now();
    UndistortImages(cameras, images, true);
    t = ms_since(t0);
    return 0.0;
  });
  timed("NormalizeReconstruction", reps, [&](double& t) {
    std::unordered_map<frame_t, Frame> fw = frames;
    std::unordered_map<track_t, Track> tw = tracks;
    for (auto& [id, im] : images) im.frame_ptr = &fw[im.frame_id];
    const auto t0 = clock::now();
    const Sim3d s = NormalizeReconstruction(rigs, cameras, fw, images, tw);
    t = ms_since(t0);
    for (auto& [id, im] : images) im.frame_ptr = &frames[im.frame_id];
    return s.scale;
  });
  return 0;
}
