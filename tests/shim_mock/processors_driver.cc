// TEST DRIVER (tests only): the shim's TrackFilter, UndistortImages and NormalizeReconstruction on a world read from a
// file, against the recording test double (mock_processors.c, tests/test_shim_processors_cpu.py) or, built against
// libb200sfm.so, against the device (tests/test_shim_processors_gpu.py).
//   processors_driver WORLD OP [ARGS]   OP: reprojection THR NORMALIZED | angle THR | triangulation THR |
//                                           undistort CLEAN | normalize FIXED EXTENT P0 P1
// WORLD (whitespace separated):
//   cameras K  then K x "id model prior nparams p..."
//   rigs R     then R x "id ref_camera n" + n x "camera qx qy qz qw tx ty tz" (calibrated non-reference sensors)
//   frames F   then F x "id rig registered qx qy qz qw tx ty tz"
//   images I   then I x "id camera frame trivial nf x y ... nu bx by bz ..."
//   tracks T   then T x "id x y z n image feature ..."
// Prints "result ..." and then the whole world after the call, in sorted id order, with %.17g.
#include <cstdio>
#include <fstream>
#include <string>

#include "estimators_shim.h"

using namespace b200sfm_shim;

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: processors_driver WORLD OP [ARGS]\n"); return 2; }
  std::unordered_map<camera_t, Camera> cameras;
  std::unordered_map<rig_t, Rig> rigs;
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  std::unordered_map<track_t, Track> tracks;
  std::ifstream in(argv[1]);
  std::string word;
  size_t n = 0;
  in >> word >> n;
  for (size_t i = 0; i < n; ++i) {
    Camera c;
    size_t np;
    int prior;
    in >> c.camera_id >> c.model_id >> prior >> np;
    c.has_prior_focal_length = prior != 0;
    c.params.resize(np);
    for (double& v : c.params) in >> v;
    cameras[c.camera_id] = c;
  }
  in >> word >> n;
  for (size_t i = 0; i < n; ++i) {
    Rig r;
    size_t ns;
    in >> r.rig_id >> r.ref_camera_id >> ns;
    for (size_t s = 0; s < ns; ++s) {
      camera_t cam;
      Rigid3d p;
      in >> cam;
      for (double& v : p.rotation.c) in >> v;
      for (double& v : p.translation) in >> v;
      r.cam_from_rig[cam] = p;
    }
    rigs[r.rig_id] = r;
  }
  in >> word >> n;
  for (size_t i = 0; i < n; ++i) {
    Frame f;
    int reg;
    in >> f.frame_id >> f.rig_id >> reg;
    f.is_registered = reg != 0;
    for (double& v : f.rig_from_world.rotation.c) in >> v;
    for (double& v : f.rig_from_world.translation) in >> v;
    frames[f.frame_id] = f;
  }
  for (auto& [id, f] : frames) f.rig_ptr = rigs.count(f.rig_id) ? &rigs[f.rig_id] : nullptr;
  in >> word >> n;
  for (size_t i = 0; i < n; ++i) {
    Image im;
    int trivial;
    size_t nf, nu;
    in >> im.image_id >> im.camera_id >> im.frame_id >> trivial >> nf;
    im.trivial_frame = trivial != 0;
    im.features.resize(nf);
    for (auto& f : im.features) in >> f[0] >> f[1];
    in >> nu;
    im.features_undist.resize(nu);
    for (auto& b : im.features_undist) in >> b[0] >> b[1] >> b[2];
    images[im.image_id] = im;
  }
  for (auto& [id, im] : images) im.frame_ptr = frames.count(im.frame_id) ? &frames[im.frame_id] : nullptr;
  in >> word >> n;
  for (size_t i = 0; i < n; ++i) {
    Track t;
    size_t no;
    in >> t.track_id >> t.xyz[0] >> t.xyz[1] >> t.xyz[2] >> no;
    t.observations.resize(no);
    for (auto& ob : t.observations) in >> ob.first >> ob.second;
    tracks[t.track_id] = t;
  }
  if (!in) { std::fprintf(stderr, "processors_driver: bad world file\n"); return 2; }

  const std::string op = argv[2];
  const ViewGraph vg;
  if (op == "reprojection") {
    std::printf("result %d\n", TrackFilter::FilterTracksByReprojection(vg, cameras, images, tracks, std::stod(argv[3]), std::stoi(argv[4]) != 0));
  } else if (op == "angle") {
    std::printf("result %d\n", TrackFilter::FilterTracksByAngle(vg, cameras, images, tracks, std::stod(argv[3])));
  } else if (op == "triangulation") {
    std::printf("result %d\n", TrackFilter::FilterTrackTriangulationAngle(vg, images, tracks, std::stod(argv[3])));
  } else if (op == "undistort") {
    UndistortImages(cameras, images, std::stoi(argv[3]) != 0);
    std::printf("result\n");
  } else if (op == "normalize") {
    const Sim3d s = NormalizeReconstruction(rigs, cameras, frames, images, tracks, std::stoi(argv[3]) != 0, std::stod(argv[4]),
                                            std::stod(argv[5]), std::stod(argv[6]));
    std::printf("result %.17g %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", s.scale, s.rotation.c[0], s.rotation.c[1], s.rotation.c[2],
                s.rotation.c[3], s.translation[0], s.translation[1], s.translation[2]);
  } else {
    std::fprintf(stderr, "processors_driver: unknown op %s\n", op.c_str());
    return 2;
  }
  std::map<rig_t, const Rig*> rs;
  for (const auto& [id, r] : rigs) rs[id] = &r;
  for (const auto& [id, r] : rs)
    for (const auto& [cam, p] : r->cam_from_rig)
      std::printf("sensor %u %u %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", id, cam, p.rotation.c[0], p.rotation.c[1], p.rotation.c[2],
                  p.rotation.c[3], p.translation[0], p.translation[1], p.translation[2]);
  std::map<frame_t, const Frame*> fs;
  for (const auto& [id, f] : frames) fs[id] = &f;
  for (const auto& [id, f] : fs) {
    const Rigid3d& p = f->rig_from_world;
    std::printf("frame %u %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", id, p.rotation.c[0], p.rotation.c[1], p.rotation.c[2],
                p.rotation.c[3], p.translation[0], p.translation[1], p.translation[2]);
  }
  std::map<image_t, const Image*> is;
  for (const auto& [id, im] : images) is[id] = &im;
  for (const auto& [id, im] : is) {
    std::printf("image %u %zu", id, im->features_undist.size());
    for (const auto& b : im->features_undist) std::printf(" %.17g %.17g %.17g", b[0], b[1], b[2]);
    std::printf("\n");
  }
  std::map<track_t, const Track*> ts;
  for (const auto& [id, t] : tracks) ts[id] = &t;
  for (const auto& [id, t] : ts) {
    std::printf("track %llu %.17g %.17g %.17g %zu", (unsigned long long)id, t->xyz[0], t->xyz[1], t->xyz[2], t->observations.size());
    for (const auto& ob : t->observations) std::printf(" %u %u", ob.first, ob.second);
    std::printf("\n");
  }
  return 0;
}
