// TEST DRIVER (tests only): builds a small world with one 2-camera rig seen in three frames plus one trivial frame,
// and runs the three shim estimators against the recording test double (mock_b200sfm.c).  The expectations are
// recomputed in Python (tests/test_shim_cpu.py) from the same closed-form construction.
#include <cmath>
#include <cstdio>
#include <limits>
#include <random>
#include <string>

#include "estimators_shim.h"

using namespace b200sfm_shim;

static void SetQuat(Quaternion& q, double ax, double ay, double az, double ang) {
  const double n = std::sqrt(ax * ax + ay * ay + az * az), s = std::sin(ang / 2) / n;
  q.c[0] = ax * s; q.c[1] = ay * s; q.c[2] = az * s; q.c[3] = std::cos(ang / 2);
}

// `shim_driver pinned`: a second world for the rules the first one never reaches.  Frame 5 holds an image that no track
// observes (a pose block for BA and GP all the same, and not BA's gauge); track 2 observes image 999, which is not in
// `images`; track 4 is shorter than min_num_view_per_track; cameras 2 and 3 of rig 1 have a cam_from_rig with a NaN
// translation and are first met as 3 then 2, the reverse of their sorted order.  GP draws its random positions and
// points, so that the centres of the unknown sensors show where they fall in the sequence of draws.
static int PinnedWorld() {
  std::unordered_map<rig_t, Rig> rigs;
  std::unordered_map<camera_t, Camera> cameras;
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  std::unordered_map<track_t, Track> tracks;
  for (camera_t c = 1; c <= 3; ++c) {
    Camera cam; cam.camera_id = c; cam.model_id = 0; cam.params = {600.0 + c, 320.0, 240.0};
    cameras[c] = cam;
  }
  Rig rig1; rig1.rig_id = 1; rig1.ref_camera_id = 1;
  const double nan = std::numeric_limits<double>::quiet_NaN();
  for (camera_t c = 2; c <= 3; ++c) {
    Rigid3d p; SetQuat(p.rotation, 0.3 * c, 1.0, -0.2, 0.1 * c); p.translation = {{nan, nan, nan}};
    rig1.cam_from_rig[c] = p;
  }
  rigs[1] = rig1;
  for (frame_t id : {5u, 10u, 20u}) {
    Frame f; f.frame_id = id; f.rig_id = 1;
    SetQuat(f.rig_from_world.rotation, 1.0, 0.01 * id, 0.3, 0.05 * id);
    f.rig_from_world.translation = {{0.1 * id, 1.0, -2.0}};
    frames[id] = f;
  }
  const image_t ids[7] = {51, 101, 102, 103, 201, 202, 203};
  for (int k = 0; k < 7; ++k) {
    Image im; im.image_id = ids[k]; im.frame_id = ids[k] < 100 ? 5 : (ids[k] / 100) * 10; im.camera_id = ids[k] % 10;
    im.trivial_frame = false;
    for (int f = 0; f < 4; ++f) {
      im.features.push_back({{5.0 * k + f, 7.0 * k - f}});
      const double b[3] = {0.02 * k - 0.01 * f, 0.01 * f + 0.005 * k, 1.0};
      const double n = std::sqrt(b[0] * b[0] + b[1] * b[1] + 1.0);
      im.features_undist.push_back({{b[0] / n, b[1] / n, 1.0 / n}});
    }
    images[ids[k]] = im;
  }
  for (auto& [id, im] : images) im.frame_ptr = &frames[im.frame_id];
  const std::vector<std::pair<image_t, feature_t>> obs[3] = {
      {{203, 0}, {102, 1}, {201, 2}, {999, 0}}, {{101, 0}, {202, 1}}, {{101, 2}, {102, 3}, {103, 0}, {201, 1}}};
  const track_t tids[3] = {2, 4, 6};
  for (int t = 0; t < 3; ++t) {
    Track tr; tr.track_id = tids[t]; tr.xyz = {{1.0 + t, -1.0, 3.0 + 0.5 * t}};
    tr.observations = obs[t];
    tracks[tids[t]] = tr;
  }
  ViewGraph vg;
  BundleAdjusterOptions bo;
  BundleAdjuster ba(bo);
  if (!ba.Solve(rigs, cameras, frames, images, tracks)) return 1;
  GlobalPositionerOptions go;   // random positions and points, seed 1
  GlobalPositioner gp(go);
  if (!gp.Solve(vg, rigs, cameras, frames, images, tracks)) return 2;
  for (camera_t c = 2; c <= 3; ++c) {
    const Rigid3d& p = rigs[1].cam_from_rig[c];
    std::printf("cfr%u %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", (unsigned)c, p.rotation.c[0], p.rotation.c[1], p.rotation.c[2],
                p.rotation.c[3], p.translation[0], p.translation[1], p.translation[2]);
  }
  std::mt19937 g(go.seed);   // the sequence GlobalPositioner draws from
  std::uniform_real_distribution<double> U(-1, 1);
  std::printf("draws");
  for (int k = 0; k < 24; ++k) std::printf(" %.17g", U(g));
  std::printf("\nshim driver ok\n");
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 1 && std::string(argv[1]) == "pinned") return PinnedWorld();
  std::unordered_map<rig_t, Rig> rigs;
  std::unordered_map<camera_t, Camera> cameras;
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  std::unordered_map<track_t, Track> tracks;
  // cameras 1, 2 (rig 1; camera 1 = reference sensor), camera 3 (trivial rig 2)
  for (camera_t c = 1; c <= 3; ++c) {
    Camera cam; cam.camera_id = c; cam.model_id = 0; cam.params = {500.0 + c, 320.0, 240.0}; cam.has_prior_focal_length = (c != 2);
    cameras[c] = cam;
  }
  Rig rig1; rig1.rig_id = 1; rig1.ref_camera_id = 1;
  Rigid3d c2r; SetQuat(c2r.rotation, 0.2, 1.0, -0.3, 0.35); c2r.translation = {{0.4, -0.1, 0.05}};
  rig1.cam_from_rig[2] = c2r;
  rigs[1] = rig1;
  Rig rig2; rig2.rig_id = 2; rig2.ref_camera_id = 3; rigs[2] = rig2;
  // frames 10, 20, 30 (rig 1) and 40 (rig 2)
  for (int k = 0; k < 4; ++k) {
    Frame f; f.frame_id = 10 * (k + 1); f.rig_id = k < 3 ? 1 : 2;
    SetQuat(f.rig_from_world.rotation, 0.1 * k, 1.0, 0.2, 0.3 + 0.4 * k);
    f.rig_from_world.translation = {{1.0 + k, -0.5 * k, 2.0 + 0.25 * k}};
    frames[f.frame_id] = f;
  }
  // images: frame 10 -> 101 (cam 1), 102 (cam 2); 20 -> 201, 202; 30 -> 301, 302; frame 40 -> 401 (cam 3, trivial)
  const image_t ids[7] = {101, 102, 201, 202, 301, 302, 401};
  for (int k = 0; k < 7; ++k) {
    Image im; im.image_id = ids[k]; im.frame_id = (ids[k] / 100) * 10; im.camera_id = k == 6 ? 3 : (ids[k] % 100);
    im.trivial_frame = (k == 6);
    for (int f = 0; f < 4; ++f) {
      im.features.push_back({{10.0 * k + f, 20.0 * k + 2.0 * f}});
      const double b[3] = {0.01 * k - 0.02 * f, 0.03 * f - 0.01 * k, 1.0};
      const double n = std::sqrt(b[0] * b[0] + b[1] * b[1] + 1.0);
      im.features_undist.push_back({{b[0] / n, b[1] / n, 1.0 / n}});
    }
    images[ids[k]] = im;
  }
  for (auto& [id, im] : images) im.frame_ptr = &frames[im.frame_id];
  // tracks 7, 3, 5: every one seen by four images
  const image_t obs[3][4] = {{101, 202, 301, 401}, {102, 201, 302, 401}, {101, 102, 201, 301}};
  const track_t tids[3] = {7, 3, 5};
  for (int t = 0; t < 3; ++t) {
    Track tr; tr.track_id = tids[t]; tr.xyz = {{0.5 * t, 1.0 - t, 4.0 + t}};
    for (int k = 0; k < 4; ++k) tr.observations.emplace_back(obs[t][k], (feature_t)((t + k) % 4));
    tracks[tids[t]] = tr;
  }
  // view graph: (101,102) lives inside one frame (self loop), the others connect frames
  ViewGraph vg;
  const image_t pr[5][2] = {{101, 102}, {101, 201}, {102, 301}, {202, 302}, {301, 401}};
  for (int k = 0; k < 5; ++k) {
    ImagePair p; p.image_id1 = pr[k][0]; p.image_id2 = pr[k][1]; p.weight = 1.0 + k;
    p.inliers.assign(10 + k, 0);
    SetQuat(p.cam2_from_cam1.rotation, 1.0, 0.1 * k, -0.2, 0.2 + 0.1 * k);
    vg.image_pairs[ImagePairToPairId(pr[k][0], pr[k][1])] = p;
  }

  BundleAdjusterOptions bo;
  BundleAdjuster ba(bo);
  if (!ba.Solve(rigs, cameras, frames, images, tracks)) return 1;
  GlobalPositionerOptions go;
  go.generate_random_positions = false; go.generate_random_points = false;
  GlobalPositioner gp(go);
  if (!gp.Solve(vg, rigs, cameras, frames, images, tracks)) return 2;
  RotationEstimatorOptions ro;
  ro.skip_initialization = true;   // the flattening checks start from the frames' own rotations
  RotationEstimator ra(ro);
  if (!ra.EstimateRotations(vg, rigs, frames, images)) return 3;
  // gravity-aligned rotation averaging: frames 20 and 40 carry a gravity prior
  frames[20].gravity_info.SetGravity({{0.1, 1.0, 0.05}});
  frames[40].gravity_info.SetGravity({{0.0, 1.0, 0.0}});
  RotationEstimatorOptions rg;
  rg.use_gravity = true;
  RotationEstimator rag(rg);
  if (!rag.EstimateRotations(vg, rigs, frames, images)) return 5;
  std::printf("q20 %.17g %.17g %.17g %.17g\n", frames[20].rig_from_world.rotation.c[0], frames[20].rig_from_world.rotation.c[1],
              frames[20].rig_from_world.rotation.c[2], frames[20].rig_from_world.rotation.c[3]);
  // trivial-frame world through the one-shot entry: only frame 40 / image 401 / camera 3
  std::unordered_map<frame_t, Frame> f2; f2[40] = frames[40];
  std::unordered_map<image_t, Image> i2; i2[401] = images[401]; i2[401].frame_ptr = &f2[40];
  std::unordered_map<camera_t, Camera> c2; c2[3] = cameras[3];
  std::unordered_map<track_t, Track> t2;
  Track tr; tr.track_id = 1; tr.observations = {{401, 0}, {401, 1}, {401, 2}}; t2[1] = tr;
  BundleAdjuster ba2(bo);
  if (!ba2.Solve(rigs, c2, f2, i2, t2)) return 4;
  // maximum-spanning-tree initialisation inside EstimateRotations (global_rotation_averaging.cc:60-63): the mock
  // records the initial theta the device solver would start from
  for (auto& [id, f] : frames) { f.rig_from_world.rotation = Quaternion(); f.gravity_info.has_gravity = false; }
  RotationEstimatorOptions rm;   // skip_initialization = false (the reference default)
  RotationEstimator ram(rm);
  if (!ram.EstimateRotations(vg, rigs, frames, images)) return 6;
  // use_gravity with an uncalibrated rig sensor must be refused (.cc:47-59)
  rigs[1].uncalibrated.push_back(9);
  RotationEstimator rag2(rg);
  if (rag2.EstimateRotations(vg, rigs, frames, images)) return 7;
  // optimize_rig_poses (bundle_adjustment.cc:162-180,296-308): the non-reference sensor (rig 1, camera 2) becomes an
  // unknown and its optimised cam_from_rig is written back into the rig; the reference sensors stay untouched
  BundleAdjusterOptions bor;
  bor.optimize_rig_poses = true;
  BundleAdjuster bar(bor);
  if (!bar.Solve(rigs, cameras, frames, images, tracks)) return 8;
  const Rigid3d& o2 = rigs[1].cam_from_rig[2];
  std::printf("c2r %.17g %.17g %.17g %.17g %.17g %.17g %.17g\n", o2.rotation.c[0], o2.rotation.c[1], o2.rotation.c[2], o2.rotation.c[3],
              o2.translation[0], o2.translation[1], o2.translation[2]);
  std::printf("nrig1 %zu\n", rigs[1].cam_from_rig.size());
  // rotation averaging with a sensor whose cam_from_rig is not known yet (global_rotation_averaging.cc:162-245,800-813):
  // camera 2 of rig 1 loses its calibration -> one extra rotation node, its estimate lands in the rig with a NaN translation
  rigs[1].uncalibrated.clear();
  rigs[1].cam_from_rig.erase(2);
  rigs[1].uncalibrated.push_back(2);
  RotationEstimator rau(ro);   // skip_initialization = true
  if (!rau.EstimateRotations(vg, rigs, frames, images)) return 9;
  const Rigid3d& e2 = rigs[1].cam_from_rig[2];
  std::printf("est2 %.17g %.17g %.17g %.17g %d\n", e2.rotation.c[0], e2.rotation.c[1], e2.rotation.c[2], e2.rotation.c[3],
              (int)std::isnan(e2.translation[0]));
  // global positioning with that sensor: its cam_from_rig translation is NaN -> RigUnknownBATA (global_positioning.cc:355-372):
  // the sensor centre is an unknown, and ConvertResults turns the estimate into a translation (.cc:578-582)
  GlobalPositionerOptions gu;
  gu.generate_random_positions = false; gu.generate_random_points = false; gu.optimize_positions = false;
  GlobalPositioner gpu(gu);
  if (!gpu.Solve(vg, rigs, cameras, frames, images, tracks)) return 10;
  const Rigid3d& g2 = rigs[1].cam_from_rig[2];
  std::printf("gpt2 %.17g %.17g %.17g\n", g2.translation[0], g2.translation[1], g2.translation[2]);
  std::printf("shim driver ok\n");
  return 0;
}
