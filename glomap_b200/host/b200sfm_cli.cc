// b200sfm_cli.cc -- stand-alone C++ driver over the estimator shim: what the
// `glomap` binary does around the three estimators, without COLMAP.
//
//   b200sfm_cli rotation_averager --relpose_path IN --output_path OUT [--mst_init 1] [--gravity_path G]
//                                 [--refine_gravity 0|1] [--use_stratified 0|1] [--weight_path W] [--use_weight 0|1]
//       mirrors glomap/exe/rotation_averager.cc:16-121: ReadRelPose (io/pose_io.cc:8-89,
//       image ids in order of first appearance), one frame per image, ReadGravity (:139-180) and ReadRelWeight
//       (:91-135), largest connected component, GravityRefiner (with --refine_gravity 1 and a gravity file) and
//       SolveRotationAveraging with use_gravity and skip_initialization = true (exe/rotation_averager.cc:58-59),
//       WriteGlobalRotation (io/pose_io.cc:182-200).  Without --gravity_path the pairs go to RotationEstimator directly,
//       which is what SolveRotationAveraging does when no frame has gravity.
//   b200sfm_cli ba --problem IN.bin --output OUT.bin [--pcg_tol T] [--fix_rotations 1]
//   b200sfm_cli gp --problem IN.bin --output OUT.bin [--pcg_tol T]
//       load a flat problem (format below) into the unordered_map world the
//       reference uses, call BundleAdjuster / GlobalPositioner ::Solve, write it back.
//
// Flat file: int64 {C,P,N,K}; int64 pt_obs_begin[P+1]; int32 obs_cam[N]; f64 obs_xy[2N];
// f64 bearings[3N]; int32 cam_intr[C]; int32 intr_model[K]; f64 intr[K*12];
// f64 quat_xyzw[4C]; f64 trans[3C]; f64 points[3P].
#include <cstring>
#include <fstream>
#include <iostream>
#include <queue>
#include <set>
#include <sstream>

#include "estimators_shim.h"

using namespace b200sfm_shim;

static std::map<std::string, std::string> ParseArgs(int argc, char** argv, int first) {
  std::map<std::string, std::string> a;
  for (int i = first; i + 1 < argc; i += 2) {
    std::string k = argv[i];
    if (k.rfind("--", 0) == 0) k = k.substr(2);
    a[k] = argv[i + 1];
  }
  return a;
}

static bool FileExists(const std::string& p) { return (bool)std::ifstream(p); }

// GetAlignRot (math/gravity.cc:11-24) with Eigen's HouseholderQR completion: column 1 is the unit gravity, columns 0
// and 2 the last two columns of the Householder reflector, column 2 negated when the determinant is negative.
static void GetAlignRotHouseholder(const double g[3], double R[9]) {
  const double n = std::sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
  const double v[3] = {g[0] / n, g[1] / n, g[2] / n};
  const double tsq = v[1] * v[1] + v[2] * v[2];
  double H[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (tsq > std::numeric_limits<double>::min()) {   // Eigen makeHouseholder; tau = 0 (H = I) otherwise
    const double beta = v[0] >= 0 ? -std::sqrt(v[0] * v[0] + tsq) : std::sqrt(v[0] * v[0] + tsq);
    const double w[3] = {1.0, v[1] / (v[0] - beta), v[2] / (v[0] - beta)};
    const double tau = (beta - v[0]) / beta;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) H[3 * r + c] -= tau * w[r] * w[c];
  }
  for (int r = 0; r < 3; ++r) { R[3 * r] = H[3 * r + 1]; R[3 * r + 1] = v[r]; R[3 * r + 2] = H[3 * r + 2]; }
  const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) + R[2] * (R[3] * R[7] - R[4] * R[6]);
  if (det < 0)
    for (int r = 0; r < 3; ++r) R[3 * r + 2] = -R[3 * r + 2];
}

static int RunRotationAverager(int argc, char** argv) {
  auto args = ParseArgs(argc, argv, 2);
  static const std::set<std::string> known = {"relpose_path", "output_path", "mst_init", "gravity_path", "weight_path",
                                              "use_stratified", "refine_gravity", "use_weight"};
  for (auto& [k, v] : args)
    if (!known.count(k)) { std::cerr << "rotation_averager: unknown option --" << k << "\n"; return 2; }
  if (!args.count("relpose_path") || !args.count("output_path")) {
    std::cerr << "usage: b200sfm_cli rotation_averager --relpose_path IN --output_path OUT [--mst_init 1] [--gravity_path G] "
                 "[--refine_gravity 0|1] [--use_stratified 0|1] [--weight_path W] [--use_weight 0|1]\n";
    return 2;
  }
  auto flag = [&](const char* k, bool dflt) { return args.count(k) ? args[k] != "0" : dflt; };
  const std::string gravity_path = args.count("gravity_path") ? args["gravity_path"] : "";
  const std::string weight_path = args.count("weight_path") ? args["weight_path"] : "";
  const bool use_stratified = flag("use_stratified", true), refine_gravity = flag("refine_gravity", false);
  const bool use_weight = flag("use_weight", false);
  // exe/rotation_averager.cc:38-56
  if (!FileExists(args["relpose_path"])) { std::cerr << "`relpose_path` is not a file\n"; return 1; }
  if (!gravity_path.empty() && !FileExists(gravity_path)) { std::cerr << "`gravity_path` is not a file\n"; return 1; }
  if (!weight_path.empty() && !FileExists(weight_path)) { std::cerr << "`weight_path` is not a file\n"; return 1; }
  if (use_weight && weight_path.empty()) { std::cerr << "Weight path is required when use_weight is set to true\n"; return 1; }
  std::unordered_map<rig_t, Rig> rigs;
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  ViewGraph view_graph;
  // ReadRelPose (io/pose_io.cc:8-89)
  std::ifstream file(args["relpose_path"]);
  if (!file) { std::cerr << "cannot open " << args["relpose_path"] << "\n"; return 1; }
  std::unordered_map<std::string, image_t> name_idx;
  image_t max_image_id = 0;
  std::string line;
  while (std::getline(file, line)) {
    std::stringstream ls(line);
    std::string f1, f2, item;
    if (!std::getline(ls, f1, ' ') || !std::getline(ls, f2, ' ')) continue;
    for (const std::string& nm : {f1, f2})
      if (!name_idx.count(nm)) {
        ++max_image_id;
        Image im;
        im.image_id = max_image_id; im.camera_id = max_image_id; im.frame_id = max_image_id; im.file_name = nm;
        images[max_image_id] = im;
        name_idx[nm] = max_image_id;
      }
    ImagePair pr;
    pr.image_id1 = name_idx[f1];
    pr.image_id2 = name_idx[f2];
    bool ok = true;
    for (int i = 0; i < 4 && ok; ++i) {                                   // QW QX QY QZ -> coeffs (x,y,z,w) (pose_io.cc:64-68)
      if (!std::getline(ls, item, ' ')) { ok = false; break; }
      pr.cam2_from_cam1.rotation.coeffs().data()[(i + 3) % 4] = std::stod(item);
    }
    for (int i = 0; i < 3 && ok; ++i) {
      if (!std::getline(ls, item, ' ')) { ok = false; break; }
      pr.cam2_from_cam1.translation[i] = std::stod(item);
    }
    if (!ok) continue;
    view_graph.image_pairs[ImagePairToPairId(pr.image_id1, pr.image_id2)] = pr;
  }
  // one rig + one frame per image (exe/rotation_averager.cc:74-86)
  for (auto& [id, im] : images) {
    Frame f;
    f.frame_id = id;
    frames[id] = f;
  }
  for (auto& [id, im] : images) im.frame_ptr = &frames[id];
  if (use_weight) {   // ReadRelWeight (io/pose_io.cc:91-135): IMAGE_NAME_1 IMAGE_NAME_2 WEIGHT; unknown names / pairs ignored
    std::ifstream wf(weight_path);
    while (std::getline(wf, line)) {
      std::stringstream ls(line);
      std::string a, b, item;
      if (!std::getline(ls, a, ' ') || !std::getline(ls, b, ' ')) continue;
      if (!name_idx.count(a) || !name_idx.count(b)) continue;
      auto it = view_graph.image_pairs.find(ImagePairToPairId(name_idx[a], name_idx[b]));
      if (it == view_graph.image_pairs.end() || !std::getline(ls, item, ' ')) continue;
      it->second.weight = std::stod(item);
    }
  }
  if (!gravity_path.empty()) {
    // ReadGravity (io/pose_io.cc:139-180): IMAGE_NAME GX GY GZ; unknown names ignored.  The prior sets R_align and the
    // initial rotation rig_from_world = R_align
    std::ifstream gf(gravity_path);
    while (std::getline(gf, line)) {
      std::stringstream ls(line);
      std::string name, item;
      std::array<double, 3> g{};
      if (!std::getline(ls, name, ' ')) continue;
      bool ok = true;
      for (int i = 0; i < 3 && ok; ++i) ok = (bool)std::getline(ls, item, ' ') && (g[i] = std::stod(item), true);
      if (!ok || !name_idx.count(name)) continue;
      Frame& f = frames[name_idx[name]];
      f.gravity_info.SetGravity(g);
      GetAlignRotHouseholder(g.data(), f.gravity_info.R_align);
      detail::RToQuat(f.gravity_info.R_align, f.RigFromWorld().rotation.coeffs().data());
    }
    KeepLargestConnectedComponents(view_graph, frames, images);                               // exe/rotation_averager.cc:95
    if (refine_gravity) {                                                                      // :99-102
      GravityRefinerOptions gopts;
      GravityRefiner refiner(gopts);
      refiner.RefineGravity(view_graph, frames, images);
      for (auto& [id, f] : frames)   // a refined prior keeps the Householder R_align (the initial rotation stays as read)
        if (f.HasGravity()) GetAlignRotHouseholder(f.gravity_info.gravity_in_rig.data(), f.gravity_info.R_align);
    }
    RotationAveragerOptions ra;
    ra.skip_initialization = true;                                                             // :58-63
    ra.use_gravity = true;
    ra.use_stratified = use_stratified;
    ra.use_weight = use_weight;
    if (!SolveRotationAveraging(view_graph, rigs, frames, images, ra)) { std::cerr << "Failed to solve global rotation averaging\n"; return 1; }
    std::ofstream out(args["output_path"]);
    std::set<image_t> sorted_ids;
    for (auto& [id, im] : images) sorted_ids.insert(id);
    for (image_t id : sorted_ids) {
      if (!images[id].IsRegistered()) continue;
      out << images[id].file_name;
      const double* c = frames[id].RigFromWorld().rotation.coeffs().data();
      for (int i = 0; i < 4; ++i) out << " " << c[(i + 3) % 4];
      out << "\n";
    }
    return 0;
  }
  // KeepLargestConnectedComponents (scene/view_graph.cc:56)
  std::unordered_map<image_t, std::vector<image_t>> adj;
  for (auto& [pid, pr] : view_graph.image_pairs) {
    adj[pr.image_id1].push_back(pr.image_id2);
    adj[pr.image_id2].push_back(pr.image_id1);
  }
  std::unordered_map<image_t, int> comp;
  std::map<int, int> comp_size;
  std::set<image_t> ids;
  for (auto& [id, im] : images) ids.insert(id);
  int ncomp = 0;
  for (image_t s : ids) {
    if (comp.count(s)) continue;
    std::queue<image_t> q;
    q.push(s);
    comp[s] = ncomp;
    while (!q.empty()) {
      image_t c = q.front(); q.pop();
      ++comp_size[ncomp];
      for (image_t nb : adj[c]) if (!comp.count(nb)) { comp[nb] = ncomp; q.push(nb); }
    }
    ++ncomp;
  }
  int best = 0;
  for (auto& [c, sz] : comp_size) if (sz > comp_size[best]) best = c;
  for (auto& [id, f] : frames) f.is_registered = comp[id] == best;
  for (auto& [pid, pr] : view_graph.image_pairs) pr.is_valid = comp[pr.image_id1] == best && comp[pr.image_id2] == best;
  if (args.count("mst_init") && args["mst_init"] == "1") {
    // extension (not in the reference CLI): BFS spanning-tree initialisation as the mapper path does
    // (global_rotation_averaging.cc:87-138); all relpose-file pairs have equal weight.
    image_t root = *ids.begin();
    for (image_t s : ids) if (comp[s] == best) { root = s; break; }
    std::queue<image_t> bfs;
    std::set<image_t> seen{root};
    bfs.push(root);
    while (!bfs.empty()) {
      image_t c = bfs.front(); bfs.pop();
      double Rc[9];
      detail::QuatToR(frames[c].RigFromWorld().rotation.coeffs().data(), Rc);
      for (image_t nb : adj[c]) {
        if (seen.count(nb)) continue;
        seen.insert(nb);
        const ImagePair& pr = view_graph.image_pairs[ImagePairToPairId(c, nb)];
        double Rr[9], Rn[9];
        detail::QuatToR(pr.cam2_from_cam1.rotation.coeffs().data(), Rr);
        for (int i = 0; i < 3; ++i)
          for (int j = 0; j < 3; ++j) {
            double s = 0;
            for (int k = 0; k < 3; ++k) s += (pr.image_id1 == c ? Rr[3 * i + k] : Rr[3 * k + i]) * Rc[3 * k + j];
            Rn[3 * i + j] = s;   // nb = image 2: R_rel R_c ; nb = image 1: R_rel^T R_c
          }
        // rotation matrix -> angle axis -> quaternion via the shim helpers
        double qw = std::sqrt(std::max(0.0, 1 + Rn[0] + Rn[4] + Rn[8])) / 2, q[4];
        if (qw > 1e-6) { q[0] = (Rn[7] - Rn[5]) / (4 * qw); q[1] = (Rn[2] - Rn[6]) / (4 * qw); q[2] = (Rn[3] - Rn[1]) / (4 * qw); q[3] = qw; }
        else {   // 180-degree case: largest diagonal pivot
          int i = 0; if (Rn[4] > Rn[0]) i = 1; if (Rn[8] > Rn[4 * i]) i = 2;
          const int j = (i + 1) % 3, k = (i + 2) % 3;
          double t = std::sqrt(Rn[4 * i] - Rn[4 * j] - Rn[4 * k] + 1.0);
          q[i] = 0.5 * t; t = 0.5 / t;
          q[3] = (Rn[3 * k + j] - Rn[3 * j + k]) * t; q[j] = (Rn[3 * j + i] + Rn[3 * i + j]) * t; q[k] = (Rn[3 * k + i] + Rn[3 * i + k]) * t;
        }
        for (int k = 0; k < 4; ++k) frames[nb].RigFromWorld().rotation.coeffs().data()[k] = q[k];
        bfs.push(nb);
      }
    }
  }
  RotationEstimatorOptions opts;
  opts.skip_initialization = true;   // exe/rotation_averager.cc:58
  opts.use_weight = use_weight;
  RotationEstimator est(opts);
  if (!est.EstimateRotations(view_graph, rigs, frames, images)) { std::cerr << "Failed to solve global rotation averaging\n"; return 1; }
  // WriteGlobalRotation (io/pose_io.cc:182-200): sorted by image id, default ostream precision
  std::ofstream out(args["output_path"]);
  for (image_t id : ids) {
    if (!images[id].IsRegistered()) continue;
    out << images[id].file_name;
    const double* c = frames[id].RigFromWorld().rotation.coeffs().data();
    for (int i = 0; i < 4; ++i) out << " " << c[(i + 3) % 4];
    out << "\n";
  }
  std::cerr << "rotation_averager: " << est.summary.num_edges << " pairs, L1 " << est.summary.l1_iterations << " IRLS "
            << est.summary.irls_iterations << " PCG " << est.summary.pcg_iterations << " its, " << est.summary.ms_total << " ms\n";
  return 0;
}

struct Flat {
  int64_t C = 0, P = 0, N = 0, K = 0;
  std::vector<int64_t> ptb;
  std::vector<int32_t> obs_cam, cam_intr, intr_model;
  std::vector<double> obs_xy, bearings, intr, quat, trans, points;
};
template <class T>
static void RW(std::fstream& f, std::vector<T>& v, size_t n, bool write) {
  if (!write) v.resize(n);
  if (n == 0) return;
  if (write) f.write(reinterpret_cast<const char*>(v.data()), n * sizeof(T));
  else f.read(reinterpret_cast<char*>(v.data()), n * sizeof(T));
}
static bool FlatIO(const std::string& path, Flat& p, bool write) {
  std::fstream f(path, std::ios::binary | (write ? std::ios::out : std::ios::in));
  if (!f) return false;
  int64_t hdr[4] = {p.C, p.P, p.N, p.K};
  if (write) f.write(reinterpret_cast<const char*>(hdr), sizeof(hdr));
  else { f.read(reinterpret_cast<char*>(hdr), sizeof(hdr)); p.C = hdr[0]; p.P = hdr[1]; p.N = hdr[2]; p.K = hdr[3]; }
  RW(f, p.ptb, p.P + 1, write); RW(f, p.obs_cam, p.N, write); RW(f, p.obs_xy, 2 * p.N, write); RW(f, p.bearings, 3 * p.N, write);
  RW(f, p.cam_intr, p.C, write); RW(f, p.intr_model, p.K, write); RW(f, p.intr, p.K * 12, write);
  RW(f, p.quat, 4 * p.C, write); RW(f, p.trans, 3 * p.C, write); RW(f, p.points, 3 * p.P, write);
  return (bool)f;
}

static int RunFlat(int argc, char** argv, bool is_ba) {
  auto args = ParseArgs(argc, argv, 2);
  Flat p;
  if (!args.count("problem") || !args.count("output") || !FlatIO(args["problem"], p, false)) {
    std::cerr << "usage: b200sfm_cli " << (is_ba ? "ba" : "gp") << " --problem IN.bin --output OUT.bin\n";
    return 2;
  }
  // what ConvertDatabaseToGlomap would hand over: ids start at 1
  std::unordered_map<rig_t, Rig> rigs;
  std::unordered_map<camera_t, Camera> cameras;
  std::unordered_map<frame_t, Frame> frames;
  std::unordered_map<image_t, Image> images;
  std::unordered_map<track_t, Track> tracks;
  ViewGraph vg;
  static const int nparams[4] = {3, 4, 4, 5};
  for (int64_t k = 0; k < p.K; ++k) {
    Camera c;
    c.camera_id = (camera_t)(k + 1);
    c.model_id = p.intr_model[k];
    c.params.assign(p.intr.begin() + k * 12, p.intr.begin() + k * 12 + nparams[c.model_id]);
    cameras[c.camera_id] = c;
  }
  for (int64_t i = 0; i < p.C; ++i) {
    Frame f;
    f.frame_id = (frame_t)(i + 1);
    for (int k = 0; k < 4; ++k) f.RigFromWorld().rotation.coeffs().data()[k] = p.quat[4 * i + k];
    for (int k = 0; k < 3; ++k) f.RigFromWorld().translation[k] = p.trans[3 * i + k];
    frames[f.frame_id] = f;
    Image im;
    im.image_id = (image_t)(i + 1); im.frame_id = f.frame_id; im.camera_id = (camera_t)(p.cam_intr[i] + 1);
    images[im.image_id] = im;
  }
  for (auto& [id, im] : images) im.frame_ptr = &frames[im.frame_id];
  for (int64_t t = 0; t < p.P; ++t) {
    Track tr;
    tr.track_id = (track_t)(t + 1);
    for (int k = 0; k < 3; ++k) tr.xyz[k] = p.points[3 * t + k];
    for (int64_t o = p.ptb[t]; o < p.ptb[t + 1]; ++o) {
      Image& im = images[(image_t)(p.obs_cam[o] + 1)];
      tr.observations.emplace_back(im.image_id, (feature_t)im.features.size());
      im.features.push_back({p.obs_xy[2 * o], p.obs_xy[2 * o + 1]});
      im.features_undist.push_back({p.bearings[3 * o], p.bearings[3 * o + 1], p.bearings[3 * o + 2]});
    }
    tracks[tr.track_id] = tr;
  }
  bool ok;
  if (is_ba) {
    BundleAdjusterOptions o;
    o.optimize_intrinsics = args.count("optimize_intrinsics") && args["optimize_intrinsics"] == "1";
    if (args.count("pcg_tol")) o.pcg_rel_tolerance = std::stod(args["pcg_tol"]);
    BundleAdjuster ba(o);
    if (args.count("fix_rotations") && args["fix_rotations"] == "1") {
      // GlobalMapper's staged use (controllers/global_mapper.cc:204-221): rotations constant first, then free
      ba.GetOptions().optimize_rotations = false;
      ok = ba.Solve(rigs, cameras, frames, images, tracks);
      ba.GetOptions().optimize_rotations = true;
      ok = ok && ba.Solve(rigs, cameras, frames, images, tracks);
    } else {
      ok = ba.Solve(rigs, cameras, frames, images, tracks);
    }
    std::cerr << "ba: " << ba.summary.iterations << " LM its, cost " << ba.summary.initial_cost << " -> " << ba.summary.final_cost << "\n";
  } else {
    GlobalPositionerOptions o;
    if (args.count("pcg_tol")) o.pcg_rel_tolerance = std::stod(args["pcg_tol"]);
    GlobalPositioner gp(o);
    ok = gp.Solve(vg, rigs, cameras, frames, images, tracks);
    std::cerr << "gp: " << gp.summary.iterations << " LM its, cost " << gp.summary.initial_cost << " -> " << gp.summary.final_cost << "\n";
  }
  if (!ok) { std::cerr << "solve failed\n"; return 1; }
  for (int64_t i = 0; i < p.C; ++i) {
    const Frame& f = frames[(frame_t)(i + 1)];
    for (int k = 0; k < 4; ++k) p.quat[4 * i + k] = f.RigFromWorld().rotation.coeffs().data()[k];
    for (int k = 0; k < 3; ++k) p.trans[3 * i + k] = f.RigFromWorld().translation[k];
  }
  for (int64_t t = 0; t < p.P; ++t)
    for (int k = 0; k < 3; ++k) p.points[3 * t + k] = tracks[(track_t)(t + 1)].xyz[k];
  for (int64_t k = 0; k < p.K; ++k) {   // refined intrinsics (optimize_intrinsics): BundleAdjuster writes camera.params in place
    const Camera& c = cameras[(camera_t)(k + 1)];
    for (size_t j = 0; j < c.params.size() && j < 12; ++j) p.intr[k * 12 + j] = c.params[j];
  }
  return FlatIO(args["output"], p, true) ? 0 : 1;
}

int main(int argc, char** argv) {
  // glomap/glomap.cc:41-75: dispatch on argv[1]
  const std::string cmd = argc > 1 ? argv[1] : "";
  if (cmd == "rotation_averager") return RunRotationAverager(argc, argv);
  if (cmd == "ba") return RunFlat(argc, argv, true);
  if (cmd == "gp") return RunFlat(argc, argv, false);
  std::cerr << "b200sfm_cli <rotation_averager|ba|gp> ...\n";
  return 2;
}
