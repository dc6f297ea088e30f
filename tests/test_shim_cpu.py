"""Host-side logic of the C++ estimator shim (glomap_b200/host/estimators_shim.h) on a box without a GPU: the shim is
linked against a recording test double of the C ABI (tests/shim_mock/mock_b200sfm.c) and driven over a small world with
a two-camera rig in three frames plus a trivial frame (tests/shim_mock/shim_driver.cc).  Checked: sorted-id flattening,
the (rig, camera) sensor table and per-observation frame / sensor indices of the known-rig BA path
(bundle_adjustment.cc:147-161), the RigBATA terms of global positioning (global_positioning.cc:294-296,339-345,
313-316) and the folding of image pairs onto frames for rotation averaging (global_rotation_averaging.cc:274-309)."""
import os
import subprocess

import numpy as np

from glomap_b200 import geometry as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _quat(ax, ay, az, ang):
    a = np.array([ax, ay, az], float)
    return np.concatenate([a / np.linalg.norm(a) * np.sin(ang / 2), [np.cos(ang / 2)]])


def _run(tmp_path, *args):
    lib, exe, dump = tmp_path / "libb200sfm_mock.so", tmp_path / "shim_driver", tmp_path / "dump.txt"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "shim_mock", "shim_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe)] + list(args), env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0 and "shim driver ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    calls, cur = [{"_name": "_stdout", "lines": r.stdout.splitlines()}], None
    for line in dump.read_text().splitlines():
        f = line.split()
        if f[0] == "call":
            cur = {"_name": f[1]}
            calls.append(cur)
        else:
            cur[f[0]] = np.array([float(x) for x in f[2:]])
            assert len(cur[f[0]]) == int(f[1])
    return calls


def stdout_line(calls, key):
    (line,) = [l for l in calls_stdout[0] if l.startswith(key + " ")]
    return line.split()[1:]


calls_stdout = [None]


def test_shim_flattening_of_a_rig_world(tmp_path):
    calls = _run(tmp_path)
    calls_stdout[0] = calls[0]["lines"]
    calls = calls[1:]
    assert [c["_name"] for c in calls] == ["ba_problem_create_rig", "ba_problem_set_state", "ba_problem_solve",
                                           "gp_problem_create", "gp_problem_set_rig_terms", "gp_problem_solve", "ra_solve",
                                           "ra_solve_gravity", "ba_solve", "ra_solve",
                                           "ba_problem_create_rig", "ba_problem_set_state", "ba_problem_set_sensor_variable",
                                           "ba_problem_solve", "ra_solve_rig",
                                           "gp_problem_create", "gp_problem_set_rig_terms", "gp_problem_set_rig_unknown",
                                           "gp_problem_solve"]
    # ---- the world of shim_driver.cc ---------------------------------------------------------------------------
    img_ids = [101, 102, 201, 202, 301, 302, 401]
    kimg = {i: k for k, i in enumerate(img_ids)}
    frame_of = {101: 0, 102: 0, 201: 1, 202: 1, 301: 2, 302: 2, 401: 3}
    sensor_of = {101: 0, 102: 1, 201: 0, 202: 1, 301: 0, 302: 1, 401: 2}       # sorted (rig, camera): (1,1) (1,2) (2,3)
    q_c2r, t_c2r = _quat(0.2, 1.0, -0.3, 0.35), np.array([0.4, -0.1, 0.05])
    q_f = np.array([_quat(0.1 * k, 1.0, 0.2, 0.3 + 0.4 * k) for k in range(4)])
    tracks = {7: [(101, 0), (202, 1), (301, 2), (401, 3)], 3: [(102, 1), (201, 2), (302, 3), (401, 0)],
              5: [(101, 2), (102, 3), (201, 0), (301, 1)]}
    order = sorted(tracks)                                                        # tracks in sorted-id order
    obs = [o for t in order for o in tracks[t]]
    # ---- BA: known-rig entry -----------------------------------------------------------------------------------
    ba = calls[0]
    assert ba["dims"].tolist() == [4, 3, 12, 3, 3, 1]                            # F P N K S min_views (1: the shim applied the rule itself)
    assert ba["pt_obs_begin"].tolist() == [0, 4, 8, 12]
    assert ba["obs_frame"].tolist() == [frame_of[i] for i, _ in obs]
    assert ba["obs_sensor"].tolist() == [sensor_of[i] for i, _ in obs]
    want_xy = np.array([[10.0 * kimg[i] + f, 20.0 * kimg[i] + 2.0 * f] for i, f in obs])
    assert np.array_equal(ba["obs_xy"].reshape(-1, 2), want_xy)
    sq = ba["sensor_quat"].reshape(3, 4)
    assert np.abs(sq[0] - [0, 0, 0, 1]).max() == 0 and np.abs(sq[2] - [0, 0, 0, 1]).max() == 0   # reference / trivial: identity
    assert np.abs(sq[1] - q_c2r).max() < 1e-15 and np.abs(ba["sensor_trans"].reshape(3, 3)[1] - t_c2r).max() == 0
    assert ba["sensor_intr"].tolist() == [0, 1, 2] and ba["intr_model"].tolist() == [0, 0, 0]
    assert ba["mask"].tolist() == [3, 0, 0, 0]                                    # first frame constant (.cc:261-266)
    # ---- GP: RigBATA terms -------------------------------------------------------------------------------------
    gp, terms = calls[3], calls[4]
    assert gp["dims"].tolist() == [4, 3, 12] and gp["obs_cam"].tolist() == ba["obs_frame"].tolist()
    Rf = G.quat_xyzw_to_rotmat(q_f)
    Rs = G.quat_xyzw_to_rotmat(np.array([[0, 0, 0, 1.0], q_c2r, [0, 0, 0, 1.0]]))
    ts = np.array([[0, 0, 0], t_c2r, [0, 0, 0]])
    want_dir, want_off, want_cal = [], [], []
    for i, f in obs:
        k = kimg[i]
        b = np.array([0.01 * k - 0.02 * f, 0.03 * f - 0.01 * k, 1.0]); b /= np.linalg.norm(b)
        Rcw = Rs[sensor_of[i]] @ Rf[frame_of[i]]
        want_dir.append(Rcw.T @ b); want_off.append(Rcw.T @ ts[sensor_of[i]])
        want_cal.append(0 if sensor_of[i] == 1 else 1)                           # camera 2 has no prior focal length
    assert np.abs(gp["obs_dir"].reshape(-1, 3) - np.array(want_dir)).max() < 1e-14
    assert np.abs(terms["obs_offset"].reshape(-1, 3) - np.array(want_off)).max() < 1e-14
    assert terms["obs_calibrated"].tolist() == want_cal
    # ---- RA: pairs folded onto frames, the same-frame pair (101,102) dropped -------------------------------------
    ra = calls[6]
    assert ra["dims"].tolist() == [4, 4]
    assert ra["ei"].tolist() == [0, 0, 1, 2] and ra["ej"].tolist() == [1, 2, 2, 3]
    assert ra["weight"].tolist() == [2.0, 3.0, 4.0, 5.0]
    R21 = G.quat_xyzw_to_rotmat(np.array([_quat(1.0, 0.1 * k, -0.2, 0.2 + 0.1 * k) for k in range(5)]))
    want_R = [R21[1], R21[2] @ Rs[1], Rs[1].T @ R21[3] @ Rs[1], R21[4]]
    assert np.abs(ra["R_rel"].reshape(-1, 3, 3) - np.array(want_R)).max() < 1e-14
    assert np.abs(G.so3_exp(ra["theta"].reshape(-1, 3)) - Rf).max() < 1e-13       # initial angle-axis of the frames
    # ---- use_gravity: frames 20 and 40 (indices 1, 3) are 1-DoF; host preparation of .cc:207-217,311-326 ------------
    from glomap_b200 import estimators as E
    rg = calls[7]
    assert rg["dims"].tolist() == [4, 4, 1]                                       # fixed frame = first gravity frame
    assert rg["has_gravity"].tolist() == [0, 1, 0, 1]
    Ra = {1: E.get_align_rot([0.1, 1.0, 0.05]), 3: E.get_align_rot([0.0, 1.0, 0.0])}
    # (the first RA call zeroed nothing: the mock leaves theta alone and the shim wrote the same rotations back)
    th = rg["theta"].reshape(-1, 3)
    for i in (1, 3):
        phi = G.so3_log((Ra[i].T @ Rf[i])[None])[0, 1]
        assert np.abs(th[i] - [0.0, phi, 0.0]).max() < 1e-12
    for i in (0, 2):
        assert np.abs(G.so3_exp(th[i][None])[0] - Rf[i]).max() < 1e-12
    want_g = []
    for (a, b), R in zip([(0, 1), (0, 2), (1, 2), (2, 3)], want_R):
        if a in Ra:
            R = R @ Ra[a]
        if b in Ra:
            R = Ra[b].T @ R
        want_g.append(R)
    assert np.abs(rg["R_rel"].reshape(-1, 3, 3) - np.array(want_g)).max() < 1e-13
    # ConvertResults for a gravity frame: R = R_align * RotY(phi) -- only the rotation about gravity survives
    q20 = np.array([float(x) for x in stdout_line(calls, "q20")])
    phi = th[1][1]
    want20 = Ra[1] @ G.so3_exp(np.array([[0.0, phi, 0.0]]))[0]
    assert np.abs(G.quat_xyzw_to_rotmat(q20[None])[0] - want20).max() < 1e-12
    # ---- trivial frames still take the one-shot entry -------------------------------------------------------------
    one = calls[8]
    assert one["dims"].tolist() == [1, 1, 3, 1] and one["obs_cam"].tolist() == [0, 0, 0] and one["cam_intr"].tolist() == [0]
    assert one["flags"].tolist() == [1, 1, 0]
    # ---- InitializeFromMaximumSpanningTree inside EstimateRotations (.cc:60-63, 87-138; math/tree.cc:78-153) -------------
    # inliers = 10 + k: Kruskal keeps all five pairs (a forest: 202-302 is not connected to the root 101); BFS from 101
    mst = calls[9]
    q21 = np.array([_quat(1.0, 0.1 * k, -0.2, 0.2 + 0.1 * k) for k in range(5)])
    Rrel = G.quat_xyzw_to_rotmat(q21)
    R = {101: np.eye(3)}
    R[102] = Rrel[0] @ R[101]            # pair (101,102): 2_R_w = 2_R_1 1_R_w
    R[201] = Rrel[1] @ R[101]
    R[301] = Rrel[2] @ R[102]
    R[401] = Rrel[4] @ R[301]

    def avg(Rs_):
        qs = np.array([G.rotmat_to_quat_xyzw(r[None])[0] for r in Rs_])
        w, v = np.linalg.eigh(qs.T @ qs)
        return G.quat_xyzw_to_rotmat(v[:, -1][None])[0]

    want = [avg([R[101], Rs[1].T @ R[102]]), R[201], R[301], R[401]]       # frame 10 averages its two images (rotation_initializer.cc:95-117)
    got = G.so3_exp(mst["theta"].reshape(-1, 3))
    assert np.abs(got - np.array(want)).max() < 1e-12, np.abs(got - np.array(want)).max()
    # ---- optimize_rig_poses: the non-reference sensor is marked as an unknown and its result lands in the rig ----------
    rp = calls[10:14]
    assert rp[0]["dims"].tolist() == [4, 3, 12, 3, 3, 1]
    assert rp[2]["sensor_variable"].tolist() == [0, 1, 0]                    # sensors sorted: (1,1) ref, (1,2), (2,3) ref
    c2r = np.array([float(x) for x in stdout_line(calls, "c2r")])
    assert np.allclose(c2r, [0, 0, 0.70710678118654757, 0.70710678118654757, 8.0, 8.0, 9.0], atol=0)   # the mock's pose of sensor 1
    assert stdout_line(calls, "nrig1") == ["1"]                              # no entry was created for the reference sensor
    # ---- rotation averaging with an uncalibrated sensor (camera 2 of rig 1): one extra rotation node -----------------
    ru = calls[14]
    assert ru["dims"].tolist() == [4, 1, 5, 0]                              # frames, unknown cameras, edges, fixed frame
    # pairs in ascending pair id: (101,102) (101,201) (102,301) (202,302) (301,401); the pair inside frame 10 is KEPT
    assert ru["ei"].tolist() == [0, 0, 0, 1, 2] and ru["ej"].tolist() == [0, 1, 2, 2, 3]
    assert ru["eci"].tolist() == [-1, -1, 4, 4, -1] and ru["ecj"].tolist() == [4, -1, -1, 4, -1]
    assert np.abs(ru["R_rel"].reshape(-1, 3, 3) - Rrel).max() < 1e-15       # no known cam_from_rig factor is left in any pair
    assert ru["cam_frames_begin"].tolist() == [0, 3] and ru["cam_frames"].tolist() == [0, 1, 2]
    assert np.abs(ru["theta"].reshape(-1, 3)[4]).max() == 0                 # no prior value: zero (.cc:239-241)
    # ---- global positioning with that sensor (translation NaN): RigUnknownBATA -------------------------------------------
    gu = calls[17]
    assert gu["dims"].tolist() == [1]
    assert gu["obs_unknown_sensor"].tolist() == [0 if sensor_of[i] == 1 else -1 for i, _ in obs]   # the images of (rig 1, camera 2)
    assert np.array_equal(gu["centers"], np.zeros(3))                      # optimize_positions = false: no random draw
    off = calls[16]["obs_offset"].reshape(-1, 3)
    assert np.abs(off[[sensor_of[i] == 1 for i, _ in obs]]).max() == 0      # no known offset is left for those observations
    # ConvertResults: translation = -(R_cr u) with the mock's centre u = (1, 2, 3) and R_cr = the 0.3 rad z-rotation RA estimated
    c3, s3 = np.cos(0.3), np.sin(0.3)
    want_t = -(np.array([[c3, -s3, 0], [s3, c3, 0], [0, 0, 1]]) @ np.array([1.0, 2.0, 3.0]))
    assert np.allclose([float(x) for x in stdout_line(calls, "gpt2")], want_t, atol=1e-15)
    est2 = stdout_line(calls, "est2")
    assert np.allclose([float(x) for x in est2[:4]], [0, 0, np.sin(0.15), np.cos(0.15)], atol=1e-15) and est2[4] == "1"


def test_shim_pose_blocks_sensors_and_draws_of_a_partly_observed_world(tmp_path):
    """The second world of shim_driver.cc: frame 5 is seen by no track, track 2 observes image 999 that is not in `images`,
    track 4 has two observations (< min_num_view_per_track = 3), and the NaN-translation sensors (rig 1, camera 3) and
    (rig 1, camera 2) are first met in that order."""
    calls = _run(tmp_path, "pinned")
    out = {l.split()[0]: np.array([float(x) for x in l.split()[1:]]) for l in calls[0]["lines"] if l != "shim driver ok"}
    calls = calls[1:]
    assert [c["_name"] for c in calls] == ["ba_problem_create_rig", "ba_problem_set_state", "ba_problem_solve",
                                           "gp_problem_create", "gp_problem_set_rig_terms", "gp_problem_set_rig_unknown",
                                           "gp_problem_solve"]
    frame_of = {101: 1, 102: 1, 103: 1, 201: 2, 202: 2, 203: 2}                 # frames 5, 10, 20
    # the observation of image 999 is dropped, the short track keeps its point but no observation (bundle_adjustment.cc:122-125)
    obs = [203, 102, 201] + [101, 102, 103, 201]
    ba = calls[0]
    assert ba["dims"].tolist() == [3, 3, 7, 3, 3, 1]                            # a pose block for frame 5 too
    assert ba["pt_obs_begin"].tolist() == [0, 3, 3, 7]
    assert ba["obs_frame"].tolist() == [frame_of[i] for i in obs]
    assert ba["obs_sensor"].tolist() == [i % 10 - 1 for i in obs]             # sorted (rig, camera): (1,1) (1,2) (1,3)
    assert ba["mask"].tolist() == [0, 3, 0]                                    # gauge: the first frame with an observation
    assert np.isnan(ba["sensor_trans"].reshape(3, 3)[1:]).all()
    gp, unk = calls[3], calls[5]
    assert gp["dims"].tolist() == [3, 3, 7] and gp["obs_cam"].tolist() == ba["obs_frame"].tolist()
    assert gp["pt_obs_begin"].tolist() == [0, 3, 3, 7]
    # unknown sensors numbered in order of first appearance: camera 3 -> 0, camera 2 -> 1
    assert unk["dims"].tolist() == [2]
    assert unk["obs_unknown_sensor"].tolist() == [{1: -1, 2: 1, 3: 0}[i % 10] for i in obs]
    # one mt19937: 3 frame positions, then the points of tracks 2 and 6 (not the short track 4), then the sensor centres
    assert np.array_equal(unk["centers"], out["draws"][15:21])
    # ConvertResults in sorted order with the mock's centre (1 + s, 2, 3) of unknown sensor s: translation = -(R_cr u)
    for cam, s in ((2, 1), (3, 0)):
        q = _quat(0.3 * cam, 1.0, -0.2, 0.1 * cam)
        assert np.abs(out["cfr%d" % cam][:4] - q).max() < 1e-15
        want = -(G.quat_xyzw_to_rotmat(q[None])[0] @ np.array([1.0 + s, 2.0, 3.0]))
        assert np.abs(out["cfr%d" % cam][4:] - want).max() < 1e-14


def test_shim_typechecks_against_the_glomap_api():
    """INTEGRATION.md section 2: inside a glomap build the shim is compiled with -DB200SFM_WITH_GLOMAP against the real scene
    types.  Those need Eigen + COLMAP (absent here), so the branch is type-checked against tests/shim_mock/glomap_stub, which
    restates the members the shim touches with their real spellings and types (Eigen::Quaterniond::coeffs().data(),
    Eigen::Vector3d, enum class CameraModelId, sensor_t, std::optional<Rigid3d> MaybeSensorFromRig, Frame::is_registered)."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(ROOT, "tests", "shim_mock", "glomap_stub"), "-I" + os.path.join(ROOT, "glomap_b200", "host"),
                        "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "shim_mock", "shim_typecheck.cc")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
