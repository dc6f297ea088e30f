"""The C++ shim's TrackFilter, UndistortImages and NormalizeReconstruction without a GPU: driven over a recording test double
(tests/shim_mock/mock_processors.c) through tests/shim_mock/processors_driver.cc, the arrays they flatten (sorted-id order,
the rig layout, the calibrated flags, the variant of the reprojection filter), the write-back of the double's results,
the failure paths (nothing changes), and the type-check against the glomap API."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK = os.path.join(ROOT, "tests", "shim_mock")
HOST = os.path.join(ROOT, "glomap_b200", "host")
IDENT = [0.0, 0.0, 0.0, 1.0]


# ---- the world file of processors_driver.cc -------------------------------------------------------------------------
def write_world(path, w):
    """w: dict of lists -- cameras (id, model, prior, params), rigs (id, ref_camera, [(camera, q4, t3)]), frames
    (id, rig, registered, q4, t3), images (id, camera, frame, trivial, features [[x, y]], features_undist [[x, y, z]]),
    tracks (id, xyz3, [(image, feature)])."""
    r = lambda v: " ".join(repr(float(x)) for x in v)   # noqa: E731
    out = [f"cameras {len(w['cameras'])}"]
    out += [f"{c} {m} {int(p)} {len(par)} {r(par)}" for c, m, p, par in w["cameras"]]
    out.append(f"rigs {len(w['rigs'])}")
    out += [f"{i} {ref} {len(s)} " + " ".join(f"{c} {r(q)} {r(t)}" for c, q, t in s) for i, ref, s in w["rigs"]]
    out.append(f"frames {len(w['frames'])}")
    out += [f"{i} {rig} {int(reg)} {r(q)} {r(t)}" for i, rig, reg, q, t in w["frames"]]
    out.append(f"images {len(w['images'])}")
    for i, c, f, triv, feat, und in w["images"]:
        out.append(f"{i} {c} {f} {int(triv)} {len(feat)} {r([v for x in feat for v in x])} {len(und)} {r([v for x in und for v in x])}")
    out.append(f"tracks {len(w['tracks'])}")
    out += [f"{i} {r(xyz)} {len(obs)} " + " ".join(f"{a} {b}" for a, b in obs) for i, xyz, obs in w["tracks"]]
    path.write_text("\n".join(out) + "\n")


def parse_output(text):
    """{'result': [...], 'sensor': {(rig, cam): [q4 + t3]}, 'frame': {id: [q4 + t3]}, 'image': {id: [[b3], ...]},
    'track': {id: (xyz3, [(image, feature)])}} of the driver's stdout."""
    res = {"sensor": {}, "frame": {}, "image": {}, "track": {}}
    for line in text.splitlines():
        tok = line.split()
        if tok[0] == "result":
            res["result"] = [float(v) for v in tok[1:]]
        elif tok[0] == "sensor":
            res["sensor"][(int(tok[1]), int(tok[2]))] = [float(v) for v in tok[3:]]
        elif tok[0] == "frame":
            res["frame"][int(tok[1])] = [float(v) for v in tok[2:]]
        elif tok[0] == "image":
            v = [float(x) for x in tok[3:]]
            res["image"][int(tok[1])] = [v[3 * k:3 * k + 3] for k in range(int(tok[2]))]
        elif tok[0] == "track":
            n = int(tok[5])
            res["track"][int(tok[1])] = ([float(v) for v in tok[2:5]], [(int(tok[6 + 2 * k]), int(tok[7 + 2 * k])) for k in range(n)])
    return res


def records(dump):
    calls, cur = [], None
    if not dump.exists():
        return calls
    for line in dump.read_text().splitlines():
        if line.startswith("call "):
            cur = {}
            calls.append((line.split()[1], cur))
            continue
        name, n, *vals = line.split()
        assert len(vals) == int(n)
        cur[name] = [float(v) for v in vals]
    return calls


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("mock")
    lib, exe = d / "libb200sfm.so", d / "processors_driver"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-Wall", "-Werror", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"),
                    "-o", str(lib), os.path.join(MOCK, "mock_processors.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + HOST, "-o", str(exe), os.path.join(MOCK, "processors_driver.cc"),
                    str(lib), "-Wl,-rpath," + str(d)], check=True, capture_output=True)
    return exe


def run(driver, tmp_path, w, *op):
    world, dump = tmp_path / "world.txt", tmp_path / "dump.txt"
    write_world(world, w)
    if dump.exists():
        dump.unlink()
    r = subprocess.run([str(driver), str(world)] + [str(a) for a in op], env=dict(os.environ, MOCK_DUMP=str(dump)),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return parse_output(r.stdout), records(dump), r.stderr


# ---- hand worlds -----------------------------------------------------------------------------------------------------
def trivial_world():
    """Images 2 (camera 3, SIMPLE_RADIAL, no prior focal) and 1 (camera 7, SIMPLE_PINHOLE, prior) on frames 20 and 10;
    camera 9 (model 4) is used by no image.  Tracks 50, 40 and the empty 60 (map order is not sorted order)."""
    return dict(
        cameras=[(7, 0, True, [100.0, 5.0, 6.0]), (3, 2, False, [200.0, 1.0, 2.0, 0.1]), (9, 4, True, [1.0] * 8)],
        rigs=[],
        frames=[(20, 0, True, [0.0, 0.6, 0.0, 0.8], [1.0, 2.0, 3.0]), (10, 0, True, IDENT, [4.0, 5.0, 6.0])],
        images=[(2, 3, 20, True, [[20.0, 21.0], [22.0, 23.0]], [[0.1, 0.2, 0.9], [0.3, 0.4, 0.8]]),
                (1, 7, 10, True, [[10.0, 11.0], [12.0, 13.0], [14.0, 15.0]], [[0.5, 0.0, 0.8], [0.0, 0.5, 0.8], [0.6, 0.0, 0.8]])],
        tracks=[(50, [1.0, 2.0, 3.0], [(2, 1), (1, 0), (1, 2)]), (40, [4.0, 5.0, 6.0], [(1, 1), (2, 0)]), (60, [7.0, 8.0, 9.0], [])])


def rig_world():
    """Rig 5: reference camera 7 and camera 3 with a known cam_from_rig; frames 20 and 10 of rig 5, two images each
    (4 = camera 3 of frame 10, 1 = camera 7 of frame 10, 2 = camera 3 of frame 20, 3 = camera 7 of frame 20)."""
    w = trivial_world()
    w["rigs"] = [(5, 7, [(3, [0.0, 0.0, 0.6, 0.8], [0.5, -0.25, 1.0])])]
    w["frames"] = [(20, 5, True, [0.0, 0.6, 0.0, 0.8], [1.0, 2.0, 3.0]), (10, 5, True, IDENT, [4.0, 5.0, 6.0])]
    f2 = [[30.0, 31.0], [32.0, 33.0]]
    u2 = [[0.0, 0.0, 1.0], [0.6, 0.0, 0.8]]
    w["images"] = [(4, 3, 10, False, f2, u2), (1, 7, 10, True, f2, u2), (2, 3, 20, False, f2, u2), (3, 7, 20, True, f2, u2)]
    w["tracks"] = [(50, [1.0, 2.0, 3.0], [(2, 1), (1, 0), (4, 1)]), (40, [4.0, 5.0, 6.0], [(3, 1), (4, 0)])]
    return w


def _unchanged(before, after):
    for k in ("sensor", "frame", "image", "track"):
        assert after[k] == before[k], k


# ---- trivial frames --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", [("reprojection", 2.5, 0), ("reprojection", 0.01, 1), ("angle", 1.5)])
def test_observation_filters_on_trivial_frames(driver, tmp_path, op):
    base, _, _ = run(driver, tmp_path, trivial_world(), "undistort", 0)
    out, calls, _ = run(driver, tmp_path, trivial_world(), *op)
    names = [c for c, _ in calls]
    kind = {("reprojection", 0): "filter_reprojection", ("reprojection", 1): "filter_reprojection_normalized"}.get(
        (op[0], op[2]) if op[0] == "reprojection" else None, "filter_angle")
    assert names == ["create", "set_state", kind]
    cr, st, fl = calls[0][1], calls[1][1], calls[2][1]
    pixels = kind == "filter_reprojection"
    # tracks 40, 50, 60 in sorted order; pose blocks = images 1 (frame 10), 2 (frame 20); min_num_view_per_track = 1
    assert cr["dims"] == [2, 3, 5, 2 if pixels else 1, 1]
    assert cr["ptb"] == [0, 2, 5, 5]
    assert cr["obs_cam"] == [0, 1, 1, 0, 0]
    # the pixel filter reads the cameras of the images (3 -> block 0, 7 -> block 1); the others one placeholder block
    if pixels:
        assert cr["obs_xy"] == [12, 13, 20, 21, 22, 23, 10, 11, 14, 15]
        assert cr["cam_intr"] == [1, 0] and cr["intr_model"] == [2, 0]
        assert st["intr"][:12] == [200, 1, 2, 0.1] + [0] * 8 and st["intr"][12:] == [100, 5, 6] + [0] * 9
    else:
        assert cr["obs_xy"] == [0] * 10
        assert cr["cam_intr"] == [0, 0] and cr["intr_model"] == [0]
    assert st["quat"] == IDENT + [0, 0.6, 0, 0.8] and st["trans"] == [4, 5, 6, 1, 2, 3]
    assert st["points"] == [4, 5, 6, 1, 2, 3, 7, 8, 9]
    assert fl["threshold"] == [op[1]]
    if kind == "filter_reprojection":
        assert fl["bearings"] == [] and fl["calibrated"] == []
    else:   # features_undist of the observations, in track order
        assert fl["bearings"] == [0, 0.5, 0.8, 0.1, 0.2, 0.9, 0.3, 0.4, 0.8, 0.5, 0, 0.8, 0.6, 0, 0.8]
        assert fl["calibrated"] == ([1, 0] if kind == "filter_angle" else [])
    # the double keeps o % 3 != 1: track 40 loses (2, 0), track 50 loses (1, 2); the count is the double's
    assert out["result"] == [7]
    assert out["track"][40][1] == [(1, 1)] and out["track"][50][1] == [(2, 1), (1, 0)] and out["track"][60][1] == []
    for t in (40, 50, 60):
        assert out["track"][t][0] == base["track"][t][0]
    for k in ("frame", "image"):
        assert out[k] == base[k]


def test_triangulation_angle_clears_rejected_tracks(driver, tmp_path):
    out, calls, _ = run(driver, tmp_path, trivial_world(), "triangulation", 2.0)
    assert [c for c, _ in calls] == ["create", "set_state", "filter_triangulation_angle"]
    assert calls[0][1]["intr_model"] == [0] and calls[2][1]["threshold"] == [2.0]
    # the double keeps p % 2 == 0: tracks 40 and 60 stay, 50 loses every observation
    assert out["result"] == [5]
    assert out["track"][40][1] == [(1, 1), (2, 0)] and out["track"][50][1] == [] and out["track"][60][1] == []


# ---- rigs ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("op", [("reprojection", 2.5, 0), ("angle", 1.5)])
def test_observation_filters_on_rigs(driver, tmp_path, op):
    out, calls, _ = run(driver, tmp_path, rig_world(), *op)
    assert [c for c, _ in calls][:2] == ["create_rig", "set_state"]
    cr, st, fl = calls[0][1], calls[1][1], calls[2][1]
    pixels = op[0] == "reprojection"
    # frames 10, 20; sensors (5, 3) -> 0 with its cam_from_rig, (5, 7) -> 1 the reference (identity)
    assert cr["dims"] == [2, 2, 5, 2 if pixels else 1, 2, 1]
    assert cr["ptb"] == [0, 2, 5]
    assert cr["obs_frame"] == [1, 0, 1, 0, 0] and cr["obs_sensor"] == [1, 0, 0, 1, 0]
    assert cr["sensor_q"] == [0, 0, 0.6, 0.8] + IDENT and cr["sensor_t"] == [0.5, -0.25, 1, 0, 0, 0]
    assert cr["sensor_intr"] == ([0, 1] if pixels else [0, 0]) and cr["intr_model"] == ([2, 0] if pixels else [0])
    assert st["quat"] == IDENT + [0, 0.6, 0, 0.8] and st["trans"] == [4, 5, 6, 1, 2, 3]
    if pixels:
        assert cr["obs_xy"] == [32, 33, 30, 31, 32, 33, 30, 31, 32, 33]
    else:   # calibrated per sensor: camera 3 has no prior focal, camera 7 has
        assert fl["calibrated"] == [0, 1]
        assert fl["bearings"] == [0.6, 0, 0.8, 0, 0, 1, 0.6, 0, 0.8, 0, 0, 1, 0.6, 0, 0.8]
    assert out["result"] == [7]
    assert out["track"][40][1] == [(3, 1)] and out["track"][50][1] == [(2, 1), (1, 0)]


# ---- UndistortImages -------------------------------------------------------------------------------------------------
def test_undistort_skips_undistorted_images_unless_clean(driver, tmp_path):
    w = trivial_world()
    w["images"][0] = w["images"][0][:5] + ([],)          # image 2: no features_undist yet
    out, calls, _ = run(driver, tmp_path, w, "undistort", 0)
    assert [c for c, _ in calls] == ["undistort_features"]
    u = calls[0][1]
    assert u["intr_model"] == [2] and u["intr"] == [200, 1, 2, 0.1] + [0] * 8
    assert u["feat_intr"] == [0, 0] and u["xy"] == [20, 21, 22, 23]
    assert out["image"][2] == [[0, 0.5, 0], [1, 0.5, -1]]
    assert out["image"][1] == [[0.5, 0, 0.8], [0, 0.5, 0.8], [0.6, 0, 0.8]]      # already full: kept
    out, calls, _ = run(driver, tmp_path, w, "undistort", 1)
    u = calls[0][1]
    # every image, sorted ids 1, 2; cameras 3 -> block 0, 7 -> block 1
    assert u["intr_model"] == [2, 0] and u["feat_intr"] == [1, 1, 1, 0, 0]
    assert u["xy"] == [10, 11, 12, 13, 14, 15, 20, 21, 22, 23]
    assert out["image"][1] == [[0, 0.5, 0], [1, 0.5, -1], [2, 0.5, -2]] and out["image"][2] == [[3, 0.5, -3], [4, 0.5, -4]]
    # nothing to do: no device call
    _, calls, _ = run(driver, tmp_path, trivial_world(), "undistort", 0)
    assert calls == []


# ---- NormalizeReconstruction -----------------------------------------------------------------------------------------
def test_normalize_on_rigs(driver, tmp_path):
    w = rig_world()
    w["frames"].append((30, 5, False, IDENT, [7.0, 8.0, 9.0]))             # posed, not registered: moved, not counted
    w["images"].append((6, 3, 30, False, [], []))
    out, calls, _ = run(driver, tmp_path, w, "normalize", 0, 10.0, 0.1, 0.9)
    assert [c for c, _ in calls] == ["create_rig", "set_state", "set_images", "normalize"]
    cr, st, si, nm = (c for _, c in calls)
    # frames 10, 20, 30; sensors in order of the registered images 1 (5, 7), 2 (5, 3); tracks 40, 50 and one
    # placeholder observation
    assert cr["dims"] == [3, 2, 1, 1, 2, 1] and cr["ptb"] == [0, 1, 1]
    assert cr["sensor_q"] == IDENT + [0, 0, 0.6, 0.8] and cr["sensor_t"] == [0, 0, 0, 0.5, -0.25, 1]
    assert st["trans"] == [4, 5, 6, 1, 2, 3, 7, 8, 9] and st["points"] == [4, 5, 6, 1, 2, 3]
    # the registered images 1, 2, 3, 4 (6 is on the unregistered frame 30)
    assert si["image_frame"] == [0, 1, 1, 0] and si["image_sensor"] == [0, 1, 0, 1]
    assert nm["args"] == [0, 10, 0.1, 0.9]
    # the double's similarity and state; cam_from_rig translations scaled on the host
    assert out["result"] == [2, 0, 0, 0, 1, 1, 2, 3]
    assert [out["frame"][f][4:] for f in (10, 20, 30)] == [[100, 101, 102], [103, 104, 105], [106, 107, 108]]
    assert out["frame"][20][:4] == [0, 0.6, 0, 0.8]
    assert out["track"][40][0] == [200, 201, 202] and out["track"][50][0] == [203, 204, 205]
    assert out["sensor"][(5, 3)] == [0, 0, 0.6, 0.8, 1.0, -0.5, 2.0]


def test_normalize_on_trivial_frames_without_tracks(driver, tmp_path):
    w = trivial_world()
    w["tracks"] = []
    out, calls, _ = run(driver, tmp_path, w, "normalize", 1, 5.0, 0.0, 1.0)
    cr, st, si, nm = (c for _, c in calls)
    # one sensor per camera of the registered images (identity), one placeholder point
    assert cr["dims"] == [2, 1, 1, 1, 2, 1] and cr["sensor_q"] == IDENT + IDENT
    assert si["image_frame"] == [0, 1] and si["image_sensor"] == [0, 1]
    assert nm["args"] == [1, 5, 0, 1]
    assert out["result"][0] == 2 and out["track"] == {}


# ---- failures: nothing changes ---------------------------------------------------------------------------------------
def _fail_cases():
    unknown = trivial_world()
    unknown["tracks"][1] = (40, [4.0, 5.0, 6.0], [(1, 1), (8, 0)])           # image 8 does not exist
    feature = trivial_world()
    feature["tracks"][1] = (40, [4.0, 5.0, 6.0], [(1, 1), (2, 5)])           # image 2 has 2 features
    model = trivial_world()
    model["images"][0] = (2, 9, 20) + model["images"][0][3:]                 # image 2 through the model-4 camera
    sensor = rig_world()
    sensor["rigs"] = [(5, 7, [])]                                            # camera 3 has no cam_from_rig
    return [(unknown, ("reprojection", 0.01, 1)), (unknown, ("angle", 1.0)), (unknown, ("triangulation", 1.0)),
            (feature, ("reprojection", 2.0, 0)), (feature, ("angle", 1.0)), (model, ("reprojection", 2.0, 0)),
            (model, ("undistort", 1)), (sensor, ("angle", 1.0)), (sensor, ("normalize", 0, 10.0, 0.1, 0.9))]


@pytest.mark.parametrize("case", range(len(_fail_cases())))
def test_failures_leave_the_maps_unchanged(driver, tmp_path, case):
    w, op = _fail_cases()[case]
    base, _, _ = run(driver, tmp_path, w, "undistort", 0)
    out, calls, err = run(driver, tmp_path, w, *op)
    assert "b200sfm:" in err
    _unchanged(base, out)
    if op[0] == "normalize":
        assert out["result"] == [1, 0, 0, 0, 1, 0, 0, 0]
    elif op[0] != "undistort":
        assert out["result"] == [0]
    # the model-4 camera is refused by the device where intrinsics are read; the other cases never reach it
    assert [c for c, _ in calls] in ([], ["create"], ["undistort_features"])


def test_model_outside_0_3_only_matters_where_intrinsics_are_read(driver, tmp_path):
    w = _fail_cases()[5][0]
    out, calls, _ = run(driver, tmp_path, w, "angle", 1.0)
    assert [c for c, _ in calls] == ["create", "set_state", "filter_angle"] and calls[0][1]["intr_model"] == [0]
    assert calls[2][1]["calibrated"] == [1, 1]                               # camera 9 has a prior focal
    assert out["result"] == [7]


def test_shim_processors_typecheck_against_the_glomap_api():
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(MOCK, "glomap_stub_processors"), "-I" + HOST,
                        os.path.join(MOCK, "processors_typecheck.cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_normalize_without_colmap_sim3_fails_with_a_message():
    """Without <colmap/geometry/sim3.h> the glomap build keeps NormalizeReconstruction declared; a call is a compile
    error that names the header, not a missing member."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(MOCK, "glomap_stub"), "-I" + HOST,
                        os.path.join(MOCK, "processors_nosim3_typecheck.cc")], capture_output=True, text=True)
    assert r.returncode != 0
    assert "needs <colmap/geometry/sim3.h>" in r.stderr, r.stderr
    assert "has no member" not in r.stderr
