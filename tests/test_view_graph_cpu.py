"""The view-graph passes of stage 3 on the CPU: the host restatements of RelPoseFilter::FilterRotations and
ViewGraph::KeepLargestConnectedComponents (glomap_b200/view_graph.py) on hand-built graphs, one case per rule (ties,
self-loop frames, no valid pair, unregistered images, NaN, the threshold itself), the mapper's camera compaction, the
argument checks of the C entries, and the C++ shim over a recording test double."""
import ctypes as ct
import math
import os
import subprocess

import numpy as np

from glomap_b200 import geometry as G, mapper as M, synthetic as S, view_graph as VG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDENTITY = [0.0, 0.0, 0.0, 1.0]


def _rot_quat(axis, deg):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    h = math.radians(deg) / 2
    return [*(a * math.sin(h)), math.cos(h)]


# ---- KeepLargestConnectedComponents -----------------------------------------------------------------------------------
def test_tie_goes_to_the_component_holding_the_smallest_frame():
    # frames {4, 5} and {1, 3}: equally large; {1, 3} holds the smaller frame
    image_frame = np.arange(6)
    valid, reg, n = VG.keep_largest_connected_components(6, image_frame, [4, 3], [5, 1])
    assert reg.tolist() == [False, True, False, True, False, False] and n == 2
    assert valid.tolist() == [False, True]


def test_a_pair_inside_one_frame_makes_that_frame_a_node():
    # images 0, 1 in frame 2 (a rig): the self-loop frame alone is the largest component (one node, two images)
    image_frame = np.array([2, 2, 0, 1])
    valid, reg, n = VG.keep_largest_connected_components(3, image_frame, [0], [1])
    assert reg.tolist() == [False, False, True] and n == 2 and valid.tolist() == [True]
    # next to a two-frame component it loses
    valid, reg, n = VG.keep_largest_connected_components(3, image_frame, [0, 2], [1, 3])
    assert reg.tolist() == [True, True, False] and n == 2 and valid.tolist() == [False, True]


def test_multi_image_frames_count_images_not_frames():
    image_frame = np.array([0, 0, 0, 1, 2, 3])          # frame 0 holds three images
    valid, reg, n = VG.keep_largest_connected_components(4, image_frame, [0, 4], [3, 5])
    assert reg.tolist() == [True, True, False, False] and n == 4


def test_no_valid_pair_changes_nothing():
    reg0 = np.array([True, False, True])
    valid, reg, n = VG.keep_largest_connected_components(3, np.arange(3), [0, 1], [1, 2], [False, False], reg0)
    assert n == 0 and reg.tolist() == reg0.tolist() and valid.tolist() == [False, False]
    valid, reg, n = VG.keep_largest_connected_components(3, np.arange(3), [], [], [], reg0)
    assert n == 0 and reg.tolist() == reg0.tolist()


def test_every_frame_outside_the_component_is_deregistered_and_its_pairs_invalidated():
    # frame 3 is registered before but has no valid pair; the invalid pair 0-1 inside the component stays invalid; the
    # valid pair 4-5 forms the smaller component and is invalidated
    valid, reg, n = VG.keep_largest_connected_components(6, np.arange(6), [0, 1, 0, 4], [1, 2, 2, 5],
                                                         [False, True, True, True], np.ones(6, bool))
    assert reg.tolist() == [True, True, True, False, False, False] and n == 3
    assert valid.tolist() == [False, True, True, False]


# ---- FilterRotations --------------------------------------------------------------------------------------------------
def _two_images(q_rel):
    q = np.array([IDENTITY, _rot_quat([0, 0, 1], 20.0)])
    return q, np.array([q_rel])


def test_angle_matches_the_trace_formula_away_from_the_threshold():
    rng = np.random.default_rng(3)
    R = G.so3_exp(rng.normal(size=(50, 3)))
    Rr = G.so3_exp(rng.normal(size=(49, 3)) * 0.3) @ R[1:] @ np.swapaxes(R[:-1], -1, -2)
    q, qr = G.rotmat_to_quat_xyzw_fast(R), G.rotmat_to_quat_xyzw_fast(Rr)
    for e in range(49):
        qa = q[e]
        qc = VG._qmul(q[e + 1], (-qa[0], -qa[1], -qa[2], qa[3]))
        want = float(G.rotation_angle_deg(R[e + 1] @ R[e].T, Rr[e]))
        assert abs(VG.rotation_angle_deg(qc, qr[e]) - want) < 1e-6
    # the quaternion sign does not matter (|d.w|)
    assert VG.rotation_angle_deg(tuple(-np.asarray(qc)), qr[48]) == VG.rotation_angle_deg(qc, qr[48])


def test_angle_equal_to_the_threshold_keeps_the_pair():
    q, qr = _two_images(_rot_quat([0, 0, 1], 7.0))
    qc = VG._qmul(q[1], (-q[0][0], -q[0][1], -q[0][2], q[0][3]))
    angle = VG.rotation_angle_deg(qc, qr[0])
    assert abs(angle - 13.0) < 1e-9
    valid, n = VG.filter_rotations(q, [0], [1], qr, angle)
    assert valid.tolist() == [True] and n == 0
    valid, n = VG.filter_rotations(q, [0], [1], qr, math.nextafter(angle, -math.inf))
    assert valid.tolist() == [False] and n == 1


def test_nan_angle_keeps_the_pair():
    q, qr = _two_images([math.nan, 0.0, 0.0, 1.0])
    valid, n = VG.filter_rotations(q, [0], [1], qr, 1.0)
    assert valid.tolist() == [True] and n == 0
    q[0, 3] = math.nan
    valid, n = VG.filter_rotations(q, [0], [1], np.array([IDENTITY]), 1.0)
    assert valid.tolist() == [True] and n == 0


def test_pairs_touching_unregistered_images_and_invalid_pairs_are_not_tested():
    q = np.array([IDENTITY, _rot_quat([1, 0, 0], 90.0), IDENTITY])
    qr = np.array([IDENTITY, IDENTITY, IDENTITY])
    valid, n = VG.filter_rotations(q, [0, 1, 0], [1, 2, 2], qr, 5.0, [True, True, False], [True, False, True])
    assert valid.tolist() == [True, True, False] and n == 0
    valid, n = VG.filter_rotations(q, [0, 1, 0], [1, 2, 2], qr, 5.0)
    assert valid.tolist() == [False, False, True] and n == 2


# ---- mapper compaction ------------------------------------------------------------------------------------------------
def test_compact_and_scatter_cameras_round_trip():
    sc = S.make_scene(8, 200, mean_track_len=5, seed=4)
    idx = np.array([0, 2, 3, 5, 7])
    part = M.compact_cameras(sc, idx)
    assert part.C == 5 and part.P == sc.P
    drop = ~np.isin(sc.obs_cam, idx)
    assert part.N == int((~drop).sum())
    assert np.array_equal(idx[part.obs_cam], sc.obs_cam[~drop]) and np.array_equal(part.obs_xy, sc.obs_xy[~drop])
    part.quat = part.quat[::-1].copy()
    back = M.scatter_cameras(sc, part, idx)
    assert np.array_equal(back.quat[idx], part.quat) and np.array_equal(back.quat[[1, 4, 6]], sc.quat[[1, 4, 6]])
    assert np.array_equal(back.obs_cam, sc.obs_cam[~drop]) and back.C == sc.C


def test_registered_view_graph_renumbers_the_images():
    vg = S.make_ring_view_graph(6, 2, seed=1)
    reg = np.array([True, False, True, True, True, True])
    valid = np.ones(vg.E, bool)
    valid[0] = False
    sub, idx = M.registered_view_graph(vg, valid, reg)
    assert idx.tolist() == [0, 2, 3, 4, 5] and sub.n_images == 5
    keep = valid & reg[vg.ei] & reg[vg.ej]
    assert np.array_equal(idx[sub.ei], vg.ei[keep]) and np.array_equal(idx[sub.ej], vg.ej[keep])


# ---- C entries: argument checks that never reach the device -----------------------------------------------------------
def test_entries_reject_a_null_context_and_null_outputs():
    from glomap_b200 import _lib
    lib = _lib.load()
    n64, n32 = ct.c_int64(7), ct.c_int32(7)
    assert lib.b200sfm_view_graph_filter_rotations(None, 0, None, None, 0, None, None, None, 1.0, None, ct.byref(n64)) == 1
    assert lib.b200sfm_view_graph_keep_largest_component(None, 0, 0, None, 0, None, None, None, None, ct.byref(n32)) == 1


# ---- C++ shim ---------------------------------------------------------------------------------------------------------
def _mock_lib(tmp_path):
    lib = tmp_path / "libb200sfm.so"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c"),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_view_graph.c")], check=True, capture_output=True)
    return lib


def test_shim_flattens_in_sorted_id_order_and_writes_back(tmp_path):
    lib, exe, dump = _mock_lib(tmp_path), tmp_path / "view_graph_driver", tmp_path / "dump.txt"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "shim_mock", "view_graph_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe)], env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    calls, cur = [], None
    for line in dump.read_text().splitlines():
        name, n, *vals = line.split()
        if name == "call":
            cur = {"_name": n}
            calls.append(cur)
            continue
        assert len(vals) == int(n)
        cur[name] = [float(v) for v in vals]
    assert [c["_name"] for c in calls] == ["view_graph_filter_rotations", "view_graph_keep_largest_component"]
    f, k = calls
    # images 101, 201, 202, 301 -> 0..3; 202 is camera 2 of the rig in frame 20: cam_from_rig (0, 0, .6, .8) * rig_from_world
    q202 = [-0.36, 0.48, 0.48, 0.64]
    assert f["max_angle"] == [5.0]
    assert np.allclose(f["cam_from_world"][:12], [0.6, 0, 0, 0.8, 0, 0.6, 0, 0.8] + q202, atol=1e-15)
    assert all(math.isnan(v) for v in f["cam_from_world"][12:])           # 301: frame 30 is not registered
    assert f["image_registered"] == [1, 1, 1, 0]
    # the valid pairs in sorted pair-id order: (101,201) (202,101) (101,301) (201,202); (201,301) is invalid
    assert f["pair_image1"] == [0, 2, 0, 1] and f["pair_image2"] == [1, 0, 3, 2]
    assert f["pair_quat"] == [0.1, 0, 0, 1, 0.2, 0, 0, 1, 0.3, 0, 0, 1, 0.4, 0, 0, 1]
    assert f["pair_valid"] == [1, 1, 1, 1]
    # frames 10, 20, 30 -> 0, 1, 2; every pair, after the filter invalidated the odd ones
    assert k["image_frame"] == [0, 1, 1, 2]
    assert k["pair_image1"] == [0, 2, 0, 1, 1] and k["pair_image2"] == [1, 0, 3, 2, 3]
    assert k["pair_valid"] == [1, 0, 1, 0, 0] and k["frame_registered"] == [1, 1, 0]
    assert r.stdout.splitlines() == ["filtered 2", "registered images 104", "frame 10 registered 1", "frame 20 registered 1",
                                     "frame 30 registered 0", "pair 101 201 valid 0", "pair 101 202 valid 0",
                                     "pair 101 301 valid 1", "pair 201 202 valid 0", "pair 201 301 valid 0",
                                     "view graph driver ok"]


def test_shim_view_graph_passes_typecheck_against_the_glomap_api():
    """Inside a glomap build the shim takes glomap's ImagePair, Frame (is_registered, RigFromWorld, RigPtr) and Image."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(ROOT, "tests", "shim_mock", "glomap_stub"),
                        "-I" + os.path.join(ROOT, "glomap_b200", "host"),
                        os.path.join(ROOT, "tests", "shim_mock", "view_graph_typecheck.cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
