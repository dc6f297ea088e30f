"""ConvertRotationsFromImageToRig and the rig pre-pass of SolveRotationAveraging without a GPU: the numpy oracle
(oracle/rig_init_oracle.py) against exact rotations, one case per rule of b200sfm_rig_rotations_from_images, the ctypes
binding against the header, and the C++ shim's pre-pass over the recording test doubles (mock_b200sfm.c and
mock_rig_init.c)."""
import os
import re
import subprocess

import numpy as np
import pytest

from glomap_b200 import _lib, geometry as G
from glomap_b200 import rotation_averager as RA
from oracle import rig_init_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rig_world(F, S, seed=0, drop=0.0):
    """F frames of one rig with S cameras (camera 0 the reference); image f * S + s, minus a random share ``drop``.
    Returns (image_frame, image_camera, cam_from_world [I,4], R_frames [F,3,3], R_cams [S,3,3])."""
    rng = np.random.default_rng(seed)
    Rf = G.so3_exp(rng.normal(size=(F, 3)))
    w = rng.normal(size=(S, 3)) * 0.4
    w[0] = 0.0
    Rs = G.so3_exp(w)
    fr = np.repeat(np.arange(F), S)
    cam = np.tile(np.arange(S), F)
    keep = rng.uniform(size=F * S) >= drop
    fr, cam = fr[keep], cam[keep]
    q = G.rotmat_to_quat_xyzw_fast(np.einsum("nij,njk->nik", Rs[cam], Rf[fr]))
    return fr, cam, q, Rf, Rs


def qangle(a, b):
    """Sign-invariant rotation angle between quaternions, 4 atan2(|a - b|, |a + b|) (exact down to rounding, unlike arccos)."""
    a = np.asarray(a) / np.linalg.norm(a, axis=-1, keepdims=True)
    b = np.asarray(b) / np.linalg.norm(b, axis=-1, keepdims=True)
    b = np.where((a * b).sum(-1, keepdims=True) < 0, -b, b)
    return 4 * np.arctan2(np.linalg.norm(a - b, axis=-1), np.linalg.norm(a + b, axis=-1))


def test_oracle_recovers_exact_rotations():
    F, S = 40, 4
    fr, cam, q, Rf, Rs = rig_world(F, S, seed=1)
    known = np.array([1, 1, 0, 0], np.uint8)
    cq0 = np.tile([0, 0, 0, 1.0], (S, 1))
    cq0[1] = G.rotmat_to_quat_xyzw_fast(Rs[1:2])[0]
    cq, cn, fq, fn = O.convert_rotations(fr, cam, q, np.zeros(F, int), known, cq0, np.tile([0, 0, 0, 1.0], (F, 1)))
    assert cn.tolist() == [0, 0, F, F] and fn.tolist() == [S] * F
    assert qangle(cq[2:], G.rotmat_to_quat_xyzw_fast(Rs[2:])).max() < 1e-12
    assert qangle(fq, G.rotmat_to_quat_xyzw_fast(Rf)).max() < 1e-12
    assert (cq[2:, 3] >= 0).all() and (fq[:, 3] >= 0).all()


def test_oracle_rules_case_by_case():
    F, S = 6, 3
    fr, cam, q, Rf, Rs = rig_world(F, S, seed=2)
    fr = fr.copy()
    est = np.ones(len(fr), bool)
    fr[0] = -1                    # frame 0: the reference image is not registered -> no camera sample, no ref sample
    fr[3 * 1 + 2] = -1            # frame 1: camera 2's image unregistered
    est[3 * 2 + 1] = False        # frame 2: camera 1's image not estimated
    est[3 * 3] = False            # frame 3: the reference image not estimated -> no camera sample from it
    known = np.zeros(S, np.uint8)
    known[0] = 1
    cam_in = np.tile([0.1, 0.2, 0.3, 0.9], (S, 1))
    fr_in = np.tile([0.5, 0.0, 0.0, 0.5], (F, 1))
    # camera 2 has one sample only (frame 2 kept; frames 0, 1, 3 give none; 4, 5 dropped below)
    m = ~((cam == 2) & (fr >= 4))
    cq, cn, fq, fn = O.convert_rotations(fr[m], cam[m], q[m], np.zeros(F, int), known, cam_in, fr_in, est[m])
    assert cn.tolist() == [0, 3, 1]                      # camera 1: frames 1, 4, 5; camera 2: frame 2
    assert qangle(cq[2], G.rotmat_to_quat_xyzw_fast(Rs[2:3])[0]) < 1e-12     # a single sample as it is
    # frame 0: its registered images of cameras 1 and 2 through the averaged cam_from_rig
    assert fn.tolist() == [2, 2, 2, 2, 2, 2]
    assert qangle(fq, G.rotmat_to_quat_xyzw_fast(Rf)).max() < 1e-12
    # a camera without a sample stays unknown (its row untouched), a frame without a sample keeps its input
    cq2, cn2, fq2, fn2 = O.convert_rotations(np.array([0, 0, -1]), np.array([1, 2, 0]), q[:3], np.zeros(2, int), known,
                                             cam_in, fr_in[:2])
    assert cn2.tolist() == [0, 0, 0] and np.array_equal(cq2, cam_in)
    assert fn2.tolist() == [0, 0] and np.array_equal(fq2, fr_in[:2])


def test_average_is_the_dominant_eigenvector():
    rng = np.random.default_rng(3)
    base = G.rotmat_to_quat_xyzw_fast(G.so3_exp(rng.normal(size=(1, 3))))[0]
    qs = [O._qmul(base, G.rotmat_to_quat_xyzw_fast(G.so3_exp(rng.normal(size=(1, 3)) * 0.01))[0]) * rng.choice([-1, 1])
          for _ in range(7)]
    a = O.average_quaternions(qs)
    M = sum(np.outer(x, x) for x in qs)
    assert a[3] >= 0 and np.allclose(M @ a, np.linalg.eigvalsh(M)[-1] * a, atol=1e-12)


def test_trivial_layout_and_folding():
    # frames 0, 1 of a 3-camera rig, camera 2 unknown; image 5 unregistered
    fr, cam = np.array([0, 0, 0, 1, 1, 1]), np.array([0, 1, 2, 0, 1, 2])
    tf, tref = RA.trivial_layout(fr, cam, [1, 1, 0], [0, 0], np.array([1, 1, 1, 1, 1, 0], bool))
    assert tf.tolist() == [0, 0, 2, 1, 1, -1] and tref.tolist() == [0, 0, 2]
    from glomap_b200.synthetic import ViewGraph
    Rr = G.so3_exp(np.random.default_rng(4).normal(size=(4, 3)))
    vg = ViewGraph(6, np.array([0, 0, 2, 1]), np.array([1, 2, 3, 5]), Rr, np.ones(4), np.tile(np.eye(3), (6, 1, 1)))
    Rc = G.so3_exp(np.array([[0, 0, 0], [0.1, 0.2, 0.3], [0, 0, 0]]))
    keep, ei, ej, R = RA.fold_pairs(vg, tf, Rc, cam)
    assert keep.tolist() == [False, True, True, False]   # inside trivial frame 0; an unregistered image
    assert ei.tolist() == [0, 2] and ej.tolist() == [2, 1]
    assert np.abs(R[0] - Rr[1]).max() < 1e-15 and np.abs(R[1] - Rr[2]).max() < 1e-15


def test_binding_matches_the_header():
    h = open(os.path.join(ROOT, "include", "b200sfm.h")).read()
    body = re.search(r"typedef struct \{([^{}]*)\} b200sfm_rig_init_stats;", h).group(1)
    names = re.findall(r"\b(?:int32_t|int64_t|double)\s+(\w+);", body)
    assert names == [f for f, _ in _lib.RigInitStats._fields_]
    decl = re.search(r"int b200sfm_rig_rotations_from_images\((.*?)\);", h, re.S).group(1)
    assert len(decl.split(",")) == len(_lib.PROTOTYPES["b200sfm_rig_rotations_from_images"][1])


@pytest.fixture(scope="module")
def shim_run(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("riginit")
    lib, exe, dump = tmp / "libb200sfm_mock.so", tmp / "rig_init_driver", tmp / "dump.txt"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c"),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_rig_init.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "shim_mock", "rig_init_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp)],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe)], env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0 and "rig init driver ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    calls, cur = [], None
    for line in dump.read_text().splitlines():
        f = line.split()
        if f[0] == "call":
            cur = {"_name": f[1]}
            calls.append(cur)
        else:
            cur[f[0]] = np.array([float(x) for x in f[2:]])
            assert len(cur[f[0]]) == int(f[1])
    out = {l.split()[0]: l.split()[1:] for l in r.stdout.splitlines() if l.split()}
    return calls, out, r.stderr


def test_shim_prepass_over_the_recording_double(shim_run):
    """World of rig_init_driver.cc: rig 1 = cameras 1 (reference), 2 (known, 90 deg about z), 3 (unknown); frames 10, 20,
    30 hold images (10·f/10 + c): 11 12 13 / 21 22 23 / 31 32 (frame 30 has no camera 3)."""
    calls, out, err = shim_run
    assert "not supported" not in err
    assert [c["_name"] for c in calls] == ["ra_mst_init", "rig_rotations_from_images", "ra_solve", "rig_rotations_from_images",
                                           "ra_solve_rig"]
    mst, conv_t, ra_t, conv, rig = calls
    # images in ascending id: 11 12 13 21 22 23 31 32 -> 0..7; the root is the smallest id
    assert mst["dims"].tolist() == [8, 7, 0]
    # trivial frames: 10, 20, 30 -> 0, 1, 2, then one per image of camera 3 (13, 23) -> 3, 4
    assert conv_t["dims"].tolist() == [8, 5, 3]
    assert conv_t["image_frame"].tolist() == [0, 0, 3, 1, 1, 4, 2, 2]
    assert conv_t["frame_ref_camera"].tolist() == [0, 0, 0, 2, 2]
    assert conv_t["camera_known"].tolist() == [1, 1, 1]
    # folded pairs: (11,12) and (21,22) and (31,32) fall inside a trivial frame and are dropped
    assert ra_t["dims"].tolist() == [5, 4]
    assert ra_t["ei"].tolist() == [0, 0, 1, 1] and ra_t["ej"].tolist() == [3, 1, 4, 2]
    # real rigs: camera 3 unknown, estimated images = all 8
    assert conv["image_frame"].tolist() == [0, 0, 0, 1, 1, 1, 2, 2]
    assert conv["camera_known"].tolist() == [1, 1, 0]
    assert conv["image_estimated"].tolist() == [1] * 8
    # the rig solve starts the camera node from the mock's average (0.25 rad about x) and the frames from theirs
    th = rig["theta"].reshape(-1, 3)
    assert rig["dims"].tolist()[:2] == [3, 1]
    assert np.allclose(th[3], [0.25, 0, 0], atol=1e-15)
    # write-back: the estimated cam_from_rig (mock: 0.3 rad about z) with a NaN translation
    c3 = [float(x) for x in out["cam3"]]
    assert np.allclose(c3[:4], [0, 0, np.sin(0.15), np.cos(0.15)], atol=1e-15) and all(np.isnan(c3[4:]))
    assert out["registered"] == ["1", "1", "1"]


def test_shim_typechecks_against_the_glomap_api():
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(ROOT, "tests", "shim_mock", "glomap_stub"), "-I" + os.path.join(ROOT, "glomap_b200", "host"),
                        "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "shim_mock", "shim_typecheck.cc")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def test_shim_links_and_refuses_without_the_prepass_entries(tmp_path):
    """A libb200sfm without b200sfm_ra_mst_init / b200sfm_rig_rotations_from_images (the entries are weak in the shim):
    the host still links, and SolveRotationAveraging reports the missing entry and returns false."""
    lib, exe = tmp_path / "libb200sfm_mock.so", tmp_path / "rig_init_driver"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "shim_mock", "rig_init_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe)], env=dict(os.environ, MOCK_DUMP=str(tmp_path / "dump.txt")), capture_output=True, text=True)
    assert r.returncode == 1 and "ok 0" in r.stdout
    assert "has no b200sfm_ra_mst_init / b200sfm_rig_rotations_from_images" in r.stderr
