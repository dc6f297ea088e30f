"""The C++ side of gravity refinement and `rotation_averager` without a GPU: the shim's GravityRefiner and
KeepLargestConnectedComponents against a recording test double of the C ABI, their type check against the glomap API,
and the CLI's gravity / weight options (argument errors, what reaches the solvers)."""
import os
import shutil
import subprocess

import numpy as np

from glomap_b200 import geometry as G, synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK = os.path.join(ROOT, "tests", "shim_mock")


def _mock_lib(tmp_path):
    lib = tmp_path / "libb200sfm.so"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(MOCK, "mock_b200sfm.c"), os.path.join(MOCK, "mock_gravity.c")], check=True, capture_output=True)
    return lib


def _calls(dump):
    calls, cur = [], None
    if not os.path.exists(dump):
        return calls
    for line in open(dump):
        f = line.split()
        if f[0] == "call":
            cur = {"_name": f[1]}
            calls.append(cur)
        else:
            cur[f[0]] = np.array([float(x) for x in f[2:]])
    return calls


def _rz(qz):
    return G.quat_xyzw_to_rotmat(np.array([[0, 0, qz, np.sqrt(1 - qz * qz)]]))[0]


def test_shim_gravity_refiner_over_the_test_double(tmp_path):
    lib = _mock_lib(tmp_path)
    exe, dump = tmp_path / "gravity_driver", tmp_path / "dump.txt"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(MOCK, "gravity_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)], check=True, capture_output=True)
    r = subprocess.run([str(exe)], env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    (c,) = [c for c in _calls(dump) if c["_name"] == "gravity_refine"]
    assert c["scalars"].tolist() == [0.5, 2.5, 7, 100, 4, 3]
    assert c["has_gravity"].tolist() == [1, 1, 1, 0]
    # valid pairs with gravity in pair-id order: (101, 202), (301 -> 101), (201, 202); 203 (uncalibrated) and 401 skipped
    assert c["frame1"].tolist() == [0, 2, 1] and c["frame2"].tolist() == [1, 0, 1]
    Rc2 = _rz(np.sqrt(0.5))
    M = c["M"].reshape(3, 3, 3)
    np.testing.assert_allclose(M[0], Rc2.T @ _rz(0.2), atol=1e-15)
    np.testing.assert_allclose(M[1], _rz(0.1), atol=1e-15)
    np.testing.assert_allclose(M[2], Rc2.T @ _rz(0.3), atol=1e-15)
    R_align = c["R_align"].reshape(4, 3, 3)
    for k, f in enumerate((10, 20, 30)):
        g = np.array([0.1 * f, 1.0, -0.02 * f])
        np.testing.assert_allclose(R_align[k][:, 1], g / np.linalg.norm(g), atol=1e-15)
    lines = r.stdout.splitlines()
    assert lines[0] == "frame 10 gravity 1 0 1 0"                      # status 2: SetGravity
    assert lines[1].startswith("frame 20 gravity 1 2 1 -0.4")         # status 3: unchanged
    assert lines[2] == "frame 30 gravity 1 0 1 2"
    assert lines[3].startswith("frame 40 gravity 0")
    assert lines[4] == "lcc images 5 registered 1 1 1 0"
    assert "gravity driver ok" in r.stdout


def test_shim_gravity_typechecks_against_the_glomap_api(tmp_path):
    """The stubs of tests/shim_mock with GravityInfo::SetGravity (glomap/scene/frame.h:18) added to a copy."""
    for d in ("glomap_stub", "glomap_stub_pairs", "glomap_stub_vgc", "glomap_stub_prune"):
        shutil.copytree(os.path.join(MOCK, d), tmp_path / d)
    base = tmp_path / "glomap_stub" / "glomap" / "scene" / "types_sfm.h"
    src = base.read_text()
    anchor = "  const Eigen::Matrix3d& GetRAlign() const { return R_align_; }\n"
    assert anchor in src
    base.write_text(src.replace(anchor, anchor + "  void SetGravity(const Eigen::Vector3d&) {}\n"))
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP", "-I" + str(tmp_path / "glomap_stub_prune"),
                        "-I" + os.path.join(ROOT, "glomap_b200", "host"), os.path.join(MOCK, "gravity_typecheck.cc")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def _cli(tmp_path):
    lib = _mock_lib(tmp_path)
    cli = tmp_path / "b200sfm_cli"
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", str(cli), os.path.join(ROOT, "glomap_b200", "host", "b200sfm_cli.cc"), str(lib),
                    "-Wl,-rpath," + str(tmp_path)], check=True, capture_output=True)
    return str(cli)


def test_cli_argument_errors(tmp_path):
    cli = _cli(tmp_path)
    vg = S.make_random_view_graph(12, 4.0, seed=2)
    rel, out = str(tmp_path / "rel.txt"), str(tmp_path / "out.txt")
    S.write_relpose_file(rel, vg)
    base = [cli, "rotation_averager", "--relpose_path", rel, "--output_path", out]
    run = lambda *a: subprocess.run(list(base) + list(a), capture_output=True, text=True)   # noqa: E731
    r = run("--gravity_path", str(tmp_path / "missing.txt"))
    assert r.returncode == 1 and "gravity_path" in r.stderr
    r = run("--weight_path", str(tmp_path / "missing.txt"))
    assert r.returncode == 1 and "weight_path" in r.stderr
    r = run("--use_weight", "1")
    assert r.returncode == 1 and "Weight path is required" in r.stderr
    r = run("--gravity", "g.txt")
    assert r.returncode == 2 and "unknown option --gravity" in r.stderr
    r = subprocess.run([cli, "rotation_averager", "--relpose_path", str(tmp_path / "none.txt"), "--output_path", out],
                       capture_output=True, text=True)
    assert r.returncode == 1 and "relpose_path" in r.stderr


def test_cli_gravity_file_reaches_the_solvers(tmp_path):
    cli = _cli(tmp_path)
    vg = S.make_random_view_graph(20, 6.0, seed=3)
    names = [f"img{i:04d}" for i in range(vg.n_images)]
    g, _ = S.make_gravity(vg.R_gt, seed=3)
    g[::2] = np.nan
    rel, grav, wts = str(tmp_path / "rel.txt"), str(tmp_path / "grav.txt"), str(tmp_path / "w.txt")
    S.write_relpose_file(rel, vg)
    S.write_gravity_file(grav, names, g)
    S.write_weight_file(wts, vg, np.arange(vg.E) + 1.0)
    dump = tmp_path / "dump.txt"
    env = dict(os.environ, MOCK_DUMP=str(dump))
    base = [cli, "rotation_averager", "--relpose_path", rel, "--output_path", str(tmp_path / "o.txt")]
    # without --gravity_path, --refine_gravity is a no-op and the plain solver runs
    r = subprocess.run(base + ["--refine_gravity", "1"], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert [c["_name"] for c in _calls(dump)] == ["ra_solve"]
    dump.unlink()
    r = subprocess.run(base + ["--gravity_path", grav, "--refine_gravity", "1", "--weight_path", wts, "--use_weight", "1"],
                       env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    calls = _calls(dump)
    names_called = [c["_name"] for c in calls]
    assert names_called[0] == "gravity_refine" and "ra_solve_gravity" in names_called
    # image ids follow first appearance in the relpose file; the frames with a prior are the file's rows
    order = []
    for e in range(vg.E):
        for i in (vg.ei[e], vg.ej[e]):
            if i not in order:
                order.append(int(i))
    assert calls[0]["has_gravity"].astype(bool).tolist() == [bool(np.isfinite(g[i]).all()) for i in order]
