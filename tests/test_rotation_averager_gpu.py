"""`b200sfm_cli rotation_averager` with gravity priors, refinement, stratification and weights on the device, against
the Python path (gravity_refinement.GravityRefiner + rotation_averager.solve_rotation_averaging)."""
import os
import subprocess

import numpy as np
import pytest

from glomap_b200 import geometry as G, synthetic as S
from glomap_b200.gravity_refinement import GravityRefiner, get_align_rot_householder
from glomap_b200.rotation_averager import RotationAveragerOptions, largest_component, solve_rotation_averaging

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "glomap_b200", "b200sfm_cli")


def _run(*args):
    r = subprocess.run([CLI, "rotation_averager", *args], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r


def _read_rotations(path):
    names, q = [], []
    for line in open(path):
        t = line.split()
        names.append(t[0])
        q.append([float(t[2]), float(t[3]), float(t[4]), float(t[1])])
    return names, G.quat_xyzw_to_rotmat(np.array(q))


def _python_path(vg, g, use_stratified=True, use_weight=False, refine=False):
    has = ~np.isnan(g).any(axis=1)
    R0 = np.tile(np.eye(3), (vg.n_images, 1, 1))
    R0[has] = get_align_rot_householder(g[has])
    if refine:   # the CLI refines on the largest component's pairs; the initial rotations stay as read
        reg = largest_component(vg.n_images, vg.ei, vg.ej)
        k = reg[vg.ei] & reg[vg.ej]
        sub = S.ViewGraph(vg.n_images, vg.ei[k], vg.ej[k], vg.R_rel[k], vg.weight[k], vg.R_gt)
        g, _, _ = GravityRefiner().RefineGravity(sub, g)
    o = RotationAveragerOptions(use_gravity=True, skip_initialization=True, use_stratified=use_stratified, use_weight=use_weight)
    ok, R, reg = solve_rotation_averaging(vg, g, o, R0)
    assert ok
    return R, reg


def _files(tmp_path, vg, g, names, weight=None):
    rel, grav = str(tmp_path / "rel.txt"), str(tmp_path / "grav.txt")
    S.write_relpose_file(rel, vg, names)
    S.write_gravity_file(grav, names, g)
    if weight is not None:
        S.write_weight_file(str(tmp_path / "w.txt"), vg, weight, names)
    return rel, grav


def _scene(seed, share, outlier_ratio=0.0, n=80):
    vg = S.make_random_view_graph(n, 10, seed=seed, noise_deg=1.0)
    g, out = S.make_gravity(vg.R_gt, noise_deg=0.0, outlier_ratio=outlier_ratio, seed=seed)
    rng = np.random.default_rng(seed)
    g[rng.uniform(size=n) >= share] = np.nan
    # the relpose file numbers images in order of first appearance: name them so that this order is the index order
    order = []
    for e in range(vg.E):
        for i in (int(vg.ei[e]), int(vg.ej[e])):
            if i not in order:
                order.append(i)
    perm = np.empty(n, np.int64)
    perm[np.array(order)] = np.arange(n)
    vg = S.ViewGraph(n, perm[vg.ei].astype(np.int32), perm[vg.ej].astype(np.int32), vg.R_rel, vg.weight, vg.R_gt[np.argsort(perm)])
    g = g[np.argsort(perm)]
    out = out[np.argsort(perm)]
    names = [f"img{i:04d}" for i in range(n)]
    return vg, g, out, names


def _aligned_diff(R_a, R_b):
    """Largest entry difference after the best global rotation R_a Q ~ R_b.  The 1-DoF gauge is the fixed frame's angle
    about its gravity, which each host reads from its own completion of R_align."""
    U, _, Vt = np.linalg.svd(np.einsum("nji,njk->ik", R_a, R_b))
    Q = U @ Vt
    return float(np.abs(R_a @ Q - R_b).max())


def _rot_err(R, R_gt):
    rot, _, _ = G.compare_reconstructions(R, np.zeros((len(R), 3)), R_gt, np.zeros((len(R), 3)))
    return rot


@pytest.mark.parametrize("share,stratified", [(1.0, True), (0.5, True), (0.5, False)])
def test_cli_with_gravity_file_matches_python(tmp_path, share, stratified):
    vg, g, _, names = _scene(31, share)
    rel, grav = _files(tmp_path, vg, g, names)
    out = str(tmp_path / "rot.txt")
    _run("--relpose_path", rel, "--output_path", out, "--gravity_path", grav, "--use_stratified", str(int(stratified)))
    got_names, R_cli = _read_rotations(out)
    g_file = S.read_gravity_file(grav, names)
    R_py, reg = _python_path(vg, g_file, use_stratified=stratified)
    assert got_names == [names[i] for i in np.nonzero(reg)[0]]
    # both hosts stop the IRLS on the same 1e-3 step threshold from differently rounded starts; the file has 6 digits
    assert _aligned_diff(R_cli, R_py[reg]) < 5e-4
    has = ~np.isnan(g_file).any(axis=1)[reg]
    gy = R_cli[has][:, :, 1]
    ref = g_file[reg][has] / np.linalg.norm(g_file[reg][has], axis=1, keepdims=True)
    assert np.abs(gy - ref).max() < 1e-4   # R_i e_y is the prior for the frames with gravity


def test_cli_refine_gravity_improves_rotations(tmp_path):
    vg, g, out_mask, names = _scene(32, 1.0, outlier_ratio=0.3, n=100)
    rel, grav = _files(tmp_path, vg, g, names)
    o1, o2 = str(tmp_path / "plain.txt"), str(tmp_path / "refined.txt")
    _run("--relpose_path", rel, "--output_path", o1, "--gravity_path", grav)
    _run("--relpose_path", rel, "--output_path", o2, "--gravity_path", grav, "--refine_gravity", "1")
    _, R1 = _read_rotations(o1)
    _, R2 = _read_rotations(o2)
    assert len(R1) == len(R2) == vg.n_images
    assert _rot_err(R2, vg.R_gt) < _rot_err(R1, vg.R_gt)
    # the refined priors reach the solver: R_i e_y is the Python refiner's gravity.  (The yaw of the refined frames starts
    # from the rotation the file's prior set, read through each host's own R_align completion, so the two hosts' IRLS
    # runs start apart and are not compared entry by entry.)
    g_ref, status, _ = GravityRefiner().RefineGravity(vg, S.read_gravity_file(grav, names))
    assert (status == 2).sum() >= 0.8 * out_mask.sum()
    ref = g_ref / np.linalg.norm(g_ref, axis=1, keepdims=True)
    assert np.abs(R2[:, :, 1] - ref).max() < 1e-4


def test_cli_weights_match_python(tmp_path):
    vg, g, _, names = _scene(33, 0.5)
    w = np.random.default_rng(33).uniform(0.5, 2.0, size=vg.E)
    rel, grav = _files(tmp_path, vg, g, names, weight=w)
    out = str(tmp_path / "rot.txt")
    _run("--relpose_path", rel, "--output_path", out, "--gravity_path", grav, "--weight_path", str(tmp_path / "w.txt"),
         "--use_weight", "1")
    _, R_cli = _read_rotations(out)
    vgw = S.ViewGraph(vg.n_images, vg.ei, vg.ej, vg.R_rel, np.array([float(f"{x:.17g}") for x in w]), vg.R_gt)
    R_py, reg = _python_path(vgw, S.read_gravity_file(grav, names), use_weight=True)
    assert _aligned_diff(R_cli, R_py[reg]) < 5e-4


def test_cli_without_gravity_flags_is_unchanged(tmp_path):
    """Without --gravity_path the new options change nothing: the plain command's output.  Compared as numbers, since
    two runs of the rotation averager differ in the last bits, which shows in printed values near zero."""
    vg, _, _, names = _scene(34, 0.0)
    rel = str(tmp_path / "rel.txt")
    S.write_relpose_file(rel, vg, names)
    a, b = str(tmp_path / "a.txt"), str(tmp_path / "b.txt")
    _run("--relpose_path", rel, "--output_path", a)
    _run("--relpose_path", rel, "--output_path", b, "--refine_gravity", "1", "--use_stratified", "0")
    la, lb = open(a).read().split(), open(b).read().split()
    assert la[::5] == lb[::5]
    np.testing.assert_allclose(np.array([float(x) for i, x in enumerate(la) if i % 5]),
                               np.array([float(x) for i, x in enumerate(lb) if i % 5]), rtol=0, atol=1e-9)
