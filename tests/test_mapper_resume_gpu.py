"""``python -m glomap_b200.mapper_resume`` end to end on the GPU: each test writes a COLMAP model to a temporary
directory, runs the command in-process and reads the output back.  Accuracy is judged as in the reference's tests
(glomap/controllers/global_mapper_test.cc:15-39, 84-86, 211-215): Sim3 alignment on the projection centres, then
rotation < 1e-2 deg and centre < 1e-4 without noise, 1e-1 / 1e-1 with 0.5 px of pixel noise."""
import os

import numpy as np
import pytest

from glomap_b200 import colmap_io as CIO, geometry as G, mapper_resume as MR, synthetic as S

pytestmark = pytest.mark.gpu


def _scramble(sc, seed=3):
    """Rotations at ground truth; translations (centres) and points scrambled."""
    rng = np.random.default_rng(seed)
    out = sc.copy()
    out.trans = rng.normal(size=out.trans.shape)
    out.points = rng.normal(size=out.points.shape)
    return out


def _run(model_dir, out_dir, *flags):
    rc = MR.main(["--input_path", str(model_dir), "--output_path", str(out_dir), *flags])
    assert rc == 0
    return str(out_dir / "0")


def _images_error(path, gt_R, gt_t, image_ids):
    _, ims, _ = CIO.read_model(path)
    q = np.array([ims[int(i)].qvec_wxyz for i in image_ids])
    R = G.quat_xyzw_to_rotmat(q[:, [1, 2, 3, 0]])
    t = np.array([ims[int(i)].tvec for i in image_ids])
    return G.compare_reconstructions(R, t, gt_R, gt_t)[:2]


def _trivial(tmp_path, pixel_sigma, seed):
    sc = S.make_scene(30, 2000, mean_track_len=6, seed=seed, pixel_sigma=pixel_sigma)
    CIO.write_model(str(tmp_path / "in"), *CIO.model_from_scene(_scramble(sc)))
    out = _run(tmp_path / "in", tmp_path / "out")
    rot, cen = _images_error(out, G.quat_xyzw_to_rotmat(sc.quat), sc.trans, np.arange(1, sc.C + 1))
    n_obs = sum(int((im.point3D_ids != CIO.INVALID_POINT3D).sum()) for im in CIO.read_model(out)[1].values())
    return sc, rot, cen, n_obs


def test_trivial_frames_without_noise(tmp_path):
    sc, rot, cen, _ = _trivial(tmp_path, 0.0, 21)
    assert rot < 1e-2 and cen < 1e-4, (rot, cen)


def test_trivial_frames_with_pixel_noise(tmp_path):
    sc, rot, cen, n_obs = _trivial(tmp_path, 0.5, 22)
    assert rot < 1e-1 and cen < 1e-1, (rot, cen)
    assert n_obs >= 0.98 * sc.N, (n_obs, sc.N)


def _rig_input(tmp_path, seed=11):
    d = S.make_rig_dataset(2, 2, 7, 100, seed=seed)
    sc = d.scene
    start = sc.copy()
    rng = np.random.default_rng(4)
    start.trans = rng.normal(size=start.trans.shape) * 0.1
    start.points = rng.normal(size=start.points.shape) * 0.1
    CIO.write_model(str(tmp_path / "in"), *CIO.model_from_scene(start))
    return sc


def _sensors(path):
    rigs, _ = CIO.read_rigs_frames(str(path))
    sensors = [s for r in sorted(rigs) for s in rigs[r].sensors]
    return np.array([s[2] for s in sensors]), np.array([s[3] for s in sensors])


@pytest.mark.parametrize("optimize_rig_poses", [False, True])
def test_rigs_without_noise(tmp_path, optimize_rig_poses):
    sc = _rig_input(tmp_path)
    out = _run(tmp_path / "in", tmp_path / "out", "--BundleAdjustment.optimize_rig_poses", str(int(optimize_rig_poses)))
    Rg, tg = sc.image_poses()
    rot, cen = _images_error(out, Rg, tg, np.arange(1, sc.I + 1))
    assert rot < 1e-2 and cen < 1e-4, (rot, cen)
    _, frames = CIO.read_rigs_frames(out)
    assert sorted(frames) == list(range(1, sc.F + 1))
    # sensor_from_rig is carried unchanged unless it is refined; NormalizeReconstruction scales its translation with
    # the world (reconstruction_normalizer.cc:70-77), so the translations keep their directions and common ratio
    q_in, t_in = _sensors(tmp_path / "in")
    q_out, t_out = _sensors(out)
    ratio = np.linalg.norm(t_out, axis=1) / np.linalg.norm(t_in, axis=1)
    unchanged = np.array_equal(q_in, q_out) and np.ptp(ratio) < 1e-12 * ratio.mean() and \
        np.abs(t_out / ratio.mean() - t_in).max() < 1e-12
    assert unchanged != optimize_rig_poses, (np.abs(q_in - q_out).max(), np.ptp(ratio))


def test_the_command_adds_nothing(tmp_path, monkeypatch):
    """What it writes is GlobalMapper.Solve's result, bit for bit; and an in-process Solve on the same scene with the
    same options and camera_prior_focal = zeros gives the same poses, points and intrinsics, to 1e-9.  Two solves are
    not compared bit for bit because the device solve is not bit-reproducible from run to run: global positioning
    accumulates its normal equations with double-precision atomicAdd (gp_kernels.cuh), whose order of additions
    varies, and the last-bit differences carry through the filters and bundle adjustment."""
    from glomap_b200 import mapper as M
    sc = _rig_input(tmp_path)
    results = []
    solve = M.GlobalMapper.Solve

    def keep(self, *a, **kw):
        ok, res = solve(self, *a, **kw)
        results.append(res)
        return ok, res
    monkeypatch.setattr(M.GlobalMapper, "Solve", keep)
    out = _run(tmp_path / "in", tmp_path / "out")
    monkeypatch.setattr(M.GlobalMapper, "Solve", solve)
    scene, index, registered = MR.read_input(str(tmp_path / "in"))
    CIO.write_model(str(tmp_path / "direct"), *CIO.model_from_scene(results[0], CIO.reindex_observations(index, scene, results[0])))
    for n in ("cameras.bin", "images.bin", "points3D.bin", "rigs.bin", "frames.bin"):
        assert (tmp_path / "direct" / n).read_bytes() == open(os.path.join(out, n), "rb").read(), n
    _, opts = MR.parse_args(["--input_path", "x", "--output_path", "y"])
    ok, res = M.GlobalMapper(opts).Solve(MR.empty_view_graph(scene.I), scene,
                                         camera_prior_focal=np.zeros(len(scene.intr_model), bool), registered=registered,
                                         keep_input_state=True)
    assert ok and res.N == results[0].N and np.array_equal(res.obs_xy, results[0].obs_xy)
    for f in ("quat", "trans", "points", "sensor_quat", "sensor_trans", "intr_params"):
        a, b = getattr(res, f), getattr(results[0], f)
        assert np.abs(a - b).max() <= 1e-9 * max(1.0, np.abs(b).max()), f
    assert sc.F == res.F


def test_unregistered_image_and_frame_keep_their_pose(tmp_path):
    d = S.make_rig_dataset(2, 2, 7, 100, seed=11)
    model = list(CIO.model_from_scene(d.scene))
    cams, ims, pts, rigs, frames = model
    # frame 14 is not stored (its images 27, 28 lose their observations); image 100 is listed by no frame
    reg = np.ones(d.scene.F, bool)
    reg[13] = False
    cams, ims, pts, rigs, frames = CIO.model_from_scene(d.scene, frame_registered=reg)
    ims[100] = CIO.Image(100, np.array([0.6, 0.8, 0, 0]), np.array([1.0, 2, 3]), 2, "lone.png",
                         np.array([[1.0, 2], [3, 4]]), np.full(2, CIO.INVALID_POINT3D, np.uint64))
    CIO.write_model(str(tmp_path / "in"), cams, ims, pts, rigs, frames)
    out = _run(tmp_path / "in", tmp_path / "out")
    _, ims_out, _ = CIO.read_model(out)
    _, frames_out = CIO.read_rigs_frames(out)
    assert 14 not in frames_out and len(frames_out) == d.scene.F - 1
    for iid in (27, 28, 100):
        a, b = ims[iid], ims_out[iid]
        assert np.array_equal(a.qvec_wxyz, b.qvec_wxyz) and np.array_equal(a.tvec, b.tvec)
        assert (b.point3D_ids == CIO.INVALID_POINT3D).all()


def test_pruning_writes_one_model_per_cluster(tmp_path):
    """Two groups of frames joined by a weak bridge: --skip_pruning 0 writes OUT/0 and OUT/1 with their images (the
    solves are skipped so that the tracks keep the shape make_cluster_tracks gives them)."""
    t = S.make_cluster_tracks([5, 6], 40, bridges=[(0, 5, 35)], seed=4)
    F, N = t["num_frames"], len(t["obs_frame"])
    R, tr = S.make_cameras(F, seed=2)
    rng = np.random.default_rng(6)
    P = len(t["track_begin"]) - 1
    cam_intr, intr_model, intr_params = S.make_intrinsics(F, S.SIMPLE_PINHOLE, 1000.0, 1000, 1)
    sc = S.Scene(G.rotmat_to_quat_xyzw_fast(R), tr, rng.normal(size=(P, 3)) * 0.5, t["track_begin"], t["obs_frame"],
                 rng.uniform(0, 1000, size=(N, 2)), cam_intr, intr_model, intr_params)
    CIO.write_model(str(tmp_path / "in"), *CIO.model_from_scene(sc))
    rc = MR.main(["--input_path", str(tmp_path / "in"), "--output_path", str(tmp_path / "out"), "--skip_pruning", "0",
                  "--skip_global_positioning", "1", "--skip_bundle_adjustment", "1"])
    assert rc == 0
    assert sorted(os.listdir(tmp_path / "out")) == ["0", "1"]
    got = [sorted(CIO.read_model(str(tmp_path / "out" / c))[1]) for c in ("0", "1")]
    groups = [sorted(int(i) + 1 for i in np.flatnonzero(t["group"] == g)) for g in (0, 1)]
    assert sorted(got) == sorted(groups) and len(got[0]) >= len(got[1])        # clusters numbered by size


def test_text_and_binary_output_hold_the_same_records(tmp_path, monkeypatch):
    """The same solve written in both layouts (the solve itself is run once: Solve is replayed for the second run)."""
    from glomap_b200 import mapper as M
    sc = S.make_scene(20, 800, mean_track_len=6, seed=23, pixel_sigma=0.5)
    CIO.write_model(str(tmp_path / "in"), *CIO.model_from_scene(_scramble(sc)))
    solve, memo = M.GlobalMapper.Solve, {}

    def once(self, *a, **kw):
        if "res" not in memo:
            memo["res"] = solve(self, *a, **kw)
        return memo["res"]
    monkeypatch.setattr(M.GlobalMapper, "Solve", once)
    b = _run(tmp_path / "in", tmp_path / "bin", "--output_format", "bin")
    t = _run(tmp_path / "in", tmp_path / "txt", "--output_format", "txt")
    assert CIO.model_format(t) == "txt"
    for x, y in zip(CIO.read_model(b), CIO.read_model(t)):
        assert x.keys() == y.keys()
        for k in x:
            for f, u in vars(x[k]).items():
                v = getattr(y[k], f)
                assert (np.array_equal(u, v) if isinstance(u, np.ndarray) else u == v), (k, f)


def _with_two_view_tracks(sc, n_short):
    """``sc`` with its first ``n_short`` tracks cut to their first 2 observations."""
    lens = np.diff(sc.pt_obs_begin)
    rank = np.arange(sc.N) - np.repeat(sc.pt_obs_begin[:-1], lens)
    pt = np.repeat(np.arange(sc.P), lens)
    from glomap_b200 import mapper as M
    return M.compact_observations(sc, (pt >= n_short) | (rank < 2))


def test_positioner_keeps_what_it_does_not_randomise():
    """Given input centres and points, GlobalPositioner randomises only the frames observed by a track of
    >= min_num_view_per_track views and those tracks (global_positioning.cc:145-151, 258-263); with optimize_positions
    off it starts from, and keeps, every input centre."""
    from glomap_b200 import estimators as E
    sc = _with_two_view_tracks(S.make_scene(20, 600, mean_track_len=5, seed=31), 100)
    lens = np.diff(sc.pt_obs_begin)
    long_obs = np.repeat(lens >= 3, lens)
    from glomap_b200 import mapper as M
    sc = M.compact_observations(sc, ~((sc.obs_cam == 19) & long_obs))        # camera 19: in 2-view tracks only
    lens = np.diff(sc.pt_obs_begin)
    short = lens < 3
    assert short[:100].all() and (sc.obs_cam == 19).any()
    rng = np.random.default_rng(8)
    c0, x0 = rng.normal(size=(sc.C, 3)), rng.normal(size=(sc.P, 3))
    R = G.quat_xyzw_to_rotmat(sc.quat)
    for optimize_positions in (True, False):
        prob = E.PositioningProblem(sc.quat, sc.pt_obs_begin, sc.obs_cam, S.bearings_from_scene(sc),
                                    centers=c0.copy(), points=x0.copy())
        gp = E.GlobalPositioner(E.GlobalPositionerOptions(optimize_positions=optimize_positions))
        assert gp.Solve(prob)
        assert np.array_equal(prob.points[short], x0[short])
        assert not np.isclose(prob.points[~short], x0[~short]).all(axis=1).any()
        if optimize_positions:
            assert np.array_equal(prob.centers[19], c0[19])
            assert not np.isclose(prob.centers[:19], c0[:19]).all(axis=1).any()
        else:
            assert np.array_equal(prob.centers, c0)
            assert np.allclose(prob.trans, -np.einsum("nij,nj->ni", R, c0))


def test_two_view_tracks_keep_their_xyz_with_fixed_positions(tmp_path):
    """--GlobalPositioning.optimize_positions 0 on a model at the ground-truth poses with 2-view tracks at their true
    xyz and the other points scrambled: the solve stays in the input's frame, the 2-view tracks are not optimised and
    keep their xyz (up to NormalizeReconstruction's similarity), and the poses meet the noise-free thresholds."""
    sc = _with_two_view_tracks(S.make_scene(30, 2000, mean_track_len=6, seed=24), 300)
    start = sc.copy()
    long = np.diff(sc.pt_obs_begin) >= 3
    start.points[long] = np.random.default_rng(9).normal(size=(int(long.sum()), 3))
    CIO.write_model(str(tmp_path / "in"), *CIO.model_from_scene(start))
    out = _run(tmp_path / "in", tmp_path / "out", "--GlobalPositioning.optimize_positions", "0")
    _, ims, pts = CIO.read_model(out)
    q = np.array([ims[i].qvec_wxyz for i in range(1, sc.C + 1)])
    R = G.quat_xyzw_to_rotmat(q[:, [1, 2, 3, 0]])
    t = np.array([ims[i].tvec for i in range(1, sc.C + 1)])
    rot, cen, (s, Ra, ta) = G.compare_reconstructions(R, t, G.quat_xyzw_to_rotmat(sc.quat), sc.trans)
    assert rot < 1e-2 and cen < 1e-4, (rot, cen)
    kept = [j for j in range(300) if j + 1 in pts]
    assert len(kept) > 200
    X = np.array([pts[j + 1].xyz for j in kept])
    assert np.abs(s * X @ Ra.T + ta - sc.points[kept]).max() < 1e-4
