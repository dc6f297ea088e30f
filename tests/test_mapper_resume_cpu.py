"""Rig-aware COLMAP model I/O and the mapper_resume command off the GPU: known-answer bytes for rigs.bin and
frames.bin, record-identical round trips through the scene in both layouts, the vectorised conversions against the
per-element code they replace, the rejections, the flags and the cluster writer on rigs (reference:
glomap/io/colmap_converter.cc:22-209, io/colmap_io.cc:8-66, exe/global_mapper.cc:110-172)."""
import os
import struct

import numpy as np
import pytest

from glomap_b200 import colmap_io as CIO, geometry as G, mapper as M, mapper_resume as MR, synthetic as S

FILES = {"bin": ("cameras.bin", "images.bin", "points3D.bin", "rigs.bin", "frames.bin"),
         "txt": ("cameras.txt", "images.txt", "points3D.txt", "rigs.txt", "frames.txt")}


# ---------------------------------------------------------------------------- the per-element conversions replaced
def legacy_scene_from_model(cameras, images, points):
    cam_ids = np.array(sorted(cameras), np.int64)
    img_ids = np.array(sorted(images), np.int64)
    pt_ids = np.array(sorted(points), np.uint64)
    cidx = {int(c): i for i, c in enumerate(cam_ids)}
    iidx = {int(i): k for k, i in enumerate(img_ids)}
    K, C, P = len(cam_ids), len(img_ids), len(pt_ids)
    intr_model = np.array([cameras[int(c)].model_id for c in cam_ids], np.int32)
    intr = np.zeros((K, S.INTR_STRIDE))
    for k, c in enumerate(cam_ids):
        p = cameras[int(c)].params
        intr[k, :len(p)] = p
    quat, trans, cam_intr = np.empty((C, 4)), np.empty((C, 3)), np.empty(C, np.int32)
    for k, i in enumerate(img_ids):
        im = images[int(i)]
        quat[k] = [im.qvec_wxyz[1], im.qvec_wxyz[2], im.qvec_wxyz[3], im.qvec_wxyz[0]]
        trans[k] = im.tvec
        cam_intr[k] = cidx[im.camera_id]
    pts = np.empty((P, 3))
    begin, obs_cam, obs_xy, obs_feat = [0], [], [], []
    for j, pid in enumerate(pt_ids):
        p = points[int(pid)]
        pts[j] = p.xyz
        for iid, fi in zip(p.image_ids, p.point2D_idxs):
            if int(iid) not in iidx:
                continue
            obs_cam.append(iidx[int(iid)]); obs_xy.append(images[int(iid)].xy[int(fi)]); obs_feat.append(int(fi))
        begin.append(len(obs_cam))
    scene = S.Scene(quat, trans, pts, np.asarray(begin, np.int64), np.asarray(obs_cam, np.int32),
                    np.asarray(obs_xy, np.float64).reshape(-1, 2), cam_intr, intr_model, intr)
    index = CIO.ModelIndex(cam_ids, np.array([[cameras[int(c)].width, cameras[int(c)].height] for c in cam_ids], np.int64),
                           img_ids, [images[int(i)].name for i in img_ids], [images[int(i)].xy for i in img_ids], pt_ids,
                           np.array([points[int(p)].rgb for p in pt_ids], np.uint8).reshape(-1, 3),
                           np.asarray(obs_feat, np.int64))
    return scene, index


def legacy_model_from_scene(scene, index=None, min_supports=2):
    from glomap_b200 import geometry as geo
    C, P, K = scene.C, scene.P, len(scene.intr_model)
    if index is None:
        index = CIO.default_index(scene)
    cameras = {}
    for k in range(K):
        m = int(scene.intr_model[k])
        cameras[int(index.camera_ids[k])] = CIO.Camera(int(index.camera_ids[k]), m, int(index.camera_size[k, 0]),
                                                        int(index.camera_size[k, 1]), scene.intr_params[k, :CIO.NUM_PARAMS[m]].copy())
    p3d_ids = [np.full(len(index.image_xy[i]), CIO.INVALID_POINT3D, np.uint64) for i in range(C)]
    R = geo.quat_xyzw_to_rotmat(scene.quat)
    pt_of_obs = np.repeat(np.arange(P), np.diff(scene.pt_obs_begin))
    Xc = np.einsum("nij,nj->ni", R[scene.obs_cam], scene.points[pt_of_obs]) + scene.trans[scene.obs_cam]
    err = np.zeros(scene.N)
    ci = scene.cam_intr[scene.obs_cam]
    for k in range(K):
        mk = ci == k
        if mk.any():
            err[mk] = np.linalg.norm(S.project(int(scene.intr_model[k]), scene.intr_params[k], Xc[mk]) - scene.obs_xy[mk], axis=1)
    points = {}
    for j in range(P):
        a, b = int(scene.pt_obs_begin[j]), int(scene.pt_obs_begin[j + 1])
        if b - a < min_supports:
            continue
        pid = int(index.point_ids[j])
        img = index.image_ids[scene.obs_cam[a:b]].astype(np.uint32)
        points[pid] = CIO.Point3D(pid, scene.points[j].copy(), index.point_rgb[j].copy(), float(err[a:b].mean()), img,
                                  index.obs_feature[a:b].astype(np.uint32))
        for o in range(a, b):
            p3d_ids[int(scene.obs_cam[o])][int(index.obs_feature[o])] = pid
    images = {}
    for i in range(C):
        q = scene.quat[i] / np.linalg.norm(scene.quat[i])
        images[int(index.image_ids[i])] = CIO.Image(int(index.image_ids[i]), np.array([q[3], q[0], q[1], q[2]]),
                                                    scene.trans[i].copy(), int(index.camera_ids[scene.cam_intr[i]]),
                                                    index.image_names[i], np.asarray(index.image_xy[i], np.float64).reshape(-1, 2),
                                                    p3d_ids[i])
    return cameras, images, points


# ---------------------------------------------------------------------------- helpers
def _files_equal(a, b, fmt):
    names = [n for n in FILES[fmt] if os.path.exists(os.path.join(a, n))]
    assert names == [n for n in FILES[fmt] if os.path.exists(os.path.join(b, n))]
    for n in names:
        assert open(os.path.join(a, n), "rb").read() == open(os.path.join(b, n), "rb").read(), n
    return names


def _read(path):
    return CIO.scene_from_model(*CIO.read_model(path), *CIO.read_rigs_frames(path))


def _round_trip(model, tmp_path, fmt):
    a, b = str(tmp_path / f"{fmt}_a"), str(tmp_path / f"{fmt}_b")
    CIO.write_model(a, *model, fmt=fmt)
    scene, index = _read(a)
    CIO.write_model(b, *CIO.model_from_scene(scene, index), fmt=fmt)
    return _files_equal(a, b, fmt), scene, index


def _rig_model(seed=11):
    d = S.make_rig_dataset(2, 2, 3, 60, seed=seed)
    return d.scene, CIO.model_from_scene(d.scene)


def _model_with_orphan():
    """A rig model with two more images (ids 100, 101, cameras 2 and 3) that no frame lists."""
    sc, (cams, ims, pts, rigs, frames) = _rig_model()
    rng = np.random.default_rng(5)
    for iid, cam in ((100, 2), (101, 3)):
        q = rng.normal(size=4)
        ims[iid] = CIO.Image(iid, q / np.linalg.norm(q), rng.normal(size=3), cam, f"lone_{iid}.png",
                             rng.uniform(0, 1000, size=(7, 2)), np.full(7, CIO.INVALID_POINT3D, np.uint64))
    return sc, (cams, ims, pts, rigs, frames)


# ---------------------------------------------------------------------------- known-answer bytes
def _kat_bytes():
    q, t = (0.5, 0.5, 0.5, 0.5), (0.1, -0.2, 0.3)
    rigs = (struct.pack("<Q", 1) + struct.pack("<II", 4, 2) + struct.pack("<iI", 0, 7)
            + struct.pack("<iIB", 0, 8, 1) + struct.pack("<4d", *q) + struct.pack("<3d", *t))
    frames = (struct.pack("<Q", 1) + struct.pack("<II", 5, 4) + struct.pack("<4d", 1.0, 0, 0, 0) + struct.pack("<3d", 1, 2, 3)
              + struct.pack("<I", 2) + struct.pack("<iIQ", 0, 7, 3) + struct.pack("<iIQ", 0, 8, 9))
    return rigs, frames


def test_known_answer_bytes_rigs_and_frames(tmp_path):
    """One rig (reference sensor: camera 7; camera 8 with a sensor_from_rig), one frame with two images."""
    rigs_b, frames_b = _kat_bytes()
    (tmp_path / "rigs.bin").write_bytes(rigs_b)
    (tmp_path / "frames.bin").write_bytes(frames_b)
    rigs = CIO.read_rigs(str(tmp_path / "rigs.bin"))
    frames = CIO.read_frames(str(tmp_path / "frames.bin"))
    r = rigs[4]
    assert r.ref_sensor == (0, 7) and len(r.sensors) == 1
    typ, sid, sq, st = r.sensors[0]
    assert (typ, sid) == (0, 8) and np.array_equal(sq, [0.5] * 4) and np.array_equal(st, [0.1, -0.2, 0.3])
    f = frames[5]
    assert f.rig_id == 4 and np.array_equal(f.qvec_wxyz, [1, 0, 0, 0]) and np.array_equal(f.tvec, [1, 2, 3])
    assert f.data_ids == [(0, 7, 3), (0, 8, 9)]
    CIO.write_rigs(str(tmp_path / "r2.bin"), rigs)
    CIO.write_frames(str(tmp_path / "f2.bin"), frames)
    assert (tmp_path / "r2.bin").read_bytes() == rigs_b and (tmp_path / "f2.bin").read_bytes() == frames_b
    # a sensor without a pose: has_pose 0 and nothing after it
    nopose = struct.pack("<Q", 1) + struct.pack("<II", 4, 2) + struct.pack("<iI", 0, 7) + struct.pack("<iIB", 0, 8, 0)
    (tmp_path / "r3.bin").write_bytes(nopose)
    assert CIO.read_rigs(str(tmp_path / "r3.bin"))[4].sensors == [(0, 8, None, None)]
    # the text layout holds the same records
    CIO.write_rigs_text(str(tmp_path / "rigs.txt"), rigs)
    CIO.write_frames_text(str(tmp_path / "frames.txt"), frames)
    assert "4 2 CAMERA 7 CAMERA 8 1 0.5 0.5 0.5 0.5 0.10000000000000001 -0.20000000000000001 0.29999999999999999" in \
        (tmp_path / "rigs.txt").read_text()
    rt, ft = CIO.read_rigs_text(str(tmp_path / "rigs.txt")), CIO.read_frames_text(str(tmp_path / "frames.txt"))
    assert rt[4].ref_sensor == (0, 7) and np.array_equal(rt[4].sensors[0][2], sq) and ft[5].data_ids == f.data_ids


def test_known_answer_model_converts_to_a_rig_scene(tmp_path):
    """The known-answer rig and frame with two cameras and images: the frame's images get composed poses."""
    rigs_b, frames_b = _kat_bytes()
    cams = {7: CIO.Camera(7, 0, 100, 100, np.array([100.0, 50, 50])), 8: CIO.Camera(8, 1, 100, 100, np.array([90.0, 95, 50, 50]))}
    ims = {3: CIO.Image(3, np.array([1.0, 0, 0, 0]), np.zeros(3), 7, "a.png", np.array([[1.0, 2], [3, 4]]), np.full(2, CIO.INVALID_POINT3D)),
           9: CIO.Image(9, np.array([1.0, 0, 0, 0]), np.zeros(3), 8, "b.png", np.array([[5.0, 6]]), np.full(1, CIO.INVALID_POINT3D))}
    pts = {11: CIO.Point3D(11, np.array([0.0, 0, 5]), np.array([1, 2, 3], np.uint8), 0.0, np.array([3, 9], np.uint32),
                           np.array([1, 0], np.uint32))}
    CIO.write_model(str(tmp_path), cams, ims, pts)
    (tmp_path / "rigs.bin").write_bytes(rigs_b)
    (tmp_path / "frames.bin").write_bytes(frames_b)
    sc, idx = _read(str(tmp_path))
    assert isinstance(sc, S.RigScene) and sc.F == 1 and sc.S == 2 and sc.I == 2
    assert sc.image_frame.tolist() == [0, 0] and sc.image_sensor.tolist() == [0, 1] and sc.rig_ref_sensor.tolist() == [0]
    assert np.array_equal(sc.sensor_quat[1], [0.5, 0.5, 0.5, 0.5]) and np.array_equal(sc.sensor_trans[1], [0.1, -0.2, 0.3])
    assert sc.obs_frame.tolist() == [0, 0] and sc.obs_sensor.tolist() == [0, 1]
    assert np.array_equal(sc.obs_xy, [[3, 4], [5, 6]]) and idx.point_rgb.tolist() == [[1, 2, 3]]
    cams2, ims2, pts2, rigs2, frames2 = CIO.model_from_scene(sc, idx)
    R, t = sc.image_poses()
    from glomap_b200 import geometry as geo
    q = geo.rotmat_to_quat_xyzw_fast(R[1:])[0]
    assert np.allclose(ims2[9].qvec_wxyz, [q[3], q[0], q[1], q[2]]) and np.allclose(ims2[9].tvec, t[1])
    assert ims2[3].point3D_ids.tolist() == [CIO.INVALID_POINT3D, 11] and ims2[9].point3D_ids.tolist() == [11]
    assert list(pts2[11].rgb) == [1, 2, 3]


# ---------------------------------------------------------------------------- round trips
@pytest.mark.parametrize("fmt", ["bin", "txt"])
def test_multi_rig_model_round_trips(tmp_path, fmt):
    sc, model = _rig_model()
    names, sc2, idx = _round_trip(model, tmp_path, fmt)
    assert len(names) == 5 and isinstance(sc2, S.RigScene)
    assert idx.frame_registered.all() and sc2.F == sc.F and sc2.I == sc.I and sc2.N == sc.N
    assert np.array_equal(sc2.obs_xy, sc.obs_xy) and np.array_equal(sc2.pt_obs_begin, sc.pt_obs_begin)
    assert np.array_equal(sc2.frame_rig, sc.frame_rig) and np.array_equal(sc2.rig_ref_sensor, sc.rig_ref_sensor)
    assert np.abs(sc2.sensor_trans - sc.sensor_trans).max() == 0


@pytest.mark.parametrize("fmt", ["bin", "txt"])
def test_unregistered_frame_round_trips(tmp_path, fmt):
    """A frame without a pose is not stored: its images stay, with their poses, unregistered and unobserved."""
    sc, model = _rig_model()
    reg = np.ones(sc.F, bool)
    reg[2] = False
    model = CIO.model_from_scene(sc, frame_registered=reg)
    assert 3 not in model[4] and len(model[1]) == sc.I
    names, sc2, idx = _round_trip(model, tmp_path, fmt)
    assert idx.frame_registered.sum() == sc.F - 1 and sc2.F == sc.F + 1     # each of its 2 images gets a frame
    unreg = np.flatnonzero(~idx.frame_registered[sc2.image_frame])
    assert len(unreg) == 2
    for k in unreg:
        im = model[1][int(idx.image_ids[k])]
        assert (im.point3D_ids == CIO.INVALID_POINT3D).all()
        assert not np.isin(sc2.image_frame[k], sc2.obs_frame)


@pytest.mark.parametrize("fmt", ["bin", "txt"])
def test_image_whose_frame_is_missing_round_trips(tmp_path, fmt):
    sc, model = _model_with_orphan()
    names, sc2, idx = _round_trip(model, tmp_path, fmt)
    orphan = np.flatnonzero(idx.frame_ids[sc2.image_frame] < 0)
    assert idx.image_ids[orphan].tolist() == [100, 101] and not idx.frame_registered[sc2.image_frame[orphan]].any()
    assert sc2.F == sc.F + 2 and idx.frame_registered.sum() == sc.F
    # the orphan frames have the rig of their cameras and the pose that reproduces the images' cam_from_world
    assert sc2.frame_rig[sc2.image_frame[orphan]].tolist() == sc2.sensor_rig[[1, 2]].tolist()
    R, t = sc2.image_poses()
    for k in orphan:
        im = model[1][int(idx.image_ids[k])]
        q = im.qvec_wxyz
        Rq = G.quat_xyzw_to_rotmat(np.array([q[1], q[2], q[3], q[0]]))
        assert np.abs(R[k] - Rq).max() < 1e-12 and np.abs(t[k] - im.tvec).max() < 1e-12


def test_binary_and_text_give_the_same_scene(tmp_path):
    sc = S.make_scene(10, 150, mean_track_len=5, seed=4, pixel_sigma=0.5, model=S.SIMPLE_RADIAL, num_intrinsics=3)
    model = CIO.model_from_scene(sc)
    CIO.write_model(str(tmp_path / "b"), *model, fmt="bin")
    CIO.write_model(str(tmp_path / "t"), *model, fmt="txt")
    assert CIO.model_format(str(tmp_path / "t")) == "txt"
    (a, ia), (b, ib) = _read(str(tmp_path / "b")), _read(str(tmp_path / "t"))
    assert isinstance(a, S.Scene) and isinstance(b, S.Scene)
    for f in ("quat", "trans", "points", "pt_obs_begin", "obs_cam", "obs_xy", "cam_intr", "intr_model", "intr_params"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert np.array_equal(ia.obs_feature, ib.obs_feature) and ia.image_names == ib.image_names
    # and the text model converted back to binary is the binary model
    CIO.write_model(str(tmp_path / "tb"), *CIO.model_from_scene(b, ib), fmt="bin")
    CIO.write_model(str(tmp_path / "bb"), *CIO.model_from_scene(a, ia), fmt="bin")
    _files_equal(str(tmp_path / "tb"), str(tmp_path / "bb"), "bin")


def _io_models():
    """The models of test_colmap_io_cpu.py."""
    sc = S.make_scene(12, 200, mean_track_len=5, seed=3, pixel_sigma=0.5, model=S.RADIAL, num_intrinsics=2)
    yield sc
    sc = S.make_scene(8, 60, mean_track_len=4, seed=5)
    lens = np.diff(sc.pt_obs_begin)
    keep = np.ones(sc.N, bool)
    keep[1:lens[0]] = False
    sc.obs_cam, sc.obs_xy = sc.obs_cam[keep], sc.obs_xy[keep]
    lens[0] = 1
    sc.pt_obs_begin = np.concatenate([[0], np.cumsum(lens)])
    yield sc


def _same_model(a, b):
    for x, y in zip(a, b):
        assert x.keys() == y.keys()
        for k in x:
            for f in dataclasses_fields(x[k]):
                u, v = getattr(x[k], f), getattr(y[k], f)
                assert (np.array_equal(u, v) if isinstance(u, np.ndarray) else u == v), (k, f)


def dataclasses_fields(obj):
    import dataclasses
    return [f.name for f in dataclasses.fields(obj)]


def test_vectorised_conversions_match_the_per_element_code():
    for sc in _io_models():
        model = legacy_model_from_scene(sc)
        _same_model(CIO.model_from_scene(sc), model)
        cams, ims, pts = model
        del ims[3]                                                        # track elements of a missing image are skipped
        for m in (model, (cams, ims, pts)):
            new, ni = CIO.scene_from_model(*m)
            old, oi = legacy_scene_from_model(*m)
            for f in ("quat", "trans", "points", "pt_obs_begin", "obs_cam", "obs_xy", "cam_intr", "intr_model", "intr_params"):
                assert np.array_equal(getattr(new, f), getattr(old, f)), f
            assert np.array_equal(ni.obs_feature, oi.obs_feature) and np.array_equal(ni.point_rgb, oi.point_rgb)
            _same_model(CIO.model_from_scene(new, ni), legacy_model_from_scene(old, oi))


# ---------------------------------------------------------------------------- rejections
def _main(argv, capsys):
    rc = MR.main(argv)
    return rc, capsys.readouterr().err


def test_rejections_name_the_problem_and_exit_2(tmp_path, capsys):
    sc, model = _rig_model()
    out = str(tmp_path / "out")
    # camera model 4 (OPENCV)
    cams, ims, pts = CIO.model_from_scene(S.make_scene(6, 40, mean_track_len=4, seed=2))
    for c in cams.values():
        c.model_id, c.params = 4, np.array([500.0, 500, 50, 50, 0, 0, 0, 0])
    CIO.write_model(str(tmp_path / "opencv"), cams, ims, pts)
    rc, err = _main(["--input_path", str(tmp_path / "opencv"), "--output_path", out], capsys)
    assert rc == 2 and "camera model 4" in err
    # a non-reference sensor without a pose that images of registered frames use
    cams, ims, pts, rigs, frames = model
    r = rigs[1]
    r.sensors[0] = (r.sensors[0][0], r.sensors[0][1], None, None)
    CIO.write_model(str(tmp_path / "nopose"), cams, ims, pts, rigs, frames)
    rc, err = _main(["--input_path", str(tmp_path / "nopose"), "--output_path", out], capsys)
    assert rc == 2 and "has no sensor_from_rig" in err
    # truncated files, every one of the five binary files (a text file cut at a line end is a smaller valid model),
    # and a text images file cut between an image and its points
    (tmp_path / "cut_txt").mkdir()
    CIO.write_model(str(tmp_path / "cut_txt"), *_rig_model()[1], fmt="txt")
    lines = (tmp_path / "cut_txt" / "images.txt").read_text().splitlines(keepends=True)
    (tmp_path / "cut_txt" / "images.txt").write_text("".join(lines[:-1]))
    rc, err = _main(["--input_path", str(tmp_path / "cut_txt"), "--output_path", out], capsys)
    assert rc == 2 and "truncated" in err
    for fmt in ("bin",):
        good = tmp_path / f"good_{fmt}"
        CIO.write_model(str(good), *_rig_model()[1], fmt=fmt)
        for name in FILES[fmt]:
            bad = tmp_path / f"trunc_{fmt}_{name}"
            bad.mkdir()
            for n in FILES[fmt]:
                data = (good / n).read_bytes()
                (bad / n).write_bytes(data[:len(data) * 2 // 3] if n == name else data)
            rc, err = _main(["--input_path", str(bad), "--output_path", out], capsys)
            assert rc == 2 and err.startswith("mapper_resume:"), (fmt, name, err)
            assert "truncated" in err, (fmt, name, err)
    # --image_path
    rc, err = _main(["--input_path", str(good), "--output_path", out, "--image_path", "/images"], capsys)
    assert rc == 2 and "colour extraction" in err
    assert not os.path.exists(out)


# ---------------------------------------------------------------------------- flags
def test_flags_parse_to_the_options_and_default_to_the_resume_options():
    _, opts = MR.parse_args(["--input_path", "a", "--output_path", "b"])
    ref = M.GlobalMapperOptions(skip_preprocessing=True, skip_view_graph_calibration=True, skip_rotation_averaging=True,
                                skip_track_establishment=True)
    assert opts == ref
    assert opts.skip_pruning and not opts.skip_global_positioning and opts.num_iteration_bundle_adjustment == 3
    values = {int: 7, float: 0.375, bool: None, str: "3"}
    argv = ["--input_path", "a", "--output_path", "b", "--retriangulation_iteration_num", "4", "--Triangulation.min_angle",
            "2.5", "--Triangulation.complete_max_reproj_error", "1", "--Triangulation.merge_max_reproj_error", "1",
            "--Triangulation.min_num_matches", "9"]
    expect = {}
    for flag, path, typ in MR._FLAGS:
        v = values[typ]
        if typ is bool:
            v = not MR._get(ref, path)
            argv += [f"--{flag}", "1" if v else "0"]
        else:
            argv += [f"--{flag}", str(v)]
        expect[path] = v
    _, opts = MR.parse_args(argv)
    for path, v in expect.items():
        assert MR._get(opts, path) == v, path
    names = {f for f, _, _ in MR._FLAGS}
    for f in ("ba_iteration_num", "skip_global_positioning", "skip_bundle_adjustment", "skip_pruning"):
        assert f in names
    for f in ("optimize_positions", "optimize_points", "optimize_scales", "thres_loss_function", "max_num_iterations",
              "gpu_index"):
        assert f"GlobalPositioning.{f}" in names
    for f in ("optimize_rig_poses", "optimize_rotations", "optimize_translation", "optimize_intrinsics",
              "optimize_principal_point", "optimize_points", "thres_loss_function", "max_num_iterations", "gpu_index"):
        assert f"BundleAdjustment.{f}" in names
    for f in ("max_angle_error", "max_reprojection_error", "min_triangulation_angle"):
        assert f"Thresholds.{f}" in names
    with pytest.raises(MR.InputError):
        MR.parse_args(["--input_path", "a", "--output_path", "b", "--skip_pruning", "maybe"])
    with pytest.raises(MR.InputError):
        MR.parse_args(["--input_path", "a", "--output_path", "b", "--output_format", "ply"])


# ---------------------------------------------------------------------------- cluster writer on rigs
@pytest.mark.parametrize("fmt", ["bin", "txt"])
def test_cluster_writer_on_rigs(tmp_path, fmt):
    sc, _ = _rig_model()                                     # 6 frames (2 rigs x 3), 12 images, 4 cameras
    idx = CIO.default_index(sc)
    cid = np.array([0, 0, 1, 1, -1, 0])
    reg = np.array([True, True, True, False, False, False])
    written = CIO.write_clustered_model(str(tmp_path), sc, idx, cid, reg, fmt)
    assert written == [str(tmp_path / "0"), str(tmp_path / "1")]
    images_of = {f: set(int(i) for i in idx.image_ids[sc.image_frame == f]) for f in range(sc.F)}
    for c, path, frames_kept, obs_frames in ((0, written[0], [0, 1, 5], [0, 1]), (1, written[1], [2], [2])):
        cams, ims, pts = CIO.read_model(path)
        rigs, frames = CIO.read_rigs_frames(path)
        # every camera and rig; the frames of cluster c (frame 5: unregistered, kept by the cluster_id != 0 rule of
        # cluster 0); frame 3 (cluster 1, unregistered) is deregistered
        assert sorted(cams) == [1, 2, 3, 4] and sorted(rigs) == [1, 2]
        assert sorted(frames) == [f + 1 for f in frames_kept]
        assert set(ims) == set().union(*(images_of[f] for f in frames_kept))
        observed = set().union(*(images_of[f] for f in obs_frames))
        for iid, im in ims.items():
            has = (im.point3D_ids != CIO.INVALID_POINT3D).any()
            assert has == (iid in observed), (c, iid)
        for p in pts.values():
            assert set(p.image_ids.tolist()) <= observed and len(p.image_ids) >= 2
    # every id -1: the registered frames, and every image (the others with their pose and no observation)
    written = CIO.write_clustered_model(str(tmp_path / "all"), sc, idx, np.full(sc.F, -1), reg, fmt)
    cams, ims, pts = CIO.read_model(written[0])
    _, frames = CIO.read_rigs_frames(written[0])
    assert sorted(frames) == [1, 2, 3] and len(ims) == sc.I
    for f in (3, 4, 5):
        for iid in images_of[f]:
            assert (ims[iid].point3D_ids == CIO.INVALID_POINT3D).all()


def test_feature_indices_follow_the_mapper_filters():
    """The filters and the compaction to registered images drop observations; each survivor keeps its feature."""
    for sc in (S.make_scene(10, 150, mean_track_len=5, seed=4), _rig_model()[0]):
        model = CIO.model_from_scene(sc)
        scene, index = CIO.scene_from_model(*model) if isinstance(sc, S.Scene) else \
            CIO.scene_from_model(*model[:3], *model[3:])
        keep = np.random.default_rng(1).uniform(size=scene.N) < 0.7
        after = M.compact_observations(scene, keep)
        assert np.array_equal(CIO.reindex_observations(index, scene, after).obs_feature, index.obs_feature[keep])
        moved = after.copy()
        moved.obs_xy = moved.obs_xy + 1.0
        with pytest.raises(ValueError, match="does not have"):
            CIO.reindex_observations(index, scene, moved)


@pytest.mark.parametrize("fmt", ["bin", "txt"])
def test_sensor_without_pose_is_accepted_when_no_registered_image_uses_it(tmp_path, fmt):
    """Global positioning reads only the sensors of registered images: an unused pose-less sensor, or one used only by
    an image that no frame lists, is carried through and written back without a pose."""
    sc, (cams, ims, pts, rigs, frames) = _rig_model()
    cams[9] = CIO.Camera(9, 0, 640, 480, np.array([500.0, 320, 240]))
    cams[10] = CIO.Camera(10, 0, 640, 480, np.array([510.0, 320, 240]))
    rigs[1].sensors.append((CIO.SENSOR_CAMERA, 9, None, None))
    rigs[2].sensors.append((CIO.SENSOR_CAMERA, 10, None, None))
    ims[200] = CIO.Image(200, np.array([0.6, 0.8, 0, 0]), np.array([1.0, 2, 3]), 10, "lone.png", np.array([[1.0, 2]]),
                         np.full(1, CIO.INVALID_POINT3D, np.uint64))
    names, sc2, idx = _round_trip((cams, ims, pts, rigs, frames), tmp_path, fmt)
    assert sc2.sensor_known.tolist() == [True] * 4 + [False] * 2
    rigs2, _ = CIO.read_rigs_frames(str(tmp_path / f"{fmt}_b"))
    assert rigs2[1].sensors[-1] == (CIO.SENSOR_CAMERA, 9, None, None)
    assert rigs2[2].sensors[-1] == (CIO.SENSOR_CAMERA, 10, None, None)


def test_identical_track_elements_keep_their_own_features():
    """A track with two elements of one image at one pixel: each survivor keeps its own feature index."""
    sc = S.make_scene(8, 60, mean_track_len=4, seed=5)
    cams, ims, pts, = CIO.model_from_scene(sc)
    p = pts[1]
    iid, f = int(p.image_ids[0]), int(p.point2D_idxs[0])
    im = ims[iid]
    im.xy = np.vstack([im.xy, im.xy[f]])
    im.point3D_ids = np.r_[im.point3D_ids, np.uint64(1)]
    p.image_ids = np.r_[p.image_ids, np.uint32(iid)]
    p.point2D_idxs = np.r_[p.point2D_idxs, np.uint32(len(im.xy) - 1)]
    scene, index = CIO.scene_from_model(cams, ims, pts)
    dup = np.flatnonzero(index.obs_feature[:scene.pt_obs_begin[1]] == len(im.xy) - 1)
    assert len(dup) == 1
    keep = np.random.default_rng(2).uniform(size=scene.N) < 0.6
    keep[[0, dup[0]]] = True
    after = M.compact_observations(scene, keep)
    feat = CIO.reindex_observations(index, scene, after).obs_feature
    assert np.array_equal(feat, index.obs_feature[keep])
    img0 = after.obs_cam[:after.pt_obs_begin[1]] == scene.obs_cam[0]
    assert sorted(feat[:after.pt_obs_begin[1]][img0].tolist()) == sorted([f, len(im.xy) - 1])
