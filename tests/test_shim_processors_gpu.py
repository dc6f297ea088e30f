"""The shim's TrackFilter, UndistortImages and NormalizeReconstruction built against libb200sfm.so
(tests/shim_mock/processors_driver.cc) on the scenes of tests/test_filters_cpu.py, against the long-double filter oracle
(exact masks and counts once the scene's decision margin clears FP64_BOUND) and the host restatements of
glomap_b200/processors.py (bearings, normalised poses and points to 1e-12 relative); and b200sfm_undistort_features
against b200sfm_ba_problem_undistort, bit for bit, with its error codes."""
import ctypes as ct
import os
import subprocess

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E, processors as PR, synthetic as S
from oracle import filter_oracle as FO
from test_filters_cpu import FP64_BOUND, bearings, image_scene, missing_sensor_rig_scene, oracle_filter, rig_dataset_scene
from test_shim_processors_cpu import parse_output, write_world

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SCENES = {"image": image_scene, "rig_dataset": rig_dataset_scene, "missing_sensor": missing_sensor_rig_scene}


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = tmp_path_factory.mktemp("drv") / "processors_driver"
    libdir = os.path.join(ROOT, "glomap_b200")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(HERE, "shim_mock", "processors_driver.cc"), "-L" + libdir, "-lb200sfm", "-Wl,-rpath," + libdir],
                   check=True, capture_output=True)
    return exe


def world_of(sc, calibrated, bear=None, undist_images=None):
    """The glomap world of a Scene / RigScene: image k has id 1000 - k (sorted order is not row order), camera = the
    image's intrinsics block (Scene) or its sensor (RigScene) with has_prior_focal_length from ``calibrated``, every
    observation is a feature of its image, track p has id 5000 - p.  features_undist holds ``bear`` for the images in
    ``undist_images`` (default: all, when ``bear`` is given)."""
    rig = hasattr(sc, "obs_sensor")
    q, t = np.asarray(sc.quat, float), np.asarray(sc.trans, float)
    if rig:
        n_img, obs_img = sc.I, sc.obs_image()
        img_cam, img_frame = np.asarray(sc.image_sensor), np.asarray(sc.image_frame)
        cams = [(s + 1, int(sc.intr_model[sc.sensor_intr[s]]), bool(calibrated[s]), list(sc.intr_params[sc.sensor_intr[s]]))
                for s in range(sc.S)]
        ref = set(int(r) for r in sc.rig_ref_sensor)
        rigs = [(r + 1, int(sc.rig_ref_sensor[r]) + 1,
                 [(s + 1, list(sc.sensor_quat[s]), list(sc.sensor_trans[s])) for s in range(sc.S)
                  if sc.sensor_rig[s] == r and s not in ref and sc.sensor_known[s]]) for r in range(len(sc.rig_ref_sensor))]
        frames = [(f + 1, int(sc.frame_rig[f]) + 1, True, list(q[f]), list(t[f])) for f in range(sc.F)]
        trivial = [int(img_cam[k]) in ref for k in range(n_img)]
    else:
        n_img, obs_img = sc.C, np.asarray(sc.obs_cam)
        img_cam, img_frame = np.asarray(sc.cam_intr), np.arange(sc.C)
        cal_of = {int(sc.cam_intr[c]): bool(calibrated[c]) for c in range(sc.C)}
        cams = [(k + 1, int(sc.intr_model[k]), cal_of.get(k, True), list(sc.intr_params[k])) for k in range(len(sc.intr_model))]
        rigs = []
        frames = [(1000 - c, 0, True, list(q[c]), list(t[c])) for c in range(sc.C)]
        trivial = [True] * n_img
    feat = [[] for _ in range(n_img)]
    und = [[] for _ in range(n_img)]
    fid = np.empty(sc.N, np.int64)
    for o in range(sc.N):
        k = int(obs_img[o])
        fid[o] = len(feat[k])
        feat[k].append(list(sc.obs_xy[o]))
        if bear is not None:
            und[k].append(list(bear[o]))
    if undist_images is not None:
        und = [u if k in undist_images else [] for k, u in enumerate(und)]
    images = [(1000 - k, int(img_cam[k]) + 1, int(img_frame[k]) + 1 if rig else 1000 - k, trivial[k], feat[k], und[k])
              for k in range(n_img)]
    b = np.asarray(sc.pt_obs_begin)
    tracks = [(5000 - p, list(sc.points[p]), [(1000 - int(obs_img[o]), int(fid[o])) for o in range(b[p], b[p + 1])])
              for p in range(sc.P)]
    return dict(cameras=cams, rigs=rigs, frames=frames, images=images, tracks=tracks), obs_img, fid


def run(driver, tmp_path, w, *op):
    path = tmp_path / "world.txt"
    write_world(path, w)
    r = subprocess.run([str(driver), str(path)] + [str(a) for a in op], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return parse_output(r.stdout), r.stderr


OPS = {"reprojection": lambda thr: ("reprojection", thr, 0), "normalized": lambda thr: ("reprojection", thr, 1),
       "angle": lambda thr: ("angle", thr), "triangulation": lambda thr: ("triangulation", thr)}


@pytest.mark.parametrize("which", sorted(SCENES))
@pytest.mark.parametrize("kind,thr", [("angle", 1.0), ("normalized", 1e-2), ("normalized", 1e-1), ("triangulation", 1.0),
                                      ("triangulation", 25.0), ("reprojection", 3.0)])
def test_track_filters_match_the_oracle(driver, tmp_path, which, kind, thr):
    sc, cal = SCENES[which]()
    bear = bearings(sc)
    margin = FO.smallest_margin(sc, [(kind, thr)], bearings=bear, calibrated=cal, project=S.project)
    assert margin > FP64_BOUND, margin
    keep, cnt = oracle_filter(sc, kind, thr, bear, cal)
    w, obs_img, fid = world_of(sc, cal, bear)
    out, _ = run(driver, tmp_path, w, *OPS[kind](thr))
    assert out["result"] == [cnt]
    b = np.asarray(sc.pt_obs_begin)
    for p in range(sc.P):
        obs = [(1000 - int(obs_img[o]), int(fid[o])) for o in range(b[p], b[p + 1])]
        want = ([ob for ob, k in zip(obs, keep[b[p]:b[p + 1]]) if k] if kind != "triangulation" else (obs if keep[p] else []))
        assert out["track"][5000 - p][1] == want, p


def test_rig_sensor_without_cam_from_rig_is_refused(driver, tmp_path):
    sc, cal = rig_dataset_scene()
    bear = bearings(sc)
    w, _, _ = world_of(sc, cal, bear)
    before, _ = run(driver, tmp_path, w, "undistort", 0)
    w["rigs"][0] = (w["rigs"][0][0], w["rigs"][0][1], [])        # rig 1's non-reference camera has no cam_from_rig
    for op in (("angle", 1.0), ("triangulation", 1.0), ("normalize", 0, 10.0, 0.1, 0.9)):
        out, err = run(driver, tmp_path, w, *op)
        assert "without cam_from_rig" in err
        assert out["track"] == before["track"] and out["frame"] == before["frame"]


@pytest.mark.parametrize("which", sorted(SCENES))
@pytest.mark.parametrize("clean", [0, 1])
def test_undistort_images_matches_the_host(driver, tmp_path, which, clean):
    sc, cal = SCENES[which]()
    want = bearings(sc)
    stale = np.full_like(want, 0.25)
    n_img = sc.I if hasattr(sc, "obs_sensor") else sc.C
    kept = set(range(0, n_img, 3))                         # images whose features_undist is already full
    w, obs_img, fid = world_of(sc, cal, stale, undist_images=kept)
    out, _ = run(driver, tmp_path, w, "undistort", clean)
    for o in range(0, sc.N):
        k = int(obs_img[o])
        got = np.array(out["image"][1000 - k][fid[o]])
        if k in kept and not clean:
            assert np.array_equal(got, stale[o])
        else:
            np.testing.assert_allclose(got, want[o], rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("which", sorted(SCENES))
@pytest.mark.parametrize("fixed", [0, 1])
def test_normalize_reconstruction_matches_the_host(driver, tmp_path, which, fixed):
    sc, cal = SCENES[which]()
    w, _, _ = world_of(sc, cal)
    ref = sc.copy()
    scale, t = PR.normalize_reconstruction(ref, fixed_scale=bool(fixed), extent=10.0, p0=0.1, p1=0.9)
    out, _ = run(driver, tmp_path, w, "normalize", fixed, 10.0, 0.1, 0.9)
    res = out["result"]
    assert res[1:5] == [0, 0, 0, 1]
    np.testing.assert_allclose(res[0], scale, rtol=1e-12)
    np.testing.assert_allclose(res[5:8], t, rtol=1e-12, atol=1e-12 * np.abs(t).max())
    rig = hasattr(sc, "obs_sensor")
    fids = [f + 1 for f in range(sc.F)] if rig else [1000 - c for c in range(sc.C)]
    got = np.array([out["frame"][f][4:] for f in fids])
    np.testing.assert_allclose(got, ref.trans, rtol=1e-12, atol=1e-12 * np.abs(ref.trans).max())
    assert np.array_equal(np.array([out["frame"][f][:4] for f in fids]), np.asarray(sc.quat, float))
    pts = np.array([out["track"][5000 - p][0] for p in range(sc.P)])
    np.testing.assert_allclose(pts, ref.points, rtol=1e-12, atol=1e-12 * np.abs(ref.points).max())
    if rig:
        for (r, cam), v in out["sensor"].items():
            np.testing.assert_allclose(v[4:], ref.sensor_trans[cam - 1], rtol=1e-12, atol=1e-15)


# ---- b200sfm_undistort_features --------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", [S.SIMPLE_PINHOLE, S.PINHOLE, S.SIMPLE_RADIAL, S.RADIAL])
def test_undistort_features_equals_the_problem_undistortion_bit_for_bit(model):
    sc = S.make_scene(30, 2000, mean_track_len=6, seed=7, pixel_sigma=0.5, model=model, num_intrinsics=4)
    prob = E.BAProblem(E.default_context(), sc, 3, E.first_frame_mask(sc.C))
    prob.set_state(sc.intr_params, sc.quat, sc.trans, sc.points)
    want = prob.undistort()
    prob.free()
    got = PR.undistort_features_device(sc.intr_model, sc.intr_params, sc.cam_intr[sc.obs_cam], sc.obs_xy)
    assert got.tobytes() == want.tobytes()


def test_undistort_features_error_codes_leave_the_output_untouched():
    ctx = E.default_context()
    lib = ctx.lib
    model = np.array([0, 4, 2], np.int32)
    params = np.zeros((3, S.INTR_STRIDE))
    params[:, 0] = 500.0
    xy = np.random.default_rng(1).uniform(0, 1000, size=(300, 2))
    ptr = lambda a: a.ctypes.data_as(ct.c_void_p)   # noqa: E731

    def call(feat, k=3):
        out = np.full((len(feat), 3), 7.0)
        fi = np.ascontiguousarray(feat, np.int32)
        rc = lib.b200sfm_undistort_features(ctx.handle, k, ptr(model), ptr(params), len(fi), ptr(fi), ptr(xy[:len(fi)]), ptr(out))
        return rc, out

    rc, out = call(np.zeros(0))
    assert rc == 0
    for bad in (-1, 3):
        feat = np.zeros(300, np.int32)
        feat[137] = bad
        rc, out = call(feat)
        assert rc == 1
        assert np.all(out == 7.0)
    feat = np.zeros(300, np.int32)
    feat[200] = 1                                             # model 4
    rc, out = call(feat)
    assert rc == 5 and np.all(out == 7.0)
    rc, out = call(np.full(300, 2, np.int32))                 # the model-4 block unused: fine
    assert rc == 0 and np.all(np.isfinite(out)) and np.allclose(np.linalg.norm(out, axis=1), 1.0)
    rc, out = call(np.zeros(5, np.int32), k=0)
    assert rc == 1 and np.all(out == 7.0)
    with pytest.raises(_lib.B200Error) as e:
        PR.undistort_features_device(model, params, feat, xy)
    assert e.value.code == 5
