"""Stage 0's UpdateImagePairsConfig without a GPU: the host restatement (glomap_b200/view_graph_manipulation.py) on
hand-built graphs, rule by rule, its F against K2^-T [t]x R K1^-1 from numpy, the object-level form over
ImagePairMatches, the C ABI's argument checks, and the C++ shim over a recording test double."""
import ctypes as ct
import os
import subprocess

import numpy as np
import pytest

from glomap_b200 import _lib, geometry as G, synthetic as S, view_graph_manipulation as VGM
from glomap_b200.image_pair_inliers import (TWO_VIEW_CALIBRATED as CAL, TWO_VIEW_PLANAR as PLANAR,
                                            TWO_VIEW_UNCALIBRATED as UNCAL)
from glomap_b200.track_establishment import ImagePairMatches
from glomap_b200.view_graph_calibration import CalibCamera

ROOT = os.path.dirname(os.path.abspath(__file__)).rsplit(os.sep, 1)[0]


def _cams(K, prior=True):
    model = np.zeros(K, np.int32)                                   # SIMPLE_PINHOLE
    params = np.zeros((K, S.INTR_STRIDE))
    params[:, 0] = 500.0 + 10 * np.arange(K)
    params[:, 1], params[:, 2] = 320.0, 240.0
    return model, params, np.full(K, prior, bool)


def _run(model, params, prior, pairs, valid=None):
    """pairs: list of (cam1, cam2, config)."""
    E = len(pairs)
    c1 = np.array([p[0] for p in pairs], np.int32)
    c2 = np.array([p[1] for p in pairs], np.int32)
    cfg = np.array([p[2] for p in pairs], np.int32)
    rng = np.random.default_rng(3)
    q = G.rotmat_to_quat_xyzw_fast(G.so3_exp(rng.normal(size=(E, 3)) * 0.3)).reshape(E, 4)
    t = rng.normal(size=(E, 3))
    F = rng.normal(size=(E, 9))
    v = np.ones(E, bool) if valid is None else np.asarray(valid, bool)
    out = VGM.update_image_pairs_config(model, params, prior, c1, c2, v, q, t, cfg, F)
    return out, dict(quat=q, trans=t, F=F, config=cfg)


def test_ratio_exactly_one_half_is_not_valid_and_just_above_is():
    m, p, pr = _cams(4)
    # camera 0: 1 CALIBRATED + 1 UNCALIBRATED with camera 1 (ratio 1/2 for both), then a promotable pair 0-1
    (cfg, F, n), _ = _run(m, p, pr, [(0, 1, CAL), (0, 1, UNCAL)])
    assert n == 0 and cfg.tolist() == [CAL, UNCAL]
    # cameras 2, 3: 2 CALIBRATED + 1 UNCALIBRATED -> 2/3 > 0.5, the UNCALIBRATED pair is promoted
    (cfg, F, n), _ = _run(m, p, pr, [(2, 3, CAL), (3, 2, CAL), (2, 3, UNCAL)])
    assert n == 1 and cfg.tolist() == [CAL, CAL, CAL]
    # 3 CALIBRATED + 3 UNCALIBRATED: exactly 0.5 again, nothing promoted
    (cfg, F, n), _ = _run(m, p, pr, [(2, 3, CAL)] * 3 + [(2, 3, UNCAL)] * 3)
    assert n == 0


def test_a_camera_without_a_prior_and_an_invalid_pair_are_not_counted():
    m, p, pr = _cams(4)
    pr[3] = False
    # camera 0: its CALIBRATED pairs are with camera 3 (no prior) or invalid: not counted, so 0 stays absent and not valid
    pairs = [(0, 3, CAL), (0, 3, CAL), (0, 1, CAL), (0, 1, UNCAL), (1, 2, CAL), (1, 2, CAL)]
    valid = [True, True, False, True, True, True]
    (cfg, F, n), _ = _run(m, p, pr, pairs, valid)
    # camera 0 counts only (0, 1, UNCAL): 0 / 1 -> not valid; camera 1: 2 CAL + 1 UNCAL -> valid
    assert n == 0 and cfg[3] == UNCAL
    # with camera 3's prior, camera 0 counts 2 / 3 -> valid
    pr[3] = True
    (cfg, F, n), _ = _run(m, p, pr, pairs, valid)
    assert n == 1 and cfg[3] == CAL
    # an invalid UNCALIBRATED pair between valid cameras is never promoted
    valid[3] = False
    (cfg, F, n), _ = _run(m, p, pr, pairs, valid)
    assert n == 0 and cfg[3] == UNCAL


def test_a_camera_absent_from_the_counter_is_not_valid():
    m, p, pr = _cams(3)
    pr[2] = False
    # camera 2 has no prior, so it never enters the counter; camera 0, 1 are valid
    (cfg, F, n), _ = _run(m, p, pr, [(0, 1, CAL), (0, 1, CAL), (0, 2, UNCAL), (2, 1, UNCAL), (0, 1, UNCAL)])
    assert cfg.tolist() == [CAL, CAL, UNCAL, UNCAL, CAL] and n == 1


def test_a_same_camera_pair_counts_twice():
    m, p, pr = _cams(2)
    # camera 0: a same-camera CALIBRATED pair (2 / 2) and two UNCALIBRATED pairs with camera 1 -> 2 / 4 = 0.5: not valid.
    # Counted once, it would be 1 / 3.  With one more same-camera CALIBRATED pair: 4 / 6 > 0.5 -> valid.
    (cfg, F, n), _ = _run(m, p, pr, [(0, 0, CAL), (0, 1, UNCAL), (1, 0, UNCAL), (1, 1, CAL), (1, 1, CAL)])
    assert n == 0
    (cfg, F, n), _ = _run(m, p, pr, [(0, 0, CAL), (0, 0, CAL), (0, 1, UNCAL), (1, 0, UNCAL), (1, 1, CAL), (1, 1, CAL)])
    assert n == 2 and cfg.tolist() == [CAL] * 6
    # a same-camera UNCALIBRATED pair of a valid camera is promoted
    (cfg, F, n), _ = _run(m, p, pr, [(0, 0, CAL), (0, 0, UNCAL), (0, 1, CAL)])
    assert n == 1 and cfg[1] == CAL


def test_planar_and_calibrated_pairs_are_never_promoted_and_keep_their_F():
    m, p, pr = _cams(2)
    pairs = [(0, 1, CAL), (0, 1, CAL), (0, 1, PLANAR), (0, 1, 0), (0, 1, 5), (0, 1, UNCAL)]
    (cfg, F, n), inp = _run(m, p, pr, pairs)
    assert n == 1 and cfg.tolist() == [CAL, CAL, PLANAR, 0, 5, CAL]
    assert np.array_equal(F[:5], inp["F"][:5])
    assert not np.array_equal(F[5], inp["F"][5])


@pytest.mark.parametrize("model1,model2", [(S.SIMPLE_PINHOLE, S.PINHOLE), (S.PINHOLE, S.SIMPLE_RADIAL), (S.RADIAL, S.RADIAL)])
def test_F_is_K2_inverse_transpose_tx_R_K1_inverse(model1, model2):
    rng = np.random.default_rng(7)
    model = np.array([model1, model2], np.int32)
    params = np.zeros((2, S.INTR_STRIDE))
    for k, mo in enumerate(model):
        n = S.MODEL_NUM_PARAMS[int(mo)]
        params[k, :n] = rng.uniform(0.01, 0.1, n)
        if mo == S.PINHOLE:
            params[k, :4] = [800 + 50 * k, 780, 300, 260]
        else:
            params[k, :3] = [900 - 30 * k, 310, 250]
    pairs = [(0, 1, CAL), (1, 0, CAL), (0, 1, CAL), (0, 1, UNCAL), (1, 0, UNCAL)]
    (cfg, F, n), inp = _run(model, params, np.ones(2, bool), pairs)
    assert n == 2

    def K(m, p):
        return S._pinhole_K(int(m), p)
    for e, (a, b) in [(3, (0, 1)), (4, (1, 0))]:
        R = G.quat_xyzw_to_rotmat(inp["quat"][e])
        t = inp["trans"][e]
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        want = np.linalg.inv(K(model[b], params[b])).T @ tx @ R @ np.linalg.inv(K(model[a], params[a]))
        np.testing.assert_allclose(F[e].reshape(3, 3), want, rtol=0, atol=1e-14 * np.abs(want).max())


def test_F_uses_the_quaternion_as_given_and_is_zero_for_the_identity_pose():
    """The reference promotes before DecomposeRelPose: a pair with the converter's identity pose gets F = 0."""
    F = VGM.fundamental_from_motion_and_cameras(0, [500, 320, 240], 0, [600, 300, 200], [0, 0, 0, 1], [0, 0, 0])
    assert np.array_equal(F, np.zeros((3, 3)))
    # Eigen's toRotationMatrix does not normalise: (1, 0, 0, 1) gives [[1, 0, 0], [0, -1, -2], [0, 2, -1]], not the
    # rotation by 90 degrees about x; with t = (1, 0, 0) and K = I, F = [t]x R
    F2 = VGM.fundamental_from_motion_and_cameras(0, [1, 0, 0], 0, [1, 0, 0], [1, 0, 0, 1], [1, 0, 0])
    assert np.array_equal(F2, np.array([[0.0, 0, 0], [0, -2, 1], [0, -1, -2]]))


def test_out_of_range_camera_raises_and_unsupported_model_only_when_promoted():
    m, p, pr = _cams(2)
    with pytest.raises(ValueError):
        _run(m, p, pr, [(0, 2, CAL)])
    m[1] = 4                                                            # OPENCV: never asked for its K
    (cfg, F, n), _ = _run(m, p, pr, [(0, 1, CAL), (0, 1, PLANAR)])
    assert n == 0
    with pytest.raises(ValueError):
        _run(m, p, pr, [(0, 1, CAL), (0, 1, CAL), (0, 1, UNCAL)])


def test_object_level_form_sets_config_and_F_in_place():
    cams = {7: CalibCamera(S.PINHOLE, np.array([500.0, 510, 320, 240]), has_prior_focal_length=True),
            3: CalibCamera(S.SIMPLE_PINHOLE, np.array([600.0, 300, 200]), has_prior_focal_length=True),
            9: CalibCamera(S.SIMPLE_RADIAL, np.array([700.0, 350, 250, 0.01]))}
    image_camera = {10: 3, 30: 3, 20: 7, 40: 9}

    def pair(a, b, cfg, valid=True):
        return ImagePairMatches(a, b, np.zeros((0, 2)), np.zeros(0, np.int64), is_valid=valid, config=cfg,
                                quat_xyzw=np.array([0.1, 0.2, 0.3, 0.9]), trans=np.array([1.0, 0.5, -0.2]),
                                F=np.full((3, 3), 7.0))
    # camera 3: 4 / 5 CALIBRATED, camera 7: 2 / 3; camera 9 has no prior
    pairs = [pair(10, 20, CAL), pair(20, 30, CAL), pair(30, 10, CAL), pair(20, 30, UNCAL), pair(40, 20, UNCAL),
             pair(10, 30, UNCAL, False)]
    n = VGM.UpdateImagePairsConfig(pairs, cams, image_camera, device=False)
    assert n == 1
    assert [p.config for p in pairs] == [CAL, CAL, CAL, CAL, UNCAL, UNCAL]
    want = VGM.fundamental_from_motion_and_cameras(S.PINHOLE, cams[7].params, S.SIMPLE_PINHOLE, cams[3].params,
                                                   pairs[3].quat_xyzw, pairs[3].trans)
    assert np.array_equal(pairs[3].F, want)
    assert all(np.array_equal(p.F, np.full((3, 3), 7.0)) for k, p in enumerate(pairs) if k != 3)
    assert VGM.UpdateImagePairsConfig([], cams, image_camera, device=True) == 0


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def test_abi_arguments_are_checked_without_a_device():
    lib = _lib.load()
    f = lib.b200sfm_view_graph_update_pairs_config
    n = ct.c_int64(5)
    assert f(None, 1, None, None, None, 1, None, None, None, None, None, None, None, ct.byref(n)) == 1
    # E == 0 needs no device and no arrays: OK with a zero count
    assert f(ct.c_void_p(1), 0, None, None, None, 0, None, None, None, None, None, None, None, ct.byref(n)) == 0
    assert n.value == 0


# ---- C++ shim ----------------------------------------------------------------------------------------------------------
def test_shim_flattens_in_sorted_id_order_and_writes_back(tmp_path):
    lib, exe, dump = tmp_path / "libb200sfm.so", tmp_path / "pairs_config_driver", tmp_path / "dump.txt"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c"),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_pairs_config.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "shim_mock", "pairs_config_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe)], env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rec = {}
    for line in dump.read_text().splitlines()[1:]:
        name, cnt, *vals = line.split()
        rec[name] = [float(v) for v in vals]
        assert len(vals) == int(cnt)
    # cameras in sorted id order: 3 (SIMPLE_PINHOLE, prior), 7 (PINHOLE, prior), 9 (SIMPLE_RADIAL, no prior)
    assert rec["intr_model"] == [0, 1, 2]
    assert rec["intr_params"][:3] == [600, 300, 200] and rec["intr_params"][12:16] == [500, 510, 320, 240]
    assert rec["intr_params"][24:28] == [700, 350, 250, 0.01]
    assert rec["has_prior_focal"] == [1, 1, 0]
    # every pair in sorted pair-id order (the pass reads all of them): (10, 20), (30, 10), (20, 30), (40, 20)
    assert rec["pair_cam1"] == [0, 0, 1, 2] and rec["pair_cam2"] == [1, 0, 0, 1]
    assert rec["pair_valid"] == [1, 1, 1, 0]
    assert rec["pair_config"] == [2, 3, 3, 2]
    assert rec["pair_quat"][:4] == [0.1, 0.2, 0.3, 0.9] and rec["pair_trans"][:3] == [10, 20, 0.5]
    assert rec["pair_F"][:9] == [10 + 0.5 * k + 0.2 for k in range(9)]
    out = r.stdout.splitlines()
    # the mock promotes every UNCALIBRATED pair and sets its F to 100 * e + k
    assert out[0] == "promoted 2"
    assert out[1:5] == ["config 2", "config 2", "config 2", "config 2"]
    assert out[5] == "F " + " ".join(f"{10 + 0.5 * k + 0.2:.17g}" for k in range(9))
    assert out[6] == "F " + " ".join(str(100 + k) for k in range(9))
    assert out[7] == "F " + " ".join(str(200 + k) for k in range(9))


def test_shim_update_image_pairs_config_typechecks_against_the_glomap_api():
    """Inside a glomap build the shim's UpdateImagePairsConfig takes glomap's ImagePair (int config, Eigen F written
    through F(r, c)) and Camera (model_id, params, has_prior_focal_length): type-checked against
    tests/shim_mock/glomap_stub_vgc and the pair type of tests/shim_mock/pairs_config_typecheck.cc."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(ROOT, "tests", "shim_mock", "glomap_stub_vgc"),
                        "-I" + os.path.join(ROOT, "glomap_b200", "host"),
                        os.path.join(ROOT, "tests", "shim_mock", "pairs_config_typecheck.cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
