"""Stage 0's UpdateImagePairsConfig on the GPU (b200sfm_view_graph_update_pairs_config, pair_config_kernels.cuh) against
the host restatement (glomap_b200/view_graph_manipulation.py): configs, validity and the promoted count exactly, F to
1e-13 of its largest entry (and in fact bit for bit); the empty graph, a graph without a valid pair, and the error paths with their outputs
untouched."""
import ctypes as ct
import dataclasses

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E, geometry as G, synthetic as S, view_graph_manipulation as VGM

pytestmark = pytest.mark.gpu


def _random_graph(E_, K, seed, prior_frac=0.8, valid_frac=0.9):
    rng = np.random.default_rng(seed)
    model = rng.integers(0, 4, K).astype(np.int32)
    params = np.zeros((K, S.INTR_STRIDE))
    params[:, :5] = rng.uniform(0.01, 0.1, (K, 5))
    params[:, 0] = rng.uniform(300, 3000, K)
    pin = model == S.PINHOLE
    params[pin, 1] = params[pin, 0] * rng.uniform(0.9, 1.1, pin.sum())
    params[pin, 2:4] = rng.uniform(100, 1000, (pin.sum(), 2))
    params[~pin, 1:3] = rng.uniform(100, 1000, ((~pin).sum(), 2))
    prior = rng.random(K) < prior_frac
    # skewed camera use, so that counts range from one pair to thousands; some same-camera pairs
    c1 = np.minimum((rng.pareto(1.2, E_) * 20).astype(np.int64), K - 1).astype(np.int32)
    c2 = rng.integers(0, K, E_).astype(np.int32)
    same = rng.random(E_) < 0.02
    c2[same] = c1[same]
    # mostly CALIBRATED / UNCALIBRATED, near 50 / 50 so that the ratio test decides both ways
    config = rng.choice(np.arange(9, dtype=np.int32), E_, p=[0.02, 0.02, 0.45, 0.43, 0.03, 0.02, 0.01, 0.01, 0.01])
    valid = rng.random(E_) < valid_frac
    quat = rng.normal(size=(E_, 4))                    # not normalised: R is Eigen's toRotationMatrix as given
    trans = rng.normal(size=(E_, 3))
    F = rng.normal(size=(E_, 9))
    return dict(intr_model=model, intr_params=params, has_prior_focal=prior, pair_cam1=c1, pair_cam2=c2, pair_valid=valid,
                pair_quat=quat, pair_trans=trans, pair_config=config, pair_F=F)


def _compare(a, ctx=None):
    cfg_h, F_h, n_h = VGM.update_image_pairs_config(**a)
    cfg_d, F_d, n_d = VGM.update_image_pairs_config_device(**a, ctx=ctx)
    assert n_d == n_h
    assert np.array_equal(cfg_d, cfg_h)
    promoted = cfg_h != a["pair_config"]
    assert np.array_equal(F_d[~promoted], a["pair_F"][~promoted])              # untouched rows, bit for bit
    scale = np.abs(F_h[promoted]).max(axis=1, initial=0.0)
    err = np.abs(F_d[promoted] - F_h[promoted]).max(axis=1, initial=0.0)
    assert (err <= 1e-13 * scale).all(), (err / np.maximum(scale, 1e-300)).max()
    # the kernel rounds every operation in the host restatement's order: the F agree bit for bit
    assert np.array_equal(F_d, F_h)
    return n_h


@pytest.mark.parametrize("seed", [1, 2])
def test_device_matches_host_on_random_pairs(seed):
    a = _random_graph(300_000, 4000, seed)
    n = _compare(a)
    assert n > 1000
    assert not np.array_equal(a["pair_valid"], np.ones(len(a["pair_valid"]), bool))


def test_device_matches_host_on_a_small_graph_with_every_camera_valid():
    a = _random_graph(500, 5, 3, prior_frac=1.0, valid_frac=1.0)
    a["pair_config"][:] = np.where(np.arange(500) % 4 == 0, 3, 2).astype(np.int32)
    assert _compare(a) == 125


def test_empty_graph_and_no_valid_pair():
    a = _random_graph(0, 4, 4)
    cfg, F, n = VGM.update_image_pairs_config_device(**a)
    assert n == 0 and cfg.shape == (0,) and F.shape == (0, 9)
    b = _random_graph(2000, 20, 5)
    b["pair_valid"][:] = False
    cfg, F, n = VGM.update_image_pairs_config_device(**b)
    assert n == 0 and np.array_equal(cfg, b["pair_config"]) and np.array_equal(F, b["pair_F"])


def _call_raw(a):
    """The C entry on the caller's own buffers: (status, config, F, count)."""
    ctx = E.default_context()
    lib = ctx.lib
    c = lambda x, t: np.ascontiguousarray(np.asarray(x).astype(t))   # noqa: E731
    model, params, prior = c(a["intr_model"], np.int32), c(a["intr_params"], np.float64), c(a["has_prior_focal"], np.uint8)
    c1, c2, valid = c(a["pair_cam1"], np.int32), c(a["pair_cam2"], np.int32), c(a["pair_valid"], np.uint8)
    quat, trans = c(a["pair_quat"], np.float64), c(a["pair_trans"], np.float64)
    config, F = c(a["pair_config"], np.int32), c(a["pair_F"], np.float64)
    n = ct.c_int64(-7)
    p = lambda x: x.ctypes.data_as(ct.c_void_p)   # noqa: E731
    rc = lib.b200sfm_view_graph_update_pairs_config(ctx.handle, len(model), p(model), p(params), p(prior), len(c1), p(c1), p(c2),
                                                    p(valid), p(quat), p(trans), p(config), p(F), ct.byref(n))
    return rc, config, F, n.value


def test_out_of_range_camera_is_an_error_and_leaves_the_outputs_untouched():
    a = _random_graph(5000, 30, 6)
    a["pair_cam2"][4321] = 30
    rc, config, F, n = _call_raw(a)
    assert rc == 1 and n == 0
    assert np.array_equal(config, a["pair_config"]) and np.array_equal(F, a["pair_F"])
    a["pair_cam2"][4321] = -1
    with pytest.raises(_lib.B200Error):
        VGM.update_image_pairs_config_device(**a)


def test_unsupported_model_of_a_promoted_pair_is_an_error_and_leaves_the_outputs_untouched():
    a = _random_graph(400, 2, 7, prior_frac=1.0, valid_frac=1.0)
    a["pair_config"][:] = np.where(np.arange(400) % 3 == 0, 3, 2).astype(np.int32)
    a["intr_model"][1] = 4                                                   # OPENCV
    rc, config, F, n = _call_raw(a)
    assert rc == 5
    assert np.array_equal(config, a["pair_config"]) and np.array_equal(F, a["pair_F"])
    # not promoted (every pair CALIBRATED): the model is never read
    a["pair_config"][:] = 2
    rc, config, F, n = _call_raw(a)
    assert rc == 0 and n == 0


def test_promoted_F_of_true_poses_is_the_true_F():
    """On a scene's true relative poses the promoted F is the true F (up to scale): F x1 . x2 = 0 on the projections."""
    sc = S.make_scene(12, 400, seed=5, num_intrinsics=12, model=S.PINHOLE)
    ei, ej = np.triu_indices(12, 1)
    uncal, _ = S.make_calibration_pairs(sc, np.stack([ei, ej], 1), seed=5, uncalibrated_frac=1.0)
    cal = [dataclasses.replace(p, config=2) for p in uncal] * 2           # every camera: 2 / 3 of its pairs CALIBRATED
    cams = {k: _cam(sc, k) for k in range(12)}
    n = VGM.UpdateImagePairsConfig(cal + uncal, cams, {i: int(sc.cam_intr[i]) for i in range(12)}, device=True)
    assert n == len(uncal) and all(p.config == 2 for p in uncal)
    R = G.quat_xyzw_to_rotmat(sc.quat)
    for p in uncal:
        Xc1 = sc.points @ R[p.image_id1].T + sc.trans[p.image_id1]
        Xc2 = sc.points @ R[p.image_id2].T + sc.trans[p.image_id2]
        x1 = np.c_[Xc1[:, :2] / Xc1[:, 2:], np.ones(len(Xc1))] @ S._pinhole_K(S.PINHOLE, sc.intr_params[sc.cam_intr[p.image_id1]]).T
        x2 = np.c_[Xc2[:, :2] / Xc2[:, 2:], np.ones(len(Xc2))] @ S._pinhole_K(S.PINHOLE, sc.intr_params[sc.cam_intr[p.image_id2]]).T
        r = np.einsum("ni,ij,nj->n", x2, p.F, x1) / np.linalg.norm(p.F)
        assert np.abs(r).max() < 1e-9 * np.abs(x1).max() ** 2


def _cam(sc, k):
    from glomap_b200.view_graph_calibration import CalibCamera
    return CalibCamera(int(sc.intr_model[k]), sc.intr_params[k, :4].copy(), has_prior_focal_length=True)
