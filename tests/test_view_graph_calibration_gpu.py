"""Device view-graph calibration (b200sfm_view_graph_calibrate, vgc_kernels.cuh / vgc_solver.cuh) against the CPU
restatement oracle/vgc_oracle.py: the LM trajectory (iteration count, termination, the cost after every iteration),
the focals, the camera and pair masks.  A pair whose squared residual lies within rounding of the threshold is reported;
the seeded inputs must have none."""
import copy
import threading

import numpy as np
import pytest

from glomap_b200 import _lib, image_pair_inliers as IP, synthetic as S, view_graph_calibration as VGC
from oracle import vgc_oracle as V

pytestmark = pytest.mark.gpu

TERM = {"function tolerance": 1, "parameter tolerance": 2, "gradient tolerance": 3, "gradient tolerance (initial)": 3,
        "max iterations": 4, "min trust region radius": 5, "too many invalid steps": 6}


def _window_pairs(C, w):
    i = np.repeat(np.arange(C), w)
    j = i + np.tile(np.arange(1, w + 1), C)
    keep = j < C
    return np.stack([i[keep], j[keep]], 1)


def _problem(model, K, C=40, seed=1, f_noise=0.2, F_sigma=0.0, outlier_frac=0.0, prior_frac=0.0, pairs=None):
    sc = S.make_scene(C, 20, seed=seed, model=model, num_intrinsics=K)
    if pairs is None:
        pairs = np.stack(np.triu_indices(C, 1), 1)
    d = S.make_vgc_pairs(sc, pairs, seed=seed, f_noise=f_noise, outlier_frac=outlier_frac, F_sigma=F_sigma)
    rng = np.random.default_rng([seed, 5])
    d["prior"] = rng.random(K) < prior_frac
    return d


def _oracle(d, max_it=100):
    return V.solve_vgc(d["principal_point"], d["focal_init"], d["prior"], d["cam1"], d["cam2"], d["F"],
                       V.VGCOptions(max_num_iterations=max_it))


def _device(d, max_it=100, **kw):
    o = VGC.ViewGraphCalibratorOptions(max_num_iterations=max_it, **kw)
    return VGC.calibrate_arrays(d["principal_point"], d["focal_init"], d["prior"], d["cam1"], d["cam2"], d["F"], o,
                                want_residual=True)


def _borderline(ref, thres=2.0):
    s = (ref["residual"] ** 2).sum(1)
    return [int(e) for e in np.flatnonzero(np.abs(s - thres * thres) <= 1e-9 * thres * thres)]


# Measured agreement: costs to 2e-10 relative (or at the rounding floor, 1e-16, of a noise-free solve); focals to 5e-8 relative (the device's Jacobi SVD and LAPACK's give Fetzer
# constants that differ by up to 5e-7 relative in the residuals, see test_zero_iterations_...).
FOCAL_RTOL = 1e-7
COST_RTOL = 1e-9


def _compare(d, dev, ref, same_trajectory=True):
    assert _borderline(ref) == [], f"pairs within rounding of the threshold: {_borderline(ref)}"
    summ, st = ref["summary"], dev["stats"]
    assert st["usable"] == int(summ.usable)
    if same_trajectory:
        assert st["iterations"] == summ.iterations, (st, summ)
        assert st["termination"] == TERM[summ.termination], (st["termination"], summ.termination)
        np.testing.assert_allclose(st["final_cost"], summ.final_cost, rtol=COST_RTOL, atol=1e-14)
    else:
        np.testing.assert_allclose(st["final_cost"], summ.final_cost, rtol=1e-4, atol=1e-14)
    np.testing.assert_allclose(dev["focal"], ref["focal"], rtol=FOCAL_RTOL if same_trajectory else 1e-4, atol=0)
    np.testing.assert_array_equal(dev["cam_accepted"], ref["cam_accepted"])
    if same_trajectory:
        np.testing.assert_array_equal(dev["pair_valid"], ref["pair_valid"])
    else:   # focals 1e-5 apart: only pairs that close to the threshold may be decided differently
        s = (ref["residual"] ** 2).sum(1)
        diff = np.flatnonzero(dev["pair_valid"] != ref["pair_valid"])
        assert np.all(np.abs(s[diff] - 4.0) <= 1e-3 * 4.0), (diff, s[diff])


CASES = [
    dict(model=S.SIMPLE_PINHOLE, K=1),
    dict(model=S.PINHOLE, K=3, F_sigma=1e-3),
    dict(model=S.SIMPLE_RADIAL, K=40, outlier_frac=0.1),
    dict(model=S.RADIAL, K=3, F_sigma=1e-3, prior_frac=0.4, seed=3),
    dict(model=S.SIMPLE_PINHOLE, K=40, outlier_frac=0.1, prior_frac=0.3, seed=2),
    dict(model=S.PINHOLE, K=1, outlier_frac=0.1, F_sigma=1e-3, seed=4),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_device_follows_the_oracle_iteration_by_iteration(case):
    d = _problem(**case)
    ref = _oracle(d)
    dev = _device(d)
    _compare(d, dev, ref)
    # the cost after every iteration: the same problem truncated at n iterations
    for n in range(1, ref["summary"].iterations):
        r_n, d_n = _oracle(d, n), _device(d, n)
        assert d_n["stats"]["iterations"] == r_n["summary"].iterations
        np.testing.assert_allclose(d_n["stats"]["final_cost"], r_n["summary"].final_cost, rtol=COST_RTOL, atol=1e-14)
        np.testing.assert_allclose(d_n["focal"], r_n["focal"], rtol=FOCAL_RTOL, atol=0)


def test_noise_free_recovery_on_the_device():
    d = _problem(S.SIMPLE_PINHOLE, 40, f_noise=0.2)
    dev = _device(d)
    np.testing.assert_allclose(dev["focal"], d["focal_true"], rtol=1e-6)
    assert dev["pair_valid"].all() and dev["cam_accepted"].all()


def test_zero_iterations_gives_the_residuals_at_the_initial_focals():
    """Pins the setup (G, the device SVD, the Fetzer constants) without a probe: the residuals of every pair at the
    initial focals against the oracle's (LAPACK SVD).  Measured: up to 5e-7 relative (1.7e-7 absolute) -- not the 1e-12
    a well-conditioned SVD would give; the Fetzer constants of these scenes amplify the SVD's rounding."""
    for model, K in ((S.SIMPLE_PINHOLE, 1), (S.PINHOLE, 3), (S.RADIAL, 40)):
        d = _problem(model, K, F_sigma=1e-3, outlier_frac=0.1)
        ref, dev = _oracle(d, 0), _device(d, 0)
        np.testing.assert_allclose(dev["residual"], ref["residual"], rtol=1e-6, atol=1e-9)
        np.testing.assert_array_equal(dev["focal"], d["focal_init"])


def test_one_shared_camera_over_a_million_pairs_is_reproducible():
    """K = 1: every pair is a same-camera pair of one camera, a single row of 1.1 M incidences split into segments.  The
    cost flattens out under the 5 % outliers, and the function-tolerance test fires two iterations apart on the device and
    the oracle (25 vs 27): the final cost and focal are compared, not the trajectory."""
    d = _problem(S.SIMPLE_PINHOLE, 1, C=1500, F_sigma=1e-3, outlier_frac=0.05)
    assert len(d["cam1"]) >= 1_000_000
    ref = _oracle(d)
    a, b = _device(d), _device(d)
    _compare(d, a, ref, same_trajectory=False)
    for k in ("focal", "residual", "pair_valid", "cam_accepted"):
        np.testing.assert_array_equal(a[k], b[k])
    assert a["stats"]["final_cost"] == b["stats"]["final_cost"]


def test_ten_thousand_cameras():
    d = _problem(S.SIMPLE_PINHOLE, 10_000, C=10_000, F_sigma=1e-3, outlier_frac=0.05, pairs=_window_pairs(10_000, 50))
    assert len(d["cam1"]) > 450_000
    ref = _oracle(d)
    dev = _device(d)
    _compare(d, dev, ref)


def test_edge_cases():
    d = _problem(S.SIMPLE_PINHOLE, 3, C=12)
    K = len(d["focal_init"])
    # no pairs: the early return writes nothing
    out = VGC.calibrate_arrays(d["principal_point"], d["focal_init"], None, [], [], np.zeros((0, 9)))
    assert out["stats"]["usable"] == 1 and not out["cam_accepted"].any()
    np.testing.assert_array_equal(out["focal"], d["focal_init"])
    # every camera a prior: the same
    out = VGC.calibrate_arrays(d["principal_point"], d["focal_init"], np.ones(K, bool), d["cam1"], d["cam2"], d["F"],
                               want_residual=True)
    assert out["stats"]["usable"] == 1 and not out["cam_accepted"].any() and out["pair_valid"].all()
    assert not out["residual"].any()
    # a camera index out of range
    bad = d["cam2"].copy()
    bad[3] = K
    with pytest.raises(_lib.B200Error) as e:
        VGC.calibrate_arrays(d["principal_point"], d["focal_init"], None, d["cam1"], bad, d["F"])
    assert e.value.code == 1
    # a non-finite F: not usable, no NaN in the focals, and the oracle's masks
    F = d["F"].copy()
    F[5, 4] = np.nan
    d2 = dict(d, F=F)
    dev, ref = _device(d2), _oracle(d2)
    assert dev["stats"]["usable"] == 0 and not ref["summary"].usable
    assert np.isfinite(dev["focal"]).all()
    np.testing.assert_array_equal(dev["focal"], ref["focal"])
    np.testing.assert_array_equal(dev["pair_valid"], ref["pair_valid"])
    np.testing.assert_array_equal(dev["cam_accepted"], ref["cam_accepted"])


def test_distributed_context_is_unsupported():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("a two-rank context needs two GPUs (NCCL ranks cannot share a device)")
    from glomap_b200.estimators import Context
    d = _problem(S.SIMPLE_PINHOLE, 3, C=12)
    nid = Context.nccl_unique_id()
    codes = [None, None]

    def rank(r):
        ctx = Context(r, r, 2, nid)
        try:
            VGC.calibrate_arrays(d["principal_point"], d["focal_init"], None, d["cam1"], d["cam2"], d["F"], ctx=ctx)
        except _lib.B200Error as e:
            codes[r] = e.code
        ctx.close()
    th = [threading.Thread(target=rank, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert codes == [5, 5]


def _calibrated_cameras(cameras, focal, accepted):
    out = {}
    for i, c in cameras.items():
        c2 = IP.Camera(c.model, np.array(c.params, np.float64))
        if accepted[i]:
            for k in VGC.focal_length_idxs(c.model):
                c2.params[k] = focal[i]
        out[i] = c2
    return out


def test_chain_calibration_then_inlier_count_matches_the_host_chain():
    """Calibration of per-image cameras with perturbed focals, then ImagePairsInlierCount on the CALIBRATED pairs with the
    refined focals: device chain and host chain (oracle calibration, host scoring) give identical masks."""
    sc = S.make_scene(30, 3000, mean_track_len=6, seed=7, num_intrinsics=30)
    md = S.make_pair_matches(sc, seed=7, outlier_frac=0.2, config_weights=(0.7, 0.3, 0.0))
    features, cameras, pairs = S.pairs_from_match_arrays(md)
    rng = np.random.default_rng(9)
    for c in cameras.values():
        c.params = np.array(c.params, np.float64)
        c.params[0] *= 1 + rng.uniform(-0.05, 0.05)
    C = len(cameras)
    pp = np.array([VGC.principal_point(cameras[i]) for i in range(C)])
    f0 = np.array([cameras[i].focal() for i in range(C)])
    qual = [p for p in pairs if p.config in (IP.TWO_VIEW_CALIBRATED, IP.TWO_VIEW_UNCALIBRATED)]
    c1 = np.array([p.image_id1 for p in qual], np.int32)
    c2 = np.array([p.image_id2 for p in qual], np.int32)
    F = np.array([np.asarray(p.F).reshape(9) for p in qual])
    ref = V.solve_vgc(pp, f0, None, c1, c2, F)
    dev_cams = {i: VGC.CalibCamera(c.model, np.array(c.params, np.float64)) for i, c in cameras.items()}
    dev_pairs = [copy.copy(p) for p in pairs]
    assert VGC.ViewGraphCalibrator().Solve(dev_pairs, dev_cams, {i: i for i in range(C)})
    host_cams = _calibrated_cameras(cameras, ref["focal"], ref["cam_accepted"])
    host_pairs = [copy.copy(p) for p in pairs]
    for p, v in zip([p for p in host_pairs if p.config in (2, 3)], ref["pair_valid"]):
        p.is_valid = bool(v)
    assert [p.is_valid for p in dev_pairs] == [p.is_valid for p in host_pairs]
    for i in range(C):
        np.testing.assert_allclose(dev_cams[i].params, host_cams[i].params, rtol=1e-10)
    cal_d = [p for p in dev_pairs if p.config == IP.TWO_VIEW_CALIBRATED]
    cal_h = [p for p in host_pairs if p.config == IP.TWO_VIEW_CALIBRATED]
    a = IP.image_pairs_inlier_count_device(cal_d, features, dev_cams)
    b = IP.image_pairs_inlier_count(cal_h, features, host_cams)
    assert len(cal_d) > 0
    for x, y in zip(a.inliers, b.inliers):
        np.testing.assert_array_equal(x, y)
