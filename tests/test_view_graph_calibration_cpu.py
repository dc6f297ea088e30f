"""View-graph calibration without a GPU: the oracle (oracle/vgc_oracle.py) against a literal scalar transcription of the
reference's cost functions, its derivatives, the SVD sign invariance, noise-free recovery, the driver rules
(ViewGraphCalibrator::Solve and its CopyBackResults / FilterImagePairs) through the object-level API with the oracle as
its back end, the C ABI's argument checks and struct layout, and the C++ shim over a recording test double."""
import ctypes as ct
import os
import subprocess

import numpy as np
import pytest

from glomap_b200 import _lib, image_pair_inliers as IP, synthetic as S, view_graph_calibration as VGC
from glomap_b200.track_establishment import ImagePairMatches
from oracle import vgc_oracle as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- literal scalar transcription of glomap/estimators/cost_function.h:138-310 ----------------------------------------
def _fetzer_d(ai, bi, aj, bj, u, v):
    return [ai[u] * aj[v] - ai[v] * aj[u], ai[u] * bj[v] - ai[v] * bj[u], bi[u] * aj[v] - bi[v] * aj[u],
            bi[u] * bj[v] - bi[v] * bj[u]]


def _fetzer_ds(s, U, V_):
    v_0, v_1, u_0, u_1 = V_[:, 0], V_[:, 1], U[:, 0], U[:, 1]
    ai = [s[0] * s[0] * (v_0[0] * v_0[0] + v_0[1] * v_0[1]), s[0] * s[1] * (v_0[0] * v_1[0] + v_0[1] * v_1[1]),
          s[1] * s[1] * (v_1[0] * v_1[0] + v_1[1] * v_1[1])]
    aj = [u_1[0] * u_1[0] + u_1[1] * u_1[1], -(u_0[0] * u_1[0] + u_0[1] * u_1[1]), u_0[0] * u_0[0] + u_0[1] * u_0[1]]
    bi = [s[0] * s[0] * v_0[2] * v_0[2], s[0] * s[1] * v_0[2] * v_1[2], s[1] * s[1] * v_1[2] * v_1[2]]
    bj = [u_1[2] * u_1[2], -(u_0[2] * u_1[2]), u_0[2] * u_0[2]]
    return _fetzer_d(ai, bi, aj, bj, 1, 0), _fetzer_d(ai, bi, aj, bj, 0, 2), _fetzer_d(ai, bi, aj, bj, 2, 1)


def _cost(d_01, d_12, fi, fj):   # FetzerFocalLengthCost::operator() (and the same-camera one with fj = fi)
    di = (fj * fj * d_01[0] + d_01[1])
    dj = (fi * fi * d_12[0] + d_12[2])
    di = 1e-6 if di == 0 else di
    dj = 1e-6 if dj == 0 else dj
    K0_01 = -(fj * fj * d_01[2] + d_01[3]) / di
    K1_12 = -(fi * fi * d_12[1] + d_12[3]) / dj
    return [(fi * fi - K0_01) / (fi * fi), (fj * fj - K1_12) / (fj * fj)]


def _random_d(rng, n):
    return rng.normal(size=(n, 4)), rng.normal(size=(n, 4))


def test_oracle_residual_equals_the_scalar_transcription():
    rng = np.random.default_rng(1)
    sc = S.make_scene(12, 20, seed=2, num_intrinsics=12)
    d = S.make_vgc_pairs(sc, np.stack(np.triu_indices(12, 1), 1), seed=2, f_noise=0.2, outlier_frac=0.2)
    pp = d["principal_point"]
    d01, d12 = V.fetzer_constants(d["F"], pp[d["cam1"]], pp[d["cam2"]])
    G = V.g_matrix(d["F"].reshape(-1, 3, 3), pp[d["cam1"]], pp[d["cam2"]])
    for e in range(len(G)):
        U, s, Vt = np.linalg.svd(G[e])
        a01, _, a12 = _fetzer_ds(s, U, Vt.T)
        assert list(d01[e]) == a01 and list(d12[e]) == a12
    f = d["focal_init"]
    r = V.residuals(d01, d12, f[d["cam1"]], f[d["cam2"]])
    for e in range(len(G)):
        assert list(r[e]) == _cost(d01[e], d12[e], f[d["cam1"][e]], f[d["cam2"][e]])
    # random constants, including exact-zero denominators (d01[0] = d01[1] = 0, d12[0] = d12[2] = 0)
    a, b = _random_d(rng, 200)
    a[:20, :2] = 0.0
    b[10:30, 0] = 0.0
    b[10:30, 2] = 0.0
    fi, fj = rng.uniform(0.5, 2.0, 200), rng.uniform(0.5, 2.0, 200)
    r = V.residuals(a, b, fi, fj)
    for e in range(200):
        assert list(r[e]) == _cost(a[e], b[e], fi[e], fj[e])


def test_analytic_jacobian_matches_central_differences():
    rng = np.random.default_rng(3)
    a, b = _random_d(rng, 300)
    a[:10, :2] = 0.0          # di replaced by the constant 1e-6 (no derivative through d01[0])
    fi, fj = rng.uniform(0.5, 2.0, 300), rng.uniform(0.5, 2.0, 300)
    _, dri, drj = V.residuals(a, b, fi, fj, True)
    h = 1e-6
    num_i = (V.residuals(a, b, fi + h * fi, fj) - V.residuals(a, b, fi - h * fi, fj)) / (2 * h * fi)[:, None]
    num_j = (V.residuals(a, b, fi, fj + h * fj) - V.residuals(a, b, fi, fj - h * fj)) / (2 * h * fj)[:, None]
    ok = np.abs(V.residuals(a, b, fi, fj)).max(1) < 1e4     # skip pairs whose residual is a near pole of 1 / di
    scale_i = np.abs(dri) + np.abs(num_i) + 1e-3
    scale_j = np.abs(drj) + np.abs(num_j) + 1e-3
    assert np.all(np.abs(dri - num_i)[ok] <= 1e-7 * scale_i[ok])
    assert np.all(np.abs(drj - num_j)[ok] <= 1e-7 * scale_j[ok])


def test_joint_sign_flip_of_the_singular_vectors_leaves_the_residuals_unchanged():
    sc = S.make_scene(10, 20, seed=5, num_intrinsics=10)
    d = S.make_vgc_pairs(sc, np.stack(np.triu_indices(10, 1), 1), seed=5, f_noise=0.2, F_sigma=1e-3)
    pp = d["principal_point"]
    G = V.g_matrix(d["F"].reshape(-1, 3, 3), pp[d["cam1"]], pp[d["cam2"]])
    U, s, Vt = np.linalg.svd(G)
    Vm = np.swapaxes(Vt, 1, 2)
    base01, base12 = V.fetzer_from_svd(s, U, Vm)
    f = d["focal_init"]
    r0 = V.residuals(base01, base12, f[d["cam1"]], f[d["cam2"]])
    for k in (0, 1, 2):
        U2, V2 = U.copy(), Vm.copy()
        U2[:, :, k] *= -1
        V2[:, :, k] *= -1
        np.testing.assert_allclose(np.abs(U2 @ (s[:, :, None] * np.swapaxes(V2, 1, 2)) - G).max(), 0, atol=1e-9 * np.abs(G).max())
        a, b = V.fetzer_from_svd(s, U2, V2)
        if k < 2:   # d_01, d_12 change sign as a whole
            np.testing.assert_allclose(a, -base01, rtol=1e-14, atol=1e-14 * np.abs(base01).max())
            np.testing.assert_allclose(b, -base12, rtol=1e-14, atol=1e-14 * np.abs(base12).max())
        r = V.residuals(a, b, f[d["cam1"]], f[d["cam2"]])
        np.testing.assert_allclose(r, r0, rtol=0, atol=1e-14 * max(1.0, np.abs(r0).max()))


def test_same_camera_cost_is_the_two_camera_cost_at_fi_equal_fj():
    rng = np.random.default_rng(6)
    a, b = _random_d(rng, 100)
    f = rng.uniform(0.5, 2.0, 100)
    r, dri, drj = V.residuals(a, b, f, f, True)
    for e in range(100):
        assert list(r[e]) == _cost(a[e], b[e], f[e], f[e])
    h = 1e-6 * f
    num = (V.residuals(a, b, f + h, f + h) - V.residuals(a, b, f - h, f - h)) / (2 * h)[:, None]
    ok = np.abs(r).max(1) < 1e4
    assert np.all(np.abs(dri + drj - num)[ok] <= 1e-7 * (np.abs(num) + 1e-3)[ok])
    # the oracle's Jacobian column of a same-camera pair is that sum
    pp = np.zeros((1, 2))
    prob = V.VGCProblem(pp, np.array([1.0]), None, np.zeros(3, np.int32), np.zeros(3, np.int32), np.zeros((3, 9)), V.VGCOptions())
    prob.d01, prob.d12 = a[:3], b[:3]
    _, rc, J = prob.evaluate(np.array([f[0]]), True)
    r3, dri3, drj3 = V.residuals(a[:3], b[:3], np.full(3, f[0]), np.full(3, f[0]), True)
    _, rho1 = V.cauchy((r3 * r3).sum(1), 1e-2)
    np.testing.assert_allclose(J.toarray().ravel(), ((dri3 + drj3) * np.sqrt(rho1)[:, None]).ravel(), rtol=1e-15)


@pytest.mark.parametrize("K", [1, 40])
def test_noise_free_recovery(K):
    sc = S.make_scene(40, 20, seed=1, num_intrinsics=K)
    for f_noise in (0.2, -0.2):
        d = S.make_vgc_pairs(sc, np.stack(np.triu_indices(40, 1), 1), seed=1)
        d["focal_init"] = d["focal_true"] * (1 + f_noise)
        out = V.solve_vgc(d["principal_point"], d["focal_init"], None, d["cam1"], d["cam2"], d["F"])
        np.testing.assert_allclose(out["focal"], d["focal_true"], rtol=1e-6)
        assert out["pair_valid"].all() and out["cam_accepted"].all() and out["summary"].usable


def test_outlier_pairs_are_invalidated_and_inliers_kept():
    sc = S.make_scene(40, 20, seed=1, num_intrinsics=40)
    d = S.make_vgc_pairs(sc, np.stack(np.triu_indices(40, 1), 1), seed=1, f_noise=0.2, outlier_frac=0.1)
    out = V.solve_vgc(d["principal_point"], d["focal_init"], None, d["cam1"], d["cam2"], d["F"])
    # the Cauchy loss bounds but does not remove the outliers' pull: 3e-5 relative here
    np.testing.assert_allclose(out["focal"], d["focal_true"], rtol=1e-4)
    assert out["pair_valid"][~d["is_outlier"]].all()
    # every invalidated pair is an outlier; a random F often stays under |r| <= 2 at the true focals (the reference's
    # loose default threshold): 36 % of them are caught on this scene
    assert (~out["pair_valid"][d["is_outlier"]]).mean() > 0.3, (~out["pair_valid"][d["is_outlier"]]).mean()


# ---- driver rules through the object-level API, with the oracle behind calibrate_arrays -----------------------------
def _oracle_backend(pp, focal, focal_constant, cam1, cam2, F, options=None, ctx=None, want_residual=False):
    o = options or VGC.ViewGraphCalibratorOptions()
    out = V.solve_vgc(pp, focal, focal_constant, cam1, cam2, F,
                      V.VGCOptions(thres_lower_ratio=o.thres_lower_ratio, thres_higher_ratio=o.thres_higher_ratio,
                                   thres_two_view_error=o.thres_two_view_error))
    usable = out["summary"].usable if out["summary"] is not None else True
    return dict(focal=out["focal"], cam_accepted=out["cam_accepted"], pair_valid=out["pair_valid"], residual=out["residual"],
                stats=dict(usable=int(usable)), problem=out["problem"])


def _world(model=S.SIMPLE_PINHOLE, C=12, f_noise=0.2, seed=3):
    """Per-image cameras (ids 100 + i), image ids 10 + i, every pair (i, j) CALIBRATED and valid."""
    sc = S.make_scene(C, 20, seed=seed, model=model, num_intrinsics=C)
    pr = np.stack(np.triu_indices(C, 1), 1)
    d = S.make_vgc_pairs(sc, pr, seed=seed, f_noise=f_noise)
    cams = {}
    for i in range(C):
        p = np.array(sc.intr_params[i, :S.MODEL_NUM_PARAMS[model]], np.float64)
        scale = d["focal_init"][i] / d["focal_true"][i]
        p[VGC.focal_length_idxs(model)] *= scale
        cams[100 + i] = VGC.CalibCamera(model, p)
    pairs = [ImagePairMatches(10 + int(a), 10 + int(b), np.zeros((0, 2)), np.zeros(0, np.int64), config=IP.TWO_VIEW_CALIBRATED,
                              F=d["F"][e].reshape(3, 3)) for e, (a, b) in enumerate(pr)]
    return sc, d, cams, pairs, {10 + i: 100 + i for i in range(C)}


def test_driver_rules(monkeypatch):
    monkeypatch.setattr(VGC, "calibrate_arrays", _oracle_backend)
    sc, d, cams, pairs, img_cam = _world()
    # an unused camera, an invalid pair and non-E/F pairs of camera 105 with a random F
    cams[999] = VGC.CalibCamera(S.SIMPLE_PINHOLE, np.array([123.0, 10.0, 20.0]))
    junk = np.arange(9.0).reshape(3, 3)
    pairs[0].is_valid = False
    pairs[0].F = junk
    pairs[1].config = IP.TWO_VIEW_PLANAR
    pairs[1].F = junk
    pairs[2].config = IP.TWO_VIEW_DEGENERATE
    pairs[2].F = junk
    # camera 100 has a prior focal (constant), half the true one: still copied back, flagged
    cams[100].has_prior_focal_length = True
    cams[100].params[0] = d["focal_true"][0] * 0.5
    f100 = cams[100].params[0]
    assert VGC.ViewGraphCalibrator().Solve(pairs, cams, img_cam)
    assert cams[100].has_refined_focal_length and cams[100].params[0] == f100
    for i in range(1, 12):
        assert cams[100 + i].has_refined_focal_length
    assert not cams[999].has_refined_focal_length and cams[999].params[0] == 123.0
    assert not pairs[0].is_valid and pairs[1].is_valid and pairs[2].is_valid
    # camera 100's wrong prior invalidates some of its pairs; the skipped ones are untouched
    assert not all(p.is_valid for p in pairs[3:])


def test_all_priors_take_the_early_return(monkeypatch):
    monkeypatch.setattr(VGC, "calibrate_arrays", _oracle_backend)
    sc, d, cams, pairs, img_cam = _world()
    for c in cams.values():
        c.has_prior_focal_length = True
    before = {k: c.params.copy() for k, c in cams.items()}
    assert VGC.ViewGraphCalibrator().Solve(pairs, cams, img_cam)
    for k, c in cams.items():
        assert not c.has_refined_focal_length and np.array_equal(c.params, before[k])
    assert all(p.is_valid for p in pairs)


def test_ratio_rejection_keeps_the_camera_and_filters_with_the_estimate(monkeypatch):
    monkeypatch.setattr(VGC, "calibrate_arrays", _oracle_backend)
    sc, d, cams, pairs, img_cam = _world(f_noise=0.0)
    cams[103].params[0] *= 3.0     # the estimate returns to the truth: ratio 1/3 < thres_lower_ratio 0.5
    before = cams[103].params.copy()
    o = VGC.ViewGraphCalibratorOptions(thres_lower_ratio=0.5)
    K = len(cams)
    ok = VGC.ViewGraphCalibrator(o).Solve(pairs, cams, img_cam)
    assert ok
    assert not cams[103].has_refined_focal_length and np.array_equal(cams[103].params, before)
    # the filter used the estimate (the truth): every pair of camera 103 stays valid, although its kept focal is 3x off
    assert all(p.is_valid for p in pairs)
    ref = V.solve_vgc(d["principal_point"], np.where(np.arange(K - 0) == 3, d["focal_true"] * 3, d["focal_true"])[:K], None,
                      d["cam1"], d["cam2"], d["F"], V.VGCOptions(thres_lower_ratio=0.5))
    assert not ref["cam_accepted"][3] and ref["cam_accepted"].sum() == K - 1
    np.testing.assert_allclose(ref["focal"][3], d["focal_true"][3], rtol=1e-6)


def test_pinhole_sets_fx_and_fy(monkeypatch):
    monkeypatch.setattr(VGC, "calibrate_arrays", _oracle_backend)
    sc, d, cams, pairs, img_cam = _world(model=S.PINHOLE)
    assert VGC.ViewGraphCalibrator().Solve(pairs, cams, img_cam)
    for c in cams.values():
        assert c.has_refined_focal_length and c.params[0] == c.params[1]


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def test_abi_null_arguments_are_invalid_without_a_device():
    lib = _lib.load()
    o = _lib.VGCOpts()
    lib.b200sfm_vgc_default_opts(ct.byref(o))
    assert o.max_num_iterations == 100 and o.thres_loss_function == 1e-2 and o.pcg_rel_tolerance == 1e-12
    assert o.thres_lower_ratio == 0.1 and o.thres_higher_ratio == 10.0 and o.thres_two_view_error == 2.0
    st = _lib.LMStats()
    assert lib.b200sfm_view_graph_calibrate(None, ct.byref(o), 1, None, None, None, 1, None, None, None, None, None, None,
                                            ct.byref(st)) == 1
    assert lib.b200sfm_view_graph_calibrate(None, None, 0, None, None, None, 0, None, None, None, None, None, None, None) == 1


def test_vgc_opts_layout_matches_ctypes(tmp_path):
    fields = [f for f, _ in _lib.VGCOpts._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200sfm.h"\nint main(void) {\n' +
                   "".join(f'  printf("%zu\\n", offsetof(b200sfm_vgc_opts, {f}));\n' for f in fields) +
                   '  printf("%zu\\n", sizeof(b200sfm_vgc_opts));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", str(exe), str(src)],
                   check=True, capture_output=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    want = [getattr(_lib.VGCOpts, f).offset for f in fields] + [ct.sizeof(_lib.VGCOpts)]
    assert got == want


# ---- C++ shim ----------------------------------------------------------------------------------------------------------
def test_shim_flattens_in_sorted_id_order_and_copies_back(tmp_path):
    lib, exe, dump = tmp_path / "libb200sfm.so", tmp_path / "vgc_driver", tmp_path / "dump.txt"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c"),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_view_graph_calibration.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "shim_mock", "vgc_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe)], env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    rec = {}
    for line in dump.read_text().splitlines()[1:]:
        name, n, *vals = line.split()
        rec[name] = [float(v) for v in vals]
        assert len(vals) == int(n)
    # cameras in sorted id order: 3 (SIMPLE_PINHOLE, prior), 7 (PINHOLE), 9 (SIMPLE_RADIAL, no qualifying pair)
    assert rec["principal_point"] == [300, 200, 320, 240, 350, 250]
    assert rec["focal"] == [600, 505, 700]
    assert rec["focal_constant"] == [1, 0, 0]
    # qualifying pairs in sorted pair-id order: (10, 20) -> cameras (3, 7), (30, 10) -> (3, 3); PLANAR and invalid skipped
    assert rec["cam1"] == [0, 0] and rec["cam2"] == [1, 0]
    assert rec["F"][:9] == [10 + 0.5 * k + 0.2 for k in range(9)]
    assert rec["F"][9:] == [30 + 0.5 * k + 0.1 for k in range(9)]
    assert rec["opts"][6] == 3.0 and rec["opts"][2] == 1e-2
    out = r.stdout.splitlines()
    assert out[0] == "usable 1"
    assert out[1] == "camera 3 refined 1 params 1000 300 200"       # accepted (index 0): FocalLengthIdxs {0}
    assert out[2] == "camera 7 refined 0 params 500 510 320 240"    # not accepted: untouched
    assert out[3] == "camera 9 refined 1 params 1002 350 250 0.01"
    assert out[4:8] == ["valid 0", "valid 1", "valid 1", "valid 0"]   # pair 0 invalidated; PLANAR kept; invalid stays invalid


def test_shim_view_graph_calibrator_typechecks_against_the_glomap_api():
    """Inside a glomap build the shim's ViewGraphCalibrator takes glomap's ImagePair and Camera (Focal(),
    PrincipalPoint(), FocalLengthIdxs(), has_refined_focal_length): type-checked against tests/shim_mock/glomap_stub_vgc."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(ROOT, "tests", "shim_mock", "glomap_stub_vgc"),
                        "-I" + os.path.join(ROOT, "glomap_b200", "host"),
                        os.path.join(ROOT, "tests", "shim_mock", "vgc_typecheck.cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
