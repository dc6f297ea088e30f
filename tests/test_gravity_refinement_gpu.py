"""Gravity refinement on the device (b200sfm_gravity_refine) against oracle/gravity_oracle.py, and the stratified
rotation averager over it."""
import ctypes as ct

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E_, synthetic as S
from glomap_b200.gravity_refinement import GravityRefiner, GravityRefinerOptions, get_align_rot_householder
from glomap_b200.rotation_averager import RotationAveragerOptions, largest_component, solve_rotation_averaging
from oracle import gravity_oracle as GO
from test_gravity_refinement_cpu import SCENES, frame_inputs, make_scene

pytestmark = pytest.mark.gpu


def angle_deg(a, b):
    a = a / np.linalg.norm(a, axis=-1, keepdims=True)
    b = b / np.linalg.norm(b, axis=-1, keepdims=True)
    return np.degrees(np.arctan2(np.linalg.norm(np.cross(a, b), axis=-1), (a * b).sum(-1)))   # accurate near 0, unlike acos


def run_device(sc, opts=None):
    ref = GravityRefiner(opts)
    g, status, st = ref.RefineGravity(sc["vg"], sc["gravity"], sc["img_frame"], sc["img_sensor"], sc["sensor_quat"])
    return g, status, st


def check_against_oracle(sc, opts=None):
    g, status, st = run_device(sc, opts)
    R_align, has, f1, f2, M = frame_inputs(sc)
    res = GO.refine_gravity(R_align, has, f1, f2, M, GO.GravityOptions(**(opts or GravityRefinerOptions()).__dict__))
    assert res["margin"] > 1e-6   # no decision of the scene is within rounding of its bound
    np.testing.assert_array_equal(status, res["status"])
    assert st["error_prone_frames"] == len(res["error_prone"])
    assert st["rectified_frames"] == int((res["status"] == 2).sum())
    assert st["too_few_terms"] == int((res["status"] == 1).sum())
    it = list(res["iterations"].values())
    assert st["lm_iterations"] == sum(it) and st["max_lm_iterations"] == (max(it) if it else 0)
    acc = status == 2
    if acc.any():
        assert angle_deg(g[acc], res["gravity"][acc]).max() < 1e-7
    np.testing.assert_array_equal(g[~acc], sc["gravity"][~acc])
    return g, status, st


@pytest.mark.parametrize("kw", SCENES)
def test_device_equals_oracle(kw):
    _, status, _ = check_against_oracle(make_scene(**kw))
    assert (status == 2).any()


def test_device_equals_oracle_with_other_options():
    o = GravityRefinerOptions(max_outlier_ratio=0.4, max_gravity_error=2.0, min_num_neighbors=5)
    check_against_oracle(make_scene(F=40, sensors=2, seed=8, pair_prob=0.2, noise_deg=0.8, outlier_ratio=0.3), o)


@pytest.mark.parametrize("sensors", [1, 2])
def test_acceptance_scene_on_device(sensors):
    sc = make_scene(F=50, sensors=sensors, seed=11, outlier_ratio=0.3)
    g, status, st = check_against_oracle(sc)
    assert angle_deg(g, sc["R_frames"][:, :, 1]).max() < 1e-2
    assert st["rectified_frames"] == sc["outlier"].sum()


def test_hub_frame_with_1e5_neighbours():
    """Frame 0 (wrong prior) is paired with 10^5 frames (correct priors); its one warp loops over all of them."""
    rng = np.random.default_rng(9)
    n = 100_001
    w = rng.normal(size=(n, 3))
    from glomap_b200 import geometry as geo
    R = geo.so3_exp(w)
    ei = np.zeros(n - 1, np.int32)
    ej = np.arange(1, n, dtype=np.int32)
    vg = S.ViewGraph(n, ei, ej, R[ej] @ np.swapaxes(R[ei], -1, -2), np.ones(n - 1), R)
    g = R[:, :, 1].copy()
    g[0] = [1.0, 0.0, 0.0]
    sc = dict(vg=vg, gravity=g, img_frame=None, img_sensor=None, sensor_quat=None)
    gn, status, st = run_device(sc)
    assert status[0] == 2 and (status[1:] == 0).all() and st["error_prone_frames"] == 1
    R_align = get_align_rot_householder(g)
    res = GO.refine_gravity(R_align, np.ones(n, bool), ei, ej, vg.R_rel)
    assert angle_deg(gn[0], res["gravity"][0]) < 1e-7
    assert st["lm_iterations"] == res["iterations"][0]
    assert angle_deg(gn[0], R[0, :, 1]) < 0.01


def test_error_prone_frame_with_too_few_terms():
    """One frame of 4 cameras and only its own 6 image pairs (noisy): 12 counted incidences, 6 terms -> status 1."""
    sc = make_scene(F=1, sensors=4, seed=14, rel_noise_deg=10.0, outlier_ratio=0.0)
    g, status, st = check_against_oracle(sc)
    assert status[0] == 1 and st["too_few_terms"] == 1 and st["lm_iterations"] == 0


@pytest.mark.parametrize("toward", [1.0, -1.0])
def test_sign_tie_on_device(toward):
    """Frame 0 sees 4 neighbours whose gravity maps to +g and 4 to -g: the average's sign follows the prior (rule (ii))."""
    from glomap_b200 import geometry as geo
    rng = np.random.default_rng(15)
    n = 9
    R = geo.so3_exp(rng.normal(size=(n, 3)))
    ei, ej = np.zeros(n - 1, np.int32), np.arange(1, n, dtype=np.int32)
    vg = S.ViewGraph(n, ei, ej, R[ej] @ np.swapaxes(R[ei], -1, -2), np.ones(n - 1), R)
    g = R[:, :, 1].copy()
    g[5:] = -g[5:]
    perp = np.cross(g[0], [0.3, 0.5, 0.8])
    g[0] = toward * 0.3 * g[0] + perp / np.linalg.norm(perp)   # wrong prior, leaning to +g or -g
    sc = dict(vg=vg, gravity=g, img_frame=None, img_sensor=None, sensor_quat=None)
    o = GravityRefinerOptions(max_outlier_ratio=0.6)
    gn, status, st = check_against_oracle(sc, o)
    assert status[0] == 2
    assert angle_deg(gn[0], toward * R[0, :, 1]) < 1e-7


def test_repeated_calls_are_bit_identical():
    sc = make_scene(F=60, sensors=2, seed=12, pair_prob=0.3, noise_deg=0.5, rel_noise_deg=0.3, outlier_ratio=0.3)
    a = run_device(sc)
    for _ in range(3):
        b = run_device(sc)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def _raw(F, R_align, has, f1, f2, M):
    ctx = E_.default_context()
    o = GravityRefinerOptions().to_c()
    out = np.full((max(F, 1), 3), 7.0)
    status = np.full(max(F, 1), 9, np.uint8)
    st = _lib.GravityStats()
    p = lambda a: a.ctypes.data_as(ct.c_void_p)   # noqa: E731
    rc = ctx.lib.b200sfm_gravity_refine(ctx.handle, ct.byref(o), F, p(np.ascontiguousarray(R_align, np.float64)),
                                        p(np.ascontiguousarray(has, np.uint8)), len(f1), p(np.ascontiguousarray(f1, np.int32)),
                                        p(np.ascontiguousarray(f2, np.int32)), p(np.ascontiguousarray(M, np.float64)), p(out),
                                        p(status), ct.byref(st))
    return rc, out, status, st


def test_edge_cases():
    sc = make_scene(F=20, seed=13, pair_prob=0.6, outlier_ratio=0.3)
    R_align, has, f1, f2, M = frame_inputs(sc)
    F = len(has)
    # E == 0: OK, nothing written
    rc, out, status, st = _raw(F, R_align, has, f1[:0], f2[:0], M[:0])
    assert rc == 0 and (out == 7.0).all() and (status == 9).all() and st.error_prone_frames == 0
    # no gravity anywhere: every pair is ignored
    rc, out, status, st = _raw(F, R_align, np.zeros(F), f1, f2, M)
    assert rc == 0 and (status == 9).all()
    g, s, st2 = GravityRefiner().RefineGravity(sc["vg"], np.full((F, 3), np.nan))
    assert (s == 0).all() and np.isnan(g).all()
    # clean priors: no error-prone frame
    clean = dict(sc, gravity=sc["R_frames"][:, :, 1].copy())
    g, s, st2 = run_device(clean)
    assert (s == 0).all() and st2["error_prone_frames"] == 0 and (g == clean["gravity"]).all()
    # a frame index out of range, on the device
    for bad in (F, -1):
        f1b = f1.copy()
        f1b[len(f1b) // 2] = bad
        rc, out, status, _ = _raw(F, R_align, has, f1b, f2, M)
        assert rc == 1 and (out == 7.0).all() and (status == 9).all()
        assert "outside" in _lib.load().b200sfm_last_error(E_.default_context().handle).decode()
    # a zero gravity prior
    gz = sc["gravity"].copy()
    gz[3] = 0.0
    with pytest.raises(_lib.B200Error) as ei:
        GravityRefiner().RefineGravity(sc["vg"], gz)
    assert ei.value.code == 1
    # the context still works
    check_against_oracle(sc)


def test_multi_rank_context_is_unsupported():
    import threading
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs for a two-rank context")
    lib = _lib.load()
    uid = ct.create_string_buffer(_lib.NCCL_ID_BYTES)
    assert lib.b200sfm_nccl_unique_id(uid) == 0
    handles, rcs = [ct.c_void_p(), ct.c_void_p()], [None, None]

    def make(r):
        rcs[r] = lib.b200sfm_create_dist(r, r, 2, uid, ct.byref(handles[r]))
    threads = [threading.Thread(target=make, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    try:
        assert rcs == [0, 0]
        o = GravityRefinerOptions().to_c()
        assert lib.b200sfm_gravity_refine(handles[0], ct.byref(o), 0, None, None, 0, None, None, None, None, None, None) == 5
    finally:
        threads = [threading.Thread(target=lib.b200sfm_destroy, args=(h,)) for h in handles if h.value]
        for t in threads:
            t.start()
        for t in threads:
            t.join()


def _gravity_vg(seed, share):
    vg = S.make_random_view_graph(80, 10, seed=seed, noise_deg=1.0)
    g, _ = S.make_gravity(vg.R_gt, noise_deg=0.0, outlier_ratio=0.0, seed=seed)
    rng = np.random.default_rng(seed)
    g[rng.uniform(size=vg.n_images) >= share] = np.nan
    return vg, g


def _r_init(g):
    has = ~np.isnan(g).any(axis=1)
    R0 = np.tile(np.eye(3), (len(g), 1, 1))
    R0[has] = get_align_rot_householder(g[has])
    return R0


@pytest.mark.parametrize("share", [0.5, 1.0])
def test_solve_rotation_averaging_equals_two_calls(share):
    vg, g = _gravity_vg(21, share)
    o = RotationAveragerOptions(use_gravity=True, skip_initialization=True)
    R0 = _r_init(g)
    ok, R, reg = solve_rotation_averaging(vg, g, o, R0)
    assert ok and reg.all()
    # the explicit composition: 1-DoF on the gravity pairs' largest component, then the whole graph
    has = ~np.isnan(g).any(axis=1)
    est_o = E_.RotationEstimatorOptions(use_gravity=True, skip_initialization=True)
    Rx = R0.copy()
    k = has[vg.ei] & has[vg.ej]
    if share < 1.0:
        m = largest_component(vg.n_images, vg.ei[k], vg.ej[k])
        idx = np.nonzero(m)[0]
        remap = np.full(vg.n_images, -1)
        remap[idx] = np.arange(len(idx))
        kk = k & m[vg.ei] & m[vg.ej]
        sub = S.ViewGraph(len(idx), remap[vg.ei[kk]].astype(np.int32), remap[vg.ej[kk]].astype(np.int32), vg.R_rel[kk],
                          vg.weight[kk], vg.R_gt[idx])
        ok1, R1 = E_.RotationEstimator(est_o).EstimateRotations(sub, Rx[idx], gravity=g[idx])
        assert ok1
        Rx[idx] = R1
    ok2, R2 = E_.RotationEstimator(est_o).EstimateRotations(vg, Rx, gravity=g)
    assert ok2
    np.testing.assert_allclose(R, R2, rtol=0, atol=1e-9)   # the rotation averager itself repeats to ~1e-14, not bit for bit
    # gravity frames keep their prior: R_i e_y is the gravity direction
    assert angle_deg(R[has][:, :, 1], g[has]).max() < 1e-6


def test_refined_gravity_improves_rotation_averaging():
    vg = S.make_random_view_graph(100, 16, seed=31, noise_deg=0.5)
    g, out = S.make_gravity(vg.R_gt, noise_deg=0.0, outlier_ratio=0.3, seed=31)
    o = RotationAveragerOptions(use_gravity=True, skip_initialization=True)
    from glomap_b200 import geometry as geo

    def err(R):
        rot, _, _ = geo.compare_reconstructions(R, np.zeros((len(R), 3)), vg.R_gt, np.zeros((len(R), 3)))
        return rot
    _, R_raw, _ = solve_rotation_averaging(vg, g, o, _r_init(g))
    g_ref, status, _ = GravityRefiner().RefineGravity(vg, g)
    assert (status[out] == 2).mean() > 0.8
    _, R_ref, _ = solve_rotation_averaging(vg, g_ref, o, _r_init(g))
    assert err(R_ref) < err(R_raw)
