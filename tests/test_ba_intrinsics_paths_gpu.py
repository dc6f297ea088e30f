"""Operator-level tests of the bundle adjuster's intrinsics paths that one camera model per problem and a held
principal point never reach, against the FP64 sparse reference, through the probe, the comparison and the bounds of
test_ba_system_gpu.py.

select_paths gives every intrinsics block its own number of variable parameters mb (SIMPLE_PINHOLE 1, PINHOLE and
SIMPLE_RADIAL 2, RADIAL 3; two more each with optimize_principal_point) and picks the kernels from the largest one, nk.
The cases here are:
  * mixed models in one problem: blocks with mb = 1 next to mb = 2 in the stored-row kernels (nk = 2), and mb = 1..3
    in one launch of the extended path; a SIMPLE_RADIAL block with k = 0 among them (the pinhole branch);
  * a free principal point: mb = 3..5, cx and cy in the slots between the focal length and the distortion;
    optimize_principal_point alone frees every parameter, exactly as with optimize_intrinsics set too;
  * one block per image with every model, and a rig whose sensors have different models;
  * an intrinsics block whose only observations lie on tracks shorter than min_num_view_per_track: it is not a
    parameter block of the problem (Jacobi scale -1, candidate equal to the start).
"""
import numpy as np
import pytest

import test_ba_system_gpu as T
from glomap_b200 import estimators as E, synthetic as S

pytestmark = pytest.mark.gpu

SP, PH, SR, RD = S.SIMPLE_PINHOLE, S.PINHOLE, S.SIMPLE_RADIAL, S.RADIAL
MIXED3 = (SP, PH, SR)                       # mb 1, 2, 2 with the principal point held
ALL4 = (SP, PH, SR, RD)                     # mb 1, 2, 2, 3 (3, 4, 4, 5 with it free)
HEAVY_CAMS = {9: 300, 10: 300, 11: 300, 12: 300}   # more than one kSeg = 256 segment each; blocks 9..12 of both cycles
K0_BLOCK = 2                                # SIMPLE_RADIAL in both cycles, k = 0: the pinhole form of the projection
UNUSED_BLOCK = T.EMPTY_CAM                  # only observations on tracks shorter than MIN_VIEWS
RIG_MODELS = (RD, PH, SP)                   # one per sensor of make_rig

_make_intrinsics = S.make_intrinsics


def _mixed_intrinsics(C, model, focal, image_size, K):
    """Per-block models (cyclic), k = 0 on K0_BLOCK, and UNUSED_BLOCK referenced by EMPTY_CAM alone: the cameras that
    share it when K < C move to the next block of the same model."""
    cam_intr, intr_model, intr_params = _make_intrinsics(C, model, focal, image_size, K)
    assert intr_model[K0_BLOCK] == SR
    intr_params = intr_params.copy()
    intr_params[K0_BLOCK, 3] = 0.0
    cam_intr = cam_intr.copy()
    other = (cam_intr == UNUSED_BLOCK) & (np.arange(C) != T.EMPTY_CAM)
    cam_intr[other] = UNUSED_BLOCK + len(model)
    return cam_intr, intr_model, intr_params


def _drop_repeated_views(sc):
    """Keep the first observation of a point by a camera (a heavy camera may be appended to a track that has it)."""
    lens = np.diff(sc.pt_obs_begin)
    pt = np.repeat(np.arange(sc.P), lens)
    keep = np.zeros(sc.N, bool)
    keep[np.unique(pt * sc.C + sc.obs_cam, return_index=True)[1]] = True
    sc.obs_cam, sc.obs_xy = sc.obs_cam[keep], sc.obs_xy[keep]
    sc.pt_obs_begin = np.concatenate([[0], np.cumsum(np.bincount(pt[keep], minlength=sc.P))]).astype(np.int64)
    return sc


def make_mixed_scene(K, models):
    """The scene of test_ba_system_gpu.make_scene with per-block models and the heavy cameras of every model."""
    with pytest.MonkeyPatch.context() as m:
        m.setattr(S, "make_intrinsics", _mixed_intrinsics)
        m.setattr(T, "SPECIAL_CAMS", {**T.SPECIAL_CAMS, **HEAVY_CAMS})
        return _drop_repeated_views(T.make_scene(K=K, model=models))


_SCENES = {}


def scene(spec):
    if spec not in _SCENES:
        kind, *arg = spec
        if kind == "mixed":
            _SCENES[spec] = make_mixed_scene(*arg)
        elif kind == "rig":
            _SCENES[spec] = T.make_rig(model=RIG_MODELS)
        else:
            _SCENES[spec] = T.make_scene(K=1, model=arg[0])
    return _SCENES[spec]


M3_300, M4_200, M4_300 = ("mixed", 300, MIXED3), ("mixed", 200, ALL4), ("mixed", 300, ALL4)
RIG = ("rig",)
INTR = dict(optimize_intrinsics=True)
PP = dict(optimize_intrinsics=True, optimize_principal_point=True)
# name: (scene, options, environment, expected path)
PATHS = {
    "kfast_nk2_mixed_K300": (M3_300, INTR, {}, dict(use_ell=1, kfast=1, nk=2, ext=1, ext_k=1)),
    "ext_kfast_off_mixed_K300": (M3_300, INTR, {"B200SFM_KFAST": "0"}, dict(ext=1, ext_k=1, kfast=0, nk=2)),
    "ext_mixed_all_models_K200": (M4_200, INTR, {}, dict(ext=1, ext_k=1, kfast=0, nk=3)),
    "pp_simple_pinhole_K1": (("one", SP), PP, {}, dict(ext=1, ext_k=1, kfast=0, nk=3)),
    "pp_pinhole_K1": (("one", PH), PP, {}, dict(ext=1, ext_k=1, kfast=0, nk=4)),
    "pp_simple_radial_K1": (("one", SR), PP, {}, dict(ext=1, ext_k=1, kfast=0, nk=4)),
    "pp_radial_K1": (("one", RD), PP, {}, dict(ext=1, ext_k=1, kfast=0, nk=5)),
    "pp_only_mixed_K200": (M4_200, dict(optimize_principal_point=True), {}, dict(ext=1, ext_k=1, kfast=0, nk=5)),
    "pp_per_image_mixed_K300": (M4_300, PP, {}, dict(ext=1, ext_k=1, kfast=0, nk=5)),
    "rig_mixed_sensors_intrinsics": (RIG, INTR, {}, dict(ext=1, ext_k=1, ext_s=0, kfast=0, nk=3)),
    "rig_mixed_sensors_intrinsics_rig_poses": (RIG, dict(INTR, optimize_rig_poses=True), {},
                                               dict(ext=1, ext_k=1, ext_s=1, kfast=0, nk=3)),
    "rig_pp": (RIG, dict(optimize_principal_point=True, optimize_rig_poses=True), {},
               dict(ext=1, ext_k=1, ext_s=1, kfast=0, nk=5)),
}


@pytest.mark.parametrize("name", list(PATHS))
def test_intrinsics_path_matches_the_fp64_reference(name, monkeypatch):
    spec, opts, env, want = PATHS[name]
    sc = scene(spec)
    # the whole comparison of test_ba_system_gpu.py on this case's scene (its scene cache is bypassed)
    monkeypatch.setitem(T.PATHS, name, ("rig" if spec == RIG else {}, opts, env, want))
    T.test_device_step_matches_the_fp64_reference(name, lambda _spec: sc, monkeypatch)


def test_principal_point_flag_alone_takes_the_same_step_as_both_flags():
    """optimize_principal_point frees every parameter whatever optimize_intrinsics says (bundle_adjustment.cc:273-293):
    the two option sets are the same problem, so the device takes the same path and forms the same numbers (up to the
    order of its atomic sums: the heavy blocks span several segments)."""
    sc = scene(M4_200)
    mask = E.first_frame_mask(sc.C)
    for c, m in T.MASKED.items():
        mask[c] = m
    runs = []
    for opts in (dict(optimize_principal_point=True), PP):
        probe = T.Probe(sc, opts, mask)
        runs.append(probe.step(T.LOOSE_K, T.FIRST_RADIUS))
    (o1, d1), (o2, d2) = runs
    for f in ("nbk", "use_v2", "use_ell", "ext", "ext_k", "ext_s", "kfast", "nk", "schur_jacobi", "pcg_iterations"):
        assert getattr(o1, f) == getattr(o2, f), f
    for f in ("cost", "model_cost_change", "cand_cost", "step_norm", "x_norm"):
        assert abs(getattr(o1, f) - getattr(o2, f)) <= 1e-12 * abs(getattr(o2, f)), f
    assert np.array_equal(d1["jscale_c"] < 0, d2["jscale_c"] < 0)
    for f, w in (("U", 21), ("g_c", 6), ("jscale_c", 6), ("V", 6), ("g_p", 3), ("Dc", 6), ("b", 6), ("Minv", 21),
                 ("px", 6), ("cand_intr", S.INTR_STRIDE), ("cand_points", 3), ("cand_trans", 3)):
        assert T.blockerr(d1[f], d2[f], w) <= 1e-12, f
