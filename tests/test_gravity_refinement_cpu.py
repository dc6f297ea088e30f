"""Gravity refinement on the CPU: the oracle against a loop-and-dict transcription of
glomap/estimators/gravity_refinement.cc, the reference's acceptance scene, the sphere manifold, the stratification rule,
and the ABI / wrapper checks that need no device."""
import ctypes as ct

import numpy as np
import pytest

from glomap_b200 import _lib, geometry as geo, synthetic as S
from glomap_b200.gravity_refinement import GravityRefiner, frame_pairs, get_align_rot_householder
from glomap_b200.rotation_averager import largest_component, stratified_branch
from oracle import gravity_oracle as GO


def random_rotations(rng, k):
    w = rng.normal(size=(k, 3))
    w /= np.linalg.norm(w, axis=1, keepdims=True)
    return geo.so3_exp(w * rng.uniform(0, np.pi, size=(k, 1)))


def make_scene(F, sensors=1, seed=1, pair_prob=1.0, noise_deg=0.0, rel_noise_deg=0.0, outlier_ratio=0.3, no_gravity=0.0):
    """F frames of ``sensors`` cameras each (sensor 0 is the rig's reference), image pairs drawn with ``pair_prob`` (pairs
    inside one frame included), gravity priors by synthetic.make_gravity, a share ``no_gravity`` of frames without one."""
    rng = np.random.default_rng(seed)
    R_frames = random_rotations(rng, F)
    R_sens = np.concatenate([np.eye(3)[None], random_rotations(rng, sensors - 1)]) if sensors > 1 else np.eye(3)[None]
    img_frame = np.repeat(np.arange(F), sensors).astype(np.int32)
    img_sensor = np.tile(np.arange(sensors), F).astype(np.int32)
    R_img = R_sens[img_sensor] @ R_frames[img_frame]
    n = F * sensors
    ei, ej = np.triu_indices(n, 1)
    keep = rng.uniform(size=len(ei)) < pair_prob
    ei, ej = ei[keep].astype(np.int32), ej[keep].astype(np.int32)
    R_rel = R_img[ej] @ np.swapaxes(R_img[ei], -1, -2)
    if rel_noise_deg > 0:
        R_rel = geo.so3_exp(rng.normal(size=(len(ei), 3)) * np.radians(rel_noise_deg) / np.sqrt(3)) @ R_rel
    vg = S.ViewGraph(n, ei, ej, R_rel, np.ones(len(ei)), R_img)
    g, out = S.make_gravity(R_frames, noise_deg, outlier_ratio, seed=seed + 100)
    g[rng.uniform(size=F) < no_gravity] = np.nan
    return dict(vg=vg, img_frame=img_frame, img_sensor=img_sensor, sensor_quat=geo.rotmat_to_quat_xyzw_fast(R_sens),
                R_sens=R_sens, gravity=g, outlier=out, R_frames=R_frames)


def frame_inputs(sc):
    """(R_align [F,3,3], has [F], frame1, frame2, M) as b200sfm_gravity_refine takes them."""
    g = sc["gravity"]
    has = ~np.isnan(g).any(axis=1)
    R_align = np.tile(np.eye(3), (len(g), 1, 1))
    R_align[has] = get_align_rot_householder(g[has])
    f1, f2, M = frame_pairs(sc["vg"], sc["img_frame"], sc["img_sensor"], sc["sensor_quat"])
    return R_align, has, f1, f2, M


def transcription(sc, opts, order=None, jacobi=True):
    """gravity_refinement.cc:9-181 over maps: images {id: (frame, cam_from_rig)}, pairs {id: (i1, i2, R_rel)}, frame
    gravities {id: g}.  ``jacobi``: the neighbours' gravities are the ones on entry (rule (i) of include/b200sfm.h);
    otherwise accepted frames update them as the loop goes, in ``order`` (ascending by default).  Returns
    (status {frame: 1|2|3}, gravity {frame: g} of the accepted frames, error-prone set, counters)."""
    vg = sc["vg"]
    images = {i: (int(sc["img_frame"][i]), sc["R_sens"][sc["img_sensor"][i]]) for i in range(vg.n_images)}
    pairs = {e: (int(vg.ei[e]), int(vg.ej[e]), vg.R_rel[e]) for e in range(vg.E)}
    frames = {f: (None if np.isnan(g).any() else g.copy()) for f, g in enumerate(sc["gravity"])}
    r_align = {f: GO_align(g) for f, g in frames.items() if g is not None}

    def has_gravity(i):
        return frames[images[i][0]] is not None

    def image_r_align(i, table):
        return images[i][1] @ table[images[i][0]]

    # IdentifyErrorProneGravity (.cc:129-181)
    counter = {f: [0, 0] for f in frames}
    for e, (i1, i2, R_rel) in pairs.items():
        if has_gravity(i1) and has_gravity(i2):
            R = image_r_align(i2, r_align).T @ R_rel @ image_r_align(i1, r_align)
            R_up = GO.angle_to_rot_up(GO.rot_up_angle(R))
            angle = np.degrees(np.arccos(np.clip((np.trace(R.T @ R_up) - 1) / 2, -1, 1)))
            counter[images[i1][0]][1] += 1
            counter[images[i2][0]][1] += 1
            if angle > opts.max_gravity_error:
                counter[images[i1][0]][0] += 1
                counter[images[i2][0]][0] += 1
    error_prone = {f for f, (m, t) in counter.items() if t >= opts.min_num_neighbors and m / t >= opts.max_outlier_ratio}
    # the pairs of every frame (.cc:29-36)
    frame_pairs_ = {}
    for e, (i1, i2, _) in pairs.items():
        for i in (i1, i2):
            frame_pairs_.setdefault(images[i][0], set()).add(e)
    entry = dict(r_align)
    current = dict(r_align)
    status, out = {}, {}
    for f in (sorted(error_prone) if order is None else [x for x in order if x in error_prone]):
        table = entry if jacobi else current
        gravities = []
        for e in sorted(frame_pairs_[f]):
            i1, i2, R_rel = pairs[e]
            if not (has_gravity(i1) and has_gravity(i2)):
                continue
            if images[i1][0] == f:
                gravities.append((images[i1][1].T @ R_rel.T @ image_r_align(i2, table))[:, 1])
            elif images[i2][0] == f:
                gravities.append((images[i2][1].T @ R_rel @ image_r_align(i1, table))[:, 1])
        if len(gravities) < opts.min_num_neighbors:
            status[f] = 1
            continue
        gs = np.array(gravities)
        x, _ = GO.solve_sphere_lm(gs, GO.average_gravity(gs, table[f][:, 1]), opts)
        outliers = sum(np.degrees(np.arccos(np.clip(g @ x, -1, 1))) > 2 * opts.max_gravity_error for g in gs)
        if outliers / len(gs) < opts.max_outlier_ratio:
            status[f] = 2
            out[f] = x
            current[f] = GO_align(x)
        else:
            status[f] = 3
    return status, out, error_prone, counter


def GO_align(g):
    return get_align_rot_householder(np.asarray(g))


SCENES = [
    dict(F=40, sensors=1, seed=1, pair_prob=0.5, noise_deg=0.3, outlier_ratio=0.3),
    dict(F=30, sensors=2, seed=2, pair_prob=0.3, noise_deg=0.2, rel_noise_deg=0.2, outlier_ratio=0.35),
    dict(F=30, sensors=3, seed=5, pair_prob=0.15, outlier_ratio=0.3, no_gravity=0.2),
    dict(F=60, sensors=1, seed=4, pair_prob=0.14, noise_deg=0.5, outlier_ratio=0.3),   # degrees around min_num_neighbors
]


@pytest.mark.parametrize("kw", SCENES)
def test_oracle_equals_transcription(kw):
    sc = make_scene(**kw)
    opts = GO.GravityOptions()
    R_align, has, f1, f2, M = frame_inputs(sc)
    res = GO.refine_gravity(R_align, has, f1, f2, M, opts)
    status, out, ep, counter = transcription(sc, opts)
    F = len(has)
    assert set(res["error_prone"].tolist()) == ep
    assert [list(counter[f]) for f in range(F)] == [[int(res["mistakes"][f]), int(res["total"][f])] for f in range(F)]
    assert {f: int(s) for f, s in enumerate(res["status"]) if s} == status
    for f, x in out.items():
        np.testing.assert_allclose(res["gravity"][f], x, rtol=0, atol=1e-12)
    assert len(ep) > 0 and 2 in status.values()


def test_scene_exercises_min_num_neighbors():
    sc = make_scene(**SCENES[3])
    R_align, has, f1, f2, M = frame_inputs(sc)
    total = GO.refine_gravity(R_align, has, f1, f2, M)["total"]
    assert ((total == 6) | (total == 7)).sum() >= 3


def test_pairs_inside_a_frame_count_twice_and_refine_once():
    sc = make_scene(F=12, sensors=2, seed=5, outlier_ratio=0.0)
    R_align, has, f1, f2, M = frame_inputs(sc)
    res = GO.refine_gravity(R_align, has, f1, f2, M)
    # 11 other frames x 4 image pairs + the frame's own pair, counted for both of its images' frames
    assert (res["total"] == 11 * 4 + 2).all()


def test_sign_tie_points_toward_the_prior():
    rng = np.random.default_rng(7)
    g = np.array([0.0, 1.0, 0.0])
    gs = np.array([g, g, -g, -g]) + rng.normal(size=(4, 3)) * 1e-3
    a = GO.average_gravity(gs, np.array([0.1, 1.0, 0.0]))
    b = GO.average_gravity(gs, np.array([0.1, -1.0, 0.0]))
    assert a[1] > 0.99 and b[1] < -0.99
    # 3 against 2: the majority decides, whatever the prior
    gs5 = np.concatenate([gs, [g]])
    assert GO.average_gravity(gs5, -g)[1] > 0.99


@pytest.mark.parametrize("sensors", [1, 2])
def test_acceptance_scene(sensors):
    """rotation_averager_test.cc:366-450: 50 frames (2 rigs x 25), all pairs, no noise, 30 % outlier priors; every
    gravity is within 1e-2 deg of the truth after refinement, also when the frames are refined one after another."""
    sc = make_scene(F=50, sensors=sensors, seed=11, outlier_ratio=0.3)
    truth = sc["R_frames"][:, :, 1]
    opts = GO.GravityOptions()
    R_align, has, f1, f2, M = frame_inputs(sc)
    res = GO.refine_gravity(R_align, has, f1, f2, M, opts)
    assert sc["outlier"].sum() >= 10

    def check(final):
        final = final / np.linalg.norm(final, axis=1, keepdims=True)
        err = np.degrees(np.arccos(np.clip((final * truth).sum(1), -1, 1)))
        assert err.max() < 1e-2, err.max()

    g = sc["gravity"].copy()
    g[res["status"] == 2] = res["gravity"][res["status"] == 2]
    check(g)
    for order in (list(range(50)), list(np.random.default_rng(3).permutation(50))):
        status, out, _, _ = transcription(sc, opts, order=order, jacobi=False)
        g = sc["gravity"].copy()
        for f, x in out.items():
            g[f] = x
        check(g)


def test_sphere_manifold_jacobian_matches_finite_differences():
    rng = np.random.default_rng(2)
    for x in [rng.normal(size=3), np.array([1e-9, -2e-9, -1.0]), np.array([0.0, 0.0, 2.0])]:
        P = GO.sphere_plus_jacobian(x)
        h = 1e-6
        fd = np.stack([(GO.sphere_plus(x, h * e) - GO.sphere_plus(x, -h * e)) / (2 * h) for e in np.eye(2)], 1)
        np.testing.assert_allclose(P, fd, atol=1e-8)
        assert abs(np.linalg.norm(GO.sphere_plus(x, rng.normal(size=2))) - np.linalg.norm(x)) < 1e-12


def test_householder_align_rot():
    rng = np.random.default_rng(4)
    g = np.concatenate([rng.normal(size=(50, 3)), [[1, 0, 0], [-1, 0, 0], [0, 0, 3]]])
    R = get_align_rot_householder(g)
    np.testing.assert_allclose(R[:, :, 1], g / np.linalg.norm(g, axis=1, keepdims=True), atol=1e-15)
    np.testing.assert_allclose(R @ np.swapaxes(R, -1, -2), np.broadcast_to(np.eye(3), R.shape), atol=1e-14)
    np.testing.assert_allclose(np.linalg.det(R), 1.0, atol=1e-14)
    assert not np.isfinite(get_align_rot_householder(np.zeros(3))).all()


@pytest.mark.parametrize("share,expect", [(0.0, False), (0.95, True), (0.96, False), (0.5, True)])
def test_stratification_branch(share, expect):
    """.cc:42-50: the 1-DoF subsystem is solved unless there is no gravity pair or they are more than 95 % of all."""
    n, E = 101, 100
    vg = S.ViewGraph(n, np.arange(E, dtype=np.int32), np.arange(1, E + 1, dtype=np.int32), np.tile(np.eye(3), (E, 1, 1)),
                     np.ones(E), np.tile(np.eye(3), (n, 1, 1)))
    g = np.full((n, 3), np.nan)
    g[: int(round(share * E)) + (1 if share > 0 else 0)] = [0, 1, 0]   # a path: k + 1 frames give k gravity pairs
    assert stratified_branch(vg, g) is expect


def test_largest_component():
    m = largest_component(7, [0, 1, 3, 4, 5], [1, 2, 4, 5, 6])
    assert m.tolist() == [False, False, False, True, True, True, True]
    assert not largest_component(3, [], []).any()


def test_abi_layout_and_null_checks():
    assert ct.sizeof(_lib.GravityOpts) == 64
    assert _lib.GravityOpts.min_num_neighbors.offset == 16 and _lib.GravityOpts.reserved.offset == 48
    assert ct.sizeof(_lib.GravityStats) == 64
    assert _lib.GravityStats.lm_iterations.offset == 16 and _lib.GravityStats.ms_refine.offset == 56
    lib = _lib.load()
    o = _lib.GravityOpts()
    lib.b200sfm_gravity_default_opts(ct.byref(o))
    assert (o.max_outlier_ratio, o.max_gravity_error, o.min_num_neighbors, o.max_num_iterations) == (0.5, 1.0, 7, 100)
    assert (o.function_tolerance, o.gradient_tolerance, o.parameter_tolerance) == (1e-5, 1e-10, 1e-8)
    assert lib.b200sfm_gravity_refine(None, ct.byref(o), 1, None, None, 0, None, None, None, None, None, None) == 1
    assert lib.b200sfm_gravity_refine(None, None, 1, None, None, 0, None, None, None, None, None, None) == 1


def test_wrapper_rejects_bad_input_before_the_device():
    sc = make_scene(F=10, seed=6)
    ref = GravityRefiner()
    vg = sc["vg"]
    bad_vg = S.ViewGraph(vg.n_images, vg.ei.astype(np.float64), vg.ej, vg.R_rel, vg.weight, vg.R_gt)
    with pytest.raises(ValueError, match="integer"):
        ref.RefineGravity(bad_vg, sc["gravity"])
    with pytest.raises(ValueError, match="rows"):
        ref.RefineGravity(vg, sc["gravity"][:-1])
    g = sc["gravity"].copy()
    g[3, 1] = np.inf
    with pytest.raises(ValueError, match="finite"):
        ref.RefineGravity(vg, g)
    g[3] = [np.nan, 1.0, 0.0]
    with pytest.raises(ValueError, match="finite"):
        ref.RefineGravity(vg, g)
    with pytest.raises(ValueError, match="img_frame"):
        ref.RefineGravity(vg, sc["gravity"], img_frame=np.zeros(3, np.int32))
    with pytest.raises(ValueError, match="int32"):
        ref.refine_frames(sc["gravity"], np.array([2 ** 32]), np.array([0]), np.eye(3)[None])
    with pytest.raises(ValueError, match="outside"):
        ref.refine_frames(sc["gravity"], np.array([10]), np.array([0]), np.eye(3)[None])


def test_gravity_file_round_trip(tmp_path):
    names = ["a.jpg", "b.jpg", "c.jpg"]
    g = np.array([[0.1, 0.9, 0.2], [np.nan] * 3, [1e-3, -1.0, 3.0]])
    S.write_gravity_file(str(tmp_path / "g.txt"), names, g)
    r = S.read_gravity_file(str(tmp_path / "g.txt"), names + ["d.jpg"])
    np.testing.assert_array_equal(r[:3], g)
    assert np.isnan(r[3]).all()
