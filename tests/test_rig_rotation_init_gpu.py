"""b200sfm_rig_rotations_from_images and solve_rotation_averaging_rig on the device against oracle/rig_init_oracle.py."""
import numpy as np
import pytest

from glomap_b200 import _lib, geometry as G
from glomap_b200 import rotation_averager as RA
from glomap_b200.synthetic import ViewGraph
from oracle import rig_init_oracle as O

pytestmark = pytest.mark.gpu


def qangle(a, b):
    """Sign-invariant rotation angle between quaternions, 4 atan2(|a - b|, |a + b|) (exact down to rounding, unlike arccos)."""
    a = np.asarray(a) / np.linalg.norm(a, axis=-1, keepdims=True)
    b = np.asarray(b) / np.linalg.norm(b, axis=-1, keepdims=True)
    b = np.where((a * b).sum(-1, keepdims=True) < 0, -b, b)
    return 4 * np.arctan2(np.linalg.norm(a - b, axis=-1), np.linalg.norm(a + b, axis=-1))


def conversion_case(F=2000, seed=0):
    """Two rigs (4 and 6 cameras: 10 cameras, 0 and 4 the references), ~30 % of the images unregistered, the images in a
    random order, image rotations R_cam R_frame with 0.02 rad of noise (the averages are estimates of one rotation;
    wider spreads are in tests/test_rig_average_gpu.py); some cameras known."""
    rng = np.random.default_rng(seed)
    rig_cams = [np.arange(0, 4), np.arange(4, 10)]
    rig_of = rng.integers(0, 2, F)
    fr, cam = [], []
    for f in range(F):
        cs = rig_cams[rig_of[f]]
        cs = cs[rng.uniform(size=len(cs)) < 0.9]
        fr += [f] * len(cs)
        cam += cs.tolist()
    perm = rng.permutation(len(fr))
    fr, cam = np.array(fr)[perm], np.array(cam)[perm]
    fr = np.where(rng.uniform(size=len(fr)) < 0.3, -1, fr)
    Rf, Rs = G.so3_exp(rng.normal(size=(F, 3))), G.so3_exp(rng.normal(size=(10, 3)) * 0.5)
    Rs[[0, 4]] = np.eye(3)
    q = G.rotmat_to_quat_xyzw_fast(G.so3_exp(rng.normal(size=(len(fr), 3)) * 0.02) @ Rs[cam] @ Rf[np.maximum(fr, 0)])
    q *= rng.choice([-1.0, 1.0], size=(len(fr), 1)) * rng.uniform(0.5, 2.0, size=(len(fr), 1))   # any sign and norm
    known = np.zeros(10, np.uint8)
    known[[0, 4, 1, 5]] = 1
    cq = G.rotmat_to_quat_xyzw_fast(Rs)
    cq[~known.astype(bool)] = [0.3, 0.1, 0.0, 0.9]                                # unknown: input rows ignored
    ref = np.where(rig_of == 0, 0, 4)
    est = (rng.uniform(size=len(fr)) < 0.95).astype(np.uint8)
    fq = np.tile([0.1, 0.2, 0.3, 0.9], (F, 1))
    return fr, cam, q, ref, known, cq, fq, est


def test_conversion_matches_the_oracle():
    args = conversion_case()
    fr, cam, q, ref, known, cq, fq, est = args
    from glomap_b200.rotation_initializer import convert_rotations_from_image_to_rig
    st = _lib.RigInitStats()
    d = convert_rotations_from_image_to_rig(fr, cam, q, ref, known, cq, fq, image_estimated=est, stats=st)
    o = O.convert_rotations(fr, cam, q, ref, known, cq, fq, image_estimated=est)
    assert np.array_equal(d[1], o[1]) and np.array_equal(d[3], o[3])             # sample counts exact
    assert (o[3] == 0).any() and (o[3] > 0).any()                                 # frames without a sample keep their input
    assert np.array_equal(d[2][o[3] == 0], fq[o[3] == 0])
    assert np.array_equal(d[0][known == 1], cq[known == 1])
    assert qangle(d[0], o[0]).max() < 1e-12 and qangle(d[2], o[2]).max() < 1e-12
    assert st.num_cam_samples == o[1].sum() and st.num_frames_averaged == (o[3] > 0).sum()
    assert st.num_ref_frames < len(ref)                                           # some frames have no reference image
    d2 = convert_rotations_from_image_to_rig(fr, cam, q, ref, known, cq, fq, image_estimated=est)
    assert all(np.array_equal(a, b) for a, b in zip(d, d2))                       # bit-identical


def test_invalid_arguments_are_rejected():
    from glomap_b200.rotation_initializer import convert_rotations_from_image_to_rig
    fr, cam, q = np.array([0, 0]), np.array([0, 1]), np.tile([0, 0, 0, 1.0], (2, 1))
    ok = dict(frame_ref_camera=[0], camera_known=[1, 0], cam_from_rig=np.tile([0, 0, 0, 1.0], (2, 1)),
              rig_from_world=[[0, 0, 0, 1.0]])
    for bad in (dict(image_frame=[0, 1]), dict(image_frame=[0, -2]), dict(image_camera=[0, 2]),
                dict(frame_ref_camera=[5])):
        a = dict(image_frame=fr, image_camera=cam, cam_from_world=q, **ok)
        a.update(bad)
        with pytest.raises(_lib.B200Error) as e:
            convert_rotations_from_image_to_rig(**a)
        assert e.value.code == 1
    from glomap_b200.estimators import default_context
    lib, h = _lib.load(), default_context().handle
    assert lib.b200sfm_rig_rotations_from_images(h, 2, 1, 2, None, None, None, None, None, None, None, None, None, None, None) == 1
    assert lib.b200sfm_rig_rotations_from_images(h, 0, 1, 2, *([None] * 10), None) == 1


def rig_scene(F=60, seed=5, noise_deg=0.3):
    """F frames of a 4-camera rig (camera 0 the reference, camera 1 known, 2 and 3 unknown); pairs between the images of
    neighbouring frames and inside each frame, cam2_from_cam1 with noise_deg of rotation noise.  Some images missing."""
    rng = np.random.default_rng(seed)
    S = 4
    Rf = G.so3_exp(rng.normal(size=(F, 3)) * 0.3)
    w = rng.normal(size=(S, 3)) * 0.5
    w[0] = 0
    Rs = G.so3_exp(w)
    fr = np.repeat(np.arange(F), S)
    cam = np.tile(np.arange(S), F)
    keep = (cam == 0) | (rng.uniform(size=F * S) < 0.9)
    fr, cam = fr[keep], cam[keep]
    Rimg = np.einsum("nij,njk->nik", Rs[cam], Rf[fr])
    ei, ej = [], []
    for i in range(len(fr)):
        for j in range(i + 1, len(fr)):
            if abs(fr[i] - fr[j]) <= 2 and rng.uniform() < 0.7:
                ei.append(i)
                ej.append(j)
    ei, ej = np.array(ei), np.array(ej)
    noise = G.so3_exp(rng.normal(size=(len(ei), 3)) * np.radians(noise_deg) / np.sqrt(3))
    R_rel = noise @ Rimg[ej] @ np.swapaxes(Rimg[ei], 1, 2)
    vg = ViewGraph(len(fr), ei.astype(np.int32), ej.astype(np.int32), R_rel, rng.integers(30, 300, len(ei)).astype(float), Rimg)
    known = np.array([1, 1, 0, 0], np.uint8)
    cq = np.tile([0, 0, 0, 1.0], (S, 1))
    cq[1] = G.rotmat_to_quat_xyzw_fast(Rs[1:2])[0]
    return vg, fr, cam, known, cq, np.zeros(F, np.int64), Rf, Rs


def test_prepass_matches_the_oracle_chain():
    vg, fr, cam, known, cq, ref, Rf, Rs = rig_scene()
    o = RA.RotationAveragerOptions(pcg_rel_tolerance=1e-12)
    info_d, info_o = {}, {}
    ok, R, Rc, reg = RA.solve_rotation_averaging_rig(vg, fr, cam, known, cq, ref, o, info=info_d)
    ok_o, R_o, Rc_o, reg_o = O.solve_rotation_averaging_rig(vg, fr, cam, known, cq, ref, o, info=info_o)
    assert ok and ok_o and np.array_equal(reg, reg_o) and reg.all()
    assert info_d == info_o and info_d["trivial"][1] > 0
    assert np.abs(R - R_o).max() < 1e-7 and np.abs(Rc - Rc_o).max() < 1e-7
    # against the truth (gauge: the first frame)
    for c in (2, 3):
        M = Rc[c].T @ Rs[c]
        assert np.degrees(np.arccos(np.clip((np.trace(M) - 1) / 2, -1, 1))) < 1.0
    A = R[0].T @ Rf[0]
    err = [np.degrees(np.arccos(np.clip((np.trace((R[f] @ A).T @ Rf[f]) - 1) / 2, -1, 1))) for f in range(len(Rf))]
    assert max(err) < 1.0


def test_skip_initialization_starts_unknown_cameras_at_zero():
    vg, fr, cam, known, cq, ref, Rf, Rs = rig_scene(F=30, seed=6)
    o = RA.RotationAveragerOptions(skip_initialization=True, pcg_rel_tolerance=1e-12)
    info_d, info_o = {}, {}
    ok, R, Rc, reg = RA.solve_rotation_averaging_rig(vg, fr, cam, known, cq, ref, o, info=info_d)
    ok_o, R_o, Rc_o, _ = O.solve_rotation_averaging_rig(vg, fr, cam, known, cq, ref, o, info=info_o)
    assert ok and ok_o and "trivial" not in info_d and info_d == info_o
    assert np.abs(R - R_o).max() < 1e-7 and np.abs(Rc - Rc_o).max() < 1e-7
    assert not RA.solve_rotation_averaging_rig(vg, fr, cam, known, cq, ref, RA.RotationAveragerOptions(use_gravity=True))[0]
