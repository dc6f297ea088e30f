"""The quaternion averages of b200sfm_rig_rotations_from_images (rig_cam_average, rig_frame_average through
rig_warp_average) and their eigen-solver quat_avg_eig (shared with ra_update_cams, run here through
b200sfm_test_device_helpers) against the mpmath restatement of oracle/gravity_mp.py: spreads with lambda2 / lambda1 from
0.1 to 0.99, warp segments of 1 to 64 samples, cam_from_rig rotations near 180 degrees (w ~ 0, where the canonical sign
decides) and samples of either sign and any norm.  The check is the angle to the mpmath eigenvector, within the
eigenvector's conditioning bound c eps / relative gap."""
import ctypes as ct

import numpy as np
import pytest

from glomap_b200 import estimators as E_, _lib
from glomap_b200.rotation_initializer import convert_rotations_from_image_to_rig
from oracle import gravity_mp as GM

pytestmark = pytest.mark.gpu
EPS = float(np.finfo(np.float64).eps)
C_EIG = 64        # the angle bound is C_EIG eps / relative gap
RATIOS = [0.1, 0.5, 0.9, 0.97, 0.99]
SEGMENTS = [1, 31, 32, 33, 64]


def ptr(a):
    return a.ctypes.data_as(ct.c_void_p)


def avg_helper(Ms, q0s):
    rows = np.ascontiguousarray(np.concatenate([Ms, q0s], axis=1), np.float64)
    out = np.full((len(rows), 4), np.nan)
    ctx = E_.default_context()
    _lib.check(ctx.handle, ctx.lib.b200sfm_test_device_helpers(ctx.handle, 4, len(rows), ptr(rows), ptr(out)))
    return out


def packed(qs):
    qs = np.asarray(qs, np.float64)
    qs = qs / np.linalg.norm(qs, axis=1, keepdims=True)
    return np.array([sum(q[a] * q[b] for q in qs) for a in range(4) for b in range(a, 4)])


def spread(rng, n, ratio, center=None):
    """n unit quaternions q = cos(phi) u +- sin(phi) w (+ a small isotropic part) with lambda2 / lambda1 ~ ratio of
    sum q q^T; u a random unit quaternion (or `center`), w orthogonal to it."""
    u = rng.normal(size=4) if center is None else np.asarray(center, np.float64)
    u /= np.linalg.norm(u)
    w = rng.normal(size=4)
    w -= (w @ u) * u
    w /= np.linalg.norm(w)
    phi = np.arctan(np.sqrt(ratio))
    sgn = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    q = np.cos(phi) * u[None] + (sgn * np.sin(phi))[:, None] * w[None] + rng.normal(size=(n, 4)) * 1e-3
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def line_angle(a, b):
    return GM.angle_to(a, b)


@pytest.mark.parametrize("ratio", RATIOS)
def test_eigen_solver_against_mpmath(ratio):
    rng = np.random.default_rng(int(ratio * 1000))
    Ms, q0s, refs = [], [], []
    for n in (2, 3, 7, 32, 200):
        for _ in range(4):
            qs = spread(rng, n, ratio) * rng.choice([-1.0, 1.0], size=(n, 1))
            Ms.append(packed(qs))
            q0s.append(qs[0])
    out = avg_helper(np.array(Ms), np.array(q0s))
    worst = 0.0
    for M, q0, v in zip(Ms, q0s, out):
        S = np.zeros((4, 4))
        S[np.triu_indices(4)] = M
        S = S + np.triu(S, 1).T
        e, gap = GM.dominant(S)
        err = line_angle(v, e)
        worst = max(worst, err * float(gap) / EPS)
        assert err <= C_EIG * EPS / float(gap), (ratio, err, float(gap))
        assert v @ q0 >= 0 and abs(np.linalg.norm(v) - 1) <= 8 * EPS      # the sign follows q0
    print(f"ratio {ratio}: worst {worst:.2f} eps / gap")


def rig_case(rng, counts, ratio, center_of=None, w_of=None):
    """Camera 0 the reference of every frame (q_ref random, any sign and norm), camera c = 1..len(counts) present in the
    first counts[c-1] frames; the cam samples of camera c spread with `ratio` about a random centre (or center_of[c])."""
    F, K = max(counts), len(counts) + 1
    fr, cam, q = [], [], []
    qref = rng.normal(size=(F, 4))
    samples = {}
    for c, n in enumerate(counts, start=1):
        centre = None if center_of is None else center_of.get(c)
        samples[c] = spread(rng, n, ratio, centre) if n > 1 or centre is None else np.asarray([centre], np.float64)
    for f in range(F):
        fr.append(f); cam.append(0); q.append(qref[f])
        for c, n in enumerate(counts, start=1):
            if f < n:
                s = samples[c][f]
                qi = np.array([float(t) for t in GM.qmul(GM.qunit(s), GM.qunit(qref[f]))])   # s (x) q_ref
                fr.append(f); cam.append(c); q.append(qi)
    q = np.array(q) * rng.choice([-1.0, 1.0], size=(len(q), 1)) * rng.uniform(0.25, 4.0, size=(len(q), 1))
    known = np.zeros(K, np.uint8); known[0] = 1
    cq = np.tile([0, 0, 0, 1.0], (K, 1))
    return np.array(fr), np.array(cam), q, np.zeros(F, np.int64), known, cq, np.tile([0, 0, 0, 1.0], (F, 1))


def check_public(fr, cam, q, ref, known, cq, fq):
    d = convert_rotations_from_image_to_rig(fr, cam, q, ref, known, cq, fq)
    cam_q, cam_n, frame_q, frame_n = d
    worst = 0.0
    for c in range(1, len(known)):
        idx = [(i, int(np.nonzero((fr == fr[i]) & (cam == 0))[0][0])) for i in np.nonzero(cam == c)[0]]
        s = [GM.cam_sample(q[i], q[r]) for i, r in idx]
        v, gap = GM.average_quaternions(s)
        assert cam_n[c] == len(s)
        err = line_angle(cam_q[c], v)
        worst = max(worst, err * float(gap) / EPS)
        assert err <= C_EIG * EPS / float(gap), (c, len(s), err, float(gap))
        assert cam_q[c][3] >= 0
        if abs(float(v[3])) > C_EIG * EPS / float(gap):   # the canonical sign is decided: it must be the reference's
            assert cam_q[c] @ np.array([float(t) for t in v]) > 0
    # the frame pass, from the device's camera averages
    for f in range(len(fq)):
        imgs = np.nonzero(fr == f)[0]
        s = []
        for i in imgs:
            if cam[i] == 0:
                s.append(GM.qunit(q[i]))
            else:
                qc = GM.qunit(cam_q[cam[i]])
                s.append(GM.qunit(GM.qmul([-qc[0], -qc[1], -qc[2], qc[3]], GM.qunit(q[i]))))
        v, gap = GM.average_quaternions(s)
        assert frame_n[f] == len(s)
        err = line_angle(frame_q[f], v)
        assert err <= C_EIG * EPS / float(gap), (f, err, float(gap))
        assert frame_q[f][3] >= 0
    d2 = convert_rotations_from_image_to_rig(fr, cam, q, ref, known, cq, fq)
    assert all(np.array_equal(a, b) for a, b in zip(d, d2))                     # bit-identical
    return worst


@pytest.mark.parametrize("ratio", RATIOS)
def test_camera_averages_through_the_public_entry(ratio):
    rng = np.random.default_rng(int(ratio * 100) + 7)
    worst = check_public(*rig_case(rng, SEGMENTS, ratio))
    print(f"ratio {ratio}: worst {worst:.2f} eps / gap")


@pytest.mark.parametrize("w", [1e-17, -1e-17, 0.0])
def test_rear_camera_at_180_degrees(w):
    """A front/back rig: the rear camera's cam_from_rig is a half turn, w ~ 0.  One sample is returned as it is, with
    the canonical sign w >= 0 (w < 0 flips, w == 0 does not); several samples about it are averaged."""
    rng = np.random.default_rng(11)
    axis = np.array([0.0, 1.0, 0.0])
    centre = np.concatenate([axis, [w]])
    fr = np.array([0, 0])
    cam = np.array([0, 1])
    q = np.array([[0, 0, 0, 1.0], centre])
    known = np.array([1, 0], np.uint8)
    cq, cn, fq, fn = convert_rotations_from_image_to_rig(fr, cam, q, np.zeros(1, np.int64), known,
                                                         np.tile([0, 0, 0, 1.0], (2, 1)), np.tile([0, 0, 0, 1.0], (1, 1)))
    want = centre if w >= 0 else -centre
    assert cn[1] == 1 and cq[1].tobytes() == want.tobytes(), (cq[1], want)
    # several noisy samples about the half turn, with either sign and any norm
    for n in (2, 33, 64):
        check_public(*rig_case(rng, [n], 0.02, center_of={1: centre}))


def test_segments_through_the_helper_and_the_entry_agree():
    """The same samples through the public entry (one warp, lane-strided sums) and through quat_avg_eig on their packed
    sum: equal to the conditioning bound; the entry's canonical sign applied to the helper's result."""
    rng = np.random.default_rng(3)
    fr, cam, q, ref, known, cq, fq = rig_case(rng, SEGMENTS, 0.9)
    d = convert_rotations_from_image_to_rig(fr, cam, q, ref, known, cq, fq)
    for c, n in enumerate(SEGMENTS, start=1):
        if n == 1:
            continue
        idx = [(i, int(np.nonzero((fr == fr[i]) & (cam == 0))[0][0])) for i in np.nonzero(cam == c)[0]]
        s = np.array([[float(t) for t in GM.cam_sample(q[i], q[r])] for i, r in idx])
        v = avg_helper(packed(s)[None], s[:1])[0]
        v = -v if v[3] < 0 else v
        _, gap = GM.average_quaternions(s)
        assert line_angle(v, d[0][c]) <= 2 * C_EIG * EPS / float(gap)
