"""Host restatement of ImagePairsInlierCount (glomap_b200/image_pair_inliers.py) against a literal per-match scalar
transcription of ImagePairInliers::ScoreErrorEssential / Fundamental / Homography (glomap/processors/
image_pair_inliers.cc:20-198, math/two_view_geometry.cc:5-93), the RelPoseFilter inlier filters, the null-argument check of
the C entry point and the C++ shim over the recording test double.  No GPU."""
import math
import os
import subprocess

import numpy as np

from glomap_b200 import geometry as G, image_pair_inliers as IP, synthetic as S
from glomap_b200.mapper import InlierThresholdOptions
from glomap_b200.track_establishment import ImagePairMatches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 1e-12


# ---- the scalar transcription -------------------------------------------------------------------------------------------
def _matvec(M, x):
    return [M[i][0] * x[0] + M[i][1] * x[1] + M[i][2] * x[2] for i in range(3)]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def ref_score(pair, features, bearings, cameras, o):
    """(inliers, score) of one valid pair, statement by statement as the reference."""
    M = [[float(v) for v in row] for row in np.asarray(pair.matches).reshape(-1, 2)]
    inliers, score = [], 0.0
    c = pair.config
    if c in (4, 5, 6):
        H = np.asarray(pair.H, float).tolist()
        sq = o.max_epipolar_error_H * o.max_epipolar_error_H
        for k, (a, b) in enumerate(M):
            p1, p2 = features[pair.image_id1][int(a)], features[pair.image_id2][int(b)]
            h = _matvec(H, [p1[0], p1[1], 1.0])
            dx, dy = h[0] / (EPS + h[2]) - p2[0], h[1] / (EPS + h[2]) - p2[1]
            r2 = dx * dx + dy * dy
            if r2 < sq:
                score += r2
                inliers.append(k)
            else:
                score += sq
        return inliers, score
    if c == 3:
        F = np.asarray(pair.F, float).tolist()
        ep = list(np.cross(F[0], F[2]))
        if not any(e > EPS or e < -EPS for e in ep):
            ep = list(np.cross(F[1], F[2]))
        sq = o.max_epipolar_error_F * o.max_epipolar_error_F
        signums, pre, errors, npos, nneg = [], [], [], 0, 0
        for k, (a, b) in enumerate(M):
            p1, p2 = features[pair.image_id1][int(a)], features[pair.image_id2][int(b)]
            Fx1 = _matvec(F, [p1[0], p1[1], 1.0])
            Ftx2 = _matvec([[F[0][i], F[1][i], F[2][i]] for i in range(3)], [p2[0], p2[1], 1.0])
            C = Fx1[0] * p2[0] + Fx1[1] * p2[1] + Fx1[2]
            r2 = C * C / ((Fx1[0] * Fx1[0] + Fx1[1] * Fx1[1]) + (Ftx2[0] * Ftx2[0] + Ftx2[1] * Ftx2[1]))
            if r2 < sq:
                signums.append((F[0][0] * p2[0] + F[1][0] * p2[1] + F[2][0]) * (ep[1] - ep[2] * p1[1]))
                if signums[-1] > 0:
                    npos += 1
                else:
                    nneg += 1
                pre.append(k)
                errors.append(r2)
            else:
                score += sq
        if npos == nneg:
            return [], 0.0
        for k in range(len(pre)):
            if (signums[k] > 0) == (npos > nneg):
                inliers.append(pre[k])
                score += errors[k]
            else:
                score += sq
        return inliers, score
    if c == 2:
        R = G.quat_xyzw_to_rotmat(np.asarray(pair.quat_xyzw, float)).tolist()
        Rt = [[R[j][i] for j in range(3)] for i in range(3)]
        t = [float(v) for v in pair.trans]
        tx = [[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]]
        E = [[tx[i][0] * R[0][j] + tx[i][1] * R[1][j] + tx[i][2] * R[2][j] for j in range(3)] for i in range(3)]
        Et = [[E[j][i] for j in range(3)] for i in range(3)]
        e12 = list(t)
        e21 = [-(R[0][i] * t[0] + R[1][i] * t[1] + R[2][i] * t[2]) for i in range(3)]
        if e12[2] < 0:
            e12 = [-v for v in e12]
        if e21[2] < 0:
            e21 = [-v for v in e21]
        thr = o.max_epipolar_error_E * 0.5 * (1. / cameras[pair.image_id1].focal() + 1. / cameras[pair.image_id2].focal())
        sq = thr * thr
        thres_epipole = math.cos(3.0 * 0.0174532925199432954743716805978692718953) + 1e-6
        for k, (a, b) in enumerate(M):
            x1, x2 = bearings[pair.image_id1][int(a)].tolist(), bearings[pair.image_id2][int(b)].tolist()
            Ex1 = [v / (EPS + x1[2]) for v in _matvec(E, x1)]
            Etx2 = [v / (EPS + x2[2]) for v in _matvec(Et, x2)]
            C = _dot(Ex1, x2)
            r2 = C * C / ((Ex1[0] * Ex1[0] + Ex1[1] * Ex1[1]) + (Etx2[0] * Etx2[0] + Etx2[1] * Etx2[1]))
            if r2 < sq:
                Rx1 = _matvec(R, x1)
                av = -_dot(Rx1, x2)
                b1 = -_dot(Rx1, t)
                b2 = _dot(x2, t)
                l1, l2 = b1 - av * b2, -av * b1 + b2
                mind, maxd = 1e-2 * (1 - av * av), 100. * (1 - av * av)
                cheir = l1 > mind and l2 > mind and l1 < maxd and l2 < maxd
                ok = _dot(x1, _matvec(Rt, x2)) < 1 + 1e-6
                ok = ok and _dot(x1, e21) < thres_epipole and _dot(x2, e12) < thres_epipole
                if cheir and ok:
                    score += r2
                    inliers.append(k)
                else:
                    score += sq
            else:
                score += sq
        return inliers, score
    return [], 0.0


def _bearings(features, cameras):
    return {i: S.bearings_from_pixels(cameras[i].model, np.asarray(cameras[i].params, float), np.asarray(features[i], float))
            for i in features}


def _check_against_transcription(pairs, features, cameras, o, clean_inliers=True):
    old = [np.asarray(p.inliers).copy() for p in pairs]
    valid = [p.is_valid for p in pairs]
    res = IP.image_pairs_inlier_count(pairs, features, cameras, o, clean_inliers)
    bear = _bearings(features, cameras)
    for k, p in enumerate(pairs):
        if not clean_inliers and len(old[k]) > 0:
            assert np.array_equal(p.inliers, old[k]) and not res.scored[k]
            continue
        if not valid[k]:
            assert len(p.inliers) == 0 and not res.scored[k]
            continue
        want_inl, want_score = ref_score(p, features, bear, cameras, o)
        assert p.inliers.tolist() == want_inl, k
        assert res.scores[k] == want_score, (k, res.scores[k], want_score)
        assert p.inliers is res.inliers[k]
    return res


# ---- scenes -------------------------------------------------------------------------------------------------------------
def _two_view_world(rng, n, cam1, cam2, behind=0, far=0, near_epipole=0):
    """Two cameras with a known cam2_from_cam1 (unit baseline) and n points: in front, some behind camera 1 or 2, some
    beyond depth 100 baselines, some within 3 degrees of the epipoles.  Returns (features {1, 2}, pose)."""
    R = G.so3_exp(np.array([[0.05, -0.2, 0.03]]))[0]
    c2 = np.array([0.8, 0.1, 0.2])
    c2 /= np.linalg.norm(c2)                                   # centre of camera 2 in camera 1
    t = -R @ c2
    X = np.column_stack([rng.uniform(-3, 3, n), rng.uniform(-3, 3, n), rng.uniform(4, 12, n)])
    k = 0
    X[k:k + behind // 2] *= -1                                  # behind camera 1 (and 2)
    X[k + behind // 2:k + behind, 2] = rng.uniform(0.02, 0.2, behind - behind // 2)   # in front of camera 1, behind camera 2
    k += behind
    X[k:k + far, 2] += 300.0; k += far                          # beyond max_depth
    for s in np.linspace(2.0, 6.0, near_epipole):               # close to the baseline, on the far side of camera 2
        X[k] = c2 * s + rng.normal(scale=0.02, size=3); k += 1
    X2 = X @ R.T + t
    proj = lambda cam, Y: S.project(cam.model, np.asarray(cam.params, float), Y)   # noqa: E731
    return {1: proj(cam1, X), 2: proj(cam2, X2)}, G.rotmat_to_quat_xyzw(R[None])[0], t


def test_essential_against_transcription_cheirality_epipoles_and_mean_focal():
    rng = np.random.default_rng(3)
    cam1 = IP.Camera(S.PINHOLE, np.array([700.0, 760.0, 320.0, 240.0]))     # fx != fy: the threshold uses the mean focal
    cam2 = IP.Camera(S.SIMPLE_RADIAL, np.array([650.0, 320.0, 240.0, 0.01]))
    features, q, t = _two_view_world(rng, 400, cam1, cam2, behind=30, far=30, near_epipole=20)
    features = {i: f + rng.normal(scale=0.3, size=f.shape) for i, f in features.items()}
    cameras = {1: cam1, 2: cam2}
    m = np.stack([np.arange(400), np.arange(400)], 1)
    m = np.concatenate([m, rng.integers(0, 400, (60, 2))])              # outliers
    pair = ImagePairMatches(1, 2, m, np.zeros(0, np.int64), config=IP.TWO_VIEW_CALIBRATED, quat_xyzw=q, trans=t)
    o = InlierThresholdOptions()
    _check_against_transcription([pair], features, cameras, o)
    d = IP.score_image_pair(pair, features, cameras, o)
    pre = d["r2"] < d["thr2"]
    cheir = (d["lambda1"] > d["min_depth"]) & (d["lambda2"] > d["min_depth"]) & (d["lambda1"] < d["max_depth"]) & \
            (d["lambda2"] < d["max_depth"])
    # every rejection reason occurs among the matches that pass the Sampson test
    assert (pre & ~cheir)[:30].sum() > 10                      # behind the cameras
    assert (pre & ~cheir)[30:60].sum() > 10                    # beyond depth 100
    near = (d["diff_epipole1"] >= IP.COS_EPIPOLE_THR) | (d["diff_epipole2"] >= IP.COS_EPIPOLE_THR)
    assert (pre & near)[60:80].sum() > 5
    assert d["thr2"] == (0.5 * (1 / 730.0 + 1 / 650.0)) ** 2
    assert 0 < len(pair.inliers) < 400


def _fundamental_pair(rng, n=300):
    cam = IP.Camera(S.SIMPLE_PINHOLE, np.array([600.0, 320.0, 240.0]))
    features, q, t = _two_view_world(rng, n, cam, cam, behind=n // 3)
    R = G.quat_xyzw_to_rotmat(q[None])[0]
    K = np.array([[600.0, 0, 320], [0, 600, 240], [0, 0, 1]])
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = np.linalg.inv(K).T @ tx @ R @ np.linalg.inv(K)
    m = np.stack([np.arange(n), np.arange(n)], 1)
    return features, {1: cam, 2: cam}, F / np.linalg.norm(F), m


def test_fundamental_against_transcription_majority_tie_and_epipole_fallback():
    rng = np.random.default_rng(4)
    features, cameras, F, m = _fundamental_pair(rng)
    o = InlierThresholdOptions()
    pair = ImagePairMatches(1, 2, np.concatenate([m, rng.integers(0, 300, (50, 2))]), np.zeros(0, np.int64),
                            config=IP.TWO_VIEW_UNCALIBRATED, F=F)
    _check_against_transcription([pair], features, cameras, o)
    d = IP.score_image_pair(pair, features, cameras, o)
    pre = d["r2"] < d["thr2"]
    pos, neg = np.flatnonzero(pre & (d["signum"] > 0)), np.flatnonzero(pre & ~(d["signum"] > 0))
    assert len(pos) > 20 and len(neg) > 20 and 0 < len(pair.inliers) < pre.sum()
    # equal signum counts: no inliers, score 0
    k = min(len(pos), len(neg))
    tie = ImagePairMatches(1, 2, pair.matches[np.concatenate([pos[:k], neg[:k], np.flatnonzero(~pre)[:7]])],
                           np.zeros(0, np.int64), config=IP.TWO_VIEW_UNCALIBRATED, F=F)
    res = _check_against_transcription([tie], features, cameras, o)
    assert len(tie.inliers) == 0 and res.scores[0] == 0.0 and res.scored[0]
    # rows 0 and 2 parallel: the epipole falls back to row 1 x row 2, which orients the matches both ways
    Fp = F.copy()
    Fp[2] = 3.0 * Fp[0]
    assert (np.abs(np.cross(Fp[0], Fp[2])) <= 1e-12).all()
    par = ImagePairMatches(1, 2, pair.matches, np.zeros(0, np.int64), config=IP.TWO_VIEW_UNCALIBRATED, F=Fp,
                           quat_xyzw=np.array([0.0, 0, 0, 1]))
    o_wide = InlierThresholdOptions(max_epipolar_error_F=1e4)
    _check_against_transcription([par], features, cameras, o_wide)
    d = IP.score_image_pair(par, features, cameras, o_wide)
    s = d["signum"][d["r2"] < d["thr2"]]
    assert (s > 0).any() and (s < 0).any()


def test_homography_both_sides_of_the_threshold_and_other_configs():
    rng = np.random.default_rng(5)
    H = np.array([[1.02, 0.01, 5.0], [-0.02, 0.99, -3.0], [1e-5, 2e-5, 1.0]])
    x1 = rng.uniform(0, 640, (200, 2))
    h = np.column_stack([x1, np.ones(200)]) @ H.T
    x2 = h[:, :2] / h[:, 2:]
    ang = rng.uniform(0, 2 * np.pi, 200)
    dist = np.where(np.arange(200) % 2 == 0, 3.99, 4.01)         # just inside / just outside 4 px
    x2 = x2 + np.column_stack([np.cos(ang), np.sin(ang)]) * dist[:, None]
    features = {1: x1, 2: x2}
    cam = IP.Camera(S.SIMPLE_PINHOLE, np.array([500.0, 320, 240]))
    m = np.stack([np.arange(200), np.arange(200)], 1)
    pairs = [ImagePairMatches(1, 2, m, np.zeros(0, np.int64), config=c, H=H) for c in (4, 5, 6)]
    pairs += [ImagePairMatches(1, 2, m, np.arange(3), config=c, H=H, F=np.eye(3)) for c in (0, 1, 7, 8)]
    res = _check_against_transcription(pairs, features, {1: cam, 2: cam}, InlierThresholdOptions())
    for p in pairs[:3]:
        assert p.inliers.tolist() == list(range(0, 200, 2))
    for k, p in enumerate(pairs[3:], 3):
        assert len(p.inliers) == 0 and res.scores[k] == 0.0


def test_invalid_pairs_and_clean_inliers_false():
    sc = S.make_scene(12, 600, mean_track_len=5, seed=8, model=S.RADIAL, pixel_sigma=0.3)
    features, cameras, pairs = S.pairs_from_match_arrays(S.make_pair_matches(sc, seed=2))
    assert {p.config for p in pairs} == {2, 3, 4}
    pairs[0].is_valid = False
    pairs[0].inliers = np.array([1, 2])
    pairs[1].inliers = np.array([0, 5])                         # kept under clean_inliers = False
    pairs[2].is_valid = False
    o = InlierThresholdOptions(max_epipolar_error_H=40.0)
    res = _check_against_transcription(pairs, features, cameras, o, clean_inliers=False)
    assert pairs[0].inliers.tolist() == [1, 2] and pairs[1].inliers.tolist() == [0, 5] and len(pairs[2].inliers) == 0
    assert res.scored.sum() == len(pairs) - 3
    _check_against_transcription(pairs, features, cameras, o, clean_inliers=True)
    assert len(pairs[0].inliers) == 0 and len(pairs[1].inliers) > 0


def test_noise_free_calibrated_pairs_keep_every_true_match_outside_the_epipole_cones():
    sc = S.make_scene(20, 2000, mean_track_len=6, seed=9, model=S.PINHOLE)
    d = S.make_pair_matches(sc, seed=4, outlier_frac=0.0, config_weights=(1, 0, 0))
    features, cameras, pairs = S.pairs_from_match_arrays(d)
    IP.image_pairs_inlier_count(pairs, features, cameras)
    R = G.quat_xyzw_to_rotmat(sc.quat)
    centres = G.centers_from_pose(R, sc.trans)
    bear = _bearings(features, cameras)
    cos3 = math.cos(math.radians(3.0))
    n_cone = 0
    for p in pairs:
        i, j = p.image_id1, p.image_id2
        e21 = R[i] @ (centres[j] - centres[i]); e21 /= np.linalg.norm(e21)     # camera j seen from camera i
        e12 = R[j] @ (centres[i] - centres[j]); e12 /= np.linalg.norm(e12)
        b1, b2 = bear[i][p.matches[:, 0]], bear[j][p.matches[:, 1]]
        cone = (np.abs(b1 @ e21) > cos3 - 1e-6) | (np.abs(b2 @ e12) > cos3 - 1e-6)
        n_cone += cone.sum()
        assert set(np.flatnonzero(~cone)) <= set(p.inliers.tolist())
        assert set(p.inliers.tolist()) <= set(np.flatnonzero(~cone | (np.abs(b1 @ e21) < cos3 + 1e-6)))
    assert sum(len(p.inliers) for p in pairs) > 0.9 * len(d["matches"])


def test_filters_thresholds_and_zero_match_pair():
    mk = lambda n_m, n_i, valid=True: ImagePairMatches(1, 2, np.zeros((n_m, 2), np.int64), np.arange(n_i), valid)   # noqa: E731
    pairs = [mk(100, 30), mk(100, 29), mk(100, 25), mk(100, 24), mk(0, 0), mk(10, 0, False)]
    assert IP.filter_inlier_num(pairs, 30.0) == 4 and [p.is_valid for p in pairs] == [True, False, False, False, False, False]
    pairs = [mk(100, 30), mk(100, 25), mk(100, 24), mk(0, 0)]
    assert IP.filter_inlier_ratio(pairs, 0.25) == 1 and [p.is_valid for p in pairs] == [True, True, False, True]
    # the reference compares size() against an int: a negative minimum becomes a huge unsigned value
    pairs = [mk(100, 30)]
    assert IP.filter_inlier_num(pairs, -1) == 1
    o = InlierThresholdOptions()
    assert (o.max_epipolar_error_E, o.max_epipolar_error_F, o.max_epipolar_error_H, o.min_inlier_num, o.min_inlier_ratio) == \
        (1.0, 4.0, 4.0, 30, 0.25)


def test_abi_entry_rejects_a_null_context_without_a_device():
    from glomap_b200 import _lib
    lib = _lib.load()
    assert lib.b200sfm_image_pairs_inlier_count(None, 1, *([None] * 3), 1, None, None, 1, *([None] * 9), 1.0, 4.0, 4.0,
                                                *([None] * 3)) == 1
    assert lib.b200sfm_image_pairs_inlier_count(None, 0, *([None] * 3), 0, None, None, 0, *([None] * 9), 1.0, 4.0, 4.0,
                                                *([None] * 3)) == 1


def test_shim_flattens_in_sorted_id_order_and_writes_inliers_back(tmp_path):
    lib, exe, dump = tmp_path / "libb200sfm_mock.so", tmp_path / "inlier_driver", tmp_path / "dump.txt"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c"),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_image_pair_inliers.c")], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "shim_mock", "inlier_driver.cc"), str(lib), "-Wl,-rpath," + str(tmp_path)],
                   check=True, capture_output=True)
    r = subprocess.run([str(exe)], env=dict(os.environ, MOCK_DUMP=str(dump)), capture_output=True, text=True)
    assert r.returncode == 0 and "inlier driver ok" in r.stdout, (r.stdout, r.stderr)
    calls = []
    for line in dump.read_text().splitlines():
        f = line.split()
        if f[0] == "call":
            calls.append({"_name": f[1]})
        else:
            calls[-1][f[0]] = np.array([float(x) for x in f[2:]])
    # the clean_inliers = false call scores nothing (both valid pairs keep old inliers) and does not reach the device
    assert [c["_name"] for c in calls] == ["image_pairs_inlier_count"]
    c = calls[0]
    assert c["dims"].tolist() == [3, 2, 2, 8] and c["thresholds"].tolist() == [2.0, 4.0, 4.0]
    # images 10, 20, 30 (sorted) with 2, 3, 4 features; cameras 3, 7 (sorted) -> blocks 0, 1
    assert c["feature_begin"].tolist() == [0, 2, 5, 9] and c["image_intr"].tolist() == [0, 1, 0]
    want_xy = [[1.0 * i + f, 2.0 * i - f] for i in (10, 20, 30) for f in range(i // 10 + 1)]
    assert c["features"].reshape(-1, 2).tolist() == want_xy
    assert c["intr_model"].tolist() == [0, 1]
    assert c["intr"].reshape(2, 12)[:, :4].tolist() == [[600.0, 300.0, 200.0, 0.0], [500.0, 510.0, 320.0, 240.0]]
    # pairs in ascending pair id: (10,20) then (30,10) [id of (10,30)]; (20,30) is invalid
    assert c["image1"].tolist() == [0, 2] and c["image2"].tolist() == [1, 0] and c["config"].tolist() == [2, 3]
    assert c["match_begin"].tolist() == [0, 5, 8]
    assert c["matches"].reshape(-1, 2).tolist() == [[k % 2, (k + 1) % 2] for k in range(5)] + [[k % 2, (k + 1) % 2] for k in range(3)]
    assert np.allclose(c["quat"].reshape(2, 4)[1], [0.1 * (30 + k) + 0.01 * 10 for k in range(4)], rtol=0, atol=1e-15)
    assert c["trans"].reshape(2, 3).tolist() == [[10.0, 20.0, -1.0], [30.0, 10.0, -1.0]]
    assert c["F"].reshape(2, 9)[1].tolist() == [30 + 0.5 * k for k in range(9)]
    assert c["H"].reshape(2, 9)[0].tolist() == [20 - 0.25 * k for k in range(9)]
    # the mock marks rows k % 3 != 1 of the call: (10,20) rows 0..4 -> 0 2 3; (30,10) rows 5..7 -> 5 6 -> local 0 1
    lines = r.stdout.splitlines()
    assert lines[:3] == ["inliers 10 20 0 2 3", "inliers 30 10 0 1", "inliers 20 30"]
    assert lines[3:7] == ["valid 0", "valid 0", "valid 0", "valid 1"]    # (10,20) 3/5 < 0.65, (30,10) 2 < 3, 0/0 stays valid


def test_shim_image_pair_functions_typecheck_against_the_glomap_api():
    """Inside a glomap build the shim's ImagePairsInlierCount / RelPoseFilter take glomap's ImagePair (config, F, H,
    Eigen::MatrixXi matches, std::vector<int> inliers) and glomap::InlierThresholdOptions: instantiated against a stub with
    those members and their real types (tests/shim_mock/glomap_stub_pairs)."""
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-DB200SFM_WITH_GLOMAP",
                        "-I" + os.path.join(ROOT, "tests", "shim_mock", "glomap_stub_pairs"),
                        "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-I" + os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "shim_mock", "inlier_typecheck.cc")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def test_a_library_override_without_the_entry_loads_and_the_entry_raises_when_called(tmp_path):
    """A library named by B200SFM_LIB may implement part of the ABI (here the estimator test double, which has no
    image-pair entry): it loads, and the missing entry raises when it is called instead of returning garbage."""
    import sys
    lib = tmp_path / "libb200sfm_mock.so"
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-O1", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", str(lib),
                    os.path.join(ROOT, "tests", "shim_mock", "mock_b200sfm.c")], check=True, capture_output=True)
    script = ("from glomap_b200 import _lib\n"
              "lib = _lib.load()\n"
              "assert lib.b200sfm_version() == 100\n"
              "try:\n"
              "    lib.b200sfm_image_pairs_inlier_count(None)\n"
              "except RuntimeError as e:\n"
              "    print('raised', e)\n")
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, B200SFM_LIB=str(lib), PYTHONPATH=ROOT),
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "raised b200sfm_image_pairs_inlier_count is not exported" in r.stdout
