"""The references of the track filters, the undistortion and the normalisation, checked without a GPU.

* ``oracle/filter_oracle.py`` against a loop-and-dict restatement of glomap/processors/track_filter.cc (images, cameras
  and tracks as dicts, one observation at a time, in plain FP64) on image scenes and multi-rig scenes, after checking
  that no decision lies within rounding of its bound; its long-double decision quantities against mpmath.
* ``filter_oracle.undistort_exact`` by round trip and against ``mpmath.findroot``, ``fold_radius`` against the
  derivative, and the production host undistortion (``synthetic.bearings_from_pixels``) against it up to the fold.
* ``processors.normalize_reconstruction`` against a restatement of reconstruction_normalizer.cc over the registered
  images for 1-5 images, duplicate centres and multi-rig tables.

The scene builders here are shared with tests/test_filters_gpu.py."""
import math

import mpmath
import numpy as np
import pytest

from glomap_b200 import geometry as G, mapper as M, processors as PR, synthetic as S
from oracle import filter_oracle as FO

FP64_BOUND = 1e-12          # relative margin every compared decision must clear (FP64 evaluation error is ~1e-15)
# the mapper's thresholds (angle, normalised reprojection 1e-2 x {1, 2, 3, 10}, triangulation, pixel reprojection), plus a
# triangulation angle that removes tracks of these wide-baseline scenes
MAPPER_FILTERS = [("angle", 1.0), ("normalized", 1e-2), ("normalized", 2e-2), ("normalized", 3e-2), ("normalized", 1e-1),
                  ("triangulation", 1.0), ("triangulation", 25.0), ("reprojection", 1.0), ("reprojection", 3.0),
                  ("reprojection", 12.0)]
RADIAL_CASES = [(S.SIMPLE_RADIAL, -0.2, 0.0), (S.SIMPLE_RADIAL, -0.25, 0.0), (S.SIMPLE_RADIAL, 0.3, 0.0),
                (S.SIMPLE_RADIAL, 0.02, 0.0), (S.RADIAL, 0.02, -0.005), (S.RADIAL, -0.3, 0.05), (S.RADIAL, -0.1, -0.02)]


# ---- scene builders ----------------------------------------------------------------------------------------------------
def _params(model, f, c, k1=0.0, k2=0.0):
    p = np.zeros(S.INTR_STRIDE)
    p[:S.MODEL_NUM_PARAMS[model]] = {S.SIMPLE_PINHOLE: [f, c, c], S.PINHOLE: [f, 1.01 * f, c, c],
                                     S.SIMPLE_RADIAL: [f, c, c, k1], S.RADIAL: [f, c, c, k1, k2]}[model]
    return p


def _spoil(sc, rng, outlier_frac=0.05, behind=40):
    """5 % outlier pixels (30 px), ``behind`` points moved far behind most cameras, unit quaternions."""
    bad = rng.uniform(size=sc.N) < outlier_frac
    sc.obs_xy[bad] += rng.normal(scale=30.0, size=(int(bad.sum()), 2))
    sc.points[:behind] *= -40.0
    sc.quat = sc.quat / np.linalg.norm(sc.quat, axis=1, keepdims=True)
    if hasattr(sc, "sensor_quat"):
        sc.sensor_quat = sc.sensor_quat / np.linalg.norm(sc.sensor_quat, axis=1, keepdims=True)
    return sc


def image_scene(C=40, P=1500, seed=51):
    """Trivial frames, one intrinsics block per image cycling through the four models, 0.5 px noise, 5 % outliers,
    points behind cameras; calibrated flags: every third image uncalibrated."""
    sc = S.make_scene(C, P, mean_track_len=6, seed=seed, num_intrinsics=C)
    rng = np.random.default_rng([seed, 9])
    sc.intr_model = (np.arange(C) % 4).astype(np.int32)
    k1 = rng.uniform(-0.08, 0.08, C)
    sc.intr_params = np.stack([_params(int(m), 1000.0 * (1 + 0.1 * np.sin(1.7 * k)), 500.0, k1[k], 0.3 * k1[k] ** 2)
                               for k, m in enumerate(sc.intr_model)])
    pt = np.repeat(np.arange(sc.P), np.diff(sc.pt_obs_begin))
    Xc = np.einsum("nij,nj->ni", G.quat_xyzw_to_rotmat(sc.quat)[sc.obs_cam], sc.points[pt]) + sc.trans[sc.obs_cam]
    for k in range(C):
        m = sc.obs_cam == k
        sc.obs_xy[m] = S.project(int(sc.intr_model[k]), sc.intr_params[k], Xc[m])
    sc.obs_xy += rng.normal(scale=0.5, size=sc.obs_xy.shape)
    return _spoil(sc, rng), (np.arange(C) % 3 != 0).astype(np.uint8)


def rig_dataset_scene(seed=3, points=300):
    """``make_rig_dataset``: 3 rigs of 2 cameras, 6 frames each (18 frames, 6 sensors, 36 of the 108 frame-sensor
    combinations are images), RADIAL intrinsics per sensor, 0.5 px noise, 5 % outliers, points behind cameras; mixed
    per-sensor calibrated flags."""
    sc = S.make_rig_dataset(3, 2, 6, points, seed=seed, model=S.RADIAL, pixel_sigma=0.5).scene
    return _spoil(sc, np.random.default_rng([seed, 9]), behind=10), np.array([1, 0, 1, 1, 0, 1], np.uint8)


def missing_sensor_rig_scene(seed=63, drop=((2, 1), (5, 1), (9, 2), (10, 0))):
    """A dense rig scene (12 frames of 3 sensors, SIMPLE_RADIAL) where the frames of ``drop`` lack that sensor's image:
    the image table and the observations lose them."""
    sc = S.make_rig_scene(12, 3, 600, mean_track_len=6, seed=seed, pixel_sigma=0.5, model=S.SIMPLE_RADIAL)
    gone = np.zeros(sc.N, bool)
    keep_img = np.ones(sc.I, bool)
    for f, s in drop:
        gone |= (sc.obs_frame == f) & (sc.obs_sensor == s)
        keep_img &= ~((sc.image_frame == f) & (sc.image_sensor == s))
    sc = M.compact_observations(sc, ~gone)
    sc.image_frame, sc.image_sensor = sc.image_frame[keep_img], sc.image_sensor[keep_img]
    return _spoil(sc, np.random.default_rng([seed, 9]), behind=20), np.array([0, 1, 1], np.uint8)


def bearings(sc):
    return PR.undistort_images(sc)


# ---- loop-and-dict restatement of track_filter.cc --------------------------------------------------------------------
def _world(sc, calibrated):
    """images {image_id: (R, t, camera_id)}, cameras {camera_id: (model, params, has_prior_focal_length)},
    tracks {track_id: [(image_id, feature_id)]}, features {(image_id, feature_id): xy}, xyz {track_id: X}."""
    if hasattr(sc, "obs_sensor"):
        R, t = sc.image_poses()
        images = {i: (R[i], t[i], int(sc.image_sensor[i])) for i in range(sc.I)}
        cam_intr, obs_img = sc.sensor_intr, sc.obs_image()
    else:
        R = G.quat_xyzw_to_rotmat(sc.quat)
        images = {i: (R[i], sc.trans[i], i) for i in range(sc.C)}
        cam_intr, obs_img = sc.cam_intr, sc.obs_cam
    cameras = {c: (int(sc.intr_model[k]), sc.intr_params[k], True if calibrated is None else bool(calibrated[c]))
               for c, k in enumerate(cam_intr)}
    tracks, features, xyz = {}, {}, {}
    for p in range(sc.P):
        tracks[p] = [(int(obs_img[o]), o) for o in range(sc.pt_obs_begin[p], sc.pt_obs_begin[p + 1])]
        xyz[p] = sc.points[p]
        for img, o in tracks[p]:
            features[(img, o)] = sc.obs_xy[o]
    return images, cameras, tracks, features, xyz


def _normalized(v):
    n = math.sqrt(sum(x * x for x in v))
    return [x / n for x in v] if n > 0 else list(v)


def restated_filter(sc, kind, thr, bearings=None, calibrated=None):
    """(kept observation ids, counter) of one TrackFilter call, one track and one observation at a time."""
    images, cameras, tracks, features, xyz = _world(sc, calibrated)
    kept, counter = set(), 0
    thres, thres_uncalib = math.cos(math.radians(thr)), math.cos(math.radians(thr * 2))
    for tid, obs in tracks.items():
        if kind == "triangulation":
            rays = []
            for img, _ in obs:
                R, t, _ = images[img]
                centre = -(R.T @ t)
                rays.append(_normalized([xyz[tid][k] - centre[k] for k in range(3)]))
            status = any(sum(a * b for a, b in zip(rays[i], rays[j])) < thres
                         for i in range(len(rays)) for j in range(i + 1, len(rays)))
            if status:
                kept.update(o for _, o in obs)
            else:
                counter += 1
            continue
        new = []
        for img, o in obs:
            R, t, cam = images[img]
            pc = R @ xyz[tid] + t
            if pc[2] < FO.EPS:
                continue
            if kind == "reprojection":
                model, params, _ = cameras[cam]
                err = float(np.linalg.norm(S.project(model, params, pc[None])[0] - features[(img, o)]))
                ok = err < thr
            elif kind == "normalized":
                b = bearings[o]
                err = math.hypot(pc[0] / pc[2] - b[0] / (b[2] + FO.EPS), pc[1] / pc[2] - b[1] / (b[2] + FO.EPS))
                ok = err < thr
            else:
                d = sum(a * b for a, b in zip(_normalized(pc), bearings[o]))
                ok = d > (thres if cameras[cam][2] else thres_uncalib)
            if ok:
                new.append(o)
        if len(new) != len(obs):
            counter += 1
        kept.update(new)
    return kept, counter


def oracle_filter(sc, kind, thr, bear=None, calibrated=None):
    if kind == "reprojection":
        return FO.filter_reprojection(sc, thr, S.project)
    if kind == "normalized":
        return FO.filter_reprojection_normalized(sc, bear, thr)
    if kind == "angle":
        return FO.filter_angle(sc, bear, thr, calibrated)
    return FO.filter_triangulation_angle(sc, thr)


@pytest.mark.parametrize("which", ["image", "rig_dataset", "missing_sensor"])
def test_oracle_filters_equal_the_loop_restatement(which):
    sc, cal = {"image": lambda: image_scene(20, 300), "rig_dataset": lambda: rig_dataset_scene(points=150),
               "missing_sensor": missing_sensor_rig_scene}[which]()
    bear = bearings(sc)
    assert FO.smallest_margin(sc, MAPPER_FILTERS, bear, cal, S.project) > FP64_BOUND
    for kind, thr in MAPPER_FILTERS:
        keep, n = oracle_filter(sc, kind, thr, bear, cal)
        kept, counter = restated_filter(sc, kind, thr, bear, cal)
        if kind == "triangulation":
            pt = np.repeat(np.arange(sc.P), np.diff(sc.pt_obs_begin))
            keep = keep[pt]
        assert set(np.flatnonzero(keep).tolist()) == kept and n == counter, (kind, thr)
        assert keep.any() and (n > 0 or (kind, thr) == ("triangulation", 1.0)), (kind, thr)


def test_rig_filters_use_the_sensor_calibration_and_pose():
    """On rigs the angle threshold follows the sensor's flag and the pose composes cam_from_rig: flipping one sensor's
    flag changes exactly its observations, and the rig scene filters like its image scene (flags per image)."""
    sc, cal = rig_dataset_scene(points=150)
    bear = bearings(sc)
    k1, _ = FO.filter_angle(sc, bear, 1.0, cal)
    flip = cal.copy(); flip[1] ^= 1
    k2, _ = FO.filter_angle(sc, bear, 1.0, flip)
    assert (k1 != k2).any() and np.all(sc.obs_sensor[k1 != k2] == 1)
    img = sc.images_scene()
    for kind, thr in MAPPER_FILTERS:
        a = oracle_filter(sc, kind, thr, bear, cal)
        b = oracle_filter(img, kind, thr, bear, cal[sc.image_sensor])
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], (kind, thr)


def test_zero_ray_counts_as_a_wide_pair():
    """A point on a camera centre: Eigen's normalized() leaves the zero ray, its dot products are 0 < cos(1 deg), and
    the track stays; without that ray the track would be removed."""
    sc = S.Scene(np.tile([0.0, 0, 0, 1], (3, 1)), np.array([[0.0, 0, 0], [-2 * np.sin(0.003), 0, -2 * np.cos(0.003)],
                                                             [-2 * np.sin(0.006), 0, -2 * np.cos(0.006)]]),
                 np.zeros((1, 3)), np.array([0, 3]), np.arange(3, dtype=np.int32), np.zeros((3, 2)),
                 np.zeros(3, np.int32), np.zeros(1, np.int32), _params(S.SIMPLE_PINHOLE, 1000.0, 500.0)[None])
    keep, n = FO.filter_triangulation_angle(sc, 1.0)
    assert keep.tolist() == [True] and n == 0
    assert restated_filter(sc, "triangulation", 1.0)[1] == 0
    sc.obs_cam = np.array([1, 2, 2], np.int32)
    assert FO.filter_triangulation_angle(sc, 1.0)[0].tolist() == [False]


def _mp(x):
    """A long double as an mpf, exactly (its shortest round-trip decimal form)."""
    return mpmath.mpf(np.format_float_scientific(x, unique=True))


def test_decision_quantities_match_mpmath():
    mpmath.mp.dps = 40
    sc, cal = rig_dataset_scene(points=60)
    bear = bearings(sc)
    rng = np.random.default_rng(4)
    Rf, Rs = G.quat_xyzw_to_rotmat(sc.quat), G.quat_xyzw_to_rotmat(sc.sensor_quat)
    pt = np.repeat(np.arange(sc.P), np.diff(sc.pt_obs_begin))

    def mp_xc(o):
        f, s = int(sc.obs_frame[o]), int(sc.obs_sensor[o])
        qf = [mpmath.mpf(x) for x in sc.quat[f]]
        qs = [mpmath.mpf(x) for x in sc.sensor_quat[s]]

        def rot(q):
            n = mpmath.sqrt(sum(x * x for x in q)); x, y, z, w = [v / n for v in q]
            return mpmath.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        X = mpmath.matrix([mpmath.mpf(v) for v in sc.points[pt[o]]])
        return rot(qs) * (rot(qf) * X + mpmath.matrix([mpmath.mpf(v) for v in sc.trans[f]])) + \
            mpmath.matrix([mpmath.mpf(v) for v in sc.sensor_trans[s]])

    z, _, mag, front = FO.decisions(sc, "z", 0.0)
    qa, _, _, _ = FO.decisions(sc, "angle", 1.0, bearings=bear, calibrated=cal)
    qn, _, _, _ = FO.decisions(sc, "normalized", 1e-2, bearings=bear)
    fidx = np.flatnonzero(front)
    for o in rng.choice(sc.N, 40, replace=False):
        xc = mp_xc(o)
        assert abs(float(xc[2] - _mp(z[o]))) <= 1e-17 * float(mag[o])
        if front[o]:
            k = int(np.searchsorted(fidx, o))
            nrm = mpmath.sqrt(sum(xc[i] ** 2 for i in range(3)))
            d = sum(xc[i] / nrm * mpmath.mpf(bear[o, i]) for i in range(3))
            assert abs(float(d - _mp(qa[k]))) <= 1e-17
            bz = mpmath.mpf(bear[o, 2]) + mpmath.mpf(FO.EPS)
            e = mpmath.sqrt((xc[0] / xc[2] - mpmath.mpf(bear[o, 0]) / bz) ** 2 + (xc[1] / xc[2] - mpmath.mpf(bear[o, 1]) / bz) ** 2)
            assert abs(float(e - _mp(qn[k]))) <= 1e-16 * max(float(e), 1e-3)


# ---- undistortion ----------------------------------------------------------------------------------------------------
def sweep_pixels(model, params, n=400, seed=0, image_size=1000):
    """Pixels from the principal point out to the distorted radius where d/dr [r d(r^2)] falls to 0.05 (for models
    without a fold: twice the image's half-diagonal), in random directions, plus a grid over the image box."""
    f, c = params[0], params[1 + (model == S.PINHOLE)]
    rng = np.random.default_rng(seed)
    if model in (S.SIMPLE_RADIAL, S.RADIAL):
        k1, k2 = params[3], params[4] if model == S.RADIAL else 0.0
        rr = np.linspace(0.0, 4.0, 40001)
        ok = np.cumprod(1 + 3 * k1 * rr ** 2 + 5 * k2 * rr ** 4 >= 0.05).astype(bool)
        r_max = rr[ok][-1]
        rd_max = r_max * (1 + k1 * r_max ** 2 + k2 * r_max ** 4)
        rd_max = min(rd_max, 2 * 0.5 * image_size * np.sqrt(2) / f) if r_max >= 4.0 else rd_max
    else:
        rd_max = image_size * np.sqrt(2) / f
    rd = np.linspace(0.0, rd_max, n)
    a = rng.uniform(0, 2 * np.pi, n)
    g = np.linspace(0, image_size, 21)
    box = np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)
    return np.concatenate([np.stack([c + f * rd * np.cos(a), c + f * rd * np.sin(a)], 1), box])


def _distort_ld(model, params, uv):
    p = np.asarray(params, FO.LD)
    if model == S.SIMPLE_PINHOLE:
        return uv * p[0] + p[1:3]
    if model == S.PINHOLE:
        return uv * p[0:2] + p[2:4]
    r2 = (uv * uv).sum(1)
    d = 1 + p[3] * r2 + (p[4] * r2 * r2 if model == S.RADIAL else 0)
    return uv * d[:, None] * p[0] + p[1:3]


ALL_CAMERAS = [(S.SIMPLE_PINHOLE, 0.0, 0.0), (S.PINHOLE, 0.0, 0.0)] + RADIAL_CASES


@pytest.mark.parametrize("model,k1,k2", ALL_CAMERAS)
def test_undistort_exact_round_trip_and_mpmath(model, k1, k2):
    p = _params(model, 1000.0, 500.0, k1, k2)
    xy = sweep_pixels(model, p)
    uv = FO.undistort_exact(model, p, xy)
    back = _distort_ld(model, p, uv)
    assert float(np.abs(back - xy).max() / np.abs(xy - 500).max()) < 1e-15
    mpmath.mp.dps = 40
    for i in np.random.default_rng(1).choice(len(xy), 12, replace=False):
        x, y = mpmath.mpf(xy[i, 0]), mpmath.mpf(xy[i, 1])
        if model in (S.SIMPLE_PINHOLE, S.PINHOLE):
            fx, fy = (p[0], p[0]) if model == S.SIMPLE_PINHOLE else (p[0], p[1])
            want = [(x - 500) / mpmath.mpf(fx), (y - 500) / mpmath.mpf(fy)]
        else:
            ud, vd = (x - 500) / mpmath.mpf(p[0]), (y - 500) / mpmath.mpf(p[0])
            rd = mpmath.sqrt(ud * ud + vd * vd)
            if rd == 0:
                want = [ud, vd]
            else:
                r = mpmath.findroot(lambda r: r * (1 + k1 * r ** 2 + k2 * r ** 4) - rd, float(np.hypot(*uv[i].astype(float))))
                want = [ud * r / rd, vd * r / rd]
        for j in range(2):
            assert abs(float(want[j]) - float(uv[i, j])) <= 1e-17 * max(1.0, abs(float(want[j])))


@pytest.mark.parametrize("model,k1,k2", RADIAL_CASES)
def test_fold_radius_is_where_the_derivative_vanishes(model, k1, k2):
    rf = FO.fold_radius(_params(model, 1.0, 0.0, k1, k2), model)
    dg = lambda r: 1 + 3 * k1 * r ** 2 + 5 * k2 * r ** 4      # noqa: E731
    rr = np.linspace(0, min(rf, 10.0), 10001)[:-1]
    assert (dg(rr) > 0).all()
    if np.isfinite(rf):
        assert abs(dg(rf)) < 1e-12
        with pytest.raises(ValueError):   # past the fold's value there is no inverse
            g_f = rf * (1 + k1 * rf ** 2 + k2 * rf ** 4)
            FO.undistort_exact(model, _params(model, 1.0, 0.0, k1, k2), np.array([[1.01 * g_f, 0.0]]))


@pytest.mark.parametrize("model,k1,k2", ALL_CAMERAS)
def test_host_undistortion_is_the_exact_inverse_up_to_the_fold(model, k1, k2):
    """The production host restatement (the one the device is compared with) against the exact inverse, bearings to
    1e-12 relative everywhere from the centre to where the derivative falls to 0.05; the fixed-point iteration it
    replaced was off by 9.5e-4 at k = -0.2."""
    p = _params(model, 1000.0, 500.0, k1, k2)
    xy = sweep_pixels(model, p)
    got = S.bearings_from_pixels(model, p, xy)
    want = FO.bearings_exact(model, p, xy).astype(np.float64)
    assert np.abs(got - want).max() <= 1e-12


# ---- normalisation ---------------------------------------------------------------------------------------------------
def restated_normalize(images, p0=0.1, p1=0.9, extent=10.0, fixed_scale=False):
    """reconstruction_normalizer.cc:16-60 over {image_id: (centre, registered)}: (scale, translation)."""
    xs, ys, zs = [], [], []
    for _, (centre, registered) in sorted(images.items()):
        if not registered:
            continue
        xs.append(np.float32(centre[0])); ys.append(np.float32(centre[1])); zs.append(np.float32(centre[2]))
    xs.sort(); ys.sort(); zs.sort()
    n = len(xs)
    P0 = int(p0 * (n - 1)) if n > 3 else 0
    P1 = int(p1 * (n - 1)) if n > 3 else n - 1
    lo = np.array([xs[P0], ys[P0], zs[P0]], np.float64)
    hi = np.array([xs[P1], ys[P1], zs[P1]], np.float64)
    mean = [0.0, 0.0, 0.0]
    for i in range(P0, P1 + 1):
        mean[0] += float(xs[i]); mean[1] += float(ys[i]); mean[2] += float(zs[i])
    mean = np.array(mean) / (P1 - P0 + 1)
    scale = 1.0
    if not fixed_scale:
        old = float(np.linalg.norm(hi - lo))
        if old >= np.finfo(np.float64).eps:
            scale = extent / old
    return scale, -scale * mean


def _image_dict(sc, registered=None):
    if hasattr(sc, "obs_sensor"):
        # every frame-sensor combination is a potential image; the table's are the registered ones
        Rf, Rs = G.quat_xyzw_to_rotmat(sc.quat), G.quat_xyzw_to_rotmat(sc.sensor_quat)
        table = set(zip(sc.image_frame.tolist(), sc.image_sensor.tolist()))
        out = {}
        for f in range(sc.F):
            for s in range(sc.S):
                R, t = Rs[s] @ Rf[f], Rs[s] @ sc.trans[f] + sc.sensor_trans[s]
                out[f * sc.S + s] = (-(R.T @ t), (f, s) in table)
        return out
    c = G.centers_from_pose(G.quat_xyzw_to_rotmat(sc.quat), sc.trans)
    return {i: (c[i], True if registered is None else bool(registered[i])) for i in range(sc.C)}


def centres_scene(n, seed=0, offset=0.0, duplicate=False):
    """n images (random poses, centres on a shell of radius 8-12 plus ``offset``, or all at one point), ten points each
    seen by up to three of them: a BA problem with min_num_view_per_track = 1 over every track."""
    R, t = S.make_cameras(n, seed=seed)
    c = G.centers_from_pose(R, t) + offset
    if duplicate:
        c[:] = c[0]
    t = -np.einsum("nij,nj->ni", R, c)
    rng = np.random.default_rng(seed)
    k = min(n, 3)
    obs_cam = np.concatenate([(np.arange(k) + p) % n for p in range(10)]).astype(np.int32)
    _, intr_model, intr_params = S.make_intrinsics(n, S.SIMPLE_PINHOLE, 1000.0, 1000, 1)
    return S.Scene(G.rotmat_to_quat_xyzw_fast(R), t, rng.normal(size=(10, 3)), np.arange(11, dtype=np.int64) * k, obs_cam,
                   rng.uniform(0, 1000, size=(len(obs_cam), 2)), np.zeros(n, np.int32), intr_model, intr_params)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 40])
@pytest.mark.parametrize("fixed_scale", [False, True])
def test_normalize_equals_the_restatement(n, fixed_scale):
    sc = centres_scene(n, seed=n)
    s_ref, t_ref = restated_normalize(_image_dict(sc), fixed_scale=fixed_scale)
    s, t = PR.normalize_reconstruction(sc.copy(), fixed_scale=fixed_scale)
    assert s == s_ref and np.abs(t - t_ref).max() <= 1e-15 * max(1.0, np.abs(t_ref).max())


def test_normalize_duplicate_centres_keep_scale_one():
    sc = centres_scene(7, duplicate=True)
    s_ref, t_ref = restated_normalize(_image_dict(sc))
    s, t = PR.normalize_reconstruction(sc.copy())
    assert s == s_ref == 1.0 and np.allclose(t, t_ref, rtol=0, atol=1e-15)


@pytest.mark.parametrize("which", ["rig_dataset", "missing_sensor"])
def test_normalize_rigs_runs_over_the_registered_images(which):
    """Only the images of the table count (reconstruction_normalizer.cc:23-29): with three rigs (36 of 108
    frame-sensor combinations) or frames that lack a sensor, all F * S combinations would give another scale."""
    sc = rig_dataset_scene()[0] if which == "rig_dataset" else missing_sensor_rig_scene()[0]
    images = _image_dict(sc)
    s_ref, t_ref = restated_normalize(images)
    s, t = PR.normalize_reconstruction(sc.copy())
    assert abs(s - s_ref) <= 1e-15 * s_ref and np.abs(t - t_ref).max() <= 1e-14 * max(1.0, np.abs(t_ref).max())
    s_all, _ = restated_normalize({k: (c, True) for k, (c, _) in images.items()})
    assert abs(s_all - s) > 1e-3 * s
