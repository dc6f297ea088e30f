"""ORACLE (test infrastructure, NOT product code) -- numpy restatement of
glomap/processors/track_filter.cc (pixel-space reprojection filter :7-52,
angle filter :54-90, triangulation-angle filter :92-127) on the flat arrays,
and the exact inverse of the radial distortion that UndistortImages needs.
PARITY UNPINNED (no golden vectors in the reference; COLMAP's ImgFromCam is
restated for the four supported models in glomap_b200.synthetic.project).

Every decision is evaluated in np.longdouble (x86-64: 64-bit mantissa), so
the masks are the exact decisions of the scene's FP64 inputs up to about 1e-19
relative, and ``decisions`` returns each quantity with its bound and the
magnitude of the terms it is made of.  ``smallest_margin`` is the smallest
|quantity - bound| / max(|bound|, magnitude) of a scene: a device evaluation
in FP64 whose rounding stays below it has to reach the same masks.

Scenes are ``synthetic.Scene`` (one image per camera, intrinsics per camera,
the angle filter's calibrated flag per camera) or ``synthetic.RigScene``
(image poses from the image table, intrinsics and the calibrated flag per
sensor, as the ABI's ``cam_calibrated`` is [S] for rig problems)."""
import numpy as np

EPS = 1e-12
LD = np.longdouble


def _rotmat(q):
    q = np.asarray(q, LD)
    q = q / np.sqrt((q * q).sum(-1, keepdims=True))
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3), LD)
    R[..., 0, 0] = 1 - 2 * (y * y + z * z); R[..., 0, 1] = 2 * (x * y - z * w); R[..., 0, 2] = 2 * (x * z + y * w)
    R[..., 1, 0] = 2 * (x * y + z * w); R[..., 1, 1] = 1 - 2 * (x * x + z * z); R[..., 1, 2] = 2 * (y * z - x * w)
    R[..., 2, 0] = 2 * (x * z - y * w); R[..., 2, 1] = 2 * (y * z + x * w); R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _norm(a):
    return np.sqrt((a * a).sum(-1))


def is_rig(scene):
    return hasattr(scene, "obs_sensor")


def observation_geometry(scene):
    """Per observation, in long double: the camera-frame point Xc [N,3], the image centre [N,3] in the world, the
    point index, the intrinsics block, the index into the calibrated flags, and the magnitude |X| + |t| (+ |t_cr|) of
    the terms Xc is made of."""
    pt = np.repeat(np.arange(scene.P), np.diff(scene.pt_obs_begin))
    X = np.asarray(scene.points, LD)[pt]
    if is_rig(scene):
        f, s = np.asarray(scene.obs_frame, np.int64), np.asarray(scene.obs_sensor, np.int64)
        Rf, Rs = _rotmat(scene.quat)[f], _rotmat(scene.sensor_quat)[s]
        tf, ts = np.asarray(scene.trans, LD)[f], np.asarray(scene.sensor_trans, LD)[s]
        R = np.einsum("nij,njk->nik", Rs, Rf)
        t = np.einsum("nij,nj->ni", Rs, tf) + ts
        intr, cal = np.asarray(scene.sensor_intr)[s], s
        mag = _norm(X) + _norm(tf) + _norm(ts)
    else:
        c = np.asarray(scene.obs_cam, np.int64)
        R, t = _rotmat(scene.quat)[c], np.asarray(scene.trans, LD)[c]
        intr, cal = np.asarray(scene.cam_intr)[c], c
        mag = _norm(X) + _norm(t)
    Xc = np.einsum("nij,nj->ni", R, X) + t
    centre = -np.einsum("nji,nj->ni", R, t)
    return dict(Xc=Xc, centre=centre, pt=pt, intr=intr, cal=cal, mag=mag)


def _keep_and_count(scene, keep, pt):
    changed = np.zeros(scene.P, bool)
    np.logical_or.at(changed, pt, ~keep)
    return keep, int(changed.sum())


def _normalized(d):
    """Eigen's normalized(): d / |d|, and a zero vector unchanged (UPSTREAM-UNVERIFIED: Eigen is not vendored)."""
    n = _norm(d)[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(n > 0, d / n, d)


def decisions(scene, kind, thr, bearings=None, calibrated=None, project=None):
    """(quantity, bound, magnitude, passes) in long double for every decision of one filter; ``passes`` is the
    comparison the reference makes (z >= EPS, error < thr, dot > thres, pair dot < thres).
      "reprojection"  pixel error (needs ``project``), "normalized" error in the normalised image plane, "angle" the
      dot product (both need ``bearings``), for observations in front of the camera, after one "z" decision each;
      "triangulation" the dot products of all pairs of rays of every track."""
    g = observation_geometry(scene)
    Xc, z = g["Xc"], g["Xc"][:, 2]
    if kind == "z":
        return z, np.full(len(z), LD(EPS)), g["mag"], ~(z < EPS)
    if kind == "triangulation":
        th = LD(np.cos(np.radians(thr)))
        ray = _normalized(np.asarray(scene.points, LD)[g["pt"]] - g["centre"])
        b = np.asarray(scene.pt_obs_begin)
        q = [np.einsum("ik,jk->ij", ray[b[p]:b[p + 1]], ray[b[p]:b[p + 1]])[np.triu_indices(b[p + 1] - b[p], 1)]
             for p in range(scene.P)]
        q = np.concatenate(q) if q else np.zeros(0, LD)
        return q, np.full(len(q), th), np.ones(len(q), LD), q < th
    front = ~(z < EPS)
    zf = z[front]
    cond = g["mag"][front] / np.abs(zf)            # the error of Xc relative to z, as seen through the division by z
    if kind == "reprojection":
        err, scale = np.zeros(len(z), LD), np.zeros(len(z), LD)
        xy = np.asarray(scene.obs_xy, LD)
        for k in np.unique(g["intr"][front]):
            m = front & (g["intr"] == k)
            px = project(int(scene.intr_model[k]), np.asarray(scene.intr_params[k], LD), Xc[m])
            err[m] = _norm(px - xy[m])
            scale[m] = (_norm(px) + _norm(xy[m])) * np.maximum(1, g["mag"][m] / np.abs(z[m]))
        q, s = err[front], scale[front]
    elif kind == "normalized":
        bf = np.asarray(bearings, LD)[front]
        bxy = bf[:, :2] / (bf[:, 2:3] + LD(EPS))
        q = _norm(Xc[front, :2] / zf[:, None] - bxy)
        s = (_norm(Xc[front, :2]) / np.abs(zf)) * np.maximum(1, cond) + _norm(bxy)
    elif kind == "angle":
        q = (_normalized(Xc[front]) * np.asarray(bearings, LD)[front]).sum(1)
        s = np.ones(len(q), LD)
    else:
        raise ValueError(kind)
    if kind == "angle":
        th, th_u = LD(np.cos(np.radians(thr))), LD(np.cos(np.radians(2 * thr)))
        b = np.full(len(q), th) if calibrated is None else \
            np.where(np.asarray(calibrated).astype(bool)[g["cal"][front]], th, th_u)
        return q, b, s, q > b
    return q, np.full(len(q), LD(thr)), s, q < thr


def _observation_filter(scene, kind, thr, **kw):
    g_pt = np.repeat(np.arange(scene.P), np.diff(scene.pt_obs_begin))
    _, _, _, front = decisions(scene, "z", 0.0)
    keep = np.zeros(scene.N, bool)
    keep[front] = decisions(scene, kind, thr, **kw)[3]
    return _keep_and_count(scene, keep, g_pt)


def filter_reprojection(scene, max_err, project):
    """FilterTracksByReprojection, in_normalized_image = false: (keep [N], #tracks changed)."""
    return _observation_filter(scene, "reprojection", max_err, project=project)


def filter_reprojection_normalized(scene, bearings, max_err):
    """in_normalized_image = true (track_filter.cc:24-31): |X_c.xy / X_c.z - b.xy / (b.z + EPS)| < max_err."""
    return _observation_filter(scene, "normalized", max_err, bearings=bearings)


def filter_angle(scene, bearings, max_angle_deg, calibrated=None):
    """FilterTracksByAngle; ``calibrated`` per camera (Scene) or per sensor (RigScene), None = all calibrated."""
    return _observation_filter(scene, "angle", max_angle_deg, bearings=bearings, calibrated=calibrated)


def filter_triangulation_angle(scene, min_angle_deg):
    """FilterTrackTriangulationAngle: (keep_track [P], #tracks removed)."""
    q, th, _, wide = decisions(scene, "triangulation", min_angle_deg)
    L = np.diff(scene.pt_obs_begin)
    npairs = L * (L - 1) // 2
    keep = np.zeros(scene.P, bool)
    nz = npairs > 0
    if nz.any():   # the pairs of the tracks with any lie back to back, in track order
        keep[nz] = np.logical_or.reduceat(wide, (np.cumsum(npairs) - npairs)[nz])
    return keep, int((~keep).sum())


def smallest_margin(scene, filters, bearings=None, calibrated=None, project=None):
    """min |quantity - bound| / max(|bound|, magnitude) over every decision of ``filters`` [(kind, thr), ...]; the
    z >= EPS test is included whenever an observation filter is."""
    out = np.inf
    kinds = [k for k, _ in filters]
    if any(k != "triangulation" for k in kinds):
        filters = [("z", 0.0)] + list(filters)
    for kind, thr in filters:
        q, b, s, _ = decisions(scene, kind, thr, bearings=bearings, calibrated=calibrated, project=project)
        if len(q):
            out = min(out, float((np.abs(q - b) / np.maximum(np.abs(b), s)).min()))
    return out


# ---- radial undistortion ---------------------------------------------------------------------------------------------
def _radial_k(model, params):
    if model == 2:
        return LD(params[3]), LD(0)
    if model == 3:
        return LD(params[3]), LD(params[4])
    raise ValueError(f"no radial distortion in model {model}")


def fold_radius(params, model=3):
    """The first undistorted radius r > 0 where d/dr [r d(r^2)] = 1 + 3 k1 r^2 + 5 k2 r^4 reaches 0 (inf if none):
    r d(r^2) increases up to it, and past its value there is no inverse."""
    k1, k2 = _radial_k(model, params)
    if k2 == 0:
        return float(np.sqrt(-1 / (3 * k1))) if k1 < 0 else np.inf
    disc = 9 * k1 * k1 - 20 * k2
    if disc < 0:
        return np.inf
    roots = [(-3 * k1 + sg * np.sqrt(disc)) / (10 * k2) for sg in (-1, 1)]
    pos = [s for s in roots if s > 0]
    return float(np.sqrt(min(pos))) if pos else np.inf


def undistort_exact(model, params, xy):
    """CamFromImg of [n,2] pixels in long double: the undistorted normalised coordinates [n,2].  Radial models invert
    rd = r d(r^2) on the radius with a bisection-safeguarded Newton iteration run to convergence in long double, on
    [0, fold_radius]; a radius past the fold's value raises (no inverse)."""
    p = np.asarray(params, LD)
    xy = np.asarray(xy, LD)
    if model == 0:
        return (xy - p[1:3]) / p[0]
    if model == 1:
        return (xy - p[2:4]) / p[0:2]
    k1, k2 = _radial_k(model, params)
    uvd = (xy - p[1:3]) / p[0]
    rd = _norm(uvd)
    g = lambda r: r * (1 + k1 * r * r + k2 * r ** 4)          # noqa: E731
    dg = lambda r: 1 + 3 * k1 * r * r + 5 * k2 * r ** 4       # noqa: E731
    rf = LD(fold_radius(params, model))
    hi = np.full(len(rd), rf) if np.isfinite(rf) else np.maximum(rd, LD(1))
    while not np.isfinite(rf) and (g(hi) < rd).any():     # no fold: g is unbounded, widen until it brackets
        hi = np.where(g(hi) < rd, 2 * hi, hi)
    if np.isfinite(rf) and (rd > g(rf)).any():
        raise ValueError("distorted radius past the fold: no inverse")
    lo = np.zeros(len(rd), LD)
    r = np.minimum(rd, hi)
    for _ in range(200):
        f = g(r) - rd
        lo, hi = np.where(f < 0, r, lo), np.where(f < 0, hi, r)
        with np.errstate(divide="ignore", invalid="ignore"):
            rn = r - f / dg(r)
        rn = np.where((rn >= lo) & (rn <= hi), rn, (lo + hi) / 2)
        if np.array_equal(rn, r):
            break
        r = rn
    with np.errstate(divide="ignore", invalid="ignore"):
        sc = np.where(rd > 0, r / rd, LD(1))
    return uvd * sc[:, None]


def bearings_exact(model, params, xy):
    """CamFromImg(xy).homogeneous().normalized() in long double, [n,3]."""
    uv = undistort_exact(model, params, xy)
    b = np.concatenate([uv, np.ones((len(uv), 1), LD)], 1)
    return b / _norm(b)[:, None]
