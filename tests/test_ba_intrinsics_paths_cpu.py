"""Host checks behind the intrinsics-path tests of tests/test_ba_intrinsics_paths_gpu.py: the scenes reach the shapes
they are built for, the FP64 reference puts every intrinsics unknown in the device slot select_paths gives it, and the
reference's projection Jacobian is right to 1e-12 against mpmath at 40 digits at the edges where it goes wrong."""
import mpmath as mp
import numpy as np
import pytest

import test_ba_intrinsics_paths_gpu as G
import test_ba_system_gpu as T
from glomap_b200 import synthetic as S
from oracle import ba_oracle as B
from oracle import ba_system as BS

mp.mp.dps = 40

# select_paths (glomap_b200/csrc/ba_solver.cuh): focal and distortion indices, then the principal point
DEVICE_FOCAL_EXTRA = {S.SIMPLE_PINHOLE: (0,), S.PINHOLE: (0, 1), S.SIMPLE_RADIAL: (0, 3), S.RADIAL: (0, 3, 4)}
DEVICE_PP = {S.SIMPLE_PINHOLE: (1, 2), S.PINHOLE: (2, 3), S.SIMPLE_RADIAL: (1, 2), S.RADIAL: (1, 2)}

MIXED = {"mixed3_K300": G.M3_300, "all4_K200": G.M4_200, "all4_per_image_K300": G.M4_300}


def _problem(sc, **opts):
    bo = B.BAOptions(min_num_view_per_track=T.MIN_VIEWS, **opts)
    mask = np.zeros(sc.C, np.uint8)
    mask[0] = 3
    if hasattr(sc, "obs_sensor"):
        return B.BAProblem(sc.quat, sc.trans, sc.points, sc.pt_obs_begin, sc.obs_frame, sc.obs_xy,
                           np.zeros(sc.F, np.int32), sc.intr_model, sc.intr_params, bo, mask, rig=sc.rig_dict())
    return B.BAProblem(sc.quat, sc.trans, sc.points, sc.pt_obs_begin, sc.obs_cam, sc.obs_xy, sc.cam_intr,
                       sc.intr_model, sc.intr_params, bo, mask)


def _used_obs_per_block(sc):
    lens = np.diff(sc.pt_obs_begin)
    valid = np.repeat(lens >= T.MIN_VIEWS, lens)
    return np.bincount(sc.cam_intr[sc.obs_cam[valid]], minlength=len(sc.intr_model))


# ---- the scenes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(MIXED))
def test_scene_reaches_the_mixed_model_shapes(name):
    spec = MIXED[name]
    sc = G.scene(spec)
    models = np.asarray(spec[2])
    K = spec[1]
    assert len(sc.intr_model) == K and set(sc.intr_model) == set(models)
    used = _used_obs_per_block(sc)
    # neighbouring cameras (neighbouring camera-order segments) have different models
    cm = sc.intr_model[sc.cam_intr]
    assert np.all(cm[9:-1] != cm[10:])
    # one point-order warp (32 points) holds observations of every model of the scene
    first_warp = sc.obs_cam[:sc.pt_obs_begin[32]]
    assert set(sc.intr_model[sc.cam_intr[first_warp]]) == set(models)
    # every model has a block with more than one kSeg = 256 segment of used observations
    for m in models:
        assert used[sc.intr_model == m].max() > 256, m
    # the block the reference leaves out: only observations on tracks shorter than MIN_VIEWS
    assert used[G.UNUSED_BLOCK] == 0 and np.count_nonzero(sc.cam_intr[sc.obs_cam] == G.UNUSED_BLOCK) > 0
    assert np.flatnonzero(sc.cam_intr == G.UNUSED_BLOCK).tolist() == [T.EMPTY_CAM]
    # a SIMPLE_RADIAL block with k = 0 (the pinhole branch) next to ones with k != 0, both used
    sr = sc.intr_model == S.SIMPLE_RADIAL
    assert sc.intr_params[G.K0_BLOCK, 3] == 0.0 and sr[G.K0_BLOCK] and used[G.K0_BLOCK] > 0
    assert np.all(sc.intr_params[sr & (np.arange(K) != G.K0_BLOCK), 3] != 0.0)
    # no camera sees a point twice
    pt = np.repeat(np.arange(sc.P), np.diff(sc.pt_obs_begin))
    assert len(np.unique(pt * sc.C + sc.obs_cam)) == sc.N
    if K == sc.C:
        assert np.array_equal(sc.cam_intr, np.arange(sc.C))


def test_rig_scene_has_one_model_per_sensor():
    rs = G.scene(G.RIG)
    assert rs.S == 3 and np.array_equal(rs.sensor_intr, np.arange(3))
    assert tuple(rs.intr_model) == G.RIG_MODELS
    assert np.all(np.bincount(rs.obs_sensor, minlength=3) > 256)


# ---- the column layout -----------------------------------------------------------------------------------------------
LAYOUTS = {f"{n}_{o}": (spec, o) for n, spec in list(MIXED.items()) + [("rig", G.RIG)]
           for o in ("intrinsics", "principal_point", "principal_point_only")}


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_every_oracle_column_maps_to_the_device_slot_of_its_parameter(name):
    spec, which = LAYOUTS[name]
    sc = G.scene(spec)
    opts = dict(optimize_intrinsics=which != "principal_point_only", optimize_principal_point=which != "intrinsics")
    prob = _problem(sc, **opts)
    C, K = prob.C, prob.K
    nbk = C + K + prob.S
    cam, pt = BS.device_index(prob, nbk)
    assert np.all((cam >= 0) ^ (pt >= 0))
    assert len(np.unique(cam[cam >= 0])) == (cam >= 0).sum()
    ci = prob.rig["obs_intr"] if prob.rig is not None else prob.cam_intr[prob.obs_cam]
    used = np.bincount(ci, minlength=K) > 0
    for k in range(K):
        m = int(prob.intr_model[k])
        # the device's pidx: focal and distortion, with the principal point when it is free, in ascending order
        pidx = sorted(DEVICE_FOCAL_EXTRA[m] + (DEVICE_PP[m] if which != "intrinsics" else ()))
        ent = prob.intr_cols[k]
        if not used[k]:
            assert ent == [], k
            assert not np.any(cam // 6 == C + k)
            continue
        assert [i for i, _ in ent] == pidx, (k, ent)
        for slot, (i, col) in enumerate(ent):
            assert cam[col] == 6 * (C + k) + slot
        slots = cam[cam // 6 == C + k] % 6
        assert sorted(slots) == list(range(len(pidx)))
    if "mixed" in name or "all4" in name:
        assert not used[G.UNUSED_BLOCK]


# ---- the projection Jacobian against mpmath -------------------------------------------------------------------------
def _mp_project(model, p, X):
    x, y, z = X
    u, v = x / z, y / z
    if model == S.SIMPLE_PINHOLE:
        return [p[0] * u + p[1], p[0] * v + p[2]]
    if model == S.PINHOLE:
        return [p[0] * u + p[2], p[1] * v + p[3]]
    r2 = u * u + v * v
    d = 1 + p[3] * r2 + (p[4] * r2 * r2 if model == S.RADIAL else 0)
    return [p[0] * u * d + p[1], p[0] * v * d + p[2]]


def _mp_jac(fn, args):
    """d fn / d args (2 x len(args)) at 40 digits."""
    args = [mp.mpf(float(a)) for a in args]
    out = np.zeros((2, len(args)))
    for j in range(len(args)):
        for a in range(2):
            out[a, j] = float(mp.diff(lambda t: fn(args[:j] + [t] + args[j + 1:])[a], args[j]))
    return out


def _rel(dev, ref):
    return float(np.abs(dev - ref).max() / np.abs(ref).max())


def _params(model, k1=0.02, k2=-0.005):
    return {S.SIMPLE_PINHOLE: [1000.0, 480.0, 530.0], S.PINHOLE: [1000.0, 1300.0, 480.0, 530.0],
            S.SIMPLE_RADIAL: [1000.0, 480.0, 530.0, k1], S.RADIAL: [1000.0, 480.0, 530.0, k1, k2]}[model]


def _edge_cases():
    """(model, params, [n,3] camera-frame points) per edge."""
    rng = np.random.default_rng(5)
    ordinary = np.column_stack([rng.uniform(-0.4, 0.4, (6, 2)), np.ones(6)]) * rng.uniform(2, 9, (6, 1))
    corner = np.array([[0.55, 0.5, 1.0], [-0.5, 0.55, 1.0], [0.56, -0.49, 1.0]]) * 3.0   # r^2 ~ 0.55
    tiny = np.array([[0.3, -0.2, 1.0], [-0.45, 0.4, 1.0]]) * (B.Z_EPS * (1 + 1e-6))       # depth just above kZEps
    cases = {}
    for m in (S.SIMPLE_PINHOLE, S.PINHOLE, S.SIMPLE_RADIAL, S.RADIAL):
        cases[f"ordinary_{m}"] = (m, _params(m), ordinary)
        cases[f"tiny_depth_{m}"] = (m, _params(m), tiny)
    for m in (S.SIMPLE_RADIAL, S.RADIAL):
        cases[f"corner_strong_{m}"] = (m, _params(m, k1=0.55, k2=-0.08), corner)     # |k1 r^2| ~ 0.3
        cases[f"k0_{m}"] = (m, _params(m, k1=0.0, k2=0.0), np.vstack([ordinary, corner]))
    cases["pinhole_fx_ne_fy_corner"] = (S.PINHOLE, [800.0, 1250.0, 480.0, 530.0], corner)
    return cases


EDGES = _edge_cases()


@pytest.mark.parametrize("name", list(EDGES))
def test_projection_jacobian_matches_mpmath(name):
    """Every column of project_with_jac -- the camera-frame point and every parameter, the principal point and k2
    included -- against 40-digit derivatives, relative to the largest entry of the observation's Jacobian."""
    model, params, Xc = EDGES[name]
    npar = S.MODEL_NUM_PARAMS[model]
    par = np.tile(np.asarray(params, float), (len(Xc), 1))
    px, Jp, Jk = B.project_with_jac(model, par, Xc)
    if name.startswith("corner_strong"):
        u, v = Xc[:, 0] / Xc[:, 2], Xc[:, 1] / Xc[:, 2]
        assert np.all(np.abs(params[3] * (u * u + v * v)) > 0.29)
    for n in range(len(Xc)):
        want = _mp_jac(lambda a: _mp_project(model, a[3:], a[:3]), list(Xc[n]) + list(params))
        ref_px = [float(t) for t in _mp_project(model, [mp.mpf(float(a)) for a in params],
                                                [mp.mpf(float(a)) for a in Xc[n]])]
        assert _rel(px[n], np.array(ref_px)) <= 1e-15
        assert _rel(Jp[n], want[:, :3]) <= 1e-12, (n, Jp[n], want[:, :3])
        assert _rel(Jk[n], want[:, 3:3 + npar]) <= 1e-12, (n, Jk[n], want[:, 3:])


def _mp_quat_rot(q, X):
    x, y, z, w = q
    R = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
         [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
         [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    return [sum(R[i][j] * X[j] for j in range(3)) for i in range(3)]


def _mp_plus(q, d):
    """EigenQuaternionManifold::Plus, as oracle/ba_oracle.quat_plus states it: exp(d) (x) q."""
    n = mp.sqrt(d[0] ** 2 + d[1] ** 2 + d[2] ** 2)
    s = mp.sin(n) / n if n != 0 else mp.mpf(1)
    a = [s * d[0], s * d[1], s * d[2], mp.cos(n)]
    ax, ay, az, aw = a
    bx, by, bz, bw = q
    return [aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
            aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz]


@pytest.mark.parametrize("model", [S.SIMPLE_PINHOLE, S.PINHOLE, S.SIMPLE_RADIAL, S.RADIAL])
def test_pose_point_and_intrinsics_columns_match_mpmath(model):
    """The chained columns of BAProblem.residuals (rotation on the quaternion manifold, translation, point, every
    intrinsic with the principal point free) for observations near the corner with strong distortion."""
    rng = np.random.default_rng(11 + model)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    t = rng.normal(size=3)
    params = _params(model, k1=0.55, k2=-0.08)
    if model == S.PINHOLE:
        params = [800.0, 1250.0, 480.0, 530.0]
    Xc = np.array([[0.55, 0.5, 1.0], [-0.5, 0.55, 1.0], [0.1, -0.2, 1.0], [-0.56, -0.49, 1.0]]) * 4.0
    R = B.quat_rotmat(q)
    X = (Xc - t) @ R                      # R^T (Xc - t): the world points that land there
    n = len(X)
    intr = np.zeros((1, S.INTR_STRIDE))
    intr[0, :len(params)] = params
    prob = B.BAProblem(q[None], t[None], X, np.arange(n + 1), np.zeros(n, np.int32), np.zeros((n, 2)),
                       np.zeros(1, np.int32), np.array([model]), intr,
                       B.BAOptions(optimize_intrinsics=True, optimize_principal_point=True, min_num_view_per_track=1))
    res, (Jrot, Jtrn, Jpt, Jk_all, valid, _, _) = prob.residuals(prob.x0, True)
    assert valid.all()
    mk, Jk = Jk_all[0]
    qm = [mp.mpf(float(a)) for a in q]
    tm = [mp.mpf(float(a)) for a in t]
    npar = len(params)
    for o in range(n):
        Xm = [mp.mpf(float(a)) for a in X[o]]

        def pix(a):   # a = (rotation tangent 3, translation step 3, point step 3, parameters)
            qn = _mp_plus(qm, a[0:3])
            Y = _mp_quat_rot(qn, [Xm[i] + a[6 + i] for i in range(3)])
            return _mp_project(model, a[9:], [Y[i] + tm[i] + a[3 + i] for i in range(3)])
        want = _mp_jac(pix, [0.0] * 9 + list(params))
        got = np.hstack([Jrot[o], Jtrn[o], Jpt[o], Jk[o, :, :npar]])
        assert _rel(got, want) <= 1e-12, (o, got - want)
