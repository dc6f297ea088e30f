"""Operator-level tests of the device rotation averager: every stage of an L1 / IRLS iteration, read through the test
probe (include/b200sfm_testing.h), against the FP64 sparse reference oracle/ra_system.py.

The trajectory tests (test_ra_gpu.py, test_rig_gpu.py, test_rotation_averager_gpu.py) run PCG to 1e-11..1e-12 and
compare the converged rotations; a wrong Jacobi diagonal, a wrong coarse correction or a wrong warm start only costs
PCG iterations there.  Here each path of the table below builds a scene that reaches the kernels' edge shapes, and the
test compares, relative to the magnitude of each compared block row:
  * the residuals and weights (L1 rows, Geman-McClure, half-norm; with and without edge weights);
  * the right-hand side and the Jacobi blocks against the exact diagonal of A^T W A;
  * on two-level paths, the inverted coarse matrix;
  * L x through the production mat-vec, M^-1 r through the production preconditioner;
  * the PCG iterate after k = 1, 2, 3, 5, 8 iterations (tolerance 0), cold and warm-started;
  * one ADMM step, and the rotation update with its sums.
The errors of every comparison are printed per path with `-s`; the worst measured values are listed beside BOUNDS.
"""
import ctypes as ct

import numpy as np
import pytest

from glomap_b200 import _lib, estimators as E
from oracle import ra_oracle as RO
from oracle import ra_system as RS

pytestmark = pytest.mark.gpu

PCG_KS = (1, 2, 3, 5, 8)
SIGMA2 = np.radians(5.0) ** 2
SPECIAL_DEG = {1: 1, 2: 31, 3: 32, 4: 33, 5: 64, 6: 65, 7: 300}   # node -> degree (CSR lane loops, unroll 2, the hub)
ISOLATED = 8                                                        # degree 0 (Jacobi-only scenes: no empty aggregate)
N_GENERAL = 1203                                                    # not a multiple of 128, n mod 8 = 3
FIXED = 517

# bound per comparison, relative to the magnitude of the compared block row; res and update in radians, Ac as
# max|Ac_dev^-1 Ac - I| in units of cond(Ac) nc 1e-16.  Worst measured on one H100 80GB HBM3 (700 W) in comments;
# a reverted fix or a broken kernel measured 1e-1 or more in the comparison that sees it
BOUNDS = dict(res=1e-13,        # 8.9e-16
              w=1e-12,          # 1.3e-13
              rhs=2e-12,        # 1.5e-13  default_large
              Minv=1e-12,       # 1.1e-13  default_large
              Ac=0.05,          # 1.3e-3   csr_2lvl
              apply=1e-12,      # 9.7e-14  default_large
              precond=1e-10,    # 1.3e-11  edge_2lvl
              pcg=1e-9,         # 5.7e-11  default_large
              pcg_warm=2e-9,    # 1.0e-10  default_large
              admm=1e-13,       # 1.0e-15
              update=1e-13,     # 1.1e-15
              sums=1e-13)       # 4.3e-16


def rand_rot(rng, n, deg):
    return RO.aa_to_R(rng.normal(size=(n, 3)) * np.radians(deg))


def general_scene(seed=1, isolated=True, gravity_frac=0.0, fixed_grav=True):
    """A view graph that reaches the shapes of the kernels (see test_scene_reaches_the_shapes_it_is_built_for)."""
    rng = np.random.default_rng(seed)
    n = N_GENERAL
    special = set(SPECIAL_DEG) | {ISOLATED}
    regular = np.array([i for i in range(n) if i not in special])
    pairs = list(zip(regular[:-1], regular[1:]))                     # a path through the regular nodes
    for s, d in SPECIAL_DEG.items():
        pairs += [(s, int(o)) for o in rng.choice(regular, d, replace=False)]
    if not isolated:
        pairs.append((ISOLATED, int(regular[3])))
    for _ in range(2 * n):
        a, b = rng.choice(regular, 2, replace=False)
        pairs.append((int(a), int(b)))
    a, b = int(regular[10]), int(regular[11])
    pairs += [(a, b), (b, a)]                                        # a duplicate and a reversed pair
    ei = np.array([p[0] for p in pairs]); ej = np.array([p[1] for p in pairs])
    flip = rng.random(len(ei)) < 0.5
    flip[-3:] = False
    ei, ej = np.where(flip, ej, ei), np.where(flip, ei, ej)
    theta = rng.normal(size=(n, 3)) * 0.4
    theta[[20, 21, 22]] = 0.0                                        # aa_to_R's first-order branch
    grav = np.zeros(n, bool)
    if gravity_frac > 0:
        grav = rng.random(n) < gravity_frac
        grav[FIXED] = fixed_grav
        grav[[30, 31, 32]] = True
        theta[grav] = np.stack([np.zeros(grav.sum()), theta[grav, 1], np.zeros(grav.sum())], 1)
        theta[30, 1], theta[31, 1], theta[32, 1] = 3.1, -3.1, 3.05  # y-only pairs around +-pi
        ei = np.append(ei, [30, 31]); ej = np.append(ej, [31, 32])
    E_ = len(ei)
    R = RO.aa_to_R(theta)
    R_rel = R[ej] @ np.swapaxes(R[ei], -1, -2) @ rand_rot(rng, E_, 2.0)
    out = rng.choice(E_ - 10, 25, replace=False)
    R_rel[out] = RO.aa_to_R(RO.R_to_aa(R_rel[out]) + rng.normal(size=(25, 3)) * 1.5)   # outliers, some beyond 120 deg
    w = rng.uniform(0.3, 3.0, E_)
    w[::17] = -1.0
    return dict(n_frames=n, ei=ei, ej=ej, R_rel=R_rel, theta=theta, fixed=FIXED, edge_w=w,
                has_grav=grav if gravity_frac > 0 else None)


def lattice_scene(side=200, seed=2):
    """The config-5 shape: a side x side lattice (two-level by default from 20 000 nodes)."""
    rng = np.random.default_rng(seed)
    n = side * side
    idx = np.arange(n).reshape(side, side)
    ei = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
    ej = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    theta = rng.normal(size=(n, 3)) * 0.3
    R = RO.aa_to_R(theta)
    R_rel = R[ej] @ np.swapaxes(R[ei], -1, -2) @ rand_rot(rng, len(ei), 1.0)
    return dict(n_frames=n, ei=ei, ej=ej, R_rel=R_rel, theta=theta, fixed=12345, edge_w=rng.uniform(0.5, 2.0, len(ei)))


def rig_scene(seed=3):
    """100 frames; sensor 0 is the reference (known), sensors 1 and 2 are unknown (nodes nf, nf + 1).  Sensor 1 is in
    every frame (more than 32: ra_update_cams' lane loop), sensor 2 in frames 0-39."""
    rng = np.random.default_rng(seed)
    nf = 100
    images = [(f, 0) for f in range(nf)] + [(f, 1) for f in range(nf)] + [(f, 2) for f in range(40)]
    cam_node = {0: -1, 1: nf, 2: nf + 1}
    pairs = set()
    for f in range(nf - 1):
        pairs.add(((f, 0), (f + 1, 0)))                            # connect the frames
        pairs.add(((f, 1), (f + 1, 1)))                            # the same unknown sensor in both images
    for f in range(40):
        pairs.add(((f, 0), (f, 2)))                                # the same frame, two sensors
        pairs.add(((f, 1), (f, 2)))
        pairs.add(((f, 2), ((f + 7) % 40, 2)))
    for _ in range(300):
        a, b = rng.choice(len(images), 2, replace=False)
        pairs.add((images[a], images[b]))
    pairs = sorted(pairs)
    th = rng.normal(size=(nf + 2, 3)) * 0.4
    th[nf:] = rng.normal(size=(2, 3)) * 0.6
    Rf = RO.aa_to_R(th)

    def R_img(f, s):
        return (Rf[cam_node[s]] if s else np.eye(3)) @ Rf[f]

    ei = np.array([p[0][0] for p in pairs]); ej = np.array([p[1][0] for p in pairs])
    eci = np.array([cam_node[p[0][1]] for p in pairs]); ecj = np.array([cam_node[p[1][1]] for p in pairs])
    R_rel = np.stack([R_img(*q) @ R_img(*p).T for p, q in pairs]) @ rand_rot(rng, len(pairs), 2.0)
    theta0 = th + rng.normal(size=th.shape) * 0.05
    cam_frames = [list(range(nf)), list(range(40))]
    return dict(n_frames=nf, ei=ei, ej=ej, R_rel=R_rel, theta=theta0, fixed=5, edge_w=rng.uniform(0.5, 2.0, len(ei)),
                n_cams=2, eci=eci, ecj=ecj, cam_frames=cam_frames)


SCENES = {
    "general": lambda: general_scene(isolated=True),
    "general_connected": lambda: general_scene(isolated=False),
    "large": lattice_scene,
    "gravity_all": lambda: general_scene(seed=4, gravity_frac=1.0),
    "gravity_mixed": lambda: general_scene(seed=5, gravity_frac=0.6),
    "gravity_fixed_without": lambda: general_scene(seed=6, gravity_frac=0.6, fixed_grav=False),
    "rig": rig_scene,
}

# name -> (scene, environment, expected flags)
PATHS = {
    "edge_jacobi": ("general", dict(B200SFM_RA_CSR="0", B200SFM_RA_2LVL="0"), dict(use_csr=0, use_2lvl=0)),
    "edge_2lvl": ("general_connected", dict(B200SFM_RA_CSR="0", B200SFM_RA_2LVL="1"), dict(use_csr=0, use_2lvl=1)),
    "csr_jacobi": ("general", dict(B200SFM_RA_2LVL="0"), dict(use_csr=1, use_2lvl=0)),
    "csr_2lvl": ("general_connected", dict(B200SFM_RA_2LVL="1"), dict(use_csr=1, use_2lvl=1, fused=0)),
    "csr_2lvl_fused": ("general_connected", dict(B200SFM_RA_2LVL="1", B200SFM_RA_FUSED="1"),
                       dict(use_csr=1, use_2lvl=1, fused=1)),
    "default_large": ("large", {}, dict(use_csr=1, use_2lvl=1, fused=0)),
    "gravity_all": ("gravity_all", {}, dict(use_csr=0, use_2lvl=0, has_grav=1)),
    "gravity_mixed": ("gravity_mixed", {}, dict(use_csr=0, use_2lvl=0, has_grav=1)),
    "gravity_fixed_without": ("gravity_fixed_without", {}, dict(use_csr=0, use_2lvl=0, has_grav=1)),
    "rig_unknown": ("rig", {}, dict(use_csr=0, use_2lvl=0, n_cams=2)),
}
ENV = ("B200SFM_RA_CSR", "B200SFM_RA_2LVL", "B200SFM_RA_FUSED")


@pytest.fixture(scope="module")
def scenes():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = SCENES[name]()
        return cache[name]
    return get


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ct.c_void_p)


def _i32(a):
    return None if a is None else np.ascontiguousarray(a, np.int32)


class Probe:
    """One resident problem (b200sfm_test_ra_problem) and its oracle counterpart."""

    def __init__(self, sc, use_weight):
        self.lib = _lib.load()
        self.ctx = E.default_context()
        self.sc = sc
        nc = sc.get("n_cams", 0)
        self.ref = RS.RASystem(sc["n_frames"], sc["ei"], sc["ej"], sc["R_rel"], sc["theta"], sc["fixed"],
                               edge_w=sc["edge_w"], use_weight=use_weight, has_grav=sc.get("has_grav"), n_cams=nc,
                               eci=sc.get("eci"), ecj=sc.get("ecj"), cam_frames=sc.get("cam_frames"))
        o = _lib.RAOpts()
        self.lib.b200sfm_ra_default_opts(ct.byref(o))
        o.use_weight = int(use_weight)
        self.keep = [_i32(sc["ei"]), _i32(sc["ej"]), _i32(sc.get("eci")), _i32(sc.get("ecj")),
                     np.ascontiguousarray(sc["R_rel"], np.float64).reshape(-1), np.ascontiguousarray(sc["edge_w"], np.float64),
                     None if sc.get("has_grav") is None else np.ascontiguousarray(sc["has_grav"], np.uint8),
                     None, None, np.ascontiguousarray(sc["theta"], np.float64).reshape(-1)]
        if nc:
            cf = sc["cam_frames"]
            self.keep[7] = np.array([0] + list(np.cumsum([len(c) for c in cf])), np.int32)
            self.keep[8] = np.array([f for c in cf for f in c], np.int32)
        k = self.keep
        h = ct.c_void_p()
        _lib.check(self.ctx.handle, self.lib.b200sfm_test_ra_problem_create(
            self.ctx.handle, ct.byref(o), sc["n_frames"], nc, len(sc["ei"]), _ptr(k[0]), _ptr(k[1]), _ptr(k[2]), _ptr(k[3]),
            _ptr(k[4]), _ptr(k[5]), _ptr(k[6]), _ptr(k[7]), _ptr(k[8]), sc["fixed"], _ptr(k[9]), ct.byref(h)))
        self.h = h
        self.n, self.E = self.ref.n, self.ref.E
        info = _lib.RAProbeInfo()
        self.agg_of = np.zeros(self.n, np.int32)
        _lib.check(self.ctx.handle, self.lib.b200sfm_test_ra_problem_info(h, ct.byref(info), _ptr(self.agg_of)))
        self.info = {f: getattr(info, f) for f, _ in info._fields_}

    def close(self):
        self.lib.b200sfm_test_ra_problem_free(self.h)

    def call(self, name, *args):
        _lib.check(self.ctx.handle, getattr(self.lib, name)(self.h, *args))

    def system(self, mode, square):
        n, E_ = self.n, self.E
        b = dict(res=np.zeros(3 * E_), w=np.zeros(E_), b=np.zeros(3 * E_), rhs=np.zeros(3 * n), deg=np.zeros(3 * n),
                 Minv=np.zeros(6 * n), Ac=np.zeros(max(self.info["nc"], 1) ** 2))
        out = _lib.RASystemProbeOut()
        for f, a in b.items():
            setattr(out, f, _ptr(a))
        self.call("b200sfm_test_ra_system", mode, SIGMA2 if mode == 1 else 0.0, square, ct.byref(out))
        b["b_norm2"] = out.b_norm2
        return b

    def vec(self, name, x):
        y = np.zeros(3 * self.n)
        self.call(name, _ptr(np.ascontiguousarray(x)), _ptr(y))
        return y

    def pcg(self, k, warm=None):
        x = np.zeros(3 * self.n)
        it = ct.c_int32()
        self.call("b200sfm_test_ra_pcg", k, _ptr(None if warm is None else np.ascontiguousarray(warm)), _ptr(x), ct.byref(it))
        return x, it.value


def blockrel(dev, ref, scale):
    """max over nodes / edges of |dev - ref| in the block, relative to the block's scale."""
    d = np.abs(np.asarray(dev) - np.asarray(ref)).reshape(len(scale), -1).max(1)
    s = np.asarray(scale)
    ok = s > 0
    assert np.all(d[~ok] == 0), "a difference where the reference block is zero"
    return float((d[ok] / s[ok]).max()) if ok.any() else 0.0


def nodemax(a):
    return np.abs(a).reshape(-1, 3).max(1)


def compare(p, err, mode, square, rng):
    ref = p.ref
    dev = p.system(mode, square)
    res = ref.residuals()
    w = ref.weights(res, mode, SIGMA2 if mode == 1 else 0.0)
    upd = lambda k, v: err.__setitem__(k, max(err.get(k, 0.0), v))   # noqa: E731
    upd("res", np.abs(dev["res"] - res.ravel()).max())              # radians
    upd("w", blockrel(dev["w"], w, np.abs(w)))
    L = ref.laplacian(w, square)
    absL = abs(L)
    rows_w = ref.row_weights(w, square)
    rhs = ref.rhs(w, square, res)
    upd("rhs", blockrel(dev["rhs"], rhs, nodemax(abs(ref.A.T) @ (rows_w * np.abs(res.ravel())))))
    if square:
        bref = np.repeat(w, 3) * res.ravel()
        upd("rhs", abs(dev["b_norm2"] - bref @ bref) / (bref @ bref))
    d, dinv = ref.jacobi(L)
    Mdev = dev["Minv"].reshape(-1, 6)
    assert np.all(Mdev[:, [1, 2, 4]] == 0)
    upd("Minv", blockrel(Mdev[:, [0, 3, 5]].ravel(), dinv, nodemax(dinv)))
    P = Ac_inv = None
    if p.info["use_2lvl"]:
        nc = p.info["nc"]
        P, Ac = ref.coarse(L, p.agg_of, nc)
        Ac_dev = dev["Ac"][:nc * nc].reshape(nc, nc)
        cond = np.linalg.cond(Ac)
        upd("Ac", np.abs(Ac_dev @ Ac - np.eye(nc)).max() / (cond * 1e-16 * nc))   # in units of cond(Ac) eps nc
        Ac_inv = np.linalg.inv(Ac)
    M = ref.precond(dinv, P, Ac_inv)
    for _ in range(3):
        x = rng.normal(size=3 * p.n)
        upd("apply", blockrel(p.vec("b200sfm_test_ra_apply", x), L @ x, nodemax(absL @ np.abs(x))))
        r = rng.normal(size=3 * p.n)
        sc = np.abs(dinv) * np.abs(r)
        if P is not None:
            sc = sc + (abs(P) @ (np.abs(Ac_inv) @ (abs(P.T) @ np.abs(r).reshape(-1, 3)))).ravel()
        upd("precond", blockrel(p.vec("b200sfm_test_ra_precond", r), M(r), nodemax(sc)))
    its, _ = ref.pcg(L, rhs, M, max(PCG_KS))
    warm = rng.normal(size=3 * p.n) * 1e-2
    warm[d == 0] = 0.0
    its_w, _ = ref.pcg(L, rhs, M, max(PCG_KS), x0=warm)
    for k in PCG_KS:
        x, it = p.pcg(k)
        assert it == k
        upd("pcg", np.abs(x - its[k - 1]).max() / np.abs(its[k - 1]).max())
        x, it = p.pcg(k, warm)
        assert it == k
        upd("pcg_warm", np.abs(x - its_w[k - 1]).max() / np.abs(its_w[k - 1]).max())
    return w, dev


def compare_admm(p, err, w, dev, rng):
    ref = p.ref
    ex = ref.row_exists.ravel()
    x = rng.normal(size=3 * p.n) * 0.05
    b = dev["b"]
    z = np.where(ex, rng.normal(size=3 * p.E) * 0.05, 0.0)
    u = np.where(ex, rng.normal(size=3 * p.E) * 0.05, 0.0)
    zr, ur, rhs, svec, uvec, nm = ref.admm_step(w, x, b, z, u, 1.0)
    zd, ud, rsu, norms = z.copy(), u.copy(), np.zeros(9 * p.n), np.zeros(5)
    p.call("b200sfm_test_ra_admm_step", 1.0, _ptr(x), _ptr(b), _ptr(zd), _ptr(ud), _ptr(rsu), _ptr(norms))
    At = abs(ref.A.T)
    W3 = np.repeat(np.abs(w), 3)
    e = max(np.abs(zd - zr).max(), np.abs(ud - ur).max()) / max(np.abs(ur).max(), 1e-300)
    for dv, rv, v in ((rsu[:3 * p.n], rhs, np.abs(b) + np.abs(zr) + np.abs(ur)), (rsu[3 * p.n:6 * p.n], svec, np.abs(zr) + np.abs(z)),
                      (rsu[6 * p.n:], uvec, np.abs(ur))):
        e = max(e, blockrel(dv, rv, nodemax(At @ (W3 * np.where(ex, v, 0.0)))))
    e = max(e, float((np.abs(norms - nm) / np.maximum(np.abs(nm), 1e-300)).max()))
    err["admm"] = max(err.get("admm", 0.0), e)


def compare_update(p, err, rng):
    ref = p.ref
    step = rng.normal(size=(p.n, 3)) * 0.02
    g = ref.grav
    step[g, 0] = step[g, 2] = 0.0
    th_ref, sums_ref = ref.update(step.ravel())
    th, sums = np.zeros(3 * p.n), np.zeros(3)
    p.call("b200sfm_test_ra_update", _ptr(step.ravel().copy()), _ptr(th), _ptr(sums))
    th = th.reshape(p.n, 3)
    # compare rotations (angle-axis near pi is ambiguous; the scenes keep |theta| small)
    err["update"] = max(err.get("update", 0.0), float(np.abs(th - th_ref).max()))
    err["sums"] = max(err.get("sums", 0.0), float((np.abs(sums - sums_ref)[:2] / sums_ref[:2]).max()))
    assert sums[2] == 0.0


def test_scene_reaches_the_shapes_it_is_built_for(scenes):
    sc = scenes("general")
    n = sc["n_frames"]
    assert n % 128 and n % 8
    deg = np.bincount(np.concatenate([sc["ei"], sc["ej"]]), minlength=n)
    for node, d in SPECIAL_DEG.items():
        assert deg[node] == d
    assert deg[ISOLATED] == 0 and deg.max() > 256
    assert scenes("general_connected")["ei"].size and np.bincount(np.concatenate(
        [scenes("general_connected")["ei"], scenes("general_connected")["ej"]]), minlength=n)[ISOLATED] == 1
    pairs = list(zip(sc["ei"], sc["ej"]))
    assert any(pairs.count(q) >= 2 for q in pairs[-3:]) and any((b, a) in pairs for a, b in pairs[-3:])
    assert sc["fixed"] != 0
    s = RS.RASystem(n, sc["ei"], sc["ej"], sc["R_rel"], sc["theta"], sc["fixed"])
    ang = np.degrees(np.linalg.norm(s.residuals(), axis=1))
    assert (ang > 120).sum() >= 2 and (ang < 10).sum() > 0.9 * len(ang)
    assert np.all(sc["theta"][[20, 21, 22]] == 0)
    for name, frac in (("gravity_all", 1.0), ("gravity_mixed", 0.6)):
        g = scenes(name)
        hg = g["has_grav"]
        assert abs(hg.mean() - frac) < 0.05
        th = g["theta"]
        both = hg[g["ei"]] & hg[g["ej"]]
        dy = th[g["ej"][both], 1] - th[g["ei"][both], 1]
        assert np.any(np.abs(dy) > np.pi)                                 # the y difference wraps around +-pi
        if frac < 1:
            assert np.any(hg[g["ei"]] != hg[g["ej"]])                     # mixed rows
    assert scenes("gravity_all")["has_grav"][FIXED] and not scenes("gravity_fixed_without")["has_grav"][FIXED]
    r = scenes("rig")
    assert np.any((r["eci"] == r["ecj"]) & (r["eci"] >= 0)) and np.any(r["ei"] == r["ej"])
    assert max(len(c) for c in r["cam_frames"]) > 32
    lg = scenes("large")
    assert lg["n_frames"] >= 20000


@pytest.mark.parametrize("name", list(PATHS))
def test_device_system_matches_the_fp64_reference(name, scenes, monkeypatch):
    scene, env, want = PATHS[name]
    for k in ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sc = scenes(scene)
    rng = np.random.default_rng(17)
    err = {}
    for use_weight in (True, False):
        p = Probe(sc, use_weight)
        try:
            info = p.info
            for k, v in want.items():
                assert info[k] == v, (k, info)
            assert info["rows_total"] == p.ref.rows_total and info["E_total"] == p.E - 1
            if info["use_2lvl"]:
                nc = info["nc"]
                assert nc > 32 and nc % 4 and nc == p.agg_of.max() + 1
                if name == "default_large":                             # ra_coarse_restrict's lane loop
                    assert np.bincount(p.agg_of).max() > 32
            w, dev = compare(p, err, 0, 1, rng)                         # the L1 stage's system
            compare_admm(p, err, w, dev, rng)
            compare(p, err, 0, 1, rng)                                   # again: the kept coarse inverse
            compare(p, err, 1, 0, rng)                                   # IRLS, Geman-McClure
            compare(p, err, 2, 0, rng)                                   # IRLS, half-norm
            compare_update(p, err, rng)
        finally:
            p.close()
    print(f"\n{name}: n={p.n} E={p.E} nc={p.info['nc']} " + " ".join(f"{k}={v:.1e}" for k, v in sorted(err.items())))
    bad = {k: v for k, v in err.items() if not v <= BOUNDS[k]}
    assert not bad, bad


def test_probe_rejects_bad_input():
    lib = _lib.load()
    ctx = E.default_context()
    o = _lib.RAOpts()
    lib.b200sfm_ra_default_opts(ct.byref(o))
    ei = np.array([0, 1], np.int32); ej_bad = np.array([1, 5], np.int32)
    R = np.tile(np.eye(3).ravel(), 2)
    th = np.zeros(9)
    h = ct.c_void_p()
    INVALID = 1
    assert lib.b200sfm_test_ra_problem_create(ctx.handle, ct.byref(o), 3, 0, 2, _ptr(ei), _ptr(ej_bad), None, None, _ptr(R),
                                              None, None, None, None, 0, _ptr(th), ct.byref(h)) == INVALID
    assert not h.value and b"out of range" in lib.b200sfm_last_error(ctx.handle)
    assert lib.b200sfm_test_ra_problem_create(ctx.handle, ct.byref(o), 3, 0, 2, _ptr(ei), _ptr(ei), None, None, _ptr(R),
                                              None, None, None, None, 3, _ptr(th), ct.byref(h)) == INVALID
    eci = np.array([-1, -1], np.int32)
    ecj_bad = np.array([-1, 1], np.int32)                                     # a frame index, not a camera node
    cfb = np.array([0, 1], np.int32); cf = np.array([0], np.int32)
    th4 = np.zeros(12)
    assert lib.b200sfm_test_ra_problem_create(ctx.handle, ct.byref(o), 3, 1, 2, _ptr(ei), _ptr(ei + 1), _ptr(eci),
                                              _ptr(ecj_bad), _ptr(R), None, None, _ptr(cfb), _ptr(cf), 0, _ptr(th4),
                                              ct.byref(h)) == INVALID
    ok = np.array([1, 2], np.int32)
    assert lib.b200sfm_test_ra_problem_create(ctx.handle, ct.byref(o), 3, 0, 2, _ptr(ei), _ptr(ok), None, None, _ptr(R),
                                              None, None, None, None, 0, _ptr(th), ct.byref(h)) == 0
    x = np.zeros(9)
    try:
        assert lib.b200sfm_test_ra_apply(h, _ptr(x), _ptr(x)) == INVALID          # no system prepared yet
        out = _lib.RASystemProbeOut()
        assert lib.b200sfm_test_ra_system(h, 3, 0.0, 1, ct.byref(out)) == INVALID
        assert lib.b200sfm_test_ra_system(h, 0, 0.0, 2, ct.byref(out)) == INVALID
        assert lib.b200sfm_test_ra_pcg(h, 0, None, _ptr(x), None) == INVALID
    finally:
        lib.b200sfm_test_ra_problem_free(h)
