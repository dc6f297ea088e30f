"""The mpmath references of oracle/gravity_mp.py against the numpy oracles on well-conditioned inputs, against closed
forms and finite differences; the ctypes mirror of the gravity probe's struct against include/b200sfm_testing.h."""
import ctypes as ct
import math
import os
import subprocess

import mpmath as mp
import numpy as np

from glomap_b200 import _lib, geometry as geo
from glomap_b200.gravity_refinement import get_align_rot_householder
from oracle import gravity_mp as GM, gravity_oracle as GO, rig_init_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = float(np.finfo(np.float64).eps)


def f(v):
    return np.array([float(t) for t in v])


def test_manifold_operations_match_the_numpy_oracle():
    rng = np.random.default_rng(1)
    for _ in range(20):
        x = rng.normal(size=3)
        v, beta, _ = GM.householder(x)
        vn, bn = GO.householder(x)
        assert np.allclose(f(v), vn, rtol=1e-13) and abs(float(beta) - bn) <= 1e-13 * abs(bn) + 1e-300
        d = rng.normal(size=2) * 0.3
        assert np.allclose(f(GM.sphere_plus(x, d)), GO.sphere_plus(x, d), rtol=1e-13, atol=1e-15)
        assert np.allclose(f(GM.sphere_plus_jacobian(x)), GO.sphere_plus_jacobian(x).ravel(), rtol=1e-13, atol=1e-15)


def test_householder_reflects_x_onto_e3_and_plus_stays_on_the_sphere():
    for x in ([0.3, -0.4, 0.5], [0.3, 0.4, -0.5], [0, 0, -2.0], [0, 0, 3.0], [2 ** -26 * 1.01, 0, 1], [1e-7, 0, -1]):
        v, beta, branch = GM.householder(x)
        with mp.workdps(50):
            xv = GM._v(x)
            vx = sum(a * b for a, b in zip(v, xv))
            hx = [xv[k] - beta * v[k] * vx for k in range(3)]
            nx = mp.sqrt(sum(t * t for t in xv))
            assert abs(hx[0]) < 1e-40 and abs(hx[1]) < 1e-40 and abs(hx[2] - nx) < 1e-40 * nx   # exact off the e3 branch
            assert branch != 0 or x[0] == x[1] == 0
            p = GM.sphere_plus(x, [0.7, -1.1])
            assert abs(mp.sqrt(sum(t * t for t in p)) - nx) < 1e-40


def test_plus_jacobian_matches_finite_differences():
    for x in ([0.3, -0.4, 0.5], [0.3, 0.4, -0.5], [0, 0, 1.0], [0, 0, -1.0], [0.6, 0.0, 0.8], [1e-9, 2e-9, -1.0]):
        J = GM.sphere_plus_jacobian(x)
        Jd = GM.sphere_plus_jacobian_fd(x)
        assert max(abs(a - b) for a, b in zip(J, Jd)) < 1e-20


def test_eigenvectors_of_a_known_basis():
    rng = np.random.default_rng(2)
    for n in (3, 4):
        Q = np.linalg.qr(rng.normal(size=(n, n)))[0]
        lam = np.array([0.1, 0.5, 2.0, 3.0][:n])
        A = Q @ np.diag(lam) @ Q.T
        E, V = GM.eig_sym(A)
        assert np.allclose(f(E), lam, atol=1e-14)
        v, gap = GM.dominant(A)
        assert GM.angle_to(v, Q[:, -1]) < 1e-14
        assert abs(float(gap) - (lam[-1] - lam[-2]) / lam[-1]) < 1e-14


def test_pair_angle_closed_forms_and_the_numpy_oracle():
    for a in (0.0, 1e-3, 1.0, 45.0, 179.0):
        for axis in (0, 2):
            w = np.zeros(3)
            w[axis] = math.radians(a)
            up, ang = GM.pair_angle(geo.so3_exp(w[None])[0])
            assert abs(float(ang) - a) < 1e-12 and abs(float(up)) < 1e-15
        R = geo.so3_exp(np.array([[0.0, math.radians(a), 0.0]]))[0]   # a pure up rotation: angle 0
        up, ang = GM.pair_angle(R)
        assert abs(float(up) - math.radians(a)) < 1e-14 and abs(float(ang)) < 1e-6
    rng = np.random.default_rng(3)
    Ra = get_align_rot_householder(rng.normal(size=(6, 3)))
    M = geo.so3_exp(rng.normal(size=(5, 3)))
    f1, f2 = np.zeros(5, np.int64), np.arange(1, 6)
    want = GO.pair_angles(Ra, f1, f2, M)
    R = np.swapaxes(Ra[f2], -1, -2) @ M @ Ra[f1]
    got = np.array([float(GM.pair_angle(r)[1]) for r in R])
    assert np.abs(got - want).max() < 1e-9


def test_average_gravity_matches_the_numpy_oracle():
    rng = np.random.default_rng(4)
    g0 = np.array([0.1, 0.98, 0.2])
    g0 /= np.linalg.norm(g0)
    for n in (7, 8):
        gs = g0[None] + rng.normal(size=(n, 3)) * 0.02
        gs[:3] *= -1
        x, gap, margin = GM.average_gravity(gs, g0)
        assert np.allclose(f(x), GO.average_gravity(gs, g0), atol=1e-13) and margin > 0.5 and float(gap) > 0.9


class _Opts:
    max_gravity_error = 1.0
    max_num_iterations = 100
    function_tolerance = 1e-5
    gradient_tolerance = 1e-10
    parameter_tolerance = 1e-8


def test_lm_restatement_matches_the_numpy_lm():
    rng = np.random.default_rng(5)
    g0 = np.array([0.2, 0.95, -0.1])
    g0 /= np.linalg.norm(g0)
    gs = g0[None] + rng.normal(size=(15, 3)) * math.radians(0.5)
    gs /= np.linalg.norm(gs, axis=1, keepdims=True)
    x0 = GO.average_gravity(gs, g0)
    ref = GM.lm_trace(gs, x0, _Opts())
    x, summ = GO.solve_sphere_lm(gs, x0, GO.GravityOptions())
    assert ref["iterations"] == summ.iterations and not ref["near"]
    assert GM.angle_to(ref["x"], x) < 1e-9
    accepted = [t[0] for t in ref["trace"] if t[4] == 1]
    assert np.allclose(accepted, summ.costs[:len(accepted)], rtol=1e-12)
    fp = GM.lm_trace(gs, x0, _Opts(), fp64=True)   # the FP64 evaluation follows the same path
    assert fp["iterations"] == ref["iterations"] and [t[4] for t in fp["trace"]] == [t[4] for t in ref["trace"]]
    assert np.allclose([t[0] for t in fp["trace"]], [t[0] for t in ref["trace"]], rtol=1e-14)


def test_rig_samples_and_average_match_the_numpy_oracle():
    rng = np.random.default_rng(6)
    base = rng.normal(size=4)
    for n in (1, 2, 9):
        qi = base[None] + rng.normal(size=(n, 4)) * 0.05
        qr = rng.normal(size=(n, 4))
        s = [GM.cam_sample(a, b) for a, b in zip(qi, qr)]
        sn = [RO._qmul(RO._unit(a), RO._conj(RO._unit(b))) for a, b in zip(qi, qr)]
        assert np.allclose(np.array([f(t) for t in s]), np.array(sn) / np.linalg.norm(sn, axis=1, keepdims=True), atol=1e-15)
        v, gap = GM.average_quaternions(s)
        assert np.allclose(f(v), RO.average_quaternions(sn), atol=1e-13) and float(v[3]) >= 0


def test_gravity_probe_struct_matches_the_header(tmp_path):
    cls = _lib.GravityProbeOut
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "b200sfm_testing.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(b200sfm_test_gravity_out));']
    lines += [f'  printf("{n} %zu\\n", offsetof(b200sfm_test_gravity_out, {n}));' for n, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                           "-I" + os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(out["size"]) == ct.sizeof(cls)
    for n, _ in cls._fields_:
        assert int(out[n]) == getattr(cls, n).offset, n


def test_gravity_probes_reject_bad_arguments_without_touching_the_device():
    lib = _lib.load()
    o, out = _lib.GravityOpts(), _lib.GravityProbeOut()
    x = (ct.c_double * 14)()
    i = (ct.c_int32 * 1)(0)
    u = (ct.c_uint8 * 1)(1)
    assert lib.b200sfm_test_gravity(None, ct.byref(o), 1, x, u, 1, i, i, x, ct.byref(out)) == 1
    assert lib.b200sfm_test_device_helpers(None, 0, 1, x, x) == 1
