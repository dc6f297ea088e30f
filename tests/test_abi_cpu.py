"""CPU checks of the drop-in boundary: the C-ABI library is built, loads, and
exports every symbol include/b200sfm.h declares (no compute calls: no GPU)."""
import ctypes as ct
import os
import re

from glomap_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "b200sfm.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200sfm_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    syms = declared_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/b200sfm.h but not exported"


def test_python_prototypes_cover_header():
    assert set(declared_symbols()) == set(_lib.PROTOTYPES), set(declared_symbols()) ^ set(_lib.PROTOTYPES)


def test_version_and_struct_sizes():
    lib = _lib.load()
    assert lib.b200sfm_version() == 100
    o = _lib.BAOpts()
    lib.b200sfm_ba_default_opts(ct.byref(o))
    # defaults mirror bundle_adjustment.h:14-32 / optimization_base.h:18-23
    assert (o.optimize_rotations, o.optimize_translation, o.optimize_intrinsics, o.optimize_principal_point,
            o.optimize_points, o.optimize_rig_poses) == (1, 1, 1, 0, 1, 0)
    assert o.min_num_view_per_track == 3 and o.max_num_iterations == 200
    assert o.thres_loss_function == 1.0 and o.function_tolerance == 1e-5


def test_no_cpu_fallback_without_device():
    """On a box without a GPU the context creation must fail loudly."""
    import torch
    if torch.cuda.is_available():
        return
    lib = _lib.load()
    h = ct.c_void_p()
    assert lib.b200sfm_create(0, ct.byref(h)) != 0
    assert not h.value


def test_ctypes_structs_match_the_c_header(tmp_path):
    """Compile a tiny C program against include/b200sfm.h and compare sizeof /
    offsetof of every struct with the ctypes mirrors (ABI drift guard)."""
    import subprocess
    structs = {"b200sfm_lm_stats": _lib.LMStats, "b200sfm_ba_opts": _lib.BAOpts, "b200sfm_gp_opts": _lib.GPOpts,
               "b200sfm_ra_opts": _lib.RAOpts, "b200sfm_ra_stats": _lib.RAStats}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "b200sfm.h")}"', "int main(void) {"]
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    subprocess.check_call(["/usr/bin/gcc", "-std=c11", "-o", str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, cls in structs.items():
        assert int(out[cname]) == ct.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(out[f"{cname}.{fname}"]) == getattr(cls, fname).offset, f"{cname}.{fname}"


def test_header_is_plain_c99(tmp_path):
    """The boundary is a C ABI: the header must compile as C (no C++-isms outside the extern "C" guards)."""
    import subprocess
    src = tmp_path / "hdr.c"
    src.write_text('#include "b200sfm.h"\nint main(void) { b200sfm_ba_opts o; b200sfm_lm_stats s; (void)o; (void)s; return 0; }\n')
    r = subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only",
                        "-I" + os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_null_arguments_are_rejected_without_touching_the_device():
    """Every entry point validates its handles before any CUDA call: callable on a box without a GPU."""
    lib = _lib.load()
    INVALID = 1   # B200SFM_ERR_INVALID_ARG
    st, ra_st = _lib.LMStats(), _lib.RAStats()
    o_ba, o_gp, o_ra = _lib.BAOpts(), _lib.GPOpts(), _lib.RAOpts()
    h = ct.c_void_p()
    assert lib.b200sfm_create(0, None) == INVALID
    assert lib.b200sfm_ba_problem_create(None, 1, 1, 1, 1, None, None, None, None, None, None, 3, ct.byref(h)) == INVALID
    assert lib.b200sfm_ba_problem_create_rig(None, 1, 1, 1, 1, 1, None, None, None, None, None, None, None, None, None, 3,
                                             ct.byref(h)) == INVALID
    assert lib.b200sfm_ba_problem_solve(None, ct.byref(o_ba), ct.byref(st)) == INVALID
    assert lib.b200sfm_ba_problem_set_state(None, None, None, None, None) == INVALID
    assert lib.b200sfm_ba_problem_filter_reprojection(None, 1.0, None, None) == INVALID
    assert lib.b200sfm_ba_problem_filter_reprojection_normalized(None, None, 1.0, None, None) == INVALID
    assert lib.b200sfm_ba_problem_filter_angle(None, None, None, 1.0, None, None) == INVALID
    assert lib.b200sfm_ba_problem_filter_triangulation_angle(None, 1.0, None, None) == INVALID
    assert lib.b200sfm_gp_problem_create(None, 1, 1, 1, None, None, None, None, None, 3, ct.byref(h)) == INVALID
    assert lib.b200sfm_gp_problem_set_rig_terms(None, None, None) == INVALID
    assert lib.b200sfm_gp_problem_solve(None, ct.byref(o_gp), ct.byref(st)) == INVALID
    assert lib.b200sfm_ba_solve(None, ct.byref(o_ba), 1, 1, 1, 1, *([None] * 10), ct.byref(st)) == INVALID
    assert lib.b200sfm_gp_solve(None, ct.byref(o_gp), 1, 1, 1, *([None] * 8), ct.byref(st)) == INVALID
    assert lib.b200sfm_ra_solve(None, ct.byref(o_ra), 1, 1, None, None, None, None, 0, None, ct.byref(ra_st)) == INVALID
    assert lib.b200sfm_last_error(None) == b"null context" or lib.b200sfm_last_error(None) is not None
    lib.b200sfm_ba_problem_free(None); lib.b200sfm_gp_problem_free(None); lib.b200sfm_destroy(None)   # no-ops
    assert lib.b200sfm_rank(None) == -1 and lib.b200sfm_world_size(None) == -1 and lib.b200sfm_kernel_launches(None) == 0


# ---- the test-only probe (include/b200sfm_testing.h): exported, mirrored, plain C, validated before any CUDA call ----
def testing_symbols():
    src = open(os.path.join(ROOT, "include", "b200sfm_testing.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200sfm_test_[a-z0-9_]+)\s*\(", src)))


def test_testing_header_symbols_are_exported_and_mirrored():
    lib = _lib.load()
    syms = testing_symbols()
    assert syms == sorted(_lib.TEST_PROTOTYPES), syms
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/b200sfm_testing.h but not exported"
    assert not set(syms) & set(declared_symbols())      # not part of the drop-in ABI


def test_testing_header_is_plain_c99_and_its_struct_matches_ctypes(tmp_path):
    import subprocess
    structs = {"b200sfm_test_ba_step_out": _lib.BAStepProbeOut, "b200sfm_test_ra_info": _lib.RAProbeInfo,
               "b200sfm_test_ra_system_out": _lib.RASystemProbeOut, "b200sfm_test_gp_step_out": _lib.GPStepProbeOut}
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "b200sfm_testing.h"', "int main(void) {"]
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        lines += [f'  printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror",
                           "-I" + os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, cls in structs.items():
        assert int(out[cname]) == ct.sizeof(cls), cname
        for f, _ in cls._fields_:
            assert int(out[f"{cname}.{f}"]) == getattr(cls, f).offset, f"{cname}.{f}"


def test_probe_rejects_a_null_problem_without_touching_the_device():
    lib = _lib.load()
    INVALID = 1   # B200SFM_ERR_INVALID_ARG
    o, out = _lib.BAOpts(), _lib.BAStepProbeOut()
    x = (ct.c_double * 6)()
    assert lib.b200sfm_test_ba_step(None, ct.byref(o), 0.0, 1e4, ct.byref(out)) == INVALID
    assert lib.b200sfm_test_ba_apply(None, x, x) == INVALID
    # rotation averaging (out-of-range indices with a live context: tests/test_ra_system_gpu.py)
    o_ra, info, sysout = _lib.RAOpts(), _lib.RAProbeInfo(), _lib.RASystemProbeOut()
    h = ct.c_void_p()
    ei = (ct.c_int32 * 1)(0)
    R = (ct.c_double * 9)(1, 0, 0, 0, 1, 0, 0, 0, 1)
    th = (ct.c_double * 6)()
    assert lib.b200sfm_test_ra_problem_create(None, ct.byref(o_ra), 2, 0, 1, ei, ei, None, None, R, None, None, None,
                                              None, 0, th, ct.byref(h)) == INVALID
    assert not h.value
    lib.b200sfm_test_ra_problem_free(None)   # no-op
    assert lib.b200sfm_test_ra_problem_info(None, ct.byref(info), None) == INVALID
    assert lib.b200sfm_test_ra_system(None, 0, 0.0, 1, ct.byref(sysout)) == INVALID
    assert lib.b200sfm_test_ra_apply(None, x, x) == INVALID
    assert lib.b200sfm_test_ra_precond(None, x, x) == INVALID
    assert lib.b200sfm_test_ra_pcg(None, 1, None, x, None) == INVALID
    assert lib.b200sfm_test_ra_admm_step(None, 1.0, x, x, x, x, x, x) == INVALID
    assert lib.b200sfm_test_ra_update(None, x, x, x) == INVALID
    # global positioning
    o_gp, gp_out = _lib.GPOpts(), _lib.GPStepProbeOut()
    assert lib.b200sfm_test_gp_step(None, ct.byref(o_gp), 0.0, 1e4, 1.0, ct.byref(gp_out)) == INVALID
    assert lib.b200sfm_test_gp_apply(None, x, x) == INVALID
