"""ctypes binding of libb200sfm.so (include/b200sfm.h).  Fails loudly when the
CUDA library has not been built -- there is no CPU fallback."""
from __future__ import annotations

import ctypes as ct
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200SFM_LIB", os.path.join(_HERE, "libb200sfm.so"))   # env override: tuning builds, other revisions, test doubles

INTR_STRIDE = 12
NCCL_ID_BYTES = 128

c_int32, c_int64, c_double, c_void_p = ct.c_int32, ct.c_int64, ct.c_double, ct.c_void_p
P = ct.POINTER


class LMStats(ct.Structure):
    _fields_ = [
        ("iterations", c_int32), ("num_successful_steps", c_int32), ("termination", c_int32), ("usable", c_int32),
        ("initial_cost", c_double), ("final_cost", c_double),
        ("num_observations", c_int64), ("pcg_iterations", c_int64), ("kernel_launches", c_int64),
        ("ms_total", c_double), ("ms_linearize", c_double), ("n_linearize", c_int64),
        ("ms_matvec", c_double), ("n_matvec", c_int64),
        ("ms_h2d", c_double), ("ms_d2h", c_double), ("h2d_bytes", c_int64), ("d2h_bytes", c_int64),
    ]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class BAOpts(ct.Structure):
    _fields_ = [
        ("optimize_rig_poses", c_int32), ("optimize_rotations", c_int32), ("optimize_translation", c_int32),
        ("optimize_intrinsics", c_int32), ("optimize_principal_point", c_int32), ("optimize_points", c_int32),
        ("min_num_view_per_track", c_int32), ("max_num_iterations", c_int32),
        ("thres_loss_function", c_double), ("function_tolerance", c_double), ("gradient_tolerance", c_double),
        ("parameter_tolerance", c_double),
        ("pcg_max_iterations", c_int32), ("pcg_min_iterations", c_int32), ("pcg_rel_tolerance", c_double),
        ("preconditioner", c_int32), ("profile_kernels", c_int32), ("fixed_num_iterations", c_int32),
        ("design", c_int32),
    ]


class GPOpts(ct.Structure):
    _fields_ = [
        ("optimize_positions", c_int32), ("optimize_points", c_int32), ("optimize_scales", c_int32),
        ("min_num_view_per_track", c_int32), ("max_num_iterations", c_int32),
        ("max_num_line_search_step_size_iterations", c_int32),
        ("thres_loss_function", c_double), ("function_tolerance", c_double), ("gradient_tolerance", c_double),
        ("parameter_tolerance", c_double),
        ("pcg_max_iterations", c_int32), ("pcg_min_iterations", c_int32), ("pcg_rel_tolerance", c_double),
        ("preconditioner", c_int32), ("profile_kernels", c_int32), ("fixed_num_iterations", c_int32),
        ("reserved0", c_int32),
    ]


class RAOpts(ct.Structure):
    _fields_ = [
        ("max_num_l1_iterations", c_int32), ("max_num_irls_iterations", c_int32), ("weight_type", c_int32),
        ("use_weight", c_int32), ("l1_step_convergence_threshold", c_double),
        ("irls_step_convergence_threshold", c_double), ("irls_loss_parameter_sigma", c_double),
        ("l1_max_admm_iterations", c_int32), ("reserved0", c_int32), ("l1_rho", c_double),
        ("l1_absolute_tolerance", c_double), ("l1_relative_tolerance", c_double),
        ("pcg_max_iterations", c_int32), ("reserved1", c_int32), ("pcg_rel_tolerance", c_double),
    ]


class VGCOpts(ct.Structure):
    _fields_ = [
        ("max_num_iterations", c_int32), ("max_num_line_search_step_size_iterations", c_int32),
        ("thres_loss_function", c_double), ("function_tolerance", c_double), ("gradient_tolerance", c_double),
        ("parameter_tolerance", c_double), ("thres_lower_ratio", c_double), ("thres_higher_ratio", c_double),
        ("thres_two_view_error", c_double),
        ("pcg_max_iterations", c_int32), ("pcg_min_iterations", c_int32), ("pcg_rel_tolerance", c_double),
        ("profile_kernels", c_int32), ("reserved0", c_int32),
    ]


class RAStats(ct.Structure):
    _fields_ = [
        ("l1_iterations", c_int32), ("irls_iterations", c_int32), ("admm_iterations", c_int32), ("usable", c_int32),
        ("num_edges", c_int64), ("pcg_iterations", c_int64), ("kernel_launches", c_int64), ("ms_total", c_double),
    ]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class MSTStats(ct.Structure):
    _fields_ = [
        ("num_reached", c_int32), ("num_tree_edges", c_int32), ("boruvka_rounds", c_int32), ("max_depth", c_int32),
        ("kernel_launches", c_int64), ("ms_total", c_double),
    ]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class RigInitStats(ct.Structure):
    _fields_ = [
        ("num_ref_frames", c_int32), ("num_cam_samples", c_int32), ("num_cams_averaged", c_int32),
        ("num_frame_samples", c_int32), ("num_frames_averaged", c_int32), ("reserved0", c_int32),
        ("kernel_launches", c_int64), ("ms_total", c_double),
    ]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_ if f != "reserved0"}


class PruneStats(ct.Structure):
    _fields_ = [
        ("covisible_pairs", c_int64), ("pairs_min5", c_int64), ("visibility_edges", c_int64), ("strong_threshold", c_double),
        ("clustering_iterations", c_int32), ("largest_component_frames", c_int32),
    ]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class GravityOpts(ct.Structure):
    _fields_ = [
        ("max_outlier_ratio", c_double), ("max_gravity_error", c_double), ("min_num_neighbors", c_int32),
        ("max_num_iterations", c_int32), ("function_tolerance", c_double), ("gradient_tolerance", c_double),
        ("parameter_tolerance", c_double), ("reserved", c_int32 * 4),
    ]


class GravityStats(ct.Structure):
    _fields_ = [
        ("error_prone_frames", c_int32), ("rectified_frames", c_int32), ("too_few_terms", c_int32),
        ("max_lm_iterations", c_int32), ("lm_iterations", c_int64), ("ms_total", c_double), ("ms_h2d", c_double),
        ("ms_error_test", c_double), ("ms_csr", c_double), ("ms_refine", c_double),
    ]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


# name -> (restype, argtypes); every symbol include/b200sfm.h declares
PROTOTYPES = {
    "b200sfm_version": (c_int32, []),
    "b200sfm_create": (c_int32, [c_int32, P(c_void_p)]),
    "b200sfm_nccl_unique_id": (c_int32, [c_void_p]),
    "b200sfm_create_dist": (c_int32, [c_int32, c_int32, c_int32, c_void_p, P(c_void_p)]),
    "b200sfm_destroy": (None, [c_void_p]),
    "b200sfm_last_error": (ct.c_char_p, [c_void_p]),
    "b200sfm_rank": (c_int32, [c_void_p]),
    "b200sfm_world_size": (c_int32, [c_void_p]),
    "b200sfm_cuda_stream": (c_void_p, [c_void_p]),
    "b200sfm_kernel_launches": (c_int64, [c_void_p]),
    "b200sfm_ba_default_opts": (None, [P(BAOpts)]),
    "b200sfm_ba_solve": (c_int32, [c_void_p, P(BAOpts), c_int32, c_int32, c_int64, c_int32] + [c_void_p] * 10 + [P(LMStats)]),
    "b200sfm_ba_problem_create": (c_int32, [c_void_p, c_int32, c_int32, c_int64, c_int32] + [c_void_p] * 6 + [c_int32, P(c_void_p)]),
    "b200sfm_ba_problem_create_rig": (c_int32, [c_void_p, c_int32, c_int32, c_int64, c_int32, c_int32] + [c_void_p] * 9 + [c_int32, P(c_void_p)]),
    "b200sfm_ba_problem_set_images": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p]),
    "b200sfm_ba_problem_set_sensor_variable": (c_int32, [c_void_p, c_void_p]),
    "b200sfm_ba_problem_get_sensor_poses": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "b200sfm_ba_problem_set_state": (c_int32, [c_void_p] * 5),
    "b200sfm_ba_problem_get_state": (c_int32, [c_void_p] * 5),
    "b200sfm_ba_problem_save_state": (c_int32, [c_void_p]),
    "b200sfm_ba_problem_restore_state": (c_int32, [c_void_p]),
    "b200sfm_ba_problem_solve": (c_int32, [c_void_p, P(BAOpts), P(LMStats)]),
    "b200sfm_ba_problem_cost": (c_int32, [c_void_p, P(BAOpts), P(c_double)]),
    "b200sfm_ba_problem_free": (None, [c_void_p]),
    "b200sfm_ba_problem_filter_reprojection": (c_int32, [c_void_p, c_double, c_void_p, P(c_int64)]),
    "b200sfm_ba_problem_filter_reprojection_normalized": (c_int32, [c_void_p, c_void_p, c_double, c_void_p, P(c_int64)]),
    "b200sfm_ba_problem_filter_angle": (c_int32, [c_void_p, c_void_p, c_void_p, c_double, c_void_p, P(c_int64)]),
    "b200sfm_ba_problem_filter_triangulation_angle": (c_int32, [c_void_p, c_double, c_void_p, P(c_int64)]),
    "b200sfm_ba_problem_normalize": (c_int32, [c_void_p, c_int32, c_double, c_double, c_double, P(c_double), c_void_p]),
    "b200sfm_ba_problem_undistort": (c_int32, [c_void_p, c_void_p]),
    "b200sfm_undistort_features": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "b200sfm_tracks_establish": (c_int32, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_double, P(c_void_p),
                                           P(c_int64), P(c_int64), P(c_int64)]),
    "b200sfm_tracks_get": (c_int32, [c_void_p] * 5),
    "b200sfm_image_pairs_inlier_count": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                                   c_int64] + [c_void_p] * 9 + [c_double] * 3 + [c_void_p] * 3),
    "b200sfm_view_graph_filter_rotations": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p, c_int64] + [c_void_p] * 3
                                            + [c_double, c_void_p, P(c_int64)]),
    "b200sfm_view_graph_keep_largest_component": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_int64] + [c_void_p] * 4
                                                  + [P(c_int32)]),
    "b200sfm_view_graph_update_pairs_config": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_int64] + [c_void_p] * 7
                                              + [P(c_int64)]),
    "b200sfm_tracks_free": (None, [c_void_p]),
    "b200sfm_tracks_select": (c_int32, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int32, c_void_p] + [c_int32] * 4
                              + [c_void_p, P(c_int64)]),
    "b200sfm_gp_default_opts": (None, [P(GPOpts)]),
    "b200sfm_gp_solve": (c_int32, [c_void_p, P(GPOpts), c_int32, c_int32, c_int64] + [c_void_p] * 8 + [P(LMStats)]),
    "b200sfm_gp_problem_create": (c_int32, [c_void_p, c_int32, c_int32, c_int64] + [c_void_p] * 5 + [c_int32, P(c_void_p)]),
    "b200sfm_gp_problem_set_rig_terms": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "b200sfm_gp_problem_set_rig_unknown": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p, c_void_p]),
    "b200sfm_gp_problem_get_rig_unknown": (c_int32, [c_void_p, c_void_p]),
    "b200sfm_gp_problem_set_state": (c_int32, [c_void_p] * 4),
    "b200sfm_gp_problem_get_state": (c_int32, [c_void_p] * 4),
    "b200sfm_gp_problem_save_state": (c_int32, [c_void_p]),
    "b200sfm_gp_problem_restore_state": (c_int32, [c_void_p]),
    "b200sfm_gp_problem_solve": (c_int32, [c_void_p, P(GPOpts), P(LMStats)]),
    "b200sfm_gp_problem_free": (None, [c_void_p]),
    "b200sfm_ra_default_opts": (None, [P(RAOpts)]),
    "b200sfm_ra_solve": (c_int32, [c_void_p, P(RAOpts), c_int32, c_int64] + [c_void_p] * 4 + [c_int32, c_void_p, P(RAStats)]),
    "b200sfm_ra_solve_rig": (c_int32, [c_void_p, P(RAOpts), c_int32, c_int32, c_int64] + [c_void_p] * 8 + [c_int32, c_void_p, P(RAStats)]),
    "b200sfm_ra_mst_init": (c_int32, [c_void_p, c_int32, c_int64] + [c_void_p] * 4 + [c_int32, c_void_p, c_void_p, P(MSTStats)]),
    "b200sfm_rig_rotations_from_images": (c_int32, [c_void_p, c_int64, c_int32, c_int32] + [c_void_p] * 10 + [P(RigInitStats)]),
    "b200sfm_vgc_default_opts": (None, [P(VGCOpts)]),
    "b200sfm_view_graph_calibrate": (c_int32, [c_void_p, P(VGCOpts), c_int32, c_void_p, c_void_p, c_void_p, c_int64]
                                     + [c_void_p] * 6 + [P(LMStats)]),
    "b200sfm_prune_weakly_connected": (c_int32, [c_void_p, c_int32, c_int64, c_void_p, c_void_p, c_void_p, c_int32, c_int64]
                                       + [c_void_p] * 3 + [P(PruneStats)]),
    "b200sfm_ra_solve_gravity": (c_int32, [c_void_p, P(RAOpts), c_int32, c_int64] + [c_void_p] * 5 + [c_int32, c_void_p, P(RAStats)]),
    "b200sfm_gravity_default_opts": (None, [P(GravityOpts)]),
    "b200sfm_gravity_refine": (c_int32, [c_void_p, P(GravityOpts), c_int32, c_void_p, c_void_p, c_int64] + [c_void_p] * 5
                               + [P(GravityStats)]),
}


class BAStepProbeOut(ct.Structure):
    """b200sfm_test_ba_step_out (include/b200sfm_testing.h)."""
    _fields_ = [(f, c_void_p) for f in ("U", "g_c", "jscale_c", "V", "g_p", "jscale_p", "Dc", "Minv", "b", "px",
                                        "cand_points", "cand_quat", "cand_trans", "cand_intr", "cand_sensor_quat",
                                        "cand_sensor_trans")] + \
              [(f, c_double) for f in ("cost", "gmax", "model_cost_change", "cand_cost", "step_norm", "x_norm")] + \
              [(f, c_int32) for f in ("pcg_iterations", "use_v2", "use_ell", "kfast", "nk", "ext", "ext_k", "ext_s",
                                      "schur_jacobi", "nbk")]


class RAProbeInfo(ct.Structure):
    """b200sfm_test_ra_info (include/b200sfm_testing.h)."""
    _fields_ = [(f, c_int32) for f in ("n", "n_frames", "n_cams", "has_grav", "use_csr", "use_2lvl", "fused", "nc")] + \
              [("rows_total", c_int64), ("E_total", c_int64)]


class RASystemProbeOut(ct.Structure):
    """b200sfm_test_ra_system_out (include/b200sfm_testing.h)."""
    _fields_ = [(f, c_void_p) for f in ("res", "w", "b", "rhs", "deg", "Minv", "Ac")] + [("b_norm2", c_double)]


class GPStepProbeOut(ct.Structure):
    """b200sfm_test_gp_step_out (include/b200sfm_testing.h)."""
    _fields_ = [(f, c_void_p) for f in ("M", "bw", "jscale_s", "ds", "Vinv", "gX", "Dp", "jscale_p", "dX", "U", "gc", "Dc",
                                        "Minv", "jscale_c", "b", "px", "resid", "cand_centers", "cand_points",
                                        "cand_scales", "cand_ucen")] + \
              [(f, c_double) for f in ("cost", "gmax", "g_dot_delta", "model_cost_change", "cand_cost", "step_norm",
                                       "x_norm")] + \
              [(f, c_int32) for f in ("pcg_iterations", "schur_jacobi", "CB", "n_us", "pcg_depth")]


class GravityProbeOut(ct.Structure):
    """b200sfm_test_gravity_out (include/b200sfm_testing.h)."""
    _fields_ = [(f, c_void_p) for f in ("mistake", "angle", "offs", "inc", "total", "mistakes", "error_prone", "ep", "gobs",
                                        "x", "status", "iterations", "trace")] + \
              [("trace_cap", c_int32), ("n_error_prone", c_int32)]


# name -> (restype, argtypes); the test-only probe of include/b200sfm_testing.h (not part of the drop-in ABI)
TEST_PROTOTYPES = {
    "b200sfm_test_ba_step": (c_int32, [c_void_p, P(BAOpts), c_double, c_double, P(BAStepProbeOut)]),
    "b200sfm_test_ba_apply": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "b200sfm_test_ra_problem_create": (c_int32, [c_void_p, P(RAOpts), c_int32, c_int32, c_int64] + [c_void_p] * 9
                                       + [c_int32, c_void_p, P(c_void_p)]),
    "b200sfm_test_ra_problem_free": (None, [c_void_p]),
    "b200sfm_test_ra_problem_info": (c_int32, [c_void_p, P(RAProbeInfo), c_void_p]),
    "b200sfm_test_ra_system": (c_int32, [c_void_p, c_int32, c_double, c_int32, P(RASystemProbeOut)]),
    "b200sfm_test_ra_apply": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "b200sfm_test_ra_precond": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "b200sfm_test_ra_pcg": (c_int32, [c_void_p, c_int32, c_void_p, c_void_p, P(c_int32)]),
    "b200sfm_test_ra_admm_step": (c_int32, [c_void_p, c_double] + [c_void_p] * 6),
    "b200sfm_test_ra_update": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "b200sfm_test_gp_step": (c_int32, [c_void_p, P(GPOpts), c_double, c_double, c_double, P(GPStepProbeOut)]),
    "b200sfm_test_gp_apply": (c_int32, [c_void_p, c_void_p, c_void_p]),
    "b200sfm_test_gravity": (c_int32, [c_void_p, P(GravityOpts), c_int32, c_void_p, c_void_p, c_int64] + [c_void_p] * 3
                             + [P(GravityProbeOut)]),
    "b200sfm_test_device_helpers": (c_int32, [c_void_p, c_int32, c_int64, c_void_p, c_void_p]),
}

_lib = None


def _not_exported(name: str):
    def call(*_args):
        raise RuntimeError(f"{name} is not exported by {LIB_PATH}")
    return call


def load() -> ct.CDLL:
    """Load libb200sfm.so and bind every prototype (the test probe's included).  Raises if the library is missing, or
    if the shipped library lacks an entry point.  A library named by B200SFM_LIB (a tuning build, another revision, a
    host-side test double) may implement part of the ABI: an entry it does not export raises when it is called."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(glomap_b200 has no CPU fallback)")
    lib = ct.CDLL(LIB_PATH)
    override = "B200SFM_LIB" in os.environ
    for name, (res, args) in PROTOTYPES.items():
        if override and not hasattr(lib, name):
            setattr(lib, name, _not_exported(name))
            continue
        fn = getattr(lib, name)      # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    # the probe is bound where it is exported (libb200sfm.so always exports it; the host-side mock library does not)
    for name, (res, args) in TEST_PROTOTYPES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
    _lib = lib
    return lib


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200sfm status {code}: {msg}")
        self.code = code


def check(ctx, rc: int):
    if rc != 0:
        msg = load().b200sfm_last_error(ctx).decode() if ctx else ""
        raise B200Error(rc, msg)
