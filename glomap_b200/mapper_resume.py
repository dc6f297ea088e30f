"""``glomap mapper_resume`` (exe/global_mapper.cc:110-172): the global mapper resumed from a COLMAP model.

    python -m glomap_b200.mapper_resume --input_path MODEL --output_path OUT [--output_format bin|txt] [options]

Reads the model (binary or text, with or without rigs.bin / frames.bin; ``colmap_io``), runs ``GlobalMapper.Solve``
with the resume skips of OptionManager::AddGlobalMapperResumeOptions (controllers/option_manager.cc:99-132: no
preprocessing, view-graph calibration, relative poses, rotation averaging, track establishment or retriangulation),
an empty view graph and the model's registration, then writes ``OUT/0``, or ``OUT/<cluster>`` with
``--skip_pruning 0`` (io/colmap_io.cc:17-66).  What runs is global positioning, the three track filters,
normalisation, the staged bundle adjustment, the final filters and pruning -- every solve, filter and normalisation
through ``libb200sfm.so``, as in ``mapper.py``; this module only parses, converts and writes.

Every camera is treated as having no prior focal length (``camera_prior_focal`` all zero): COLMAP's model files do
not store Camera::has_prior_focal_length (UPSTREAM-UNVERIFIED), so on resume the reference gives every camera the
down-weighted positioning loss (global_positioning.cc:313-316) and the doubled angle-filter threshold
(track_filter.cc:74).  Global positioning starts from the model's centres and points and randomises only what the
reference does (global_positioning.cc:145-151, 258-263): with ``--GlobalPositioning.optimize_positions 0`` every centre
is kept, and tracks shorter than ``min_num_view_per_track`` are not optimised and keep their input xyz; they are
written when they have at least 2 observations.

The reference's flags are accepted with their names and defaults.  ``--retriangulation_iteration_num`` and the
``--Triangulation.*`` options are accepted and ignored (resume skips retriangulation, option_manager.cc:112);
``--image_path`` is refused, as colour extraction is not supported.  Exit codes: 0 done, 1 a stage failed (nothing is
written), 2 bad input (a message names it)."""
from __future__ import annotations

import argparse
import sys

import numpy as np

from . import colmap_io as CIO, mapper as M, synthetic as S

# (flag, options path, type) for every resume flag the mapper implements (option_manager.cc:114-122, 180-270)
_FLAGS = [
    ("ba_iteration_num", "num_iteration_bundle_adjustment", int),
    ("skip_global_positioning", "skip_global_positioning", bool),
    ("skip_bundle_adjustment", "skip_bundle_adjustment", bool),
    ("skip_pruning", "skip_pruning", bool),
    ("GlobalPositioning.optimize_positions", "opt_gp.optimize_positions", bool),
    ("GlobalPositioning.optimize_points", "opt_gp.optimize_points", bool),
    ("GlobalPositioning.optimize_scales", "opt_gp.optimize_scales", bool),
    ("GlobalPositioning.thres_loss_function", "opt_gp.thres_loss_function", float),
    ("GlobalPositioning.max_num_iterations", "opt_gp.solver_options.max_num_iterations", int),
    ("GlobalPositioning.gpu_index", "opt_gp.gpu_index", str),
    ("BundleAdjustment.optimize_rig_poses", "opt_ba.optimize_rig_poses", bool),
    ("BundleAdjustment.optimize_rotations", "opt_ba.optimize_rotations", bool),
    ("BundleAdjustment.optimize_translation", "opt_ba.optimize_translation", bool),
    ("BundleAdjustment.optimize_intrinsics", "opt_ba.optimize_intrinsics", bool),
    ("BundleAdjustment.optimize_principal_point", "opt_ba.optimize_principal_point", bool),
    ("BundleAdjustment.optimize_points", "opt_ba.optimize_points", bool),
    ("BundleAdjustment.thres_loss_function", "opt_ba.thres_loss_function", float),
    ("BundleAdjustment.max_num_iterations", "opt_ba.solver_options.max_num_iterations", int),
    ("BundleAdjustment.gpu_index", "opt_ba.gpu_index", str),
    ("Thresholds.max_angle_error", "inlier_thresholds.max_angle_error", float),
    ("Thresholds.max_reprojection_error", "inlier_thresholds.max_reprojection_error", float),
    ("Thresholds.min_triangulation_angle", "inlier_thresholds.min_triangulation_angle", float),
]
# accepted and ignored: resume skips retriangulation
_IGNORED = ["retriangulation_iteration_num", "Triangulation.complete_max_reproj_error",
            "Triangulation.merge_max_reproj_error", "Triangulation.min_angle", "Triangulation.min_num_matches"]


class InputError(Exception):
    """Bad input: exit code 2."""


def resume_options() -> M.GlobalMapperOptions:
    """GlobalMapperOptions with the resume skips (option_manager.cc:107-112)."""
    return M.GlobalMapperOptions(skip_preprocessing=True, skip_view_graph_calibration=True,
                                 skip_rotation_averaging=True, skip_track_establishment=True)


def _get(obj, path):
    for part in path.split("."):
        obj = getattr(obj, part)
    return obj


def _set(obj, path, value):
    *head, last = path.split(".")
    for part in head:
        obj = getattr(obj, part)
    setattr(obj, last, value)


def _bool(v: str) -> bool:
    t = v.strip().lower()
    if t in ("1", "true", "yes"):
        return True
    if t in ("0", "false", "no"):
        return False
    raise argparse.ArgumentTypeError(f"not a boolean: {v!r}")


class _Parser(argparse.ArgumentParser):
    def error(self, message):
        raise InputError(message)


def _parser() -> argparse.ArgumentParser:
    ap = _Parser(prog="glomap_b200.mapper_resume", description=__doc__.split("\n\n")[0])
    ap.add_argument("--input_path", required=True)
    ap.add_argument("--output_path", required=True)
    ap.add_argument("--output_format", default="bin", choices=("bin", "txt"))
    ap.add_argument("--image_path", default="")
    defaults = resume_options()
    for flag, path, typ in _FLAGS:
        d = _get(defaults, path)
        ap.add_argument(f"--{flag}", dest=path, type=_bool if typ is bool else typ, default=d, metavar=typ.__name__.upper())
    for flag in _IGNORED:
        ap.add_argument(f"--{flag}", help=argparse.SUPPRESS)
    return ap


def parse_args(argv=None):
    """(args, GlobalMapperOptions) of the command line; bad flags raise InputError."""
    args = _parser().parse_args(argv)
    if args.image_path:
        raise InputError("--image_path: colour extraction from the images is not supported; the colours of the input "
                         "model are written back")
    opts = resume_options()
    for _, path, _ in _FLAGS:
        _set(opts, path, getattr(args, path))
    return args, opts


def read_input(path: str):
    """(scene, index, registration) of the model in ``path``; a model that cannot be used raises InputError."""
    try:
        cameras, images, points = CIO.read_model(path)
        rigs, frames = CIO.read_rigs_frames(path)
        scene, index = CIO.scene_from_model(cameras, images, points, rigs, frames)
    except (OSError, ValueError) as e:
        raise InputError(str(e)) from None
    registered = index.frame_registered if isinstance(scene, S.RigScene) else np.ones(scene.C, bool)
    return scene, index, registered


def empty_view_graph(n_images: int) -> S.ViewGraph:
    return S.ViewGraph(n_images, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 3, 3)), np.zeros(0), None)


def solve(scene, registered, opts: M.GlobalMapperOptions, ctx=None):
    """GlobalMapper.Solve as mapper_resume runs it: (ok, scene, mapper)."""
    mapper = M.GlobalMapper(opts, ctx)
    n_images = scene.I if isinstance(scene, S.RigScene) else scene.C
    ok, out = mapper.Solve(empty_view_graph(n_images), scene, camera_prior_focal=np.zeros(len(scene.intr_model), bool),
                           registered=registered, keep_input_state=True)
    return ok, out, mapper


def write_output(path: str, scene_in, scene, index, mapper, registered, fmt: str) -> list:
    """WriteGlomapReconstruction of ``scene``, the mapper's result on ``scene_in``: the clusters of stage 8, or every
    registered frame in ``path/0``."""
    if mapper.frame_cluster_id is not None:
        cid, reg = mapper.frame_cluster_id, mapper.frame_registered
    else:
        cid, reg = np.full(len(registered), -1, np.int64), registered
    return CIO.write_clustered_model(path, scene, CIO.reindex_observations(index, scene_in, scene), cid, reg, fmt)


def main(argv=None) -> int:
    try:
        args, opts = parse_args(argv)
        scene, index, registered = read_input(args.input_path)
    except InputError as e:
        print(f"mapper_resume: {e}", file=sys.stderr)
        return 2
    rig = isinstance(scene, S.RigScene)
    print(f"read {args.input_path}: {len(scene.intr_model)} cameras, "
          + (f"{len(scene.rig_ref_sensor)} rigs, {int(registered.sum())} / {scene.F} frames registered, {scene.I} images, "
             if rig else f"{scene.C} images, ")
          + f"{scene.P} points, {scene.N} observations")
    ok, out, mapper = solve(scene, registered, opts)
    for line in mapper.log:
        print(line)
    if not ok:
        print("mapper_resume: the global mapper failed; nothing is written", file=sys.stderr)
        return 1
    for path in write_output(args.output_path, scene, out, index, mapper, registered, args.output_format):
        print(f"wrote {path}")
    print(f"{out.P} points, {out.N} observations after the mapper")
    return 0


if __name__ == "__main__":
    sys.exit(main())
