"""Where mapper_resume spends its time at config-2 size (1 000 images, 200 000 points, ~2 M observations, seed 1).

Builds the model on disk twice -- trivial frames (``make_scene(1000, 200000)``) and rigs (``make_rig_scene``: 250
frames of one 4-camera rig) -- with the poses at ground truth and the points perturbed, runs the command in-process and
reports, separately: model read and flatten (host), global positioning, the track filters and each bundle adjustment
stage (device, synchronised), pruning, and the model write (host).  The per-element conversion the vectorised one
replaced (kept in tests/test_mapper_resume_cpu.py as its reference) is timed on the same trivial model.  The GPU name
and power limit are recorded in the same run.

    python profiles/mapper_resume_bench.py [--points 200000] [--images 1000] [--skip_pruning 0]
"""
import argparse
import contextlib
import importlib.util
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from glomap_b200 import colmap_io as CIO, estimators as E, mapper as M, mapper_resume as MR  # noqa: E402
from glomap_b200 import reconstruction_pruning as RP, synthetic as S  # noqa: E402


def _sync():
    import torch
    if torch.cuda.is_available():
        torch.cuda.synchronize()


class Timer:
    def __init__(self):
        self.t = {}

    @contextlib.contextmanager
    def span(self, name):
        _sync()
        t0 = time.perf_counter()
        try:
            yield
        finally:
            _sync()
            self.t[name] = self.t.get(name, 0.0) + time.perf_counter() - t0


def _wrap(obj, attr, timer, name_of):
    orig = getattr(obj, attr)

    def wrapped(*a, **kw):
        with timer.span(name_of(*a, **kw)):
            return orig(*a, **kw)
    setattr(obj, attr, wrapped)
    return lambda: setattr(obj, attr, orig)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run_once(model_dir, out_dir, skip_pruning):
    timer = Timer()
    ba_calls = {"n": 0}

    def ba_name(self, *a, **kw):
        ba_calls["n"] += 1
        return f"bundle adjustment solve {ba_calls['n']}"
    undo = [_wrap(E.GlobalPositioner, "Solve", timer, lambda *a, **k: "global positioning"),
            _wrap(E.BundleAdjuster, "Solve", timer, ba_name),
            _wrap(M.GlobalMapper, "_filters", timer, lambda self, scene, what: "filters " + "+".join(k for k, _ in what)),
            _wrap(RP, "prune_weakly_connected_images", timer, lambda *a, **k: "pruning")]
    try:
        with timer.span("read + flatten (host)"):
            scene, index, registered = MR.read_input(model_dir)
        _, opts = MR.parse_args(["--input_path", model_dir, "--output_path", out_dir, "--skip_pruning", str(skip_pruning)])
        with timer.span("GlobalMapper.Solve (total)"):
            ok, out, mapper = MR.solve(scene, registered, opts)
        assert ok, mapper.log
        with timer.span("write (host)"):
            MR.write_output(out_dir, scene, out, index, mapper, registered, "bin")
    finally:
        for u in undo:
            u()
    return {k: round(v, 4) for k, v in timer.t.items()}, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--points", type=int, default=200_000)
    ap.add_argument("--skip_pruning", type=int, default=0)
    args = ap.parse_args()
    res = {"gpu": gpu_info(), "images": args.images, "points": args.points}
    spec = importlib.util.spec_from_file_location("resume_cpu", os.path.join(ROOT, "tests", "test_mapper_resume_cpu.py"))
    legacy = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(legacy)
    with tempfile.TemporaryDirectory() as tmp:
        sc = S.make_scene(args.images, args.points, mean_track_len=10, seed=1, pixel_sigma=0.5)
        start = S.perturb_scene(sc, rot_deg=0.0, center_frac=0.0, point_frac=0.01)
        t0 = time.perf_counter()
        CIO.write_model(os.path.join(tmp, "trivial"), *CIO.model_from_scene(start))
        res["trivial_build_write_s"] = round(time.perf_counter() - t0, 3)
        res["trivial_N"] = int(sc.N)
        res["trivial"], _ = run_once(os.path.join(tmp, "trivial"), os.path.join(tmp, "out_trivial"), args.skip_pruning)
        # the per-element conversion on the same model
        model = CIO.read_model(os.path.join(tmp, "trivial"))
        t0 = time.perf_counter()
        old_scene, old_index = legacy.legacy_scene_from_model(*model)
        t1 = time.perf_counter()
        legacy.legacy_model_from_scene(old_scene, old_index)
        t2 = time.perf_counter()
        new_scene, new_index = CIO.scene_from_model(*model)
        t3 = time.perf_counter()
        CIO.model_from_scene(new_scene, new_index)
        t4 = time.perf_counter()
        res["conversion_s"] = {"scene_from_model per-element": round(t1 - t0, 3), "scene_from_model vectorised": round(t3 - t2, 3),
                               "model_from_scene per-element": round(t2 - t1, 3), "model_from_scene vectorised": round(t4 - t3, 3)}
        F = args.images // 4
        rs = S.make_rig_scene(F, 4, args.points, mean_track_len=10, seed=1, pixel_sigma=0.5)
        rstart = rs.copy()
        rstart.points = rs.points + np.random.default_rng(2).normal(size=rs.points.shape) * 0.01
        CIO.write_model(os.path.join(tmp, "rig"), *CIO.model_from_scene(rstart))
        res["rig_N"] = int(rs.N)
        res["rig"], _ = run_once(os.path.join(tmp, "rig"), os.path.join(tmp, "out_rig"), args.skip_pruning)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
