#!/usr/bin/env python
"""Gravity refinement on the GPU (b200sfm_gravity_refine) at config-5 size.

  python profiles/gravity_refine_bench.py [--frames 100000] [--neighbours 50] [--reps 5] [--oracle-frames 200]

Scene: make_lattice_view_graph(frames, neighbours) (2 deg relative-rotation noise, 5 % outlier pairs), a gravity prior on
every frame from synthetic.make_gravity with 30 % outlier priors.  Reported: the call end to end (host clock around the
synchronous call, median of --reps after a warm-up), its device split from the call's CUDA events (H2D, error test, CSR,
refinement), the frame counts and LM iterations, and the CPU oracle's time on the first --oracle-frames error-prone
frames only (stated as measured on that sample, not extrapolated).  The card name and power limit are read in the same
process.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100_000)
    ap.add_argument("--neighbours", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-frames", type=int, default=200)
    a = ap.parse_args()
    import numpy as np
    from glomap_b200 import synthetic as S
    from glomap_b200.gravity_refinement import GravityRefiner, get_align_rot_householder
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    vg = S.make_lattice_view_graph(a.frames, a.neighbours, seed=1)
    g, _ = S.make_gravity(vg.R_gt, noise_deg=0.0, outlier_ratio=0.3, seed=1)
    ref = GravityRefiner()
    ref.RefineGravity(vg, g)                                               # warm-up
    times, stats = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        g_new, status, st = ref.RefineGravity(vg, g)
        times.append((time.perf_counter() - t0) * 1e3)
        stats.append(st)
    st = stats[len(stats) // 2]
    out = dict(card=card, frames=a.frames, pairs=int(vg.E), call_ms_median=float(np.median(times)),
               abi_ms_total=st["ms_total"], ms_h2d=st["ms_h2d"], ms_error_test=st["ms_error_test"], ms_csr=st["ms_csr"],
               ms_refine=st["ms_refine"], error_prone=st["error_prone_frames"], rectified=st["rectified_frames"],
               lm_iterations=st["lm_iterations"], max_lm_iterations=st["max_lm_iterations"])
    if a.oracle_frames > 0:
        from oracle import gravity_oracle as GO
        ep = np.nonzero(status)[0][: a.oracle_frames]
        keep = np.isin(vg.ei, ep) | np.isin(vg.ej, ep)                      # the sampled frames' pairs
        R_align = get_align_rot_householder(g)
        t0 = time.perf_counter()
        res = GO.refine_gravity(R_align, np.ones(len(g), bool), vg.ei[keep], vg.ej[keep], vg.R_rel[keep])
        out["oracle_s"] = time.perf_counter() - t0
        out["oracle_error_prone"] = int(len(res["error_prone"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
