#!/usr/bin/env python
"""Stage 3 of the mapper (two rotation averaging runs with their filters) with and without gravity priors.

  python profiles/mapper_gravity_bench.py [--rigs 2] [--cams 2] [--rig-frames 100] [--frames 100000] [--neighbours 50]
                                          [--reps 3]

Scenes: camera rigs from synthetic.make_rig_dataset (--rigs rigs of --cams cameras, --rig-frames frames each, 3 deg of
relative-rotation noise), and trivial frames on make_lattice_view_graph(--frames, --neighbours) (2 deg noise, 5 %
outlier pairs), the largest lattice profiles/ uses.  Priors from synthetic.make_frame_gravity on 70 % of the frames at
0.5 deg.  ``GlobalMapper.Solve`` runs with global positioning and bundle adjustment skipped, once with
``opt_ra.use_gravity`` and once without; reported per scene: the median host-to-host time of --reps calls after a
warm-up of each, the b200sfm_ra_solve_gravity calls of one call, and the median rotation error after the best global
rotation.  --rig-frames 0 or --frames 0 leaves that scene out.  The card name and power limit are read in the same
process.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _median_error(R, R_gt):
    import numpy as np
    from glomap_b200 import geometry as G
    U, _, Vt = np.linalg.svd(np.einsum("nji,njk->ik", R, R_gt))
    return float(np.median(G.rotation_angle_deg(R @ (U @ Vt), R_gt)))


def _time(vg, scene, g, R_gt, reps, lib):
    import numpy as np
    from glomap_b200 import geometry as G, mapper as M, synthetic as S
    calls = [0]
    solve = lib.b200sfm_ra_solve_gravity

    def counted(*args):
        calls[0] += 1
        return solve(*args)

    out = {}
    lib.b200sfm_ra_solve_gravity = counted
    try:
        for use in (False, True):
            o = M.GlobalMapperOptions(skip_global_positioning=True, skip_bundle_adjustment=True)
            o.opt_ra.use_gravity = use
            M.GlobalMapper(o).Solve(vg, scene, gravity=g)                          # warm-up
            times = []
            for _ in range(reps):
                calls[0] = 0
                mapper = M.GlobalMapper(o)
                t0 = time.perf_counter()
                ok, res = mapper.Solve(vg, scene, gravity=g)
                times.append((time.perf_counter() - t0) * 1e3)
                assert ok, mapper.log
            reg = mapper.frame_in_component if isinstance(scene, S.RigScene) else mapper.image_registered
            R = G.quat_xyzw_to_rotmat(res.quat)
            key = "gravity" if use else "plain"
            out[key] = dict(ms_median=float(np.median(times)), ms_all=[round(t, 1) for t in times],
                            ra_solve_gravity_calls=calls[0], registered=int(reg.sum()),
                            median_rotation_error_deg=_median_error(R[reg], R_gt[reg]),
                            log=[line for line in mapper.log if "gravity" in line])
    finally:
        lib.b200sfm_ra_solve_gravity = solve
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rigs", type=int, default=2)
    ap.add_argument("--cams", type=int, default=2)
    ap.add_argument("--rig-frames", type=int, default=100)
    ap.add_argument("--frames", type=int, default=100_000)
    ap.add_argument("--neighbours", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    from glomap_b200 import estimators as E
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    lib = E.default_context().lib
    res = dict(card=card)
    if a.rig_frames > 0:
        _rigs(a, res, lib)
    if a.frames > 0:
        _trivial(a, res, lib)
    print(json.dumps(res))


def _rigs(a, res, lib):
    import numpy as np
    from glomap_b200 import geometry as G, synthetic as S
    d = S.make_rig_dataset(a.rigs, a.cams, a.rig_frames, 300, seed=1, rotation_noise_deg=3.0)
    R_gt = G.quat_xyzw_to_rotmat(d.scene.quat)
    start = d.scene.copy()
    start.quat[:] = [0, 0, 0, 1]
    g = S.make_frame_gravity(R_gt, share=0.7, noise_deg=0.5, seed=1)
    res["rigs"] = dict(frames=int(d.scene.F), images=int(d.scene.I), pairs=int(d.view_graph.E),
                       priors=int((~np.isnan(g).any(axis=1)).sum()), **_time(d.view_graph, start, g, R_gt, a.reps, lib))
    print(json.dumps(res), flush=True)


def _trivial(a, res, lib):
    import numpy as np
    from glomap_b200 import synthetic as S
    vg = S.make_lattice_view_graph(a.frames, a.neighbours, seed=1, noise_deg=2.0, outlier_ratio=0.05)
    n = vg.n_images
    scene = S.Scene(np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)), np.zeros((n, 3)), np.zeros((0, 3)), np.zeros(1, np.int64),
                    np.zeros(0, np.int32), np.zeros((0, 2)), np.zeros(n, np.int32), np.zeros(1, np.int32),
                    np.zeros((1, S.INTR_STRIDE)))
    g = S.make_frame_gravity(vg.R_gt, share=0.7, noise_deg=0.5, seed=1)
    res["trivial"] = dict(frames=n, pairs=int(vg.E), priors=int((~np.isnan(g).any(axis=1)).sum()),
                          **_time(vg, scene, g, np.asarray(vg.R_gt), a.reps, lib))


if __name__ == "__main__":
    main()
