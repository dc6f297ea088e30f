#!/usr/bin/env python
"""The shim's TrackFilter, UndistortImages and NormalizeReconstruction timed host to host on a config-4-sized scene,
against the host restatements.

  python profiles/shim_processors_bench.py [--cameras 10000] [--points 2000000] [--reps 3] [--host-frac 0.1]

Scene: ``synthetic.make_scene(cameras, points, 10, seed=1, pixel_sigma=0.5)`` (config 4 of bench.py: about 20 M
observations) perturbed by ``perturb_scene`` so that the filters remove observations; one intrinsics block per 100
images, every third block without a prior focal length.  The scene is written as raw arrays to a temporary directory
and profiles/shim_processors_bench.cc, built there against libb200sfm.so, turns it into the glomap maps and times each
shim call (median of --reps, each on a fresh copy of the maps it changes).  Host restatements in this process:
``processors.undistort_images`` and ``processors.normalize_reconstruction`` on the whole scene, and the long-double
filter oracle (``oracle.filter_oracle``) on the first --host-frac of the points (its memory grows with 16-byte
3x3 matrices per observation).  The card name and power limit are read in the same run.  Prints one JSON line per
measurement; writes nothing outside the temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def subscene(sc, P):
    from glomap_b200 import synthetic as S
    n = int(sc.pt_obs_begin[P])
    return S.Scene(sc.quat, sc.trans, sc.points[:P], sc.pt_obs_begin[:P + 1], sc.obs_cam[:n], sc.obs_xy[:n], sc.cam_intr,
                   sc.intr_model, sc.intr_params)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, default=10000)
    ap.add_argument("--points", type=int, default=2_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-frac", type=float, default=0.1)
    args = ap.parse_args()
    from glomap_b200 import processors as PR, synthetic as S
    from oracle import filter_oracle as FO

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    t0 = time.perf_counter()
    K = max(args.cameras // 100, 1)
    sc = S.perturb_scene(S.make_scene(args.cameras, args.points, 10, seed=1, pixel_sigma=0.5, num_intrinsics=K))
    prior = (np.arange(K) % 3 != 0).astype(np.uint8)
    gen_s = time.perf_counter() - t0
    out = dict(card=card, cameras=sc.C, points=sc.P, observations=sc.N, scene_generation_s=round(gen_s, 1))
    print(json.dumps(out), flush=True)

    def host(name, fn, scene):
        t = time.perf_counter()
        fn()
        print(json.dumps(dict(card=card, host=name, observations=scene.N, ms=round(1e3 * (time.perf_counter() - t), 1))), flush=True)

    box = {}
    host("processors.undistort_images", lambda: box.setdefault("b", PR.undistort_images(sc)), sc)
    bear = box["b"]
    host("processors.normalize_reconstruction", lambda: PR.normalize_reconstruction(sc.copy()), sc)
    sub = subscene(sc, max(1, int(args.host_frac * sc.P)))
    nsub = sub.N
    cal = prior[sub.cam_intr]
    host("filter_oracle.filter_reprojection_normalized(1e-2)", lambda: FO.filter_reprojection_normalized(sub, bear[:nsub], 1e-2), sub)
    host("filter_oracle.filter_reprojection(3)", lambda: FO.filter_reprojection(sub, 3.0, S.project), sub)
    host("filter_oracle.filter_angle(1)", lambda: FO.filter_angle(sub, bear[:nsub], 1.0, cal), sub)
    host("filter_oracle.filter_triangulation_angle(1)", lambda: FO.filter_triangulation_angle(sub, 1.0), sub)

    with tempfile.TemporaryDirectory() as d:
        arrays = dict(quat=(sc.quat, np.float64), trans=(sc.trans, np.float64), points=(sc.points, np.float64),
                      ptb=(sc.pt_obs_begin, np.int64), obs_cam=(sc.obs_cam, np.int32), obs_xy=(sc.obs_xy, np.float64),
                      cam_intr=(sc.cam_intr, np.int32), intr_model=(sc.intr_model, np.int32),
                      intr_params=(sc.intr_params, np.float64), bearings=(bear, np.float64), prior=(prior, np.uint8))
        for name, (a, dt) in arrays.items():
            np.ascontiguousarray(a, dt).tofile(os.path.join(d, name + ".bin"))
        with open(os.path.join(d, "dims.txt"), "w") as f:
            f.write(f"{sc.C} {sc.P} {sc.N} {len(sc.intr_model)}\n")
        exe = os.path.join(d, "shim_processors_bench")
        libdir = os.path.join(ROOT, "glomap_b200")
        subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I" + os.path.join(ROOT, "glomap_b200", "host"), "-o", exe,
                        os.path.join(ROOT, "profiles", "shim_processors_bench.cc"), "-L" + libdir, "-lb200sfm",
                        "-Wl,-rpath," + libdir], check=True)
        r = subprocess.run([exe, d, str(args.reps)], capture_output=True, text=True)
        sys.stderr.write(r.stderr)
        for line in r.stdout.splitlines():
            rec = json.loads(line)
            rec.update(card=card, observations=sc.N)
            print(json.dumps(rec), flush=True)
        if r.returncode:
            sys.exit(r.returncode)


if __name__ == "__main__":
    main()
