#!/usr/bin/env python
"""ConvertRotationsFromImageToRig on the GPU (b200sfm_rig_rotations_from_images) and the rig pre-pass of
solve_rotation_averaging_rig, each against its numpy restatement in oracle/rig_init_oracle.py.

  python profiles/rig_rotation_init_bench.py [--frames 100000] [--cams 6] [--prepass-frames 300] [--reps 7]

Workloads:
  conversion  --frames frames of one --cams-camera rig (config 5: 100 000 frames x 6 cameras), camera 0 the reference,
              cameras 1..cams/2 known and the others unknown, 10 % of the images missing, 0.5 deg of noise on the image
              rotations.  Reported: the device call from host to host (wall clock around the synchronous call, copies
              included; median of --reps after a warm-up), its ms_total, the host restatement's time (one run), whether
              the sample counts are equal and the largest sign-invariant rotation difference.
  prepass     the whole pre-pass on a --prepass-frames-frame 4-camera rig (2 cameras unknown, 0.3 deg of pair noise):
              solve_rotation_averaging_rig from host to host (median of 3 after a warm-up) against the oracle chain
              (one run), their L1 / IRLS counts and the largest rotation difference.
The card name and power limit are read in the same process.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def conversion_workload(F, S, seed=0):
    import numpy as np
    from glomap_b200 import geometry as G
    rng = np.random.default_rng(seed)
    Rf = G.so3_exp(rng.normal(size=(F, 3)))
    w = rng.normal(size=(S, 3)) * 0.4
    w[0] = 0
    Rs = G.so3_exp(w)
    fr, cam = np.repeat(np.arange(F), S), np.tile(np.arange(S), F)
    keep = (cam == 0) | (rng.uniform(size=F * S) >= 0.1)
    fr, cam = fr[keep], cam[keep]
    noise = G.so3_exp(rng.normal(size=(len(fr), 3)) * np.radians(0.5) / np.sqrt(3))
    q = G.rotmat_to_quat_xyzw_fast(noise @ np.einsum("nij,njk->nik", Rs[cam], Rf[fr]))
    known = (np.arange(S) <= S // 2).astype(np.uint8)
    cq = G.rotmat_to_quat_xyzw_fast(Rs)
    return fr, cam, q, np.zeros(F, np.int64), known, cq, np.tile([0, 0, 0, 1.0], (F, 1))


def qangle(a, b):
    """Sign-invariant rotation angle between quaternions, 4 atan2(|a - b|, |a + b|) (exact down to rounding, unlike arccos)."""
    import numpy as np
    a = np.asarray(a) / np.linalg.norm(a, axis=-1, keepdims=True)
    b = np.asarray(b) / np.linalg.norm(b, axis=-1, keepdims=True)
    b = np.where((a * b).sum(-1, keepdims=True) < 0, -b, b)
    return 4 * np.arctan2(np.linalg.norm(a - b, axis=-1), np.linalg.norm(a + b, axis=-1))


def run_conversion(F, S, reps, card):
    import numpy as np
    from glomap_b200 import _lib
    from glomap_b200.rotation_initializer import convert_rotations_from_image_to_rig as conv
    from oracle import rig_init_oracle as O
    args = conversion_workload(F, S)
    st = _lib.RigInitStats()
    conv(*args)                                                                  # warm-up
    times, inner = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        d = conv(*args, stats=st)
        times.append(1e3 * (time.perf_counter() - t0))
        inner.append(st.ms_total)
    t0 = time.perf_counter()
    o = O.convert_rotations(*args)
    host = 1e3 * (time.perf_counter() - t0)
    return dict(card=card, workload="conversion", frames=F, cameras=S, images=int(len(args[0])),
                device_call_ms_median=round(float(np.median(times)), 3), device_call_ms_all=[round(t, 3) for t in times],
                ms_total_median=round(float(np.median(inner)), 3), kernel_launches=st.kernel_launches,
                host_ms=round(host, 1), counts_equal=bool(np.array_equal(d[1], o[1]) and np.array_equal(d[3], o[3])),
                max_angle_diff_rad=float(max(qangle(d[0], o[0]).max(), qangle(d[2], o[2]).max())))


def run_prepass(F, card):
    import numpy as np
    from glomap_b200 import rotation_averager as RA
    from oracle import rig_init_oracle as O
    from test_rig_rotation_init_gpu import rig_scene
    vg, fr, cam, known, cq, ref, _, _ = rig_scene(F=F)
    o = RA.RotationAveragerOptions(pcg_rel_tolerance=1e-12)
    RA.solve_rotation_averaging_rig(vg, fr, cam, known, cq, ref, o)             # warm-up
    times = []
    for _ in range(3):
        info = {}
        t0 = time.perf_counter()
        ok, R, Rc, _ = RA.solve_rotation_averaging_rig(vg, fr, cam, known, cq, ref, o, info=info)
        times.append(1e3 * (time.perf_counter() - t0))
    info_o = {}
    t0 = time.perf_counter()
    ok_o, R_o, Rc_o, _ = O.solve_rotation_averaging_rig(vg, fr, cam, known, cq, ref, o, info=info_o)
    host = 1e3 * (time.perf_counter() - t0)
    return dict(card=card, workload="prepass", frames=F, images=int(len(fr)), pairs=int(vg.E), ok=bool(ok and ok_o),
                device_call_ms_median=round(float(np.median(times)), 3), host_ms=round(host, 1),
                iterations=info, iterations_oracle=info_o,
                max_abs_diff=float(max(np.abs(R - R_o).max(), np.abs(Rc - Rc_o).max())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100000)
    ap.add_argument("--cams", type=int, default=6)
    ap.add_argument("--prepass-frames", type=int, default=300)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    print(json.dumps(run_conversion(args.frames, args.cams, args.reps, card)), flush=True)
    print(json.dumps(run_prepass(args.prepass_frames, card)), flush=True)


if __name__ == "__main__":
    main()
