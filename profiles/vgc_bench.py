#!/usr/bin/env python
"""View-graph calibration on the GPU (b200sfm_view_graph_calibrate) on seeded view graphs.

  python profiles/vgc_bench.py [--scenes config2,config5] [--cameras shared,per_image] [--reps 5] [--oracle]

Scenes: config2 = the pairs of make_scene(1000, 200k) that share >= 30 points (view_graph_from_scene, about 100 k pairs);
config5 = 100 k images, image i paired with i+1 .. i+50 (about 5 M pairs).  Each runs with one camera shared by every image
(K = 1: every pair is a same-camera pair, one row of E incidences) and with one camera per image (K = images).  F is the
true fundamental matrix with 1e-3 multiplicative noise, 5 % random-F outlier pairs, initial focals 20 % off.
Reported per run: the ABI call end to end from pinned host buffers (host clock around the call, which ends in a stream
synchronise; median of --reps after a warm-up) with the H2D / D2H copy times the call measures with CUDA events, the
device solve time (CUDA events), LM and PCG iterations, per-kernel device times from torch.profiler (one profiled call in
the same process after the timed ones), the byte model below per kernel, the CPU oracle's time (--oracle; config2 only),
and the card name and power limit read in the same process.  Writes nothing.

Byte model (HBM, per launch): setup reads F and the camera indices and writes the constants (9*8 + 8 + 64 B per pair);
linearize reads 64 + 8 B and writes 32 + 8 B per pair; cost, model and filter read 72 B per pair (filter also writes 17 B);
seg_sums reads 4 B and gathers 32 B per incidence; the mat-vec's first pass reads 8 B and gathers 8 B per incidence.
Camera-sized vectors (K doubles) are not counted.
"""
import argparse
import ctypes as ct
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BW = 3.35e12


def make(scene, cameras):
    import numpy as np
    from glomap_b200 import synthetic as S
    if scene == "config2":
        sc = S.make_scene(1000, 200_000, 10.0, seed=1, num_intrinsics=1 if cameras == "shared" else 1000)
        vg = S.view_graph_from_scene(sc, min_shared=30)
        pairs = np.stack([vg.ei, vg.ej], 1)
    else:
        C = 100_000 if scene == "config5" else 2_000
        sc = S.make_scene(C, 10, 10.0, seed=1, num_intrinsics=1 if cameras == "shared" else C)
        i = np.repeat(np.arange(C), 50)
        j = i + np.tile(np.arange(1, 51), C)
        pairs = np.stack([i[j < C], j[j < C]], 1)
    return S.make_vgc_pairs(sc, pairs, seed=1, f_noise=0.2, outlier_frac=0.05, F_sigma=1e-3)


def byte_model(E, n_inc):
    return {"vgc_setup": 144 * E, "vgc_linearize": 112 * E, "vgc_cost": 72 * E, "vgc_model": 72 * E, "vgc_filter": 89 * E,
            "vgc_seg_sums": 36 * n_inc, "vgc_mv_seg": 16 * n_inc}


def run(scene, cameras, reps, with_oracle):
    import numpy as np
    import torch
    from glomap_b200 import _lib, estimators as E_, view_graph_calibration as VGC
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    torch.cuda.set_device(0)
    torch.cuda.init()
    t0 = time.perf_counter()
    d = make(scene, cameras)
    t_gen = time.perf_counter() - t0
    Ep, K = len(d["cam1"]), len(d["focal_init"])
    n_inc = int(2 * (d["cam1"] != d["cam2"]).sum() + (d["cam1"] == d["cam2"]).sum())
    ctx = E_.Context(0, 0, 1, None)

    def pinned(a):
        t = torch.empty(a.shape, dtype=getattr(torch, a.dtype.name), pin_memory=True)
        t.numpy()[...] = a
        return t
    keep = {k: pinned(np.ascontiguousarray(d[k])) for k in ("principal_point", "cam1", "cam2", "F")}
    focal = pinned(np.ascontiguousarray(d["focal_init"]))
    out = {"valid": torch.empty(Ep, dtype=torch.uint8, pin_memory=True), "acc": torch.empty(K, dtype=torch.uint8, pin_memory=True)}
    p = lambda t: ct.c_void_p(t.data_ptr())   # noqa: E731
    o = VGC.ViewGraphCalibratorOptions().to_c()
    st = _lib.LMStats()

    def call():
        focal.numpy()[...] = d["focal_init"]
        rc = ctx.lib.b200sfm_view_graph_calibrate(ctx.handle, ct.byref(o), K, p(keep["principal_point"]), p(focal), None, Ep,
                                                  p(keep["cam1"]), p(keep["cam2"]), p(keep["F"]), p(out["valid"]),
                                                  p(out["acc"]), None, ct.byref(st))
        assert rc == 0, ctx.lib.b200sfm_last_error(ctx.handle)
    call()   # warm-up (module load, pool growth)
    ms, solve_ms, h2d, d2h = [], [], [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        ms.append(1e3 * (time.perf_counter() - t0))
        solve_ms.append(st.ms_total)
        h2d.append(st.ms_h2d)
        d2h.append(st.ms_d2h)
    stats = st.as_dict()
    first = (focal.numpy().copy(), out["valid"].numpy().copy())
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    assert np.array_equal(first[0].view(np.uint64), focal.numpy().view(np.uint64)) and np.array_equal(first[1], out["valid"].numpy())
    kern, calls, copies = {}, {}, {"h2d": 0.0, "d2h": 0.0}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or not ev.name:
            continue
        if ev.name.startswith("Memcpy HtoD"):
            copies["h2d"] += ev.device_time_total / 1e3
        elif ev.name.startswith("Memcpy DtoH"):
            copies["d2h"] += ev.device_time_total / 1e3
        else:
            name = ev.name.split("(")[0].replace("void ", "").replace("b200::", "").split("<")[0]
            kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1e3
            calls[name] = calls.get(name, 0) + 1
    if not any(k.startswith("vgc_") for k in kern):
        raise RuntimeError("no vgc_* kernel in the profile: " + str(sorted(kern)[:20]))
    model = byte_model(Ep, n_inc)
    per_kernel = {k: dict(ms=round(v, 3), launches=calls[k],
                          tb_per_s=round(model[k] * calls[k] / (v * 1e-3) / 1e12, 3) if k in model and v > 0 else None)
                  for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}
    f = focal.numpy()
    rec = dict(scene=scene, cameras=cameras, card=card, images=int(max(d["img1"].max(), d["img2"].max()) + 1), K=K, pairs=Ep,
               incidences=n_inc, generate_s=round(t_gen, 1), call_ms_median=round(float(np.median(ms)), 2),
               call_ms_all=[round(x, 2) for x in ms], solve_ms_median=round(float(np.median(solve_ms)), 2),
               h2d_ms_median=round(float(np.median(h2d)), 2), d2h_ms_median=round(float(np.median(d2h)), 2),
               h2d_bytes=stats["h2d_bytes"], lm_iterations=stats["iterations"], pcg_iterations=stats["pcg_iterations"],
               termination=VGC.TERMINATION[stats["termination"]], kernel_launches=stats["kernel_launches"],
               kernel_total_ms=round(sum(kern.values()), 3), kernels=per_kernel,
               profiled_h2d_ms=round(copies["h2d"], 2), profiled_d2h_ms=round(copies["d2h"], 2),
               focal_rel_err_max=float(np.abs(f / d["focal_true"] - 1).max()),
               pairs_invalidated=int((out["valid"].numpy() == 0).sum()), outliers=int(d["is_outlier"].sum()))
    if with_oracle and scene == "config2":
        from oracle import vgc_oracle as V
        t0 = time.perf_counter()
        ref = V.solve_vgc(d["principal_point"], d["focal_init"], None, d["cam1"], d["cam2"], d["F"])
        rec["oracle_cpu_s"] = round(time.perf_counter() - t0, 2)
        rec["oracle_lm_iterations"] = ref["summary"].iterations
        rec["focal_vs_oracle_rel"] = float(np.abs(f / ref["focal"] - 1).max())
    print(json.dumps(rec), flush=True)
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="config2,config5")
    ap.add_argument("--cameras", default="shared,per_image")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--one", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.one:
        run(args.scenes, args.cameras, args.reps, args.oracle)
        return
    for scene in args.scenes.split(","):   # one process per run: a second torch.profiler session records no kernels
        for cameras in args.cameras.split(","):
            cmd = [sys.executable, os.path.abspath(__file__), "--one", "--scenes", scene, "--cameras", cameras,
                   "--reps", str(args.reps)] + (["--oracle"] if args.oracle else [])
            subprocess.check_call(cmd)


if __name__ == "__main__":
    main()
