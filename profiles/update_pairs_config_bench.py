#!/usr/bin/env python
"""Stage 0's UpdateImagePairsConfig on the GPU (b200sfm_view_graph_update_pairs_config) against its host restatement
(view_graph_manipulation.update_image_pairs_config, the reference's loops), on the pairs of
synthetic.make_lattice_view_graph with random configs, validity and priors.

  python profiles/update_pairs_config_bench.py [--sizes 100:10,1000:10,100000:100] [--reps 5] [--host-max 300000]

A size is frames:neighbours; 100000:100 is config 5 (100 k frames, about 5 M pairs).  One SIMPLE_RADIAL intrinsics block
per frame, 80 % of them with a prior focal; pairs 90 % valid, CALIBRATED / UNCALIBRATED / PLANAR at 50 / 45 / 5 %.  The
mapper's cut-over (mapper.UPDATE_PAIRS_CONFIG_DEVICE_MIN_PAIRS, 100 pairs) is the 10:10 size's pair count.  Reported
per size, median of --reps after a warm-up:
  device_ms    the device call, host arrays in and out (host clock around the synchronous call)
  kernel_ms    device time of the pc_* kernels of one profiled run (torch.profiler), copies excluded
  host_ms      the host restatement (only up to --host-max pairs)
  same         configs and count equal, F within 1e-13 of its largest entry, against the host restatement
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


def _median_ms(f, reps):
    import numpy as np
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(ts)), 3)


def _problem(frames, neighbours, seed=1):
    import numpy as np
    from glomap_b200 import synthetic as S
    vg = S.make_lattice_view_graph(frames, neighbours, seed=seed, noise_deg=0.0, outlier_ratio=0.0)
    rng = np.random.default_rng(seed)
    K, E = vg.n_images, vg.E
    params = np.zeros((K, S.INTR_STRIDE))
    params[:, :4] = np.c_[rng.uniform(500, 1500, K), rng.uniform(300, 700, (K, 2)), rng.uniform(-0.05, 0.05, K)]
    return dict(intr_model=np.full(K, S.SIMPLE_RADIAL, np.int32), intr_params=params, has_prior_focal=rng.random(K) < 0.8,
                pair_cam1=vg.ei, pair_cam2=vg.ej, pair_valid=rng.random(E) < 0.9, pair_quat=rng.normal(size=(E, 4)),
                pair_trans=rng.normal(size=(E, 3)),
                pair_config=rng.choice(np.array([2, 3, 4], np.int32), E, p=[0.5, 0.45, 0.05]), pair_F=rng.normal(size=(E, 9)))


def run(frames, neighbours, reps, host_max):
    import numpy as np
    import torch
    from glomap_b200 import estimators as E_, view_graph_manipulation as VGM
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    a = _problem(frames, neighbours)
    ctx = E_.default_context()
    out = {}

    def device():
        out["dev"] = VGM.update_image_pairs_config_device(**a, ctx=ctx)

    rec = dict(card=card, frames=frames, pairs=int(len(a["pair_cam1"])), device_ms=_median_ms(device, reps))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        device()
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0 and "pc_" in ev.key:
            kern[ev.key.split("(")[0][:40]] = round(t / 1e3, 4)
    rec["kernel_ms"] = round(sum(kern.values()), 4)
    rec["kernels"] = kern
    cfg_d, F_d, n_d = out["dev"]
    rec["promoted"] = n_d
    if rec["pairs"] <= host_max:
        def host():
            out["host"] = VGM.update_image_pairs_config(**a)
        rec["host_ms"] = _median_ms(host, max(1, min(reps, 3)))
        cfg_h, F_h, n_h = out["host"]
        pr = cfg_h != a["pair_config"]
        err = np.abs(F_d[pr] - F_h[pr]).max(axis=1, initial=0.0) / np.maximum(np.abs(F_h[pr]).max(axis=1, initial=0.0), 1e-300)
        rec["same"] = bool(n_d == n_h and np.array_equal(cfg_d, cfg_h) and (err <= 1e-13).all()
                           and np.array_equal(F_d[~pr], a["pair_F"][~pr]))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10:10,100:10,1000:10,10000:50,100000:100")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-max", type=int, default=300_000, help="largest pair count the host restatement is timed at")
    args = ap.parse_args()
    for s in args.sizes.split(","):
        f, k = (int(x) for x in s.split(":"))
        print(json.dumps(run(f, k, args.reps, args.host_max)), flush=True)


if __name__ == "__main__":
    main()
