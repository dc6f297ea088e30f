#!/usr/bin/env python
"""Reconstruction pruning on the GPU (b200sfm_prune_weakly_connected) on seeded track sets.

  python profiles/prune_bench.py [--scenes config2,config4,long100] [--reps 5] [--oracle] [--per-pass N]

Scenes: config2 = the tracks of make_scene(1000, 200k, mean length 10); config4 = make_scene(10k, 2M, mean length 10);
long100 = make_scene(10k, 100k) with every track 100 views long.  Frames are the scene's images (trivial frames).
Reported per scene: the call end to end (host clock around the synchronous call, median of --reps after a warm-up),
per-kernel device times from torch.profiler (one profiled call after the timed ones, same process), the exact number of
pair slots (sum of L (L - 1) / 2 over the tracks longer than 2) and distinct covisible pairs, the byte model below, the
CPU oracle's time (--oracle; config2 only), and the card name and power limit read in the same process.  Writes nothing.

Byte model (HBM), per pair slot: the key kernel reads 2 frames (8 B, mostly cached) and writes the 8-B key; the radix
sort reads and writes 8 B per key per 8-bit digit of end_bit = bit width of F^2 - 1 (plus one read for the histogram);
run-length encoding reads the sorted key (8 B).  Per observation: 4 B of obs_frame and the 8-B binary-search hit.
Edge- and frame-sized work is not counted.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BW = 3.35e12


def make(scene):
    from glomap_b200 import synthetic as S
    if scene == "config2":
        sc = S.make_scene(1000, 200_000, 10.0, seed=1, chunk=25_000)
    elif scene == "config4":
        sc = S.make_scene(10_000, 2_000_000, 10.0, seed=1, chunk=50_000)
    else:
        sc = S.make_scene(10_000, 100_000, 100.0, seed=1, ragged=False, chunk=10_000)
    return sc.pt_obs_begin, sc.obs_cam, sc.C


def byte_model(tb, F):
    import numpy as np
    L = np.diff(tb)
    slots = int((L[L > 2] * (L[L > 2] - 1) // 2).sum())
    end_bit = int(F * F - 1).bit_length()
    digits = (end_bit + 7) // 8
    return slots, {"keys": 16 * slots, "sort": slots * 8 * (2 * digits + 1), "rle": 8 * slots, "obs": 12 * int(tb[-1])}


def run(scene, reps, with_oracle, per_pass):
    import numpy as np
    import torch
    from glomap_b200 import reconstruction_pruning as RP
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    tb, of, F = make(scene)
    slots, model = byte_model(tb, F)
    out = RP.prune_weakly_connected_images(tb, of, F, max_pair_keys_per_pass=per_pass)   # warm-up
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        again = RP.prune_weakly_connected_images(tb, of, F, max_pair_keys_per_pass=per_pass)
        times.append(time.perf_counter() - t0)
        assert again["cluster_id"].tobytes() == out["cluster_id"].tobytes() and again["stats"] == out["stats"]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        RP.prune_weakly_connected_images(tb, of, F, max_pair_keys_per_pass=per_pass)
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            kern[ev.key[:60]] = round(t / 1e3, 3)
    kernel_ms = sum(v for k, v in kern.items() if "Memcpy" not in k and "Memset" not in k)
    rec = dict(scene=scene, card=card, frames=F, tracks=len(tb) - 1, observations=int(tb[-1]), pair_slots=slots,
               covisible_pairs=out["stats"]["covisible_pairs"], visibility_edges=out["stats"]["visibility_edges"],
               clusters=out["num_clusters"], clustering_iterations=out["stats"]["clustering_iterations"],
               strong_threshold=out["stats"]["strong_threshold"], call_ms_median=round(1e3 * float(np.median(times)), 3),
               call_ms_all=[round(1e3 * t, 3) for t in times], kernel_ms=round(kernel_ms, 3),
               model_bytes=sum(model.values()), model_TBps=round(sum(model.values()) / (kernel_ms * 1e-3) / 1e12, 3),
               model_share_of_peak=round(sum(model.values()) / (kernel_ms * 1e-3) / PEAK_BW, 3),
               kernels=dict(sorted(kern.items(), key=lambda kv: -kv[1])[:12]))
    if with_oracle and scene == "config2":
        from oracle import pruning_oracle as O
        t0 = time.perf_counter()
        ref = O.prune(tb, of, F)
        rec["cpu_oracle_s"] = round(time.perf_counter() - t0, 3)
        rec["oracle_equal"] = bool(ref["cluster_id"].tolist() == out["cluster_id"].tolist()
                                   and ref["is_registered"].tolist() == out["is_registered"].tolist())
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="config2,config4,long100")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle", action="store_true")
    ap.add_argument("--per-pass", type=int, default=0, help="max_pair_keys_per_pass (0: the library default, 2^27)")
    args = ap.parse_args()
    for scene in args.scenes.split(","):
        print(json.dumps(run(scene, args.reps, args.oracle, args.per_pass)), flush=True)


if __name__ == "__main__":
    main()
