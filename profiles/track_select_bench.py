#!/usr/bin/env python
"""Track selection on the GPU (b200sfm_tracks_select, TrackEngine::FindTracksForProblem) on a seeded config-4-sized
track set.

  python profiles/track_select_bench.py [--tracks 2000000] [--images 10000] [--reps 5] [--check-frac 0.1]

Tracks: lengths uniform in 2..15 (about 17 M observations at 2 M tracks), images drawn uniformly from --images ids (so
a track may repeat an image), 5 % of the images unregistered, track ids scattered over 64 bits.  Two runs: the default
options (no per-image quota) and min_num_tracks_per_view = 100.  Reported per run: the ABI call end to end (host clock
around the synchronous call, median of --reps after a warm-up), per-kernel device times from torch.profiler (one
profiled call, same process), the host-to-device copy of the same input arrays by torch (pageable memory, the path the
call takes) as the upload estimate, the number selected, whether the device mask equals the host loop
(track_establishment.find_tracks_for_problem) on the first --check-frac of the tracks, and that loop's time.  The card
name and power limit are read in the same process.  Writes nothing.
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


def make(T, I, seed=1):
    import numpy as np
    from glomap_b200 import track_establishment as TE
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 16, T)
    n = int(lens.sum())
    ids = np.arange(T, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)       # odd multiplier: distinct ids
    tracks = TE.Tracks(ids, np.concatenate([[0], np.cumsum(lens)]).astype(np.int64),
                       rng.integers(0, I, n).astype(np.uint32), np.zeros(n, np.uint32))
    registered = np.sort(rng.choice(I, int(0.95 * I), replace=False)).astype(np.uint32)
    return tracks, registered


def subset(tracks, k):
    from glomap_b200 import track_establishment as TE
    e = int(tracks.begin[k])
    return TE.Tracks(tracks.track_ids[:k], tracks.begin[:k + 1], tracks.obs_image[:e], tracks.obs_feature[:e])


def call(ctx, tracks, reg, o):
    import numpy as np
    from glomap_b200 import _lib
    keep, num = np.zeros(len(tracks), np.uint8), ct.c_int64()
    p = lambda a: a.ctypes.data_as(ct.c_void_p)   # noqa: E731
    _lib.check(ctx.handle, ctx.lib.b200sfm_tracks_select(ctx.handle, len(tracks), p(tracks.track_ids), p(tracks.begin),
                                                         p(tracks.obs_image), len(reg), p(reg), o.min_num_tracks_per_view,
                                                         o.min_num_view_per_track, o.max_num_view_per_track, o.max_num_tracks,
                                                         p(keep), ct.byref(num)))
    return keep, num.value


def run(name, o, tracks, reg, reps, frac, card):
    import numpy as np
    import torch
    from glomap_b200 import estimators as E, track_establishment as TE
    ctx = E.default_context()
    keep, num = call(ctx, tracks, reg, o)                      # warm-up
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        again, _ = call(ctx, tracks, reg, o)
        times.append(time.perf_counter() - t0)
        assert again.tobytes() == keep.tobytes()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call(ctx, tracks, reg, o)
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            kern[ev.key[:60]] = round(t / 1e3, 3)
    kernel_ms = sum(v for k, v in kern.items() if "Memcpy" not in k and "Memset" not in k)
    up = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for a in (tracks.track_ids.view(np.int64), tracks.begin, tracks.obs_image.view(np.int32), reg.view(np.int32)):
            torch.from_numpy(a).to("cuda")
        torch.cuda.synchronize()
        up.append(time.perf_counter() - t0)
    k = max(1, int(frac * len(tracks)))
    sub = subset(tracks, k)
    sub_keep, _ = call(ctx, sub, reg, o)
    t0 = time.perf_counter()
    host = TE.find_tracks_for_problem(sub, reg.tolist(), o)
    host_s = time.perf_counter() - t0
    equal = bool(sub_keep.astype(bool).tolist() == np.isin(sub.track_ids, host.track_ids).tolist())
    return dict(run=name, card=card, tracks=len(tracks), observations=int(tracks.begin[-1]), registered=len(reg),
                min_num_tracks_per_view=o.min_num_tracks_per_view, selected=int(num),
                call_ms_median=round(1e3 * float(np.median(times)), 3), call_ms_all=[round(1e3 * t, 3) for t in times],
                kernel_ms=round(kernel_ms, 3), upload_ms_torch=round(1e3 * min(up), 3),
                check_tracks=k, host_equal=equal, host_loop_s=round(host_s, 3),
                kernels=dict(sorted(kern.items(), key=lambda kv: -kv[1])[:12]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=2_000_000)
    ap.add_argument("--images", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--check-frac", type=float, default=0.1)
    args = ap.parse_args()
    from glomap_b200 import track_establishment as TE
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    tracks, reg = make(args.tracks, args.images)
    for name, o in (("default", TE.TrackEstablishmentOptions()),
                    ("quota100", TE.TrackEstablishmentOptions(min_num_tracks_per_view=100))):
        print(json.dumps(run(name, o, tracks, reg, args.reps, args.check_frac, card)), flush=True)


if __name__ == "__main__":
    main()
