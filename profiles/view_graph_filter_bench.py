#!/usr/bin/env python
"""The view-graph passes of stage 3 (RelPoseFilter::FilterRotations + ViewGraph::KeepLargestConnectedComponents) on the
GPU against the numpy / scipy path the mapper used before, on the lattice view graphs of synthetic.make_lattice_view_graph.

  python profiles/view_graph_filter_bench.py [--sizes 10:45,100:1000,10000:50,100000:100] [--reps 5]

A size is frames:neighbours; 100000:100 is config 5 (100 k frames, about 5 M pairs).  Rotations: the ground truth, so
the filter removes the outlier pairs (5 %).  Reported per size, median of --reps after a warm-up, host clock around the
synchronous calls:
  device_ms      both device calls, host arrays in and out (b200sfm_view_graph_filter_rotations, then
                 b200sfm_view_graph_keep_largest_component), plus the quaternion conversion they need
  kernel_ms      device time of the vg_* kernels of one profiled run (torch.profiler), copies excluded
  numpy_scipy_ms mapper.filter_rotations (trace formula on rotation matrices) + mapper.largest_connected_component
  host_loop_ms   the host restatements of view_graph.py (the reference's loops; only up to --host-max pairs)
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


def run(frames, neighbours, reps, host_max):
    import numpy as np
    import torch
    from glomap_b200 import estimators as E, geometry as G, mapper as M, synthetic as S, view_graph as VG
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    vg = S.make_lattice_view_graph(frames, neighbours, seed=1, noise_deg=2.0, outlier_ratio=0.05)
    R = vg.R_gt
    ctx = E.default_context()
    q_rel = G.rotmat_to_quat_xyzw_fast(vg.R_rel)                # converted once per view graph by the mapper
    frame = np.arange(vg.n_images, dtype=np.int32)
    out = {}

    def device():
        q = G.rotmat_to_quat_xyzw_fast(R)
        v, n = VG.filter_rotations_device(q, vg.ei, vg.ej, q_rel, 10.0, ctx=ctx)
        out["dev"] = (v, n) + VG.keep_largest_connected_components_device(vg.n_images, frame, vg.ei, vg.ej, v, ctx=ctx)

    def numpy_scipy():
        v = M.filter_rotations(vg, R, 10.0)
        out["np"] = (v, M.largest_connected_component(vg.n_images, vg.ei[v], vg.ej[v]))

    rec = dict(card=card, frames=vg.n_images, pairs=int(vg.E), device_ms=_median_ms(device, reps),
               numpy_scipy_ms=_median_ms(numpy_scipy, reps))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        device()
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0 and "vg_" in ev.key:
            kern[ev.key.split("(")[0][:40]] = round(t / 1e3, 4)
    rec["kernel_ms"] = round(sum(kern.values()), 4)
    rec["kernels"] = kern
    v, n, v2, reg, num = out["dev"]
    rec.update(invalidated=n, registered_images=num)
    # the trace formula and angularDistance agree away from the threshold
    rec["same_filter_as_numpy"] = bool(np.array_equal(v, out["np"][0]))
    rec["same_component_as_scipy"] = bool(np.array_equal(reg, out["np"][1]))
    if vg.E <= host_max:
        def host():
            q = G.rotmat_to_quat_xyzw_fast(R)
            hv, _ = VG.filter_rotations(q, vg.ei, vg.ej, q_rel, 10.0)
            VG.keep_largest_connected_components(vg.n_images, frame, vg.ei, vg.ej, hv)
        rec["host_loop_ms"] = _median_ms(host, max(1, min(reps, 3)))
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10:45,30:20,100:1000,10000:50,100000:100")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-max", type=int, default=300_000, help="largest pair count the host loops are timed at")
    args = ap.parse_args()
    for s in args.sizes.split(","):
        f, k = (int(x) for x in s.split(":"))
        print(json.dumps(run(f, k, args.reps, args.host_max)), flush=True)


if __name__ == "__main__":
    main()
