#!/usr/bin/env python
"""Maximum-spanning-tree initialisation of rotation averaging on the GPU (b200sfm_ra_mst_init) against the host
function initialize_from_maximum_spanning_tree, on the lattice view graphs of synthetic.make_lattice_view_graph
(all weights equal, so the edge index decides every tie).

  python profiles/mst_init_bench.py [--frames 10,30,100,1000,10000,100000] [--reps 7]

The sizes straddle RotationEstimator's MST_DEVICE_MIN_EDGES gate and reach config 5 (100 000 frames).  Reported per
size: the device call from host to host (wall clock around the synchronous call, copies included; median of --reps after
a warm-up), the call's own ms_total, rounds and launches, the host function's time (median of up to --reps runs, one run
where it takes over a second), whether the device parents equal the host tree's (scipy MST + BFS from frame 0) and the
largest rotation difference.  The card name and power limit are read in the same process.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def host_parents(vg):
    import numpy as np
    import scipy.sparse as sp
    from scipy.sparse.csgraph import breadth_first_order, minimum_spanning_tree
    n, m = vg.n_images, vg.E
    cost = (float(vg.weight.max()) - vg.weight) + 1e-9 * (1 + np.arange(m) / max(m, 1))
    G = sp.coo_matrix((cost, (vg.ei, vg.ej)), shape=(n, n)).tocsr()
    T = minimum_spanning_tree(G.maximum(G.T))
    _, pred = breadth_first_order(T.maximum(T.T).tocsr(), 0, directed=False)
    par = np.where(pred < 0, -1, pred)
    par[0] = 0
    return par


def run(n, reps, card):
    import numpy as np
    from glomap_b200 import _lib, estimators as E, synthetic as S
    ctx = E.default_context()
    vg = S.make_lattice_view_graph(n)
    st = _lib.MSTStats()
    E.initialize_from_maximum_spanning_tree_device(vg, None, ctx)               # warm-up
    times, inner = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        R, par = E.initialize_from_maximum_spanning_tree_device(vg, None, ctx, stats=st)
        times.append(1e3 * (time.perf_counter() - t0))
        inner.append(st.ms_total)
    host = []
    for _ in range(reps):
        t0 = time.perf_counter()
        R_host = E.initialize_from_maximum_spanning_tree(vg)
        host.append(1e3 * (time.perf_counter() - t0))
        if host[-1] > 1000:
            break
    return dict(card=card, frames=n, edges=int(vg.E), device_call_ms_median=round(float(np.median(times)), 3),
                device_call_ms_all=[round(t, 3) for t in times], ms_total_median=round(float(np.median(inner)), 3),
                boruvka_rounds=st.boruvka_rounds, max_depth=st.max_depth, kernel_launches=st.kernel_launches,
                host_ms_median=round(float(np.median(host)), 3), host_runs=len(host),
                parents_equal=bool(np.array_equal(par, host_parents(vg))), max_abs_diff_R=float(np.abs(R - R_host).max()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="10,30,100,1000,10000,100000")
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    from glomap_b200 import estimators as E, synthetic as S
    E.initialize_from_maximum_spanning_tree(S.make_lattice_view_graph(10))      # the host function's first call imports scipy
    for n in (int(x) for x in args.frames.split(",")):
        print(json.dumps(run(n, args.reps, card)), flush=True)


if __name__ == "__main__":
    main()
