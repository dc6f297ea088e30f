#!/usr/bin/env python
"""Per-kernel device time of the resident BA solve, from torch.profiler (CUPTI), on the scene bench.py builds.

  python profiles/kernel_times.py --workload config4 [--optimize-intrinsics 1] [--solves 2]

Prints, per kernel, launches, total and average device time over the profiled solves (after one warm-up solve), the
LM / PCG iteration counts, and the device memory the resident problem holds (torch.cuda.mem_get_info before problem
creation and after the warm-up solve).  Environment switches (B200SFM_*) apply as in bench.py.  Writes nothing.
"""
import argparse
import collections
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config4")
    ap.add_argument("--optimize-intrinsics", type=int, default=0)
    ap.add_argument("--solves", type=int, default=2)
    ap.add_argument("--top", type=int, default=14)
    args = ap.parse_args()
    import torch
    from bench import WORKLOADS
    from glomap_b200 import estimators as E, synthetic as S

    C, P, L, chunk = WORKLOADS[args.workload]
    sc = S.make_scene(C, P, L, seed=1, pixel_sigma=0.5, chunk=chunk, point_range=(0, P))
    init = S.perturb_scene(sc, chunk=chunk, point_offset=0)
    mask = E.first_frame_mask(C)
    torch.cuda.set_device(0)
    ctx = E.Context(0, 0, 1, None)
    opts = E.BundleAdjusterOptions(optimize_intrinsics=bool(args.optimize_intrinsics))
    opts.solver_options.max_num_iterations = 20
    opts.solver_options.pcg_rel_tolerance = 0.05
    opts.solver_options.pcg_max_iterations = 200
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    prob = E.BAProblem(ctx, sc, 3, mask)
    prob.set_state(init.intr_params, init.quat, init.trans, init.points)
    prob.save_state()
    prob.solve(opts)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    its = []
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.solves):
            prob.restore_state()
            st = prob.solve(opts).as_dict()
            its.append((st["iterations"], st["pcg_iterations"]))
        torch.cuda.synchronize()
    agg = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.name and not ev.name.startswith("Memcpy") \
                and not ev.name.startswith("Memset"):
            name = ev.name.split("(")[0].replace("void ", "").replace("b200::", "")
            agg[name][0] += 1
            agg[name][1] += ev.device_time_total
    tot = sum(v[1] for v in agg.values())
    print(f"{args.workload} optimize_intrinsics={args.optimize_intrinsics} env="
          f"{ {k: v for k, v in os.environ.items() if k.startswith('B200SFM_')} } LM/PCG per solve {its}")
    print(f"device memory held by the resident problem after one solve: {(free0 - free1) / 1e9:.3f} GB")
    print("| kernel | launches | total ms | avg us |\n|---|---|---|---|")
    for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:args.top]:
        print(f"| `{k}` | {n} | {us / 1e3:.3f} | {us / n:.1f} |")
    print(f"total kernel time {tot / 1e3 / args.solves:.2f} ms per solve\n")
    prob.free()
    ctx.close()


if __name__ == "__main__":
    main()
