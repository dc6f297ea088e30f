#!/usr/bin/env python
"""ImagePairsInlierCount on the GPU (b200sfm_image_pairs_inlier_count) on seeded match sets.

  python profiles/inlier_count_bench.py [--sizes config2,config4] [--reps 5] [--host-pairs 300]

Match set: every pair of observations inside a track of ``synthetic.make_scene`` is a match, plus 20 % random outlier
matches; pairs are 80 % CALIBRATED, 15 % UNCALIBRATED, 5 % PLANAR (``synthetic.make_pair_matches``).  Sizes: config2 =
make_scene(1000, 200k) (about 9 M matches), config4 = make_scene(1000, 2M) (about 90 M matches; the 1000-camera view
graph keeps about 180 matches per pair, where 10k cameras with random candidate sets would leave about 2).
Reported per size: the device time of each kernel (torch.profiler / CUPTI, one profiled call after a warm-up), the ABI
call end to end from pinned host buffers (host clock around the call, which ends in a stream synchronise; median of
--reps), matches per second for both, the byte model below over kernel time against the 3.35 TB/s data-sheet HBM
bandwidth, the host restatement's time per match on a sample of pairs, and the card name and power limit.  Writes nothing.

Byte model (per call, HBM): a CALIBRATED match reads 8 B of indices, gathers two 24-B bearings and writes a 1-B mask
(57 B); an F / H match gathers two 16-B pixels instead (41 B) and an F match re-reads and re-writes its mask byte (2 B);
a feature of an image of a CALIBRATED pair is read (16 B) and its bearing written (24 B); a pair costs about 200 B
(inputs, 256-B record written and read, outputs).
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

SIZES = {"config2": (1000, 200_000), "config4": (1000, 2_000_000), "tiny": (50, 5_000)}
PEAK_BW = 3.35e12


def byte_model(d):
    cfg, mb = d["config"], d["match_begin"]
    n = mb[1:] - mb[:-1]
    m_e, m_f, m_h = int(n[cfg == 2].sum()), int(n[cfg == 3].sum()), int(n[(cfg >= 4) & (cfg <= 6)].sum())
    import numpy as np
    need = np.zeros(len(d["image_intr"]), bool)
    need[d["img1"][cfg == 2]] = True
    need[d["img2"][cfg == 2]] = True
    nf_e = int((d["feature_begin"][1:] - d["feature_begin"][:-1])[need].sum())
    return 57 * m_e + 41 * (m_f + m_h) + 2 * m_f + 40 * nf_e + 200 * len(cfg), dict(M_E=m_e, M_F=m_f, M_H=m_h, nf_E=nf_e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="config2,config4")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-pairs", type=int, default=300)
    args = ap.parse_args()
    sizes = args.sizes.split(",")
    if len(sizes) > 1:   # one process per size: a second torch.profiler session in a process records no kernels
        for size in sizes:
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--sizes", size, "--reps", str(args.reps),
                                   "--host-pairs", str(args.host_pairs)])
        return
    import numpy as np
    import torch
    from glomap_b200 import estimators as E, image_pair_inliers as IP, synthetic as S
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    torch.cuda.set_device(0)
    torch.cuda.init()
    ctx = E.Context(0, 0, 1, None)
    o = IP.InlierThresholdOptions()
    for size in sizes:
        C, P = SIZES[size]
        t0 = time.perf_counter()
        d = S.make_pair_matches(S.make_scene(C, P, 10.0, seed=1, pixel_sigma=0.5), seed=1)
        t_gen = time.perf_counter() - t0
        Ep, M = len(d["img1"]), len(d["matches"])

        def pinned(a):
            t = torch.empty(a.shape, dtype=getattr(torch, a.dtype.name), pin_memory=True)
            t.numpy()[...] = a
            return t
        keep = {k: pinned(np.ascontiguousarray(d[k])) for k in ("feature_begin", "features", "image_intr", "intr_model",
                                                                   "intr_params", "img1", "img2", "config", "quat", "trans", "F",
                                                                   "H", "match_begin", "matches")}
        out = {"mask": torch.empty(M, dtype=torch.uint8, pin_memory=True), "n": torch.empty(Ep, dtype=torch.int32, pin_memory=True),
               "score": torch.empty(Ep, dtype=torch.float64, pin_memory=True)}
        p = lambda k: ct.c_void_p(keep[k].data_ptr())   # noqa: E731
        q = lambda k: ct.c_void_p(out[k].data_ptr())    # noqa: E731

        def call():
            rc = ctx.lib.b200sfm_image_pairs_inlier_count(
                ctx.handle, len(d["image_intr"]), p("feature_begin"), p("features"), p("image_intr"), len(d["intr_model"]),
                p("intr_model"), p("intr_params"), Ep, p("img1"), p("img2"), p("config"), p("quat"), p("trans"), p("F"), p("H"),
                p("match_begin"), p("matches"), o.max_epipolar_error_E, o.max_epipolar_error_F, o.max_epipolar_error_H,
                q("mask"), q("n"), q("score"))
            assert rc == 0, ctx.lib.b200sfm_last_error(ctx.handle)
        call()   # warm-up (module load, pool growth)
        ms = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            call()
            ms.append(1e3 * (time.perf_counter() - t0))
        first = (out["mask"].numpy().copy(), out["score"].numpy().copy())
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        assert np.array_equal(first[0], out["mask"].numpy()) and np.array_equal(first[1].view(np.uint64),
                                                                                 out["score"].numpy().view(np.uint64))
        kern, copies = {}, {"h2d": 0.0, "d2h": 0.0}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA or not ev.name:
                continue
            if ev.name.startswith("Memcpy HtoD"):
                copies["h2d"] += ev.device_time_total / 1e3
            elif ev.name.startswith("Memcpy DtoH"):
                copies["d2h"] += ev.device_time_total / 1e3
            elif "pair_" in ev.name:
                name = ev.name.split("(")[0].replace("void ", "").replace("b200::", "")
                kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1e3
        k_ms = sum(kern.values())
        if not kern:
            raise RuntimeError("no pair_* kernel in the profile: " + str(sorted({ev.name for ev in prof.events()})[:20]))
        nbytes, parts = byte_model(d)
        # host restatement on a sample of pairs
        features, cameras, pairs = S.pairs_from_match_arrays({**d, "img1": d["img1"][:args.host_pairs],
                                                              "match_begin": d["match_begin"][:args.host_pairs + 1]})
        m_host = int(d["match_begin"][min(args.host_pairs, Ep)])
        t0 = time.perf_counter()
        IP.image_pairs_inlier_count(pairs, features, cameras, o)
        host_s = time.perf_counter() - t0
        n_inl = out["n"].numpy()
        host_inl = np.array([len(x.inliers) for x in pairs])
        rec = dict(size=size, card=card, images=C, pairs=Ep, matches=M, **parts, inliers=int(n_inl.sum()),
                   host_sample_agrees=bool(np.array_equal(host_inl, n_inl[:len(pairs)])), generate_s=round(t_gen, 1),
                   kernel_ms={k: round(v, 3) for k, v in kern.items()}, kernel_total_ms=round(k_ms, 3),
                   kernel_gmatch_per_s=round(M / k_ms / 1e6, 2), call_ms_median=round(float(np.median(ms)), 2),
                   call_ms_all=[round(x, 2) for x in ms], call_gmatch_per_s=round(M / float(np.median(ms)) / 1e6, 3),
                   profiled_h2d_ms=round(copies["h2d"], 2), profiled_d2h_ms=round(copies["d2h"], 2),
                   model_bytes=nbytes, model_tb_per_s=round(nbytes / (k_ms * 1e-3) / 1e12, 3),
                   frac_of_3p35=round(nbytes / (k_ms * 1e-3) / PEAK_BW, 3),
                   host_sample_matches=m_host, host_us_per_match=round(1e6 * host_s / max(m_host, 1), 3))
        print(json.dumps(rec), flush=True)
        del keep, out, d
    ctx.close()


if __name__ == "__main__":
    main()
