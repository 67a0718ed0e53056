#!/usr/bin/env python
"""Where the BAL point leaves spend their time: per-kernel times with a byte model, and a sweep of the leaf run length.

    python profiles/point_leaf_stream.py --out DIR [--workloads bal_c5_metis,bal_1m,bal_c3] [--steps 10]
                                         [--sweep 32,64,128,256,1024] [--sweep-workloads bal_c5_metis,bal_1m]

Pass 1 (torch.profiler, CUDA activities, a pass of its own): per workload at the default run length, the device time per
LM step of the point-leaf kernels and their neighbours, and for the two kernels that stream the point conditionals the
achieved GB/s against the bytes they have to move:
  * leaf_point_fused_mma_kernel reads [A_c A_p b] of every leaf factor (2 rows x (DC + 4) columns, in the Jacobian storage
    precision) and writes every point's conditional [R S' d'] (3 x (s + 4) doubles, s = DC x cameras of the point);
  * backsub_point_kernel reads the same conditionals, the separator's slice of delta (s doubles per point) and writes the
    point's 3 unknowns.
Pass 2 (the library's phase timers, as bench.py reports them): per --sweep-workloads and B200_LEAF_RUN_MAX in --sweep
(plus the default, "auto"), ms per step (event pairs, L2 flushed in between) and phases_ms_per_step.leaf_fused /
back_substitute.  The card's name, power limit and maximum SM clock are read in the same process.
Writes DIR/point_leaf_stream.json and prints a summary."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = ("leaf_point_fused_mma_kernel", "backsub_point_kernel", "backsub_large_kernel", "front_df_kernel", "linerr_kernel")


def leaf_bytes(prob, jb):
    """(bytes of the fused point-leaf kernel, bytes of the point back-substitution) per launch: BAL projection groups."""
    from gtsam_b200 import problem as P
    obs = None
    dc = 6
    for g in prob.groups:
        if g.keys.shape[1] != 2 or P.FACTOR_DIM[g.type] != 2:
            continue
        dc = P.factor_ncols(g.type) - 4          # [A_c A_p b]: DC + 3 + 1 columns
        c = np.bincount(g.keys[:, 1], minlength=prob.nvars)
        obs = c if obs is None else obs + c
    m = obs[obs > 0].astype(np.int64)           # cameras per point
    s = dc * m
    cond = 3 * (s + 4) * 8                      # [R S' d'] per point, FP64
    fused = int(np.sum(m * 2 * (dc + 4) * jb + cond))
    backsub = int(np.sum(cond + s * 8 + 3 * 8))
    return fused, backsub, int(m.size)


def run_steps(ctx, dev, lm, stream, flush_buf, steps, phases=False):
    """steps LM iterations from the same start; returns (ms per step from event pairs, phase profile or None)."""
    import torch
    from gtsam_b200 import capi
    L = dev.L
    ms = 0.0
    for it in range(steps):
        dev.restore_values()
        capi._check(L.b200_lm_reset(lm.h))
        with torch.cuda.stream(stream):
            flush_buf.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if phases:
            dev.profile_enable(1 if it == 0 else 2)
        a.record(stream)
        lm.iterate()
        b.record(stream)
        dev.synchronize()
        if phases:
            dev.profile_enable(0)
        ms += a.elapsed_time(b)
    return ms / steps, (dev.profile() if phases else None)


def open_problem(ctx, prob, jac32):
    import torch
    from gtsam_b200 import capi, optimizer
    dev = capi.DeviceProblem(ctx, prob)
    if jac32:
        dev.set_jacobian_precision(True)
    dev.synchronize()
    lm = optimizer.LevenbergMarquardtOptimizer(ctx, prob, device_problem=dev)
    dev.save_values()
    stream = torch.cuda.ExternalStream(ctx.stream(), device=torch.device("cuda", 0))
    return dev, lm, stream


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--workloads", default="bal_c5_metis,bal_1m,bal_c3")
    ap.add_argument("--sweep-workloads", default="bal_c5_metis,bal_1m")
    ap.add_argument("--sweep", default="32,64,128,256,1024")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from gtsam_b200 import capi, datasets

    os.makedirs(a.out, exist_ok=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", smi, flush=True)
    ctx = capi.Context(0)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out = {"gpu": smi, "steps": a.steps, "profile": {}, "sweep": {}}
    names = list(dict.fromkeys(a.workloads.split(",") + [w for w in a.sweep_workloads.split(",") if w]))
    for wl in names:
        t0 = time.perf_counter()
        prob = datasets.make(wl)
        jac32 = wl.startswith("bal_c5")
        jb = 4 if jac32 else 8
        fused_b, back_b, npts = leaf_bytes(prob, jb)
        print(f"{wl}: {prob.nfactors} factors, {npts} points, generated in {time.perf_counter() - t0:.1f} s", flush=True)
        if wl in a.workloads.split(","):
            os.environ.pop("B200_LEAF_RUN_MAX", None)
            dev, lm, stream = open_problem(ctx, prob, jac32)
            run_steps(ctx, dev, lm, stream, flush_buf, a.warmup)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run_steps(ctx, dev, lm, stream, flush_buf, a.steps)
            rec = {"jacobian_bytes": jb, "points": npts, "model_bytes": {"leaf_point_fused_mma_kernel": fused_b,
                                                                         "backsub_point_kernel": back_b}, "kernels": {}}
            for ev in prof.key_averages():
                k = next((k for k in KERNELS if k in ev.key), None)
                if k is None:
                    continue
                us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                e = rec["kernels"].setdefault(k, {"ms_per_step": 0.0, "launches_per_step": 0.0})
                e["ms_per_step"] += us * 1e-3 / a.steps
                e["launches_per_step"] += ev.count / a.steps
            for k, e in rec["kernels"].items():
                if k in rec["model_bytes"] and e["launches_per_step"]:
                    e["gb_per_s"] = rec["model_bytes"][k] / (e["ms_per_step"] / e["launches_per_step"] * 1e-3) / 1e9
            out["profile"][wl] = rec
            print(wl, json.dumps({k: {x: round(y, 4) for x, y in e.items()} for k, e in rec["kernels"].items()}), flush=True)
            del lm
            dev.close()
        if wl in a.sweep_workloads.split(","):
            out["sweep"][wl] = {}
            for rm in ["auto"] + a.sweep.split(","):
                if rm == "auto":
                    os.environ.pop("B200_LEAF_RUN_MAX", None)
                else:
                    os.environ["B200_LEAF_RUN_MAX"] = rm
                dev, lm, stream = open_problem(ctx, prob, jac32)
                run_steps(ctx, dev, lm, stream, flush_buf, a.warmup)
                ms, _ = run_steps(ctx, dev, lm, stream, flush_buf, a.steps)
                _, ph = run_steps(ctx, dev, lm, stream, flush_buf, a.steps, phases=True)
                r = {"ms_per_step": ms, "leaf_fused": ph["leaf_fused"][0] / a.steps,
                     "back_substitute": ph["back_substitute"][0] / a.steps}
                out["sweep"][wl][rm] = r
                print(wl, "run max", rm, {k: round(v, 4) for k, v in r.items()}, flush=True)
                del lm
                dev.close()
            os.environ.pop("B200_LEAF_RUN_MAX", None)
        del prob
    with open(os.path.join(a.out, "point_leaf_stream.json"), "w") as f:
        json.dump(out, f, indent=1)
    ctx.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
