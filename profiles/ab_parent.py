#!/usr/bin/env python
"""A/B of bench.py between builds of libgtsam_b200.so, run alternately in one session.

    python profiles/ab_parent.py --out DIR --arm parent=PATH/libgtsam_b200.so [--arm NAME=LIB ...] [--runs 3]
                                 [--bench-args "..."]

The in-tree library (gtsam_b200/libgtsam_b200.so, as build() left it) is arm "new".  Every run is one
`bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline --dump-outputs TMP/<arm>_<i>` in its own process with
gtsam_b200.capi.LIB_PATH pointed at the arm's library; the arms take turns (new, parent, ..., new, parent, ...) so that
drift of the shared machine falls on all of them.  The card's name, power limit and maximum SM clock are recorded in the
same session (nvidia-smi, read-only query).  Writes DIR/ab.json: per arm and workload every ms_per_step, the median,
max - min, the point-leaf phase times, and the largest difference of the dumped Values / LM state against the first run
of the first --arm (and that arm's spread against itself), and every run's bench.py line as DIR/<arm>_<i>.json.  The dumped
Values (about 22 MB per run) go to a temporary directory that is removed at the end."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNNER = ("import runpy, sys; sys.path.insert(0, {root!r}); from gtsam_b200 import capi; capi.LIB_PATH = {lib!r}; "
          "sys.argv = ['bench.py'] + {args!r}; runpy.run_path({bench!r}, run_name='__main__')")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--arm", action="append", default=[], help="NAME=path of a libgtsam_b200.so")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--bench-args", default="--gpus 1 --steps 20 --warmup 3 --no-cpu-baseline")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="ab_parent_")
    arms = {"new": os.path.join(ROOT, "gtsam_b200", "libgtsam_b200.so")}
    for spec in a.arm:
        name, path = spec.split("=", 1)
        arms[name] = os.path.abspath(path)
    ref_arm = next(n for n in arms if n != "new") if len(arms) > 1 else "new"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", smi, flush=True)
    recs = {n: [] for n in arms}
    for i in range(a.runs):
        for name, lib in arms.items():
            dump = os.path.join(tmp, f"{name}_{i}")
            args = a.bench_args.split() + ["--dump-outputs", dump]
            cmd = [sys.executable, "-c", RUNNER.format(root=ROOT, lib=lib, args=args, bench=os.path.join(ROOT, "bench.py"))]
            out = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
            line = next((l for l in reversed(out.stdout.splitlines()) if l.startswith("{")), None)
            if out.returncode != 0 or line is None:
                print(f"{name} run {i}: exit {out.returncode}\n{out.stderr[-3000:]}", flush=True)
                sys.exit(1)
            rec = json.loads(line)
            with open(os.path.join(a.out, f"{name}_{i}.json"), "w") as f:
                f.write(line + "\n")
            recs[name].append((rec, dump))
            print(f"{name} run {i}: ms_per_step {rec['ms_per_step']:.4f}", flush=True)

    def workloads(rec):     # (name as in the dump files, record): the primary workload, then bench.py's other_workloads
        yield str(rec["config"]["workload"]).split(":")[0], rec
        for name, o in (rec.get("other_workloads") or {}).items():
            if isinstance(o, dict) and "ms_per_step" in o:
                yield name, o

    def dumped(dump, wl):
        return (np.load(os.path.join(dump, f"{wl}.values.npy")), np.load(os.path.join(dump, f"{wl}.lm_state.npy")))

    def diff(x, y):
        (v0, s0), (v1, s1) = x, y
        return {"values_max_abs": float(np.max(np.abs(v1 - v0))),
                "values_rel2": float(np.linalg.norm(v1 - v0) / max(np.linalg.norm(v0), 1e-300)),
                "error_rel": float(abs(s1[0] - s0[0]) / abs(s0[0])), "lambda_equal": bool(s1[1] == s0[1])}

    summary = {"gpu": smi, "bench_args": a.bench_args, "runs": a.runs, "arms": list(arms), "workloads": {}}
    base_rec, base_dump = recs[ref_arm][0]
    for wl, _ in workloads(base_rec):
        base = dumped(base_dump, wl)
        entry = {}
        for name in arms:
            ms, ph, d = [], [], []
            for rec, dump in recs[name]:
                r = dict(workloads(rec)).get(wl)
                if r is None:
                    continue
                ms.append(r["ms_per_step"])
                p = r.get("phases_ms_per_step", {})
                ph.append({k: p.get(k) for k in ("leaf_fused", "leaf_schur", "eliminate_large", "back_substitute")})
                d.append(diff(base, dumped(dump, wl)))
            if ms:
                entry[name] = {"ms_per_step": ms, "median": float(np.median(ms)), "spread": float(max(ms) - min(ms)),
                               "phases": ph, "vs_" + ref_arm + "_run0": d}
        summary["workloads"][wl] = entry
    shutil.rmtree(tmp)
    with open(os.path.join(a.out, "ab.json"), "w") as f:
        json.dump(summary, f, indent=1)
    for wl, e in summary["workloads"].items():
        print(wl, {n: (round(v["median"], 4), round(v["spread"], 4)) for n, v in e.items()})
    return 0


if __name__ == "__main__":
    sys.exit(main())
