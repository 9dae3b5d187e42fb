"""Per-solve device time of the two solvers of the reduced camera system (the default PCG policy and the dense Cholesky,
Engine.set_linear_solver) on the lambda ladder 1e3 / 10 / 0.1, and optimize(10) per LM step for both.

  python tools/dense_solve_timing.py [--reps 3] [--solves 5] [--out DIR]

Per solve: cuba_bench_stage 4 (the solve alone, CUDA events, L2 flushed before each solve) after one stage solve at the same lambda
(its Schur complement is what the timed solves factor).  The two solvers alternate, repetition by repetition; every number is the
median over the repetitions with the min .. max spread.  The factorisation rate is the algorithmic work n^3/3 multiply-adds (2 n^3/3
flop, n = 6 numP) over the whole dense solve (scatter and both substitutions included), against the data sheet's 67 TFLOP/s of the
H100 SXM's FP64 tensor cores.  The card name and power limit are read in the same run.  Writes dense_solve_timing.json into --out.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

LADDER = (1e3, 10.0, 0.1)
GRAPHS = ("local_ba", "kitti07_shaped", "orbit_600", "covis_1000", "kitti00_shaped", "covis_2000", "ba_kitti_07", "ba_kitti_00")
DENSE_ONLY = ("covis_2000",)
PEAK_FP64_TC = 67e12
HUBER = ((1, 1), (5.991 ** 0.5, 7.815 ** 0.5))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def load(pkg, name):
    if name.startswith("ba_"):
        path = os.path.join(ROOT, "oracle", "_ref", "fixtures", name + ".cubagraph")
        if not os.path.exists(path):
            return None
        return pkg.graphio.flatten(pkg.graphio.read_graph(path))
    return pkg.graphio.flatten(pkg.synth.make_config(name))


def engine(pkg, prob, solver):
    eng = pkg.Engine(device=0)
    for et in (0, 1):
        eng.set_robust_kernels(HUBER[0][et], HUBER[1][et], et)
    eng.set_linear_solver(solver)
    eng.initialize(prob)
    return eng


def spread(v):
    v = np.asarray(v, dtype=np.float64)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--solves", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--graphs", default=",".join(GRAPHS))
    ap.add_argument("--out", default=".")
    a = ap.parse_args()
    pkg = ge.load_package()
    pkg.load_library()
    res = {"card": card(), "graphs": {}}
    print("card:", res["card"], flush=True)
    for name in a.graphs.split(","):
        prob = load(pkg, name)
        if prob is None:
            print("%s: no fixture, not measured" % name, flush=True)
            continue
        solvers = ("dense",) if name in DENSE_ONLY else ("pcg", "dense")
        n = 6 * prob.numP
        engs = {s: engine(pkg, prob, s) for s in solvers}
        for e in engs.values():
            e.linearize()
        solve = {s: {lam: [] for lam in LADDER} for s in solvers}
        kernel = {s: {} for s in solvers}
        step = {s: [] for s in solvers}
        for rep in range(a.reps):
            order = solvers if rep % 2 == 0 else solvers[::-1]
            for s in order:
                e = engs[s]
                for lam in LADDER:
                    e.solve(lam)
                    solve[s][lam].append(e.bench_stage(4, reps=a.solves, flush_l2=True, lam=lam))
                    info = e.pcg_info()
                    kernel[s][lam] = "%s%s it=%d st=%d" % (info["kernel"], "/2L" if info["two_level"] else "", info["iters"], info["status"])
            for s in order:
                e = engs[s]
                e.reset_state()
                t0 = time.perf_counter()
                st = e.optimize(a.steps)
                dt = time.perf_counter() - t0
                step[s].append(1e3 * dt / max(len(st), 1))
        g = {"numP": prob.numP, "n": n, "solvers": {}}
        for s in solvers:
            d = {"solve_ms": {str(lam): spread(solve[s][lam]) for lam in LADDER}, "kernel": {str(k): v for k, v in kernel[s].items()},
                 "step_ms": spread(step[s])}
            if s == "dense":
                tmin = min(np.median(solve[s][lam]) for lam in LADDER) * 1e-3
                flop = 2.0 * n ** 3 / 3.0
                d["factor_tflops"] = flop / tmin / 1e12
                d["share_of_67tf"] = flop / tmin / PEAK_FP64_TC
            g["solvers"][s] = d
        res["graphs"][name] = g
        for s in solvers:
            d = g["solvers"][s]
            print("%-15s %-5s n=%5d  solve ms %s  step ms %.3f [%.3f..%.3f]  %s%s" % (
                name, s, n, "  ".join("%g: %.3f [%.3f..%.3f]" % (lam, d["solve_ms"][str(lam)]["median"], d["solve_ms"][str(lam)]["min"],
                                                                  d["solve_ms"][str(lam)]["max"]) for lam in LADDER),
                d["step_ms"]["median"], d["step_ms"]["min"], d["step_ms"]["max"], d["kernel"],
                ("  %.2f TFLOP/s (%.1f %% of 67)" % (d["factor_tflops"], 100 * d["share_of_67tf"])) if s == "dense" else ""), flush=True)
        for e in engs.values():
            e.close()
    res["card_after"] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "dense_solve_timing.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
