#!/usr/bin/env python3
"""ORB-SLAM2's OptimizeSim3 (optimize(5), the pair test, optimize(10 or 5), the test again) on keyframe pairs of ba_kitti_00
(kitti00_shaped when the fixture is absent): every pose pair (i, i + k), k = 1 .. --kmax, with at least 20 shared landmarks, from
graphio.sim3_problems with a scale drift s0 in [0.8, 1.25], the initial S12 perturbed (about 1 degree, 5 % of |t|, 3 % in scale) and
10-20 % of the matches wrong (keypoint moved 30-80 px, or the point of another match).

  call     Engine.optimize_sim3 on the first B problems, B = 1, 8, 64 and all: host clock around the whole call (packing, the copies,
           the launch and the unpacking)
  kernel   k_sim3_batch's device time from torch.profiler, in a pass of its own

Prints one JSON line: microseconds per problem per arm, the card and its power limit.
Usage: python tools/sim3_batch_timing.py [--reps 3] [--kmax 5] [--out path.json]"""
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

BATCHES = (1, 8, 64, None)       # None: every problem


def workload(pkg, prob, kmax, seed=1):
    P = np.concatenate([prob.idx2[:, 0], prob.idx3[:, 0]]); L = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    sets = [set(L[P == i].tolist()) for i in range(prob.Pall)]
    pairs = [(i, i + k) for k in range(1, kmax + 1) for i in range(prob.Pall - k) if len(sets[i] & sets[i + k]) >= 20]
    rng = np.random.default_rng(seed)
    problems = pkg.graphio.sim3_problems(prob, pairs, scale=np.exp(rng.uniform(np.log(0.8), np.log(1.25), len(pairs))))
    for p in problems:
        w = rng.normal(0, 0.01, 3)
        th = np.linalg.norm(w)
        dq = np.concatenate([np.sin(th / 2) * w / th, [np.cos(th / 2)]])
        x, y, z, qw = p.q
        a, b, c, d = dq
        p.q = np.array([d * x + a * qw + b * z - c * y, d * y + b * qw + c * x - a * z, d * z + c * qw + a * y - b * x, d * qw - a * x - b * y - c * z])
        p.t = p.t + rng.normal(0, 1, 3) * 0.05 * np.linalg.norm(p.t) / np.sqrt(3)
        p.s *= np.exp(rng.uniform(-0.03, 0.03))
        n = len(p.omega1)
        bad = rng.random(n) < rng.uniform(0.1, 0.2)
        move = bad & (rng.random(n) < 0.5)
        p.obs1[move] += rng.uniform(30, 80, (int(move.sum()), 2))
        swap = np.nonzero(bad & ~move)[0]
        if len(swap) > 1:
            p.X2[swap] = p.X2[np.roll(swap, 1)]
    return problems


def kernel_ms(eng, problems, calls):
    """mean device ms of k_sim3_batch over `calls` calls, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            eng.optimize_sim3(problems)
        torch.cuda.synchronize()
    tot, n = 0.0, 0
    for ev in prof.events():
        if "k_sim3_batch" in ev.name and ev.device_type.name == "CUDA":
            tot += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            n += 1
    if n != calls:
        raise RuntimeError("torch.profiler saw %d k_sim3_batch launches, expected %d" % (n, calls))
    return tot / n / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kmax", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pkg = ge.load_package()
    fx = os.path.join(ROOT, "oracle", "_ref", "fixtures", "ba_kitti_00.cubagraph")
    if os.path.exists(fx):
        graph, g = "ba_kitti_00", pkg.graphio.read_graph(fx)
    else:
        graph, g = "kitti00_shaped", pkg.synth.make_config("kitti00_shaped")
    problems = workload(pkg, pkg.graphio.flatten(g), args.kmax)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    eng = pkg.Engine(device=0)
    for B in BATCHES:          # warm-up: every shape the timed window uses
        eng.optimize_sim3(problems[:B])
    res = eng.optimize_sim3(problems)
    rec = {"graph": graph, "problems": len(problems), "pairs_per_problem": float(np.mean([len(p.omega1) for p in problems])),
           "inlier_fraction": float(np.mean([r["ninliers"] / max(1, len(p.omega1)) for p, r in zip(problems, res)])),
           "card": card, "reps": []}
    for _ in range(args.reps):
        rep = {}
        for B in BATCHES:
            pr = problems[:B]
            calls = max(1, min(200, 2000 // len(pr)))
            t0 = time.perf_counter()
            for _ in range(calls):
                eng.optimize_sim3(pr)
            dt = (time.perf_counter() - t0) / calls
            rep["batch_%d" % len(pr)] = dict(calls=calls, ms=1e3 * dt, us_per_problem=1e6 * dt / len(pr))
        rec["reps"].append(rep)
    rec["kernel"] = {}
    for B in BATCHES:          # the kernel alone, in a pass of its own (tracing slows the host)
        pr = problems[:B]
        ms = kernel_ms(eng, pr, max(3, min(50, 500 // len(pr))))
        rec["kernel"]["batch_%d" % len(pr)] = dict(ms=ms, us_per_problem=1e3 * ms / len(pr))
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
