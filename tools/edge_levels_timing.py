#!/usr/bin/env python3
"""ORB-SLAM2's two-round local-BA protocol on ba_kitti_00 (kitti00_shaped when the fixture is absent), three ways:

  Huber optimize(5) -> outlier test (chi2 > 5.991 / 7.815 or landmark behind the camera) -> NONE optimize(10) -> outlier test

  (a) levels    classify_edges on the device, the state stays on the device
  (b) zero-omega get_chi2 + get_state -> numpy test with the depth -> set_problem with omega 0 on the outliers (structure reuse)
  (c) sub-problem get_chi2 + get_state -> numpy test -> the graph without the outliers, flattened, through a fresh set_problem

The arms alternate in one process, each on a fresh engine warmed up on the problem.  Prints the wall ms of the step between the rounds and of the whole protocol per arm, the device
time of one classify_edges (CUDA events on the engine's stream), the card and its power limit, and whether (a) and (b) gave
bitwise-equal trajectories, states and levels in every repetition.  Usage: python tools/edge_levels_timing.py [--reps 3] [--classify-reps 200]"""
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

HUBER = ((1, 1), (5.991 ** 0.5, 7.815 ** 0.5))
NONE = ((0, 0), (0.0, 0.0))
THR = (5.991, 7.815)


def set_kernel(eng, rk):
    for et in (0, 1):
        eng.set_robust_kernels(rk[0][et], rk[1][et], et)


def host_test(pkg, prob, eng, old):
    """the outlier test on the host: per-edge chi2 and the estimate come down, depth from q, t, Xw"""
    chi = eng.chi_squared()
    q, t, Xw = eng.state()
    ip = np.concatenate([prob.idx2[:, 0], prob.idx3[:, 0]]); il = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    z = (pkg.synth._rotate(q[ip], Xw[il]) + t[ip])[:, 2]
    thr = np.where(np.arange(prob.nedges) < prob.E2, THR[0], THR[1])
    return (old.astype(bool) | (chi > thr) | (z <= 0)).astype(np.uint8), (q, t, Xw)


def arm_levels(pkg, prob, eng):
    t0 = time.perf_counter()
    set_kernel(eng, HUBER); eng.initialize(prob)
    s1 = eng.optimize(5)
    t1 = time.perf_counter()
    eng.classify_edges(*THR, depth=True)
    t2 = time.perf_counter()
    set_kernel(eng, NONE)
    s2 = eng.optimize(10)
    eng.classify_edges(*THR, depth=True)
    t3 = time.perf_counter()
    return dict(step_ms=1e3 * (t2 - t1), total_ms=1e3 * (t3 - t0), stats=s1 + s2, state=eng.state(), levels=eng.edge_levels())


def arm_zero_omega(pkg, prob, eng):
    t0 = time.perf_counter()
    set_kernel(eng, HUBER); eng.initialize(prob)
    s1 = eng.optimize(5)
    t1 = time.perf_counter()
    mask, (q, t, Xw) = host_test(pkg, prob, eng, np.zeros(prob.nedges, np.uint8))
    p2 = prob.copy(); p2.q, p2.t, p2.Xw = q, t, Xw
    p2.omega2 = np.where(mask[:prob.E2] != 0, 0.0, prob.omega2); p2.omega3 = np.where(mask[prob.E2:] != 0, 0.0, prob.omega3)
    eng.initialize(p2)
    t2 = time.perf_counter()
    set_kernel(eng, NONE)
    s2 = eng.optimize(10)
    # (the engine now reports chi2 0 for the zeroed edges; they are at level 1 already and stay there)
    mask2, _ = host_test(pkg, prob, eng, mask)
    t3 = time.perf_counter()
    return dict(step_ms=1e3 * (t2 - t1), total_ms=1e3 * (t3 - t0), stats=s1 + s2, state=eng.state(), levels=mask2)


def arm_sub_problem(pkg, g, prob, eng):
    t0 = time.perf_counter()
    set_kernel(eng, HUBER); eng.initialize(prob)
    eng.optimize(5)
    t1 = time.perf_counter()
    mask, (q, t, Xw) = host_test(pkg, prob, eng, np.zeros(prob.nedges, np.uint8))
    g2 = dict(g); g2["q"] = g["q"].copy(); g2["t"] = g["t"].copy(); g2["Xw"] = g["Xw"].copy()
    pkg.graphio.write_back(g2, prob, q, t, Xw)
    km = np.ones(len(g["mono_vP"]), bool); ks = np.ones(len(g["stereo_vP"]), bool)
    km[prob.mono_rows[mask[:prob.E2] != 0]] = False; ks[prob.stereo_rows[mask[prob.E2:] != 0]] = False
    for k in ("mono_vP", "mono_vL", "mono_meas", "mono_info"):
        g2[k] = g[k][km]
    for k in ("stereo_vP", "stereo_vL", "stereo_meas", "stereo_info"):
        g2[k] = g[k][ks]
    sub = pkg.graphio.flatten(g2)
    eng.initialize(sub)
    t2 = time.perf_counter()
    set_kernel(eng, NONE)
    eng.optimize(10)
    host_test(pkg, sub, eng, np.zeros(sub.nedges, np.uint8))
    t3 = time.perf_counter()
    return dict(step_ms=1e3 * (t2 - t1), total_ms=1e3 * (t3 - t0))


def classify_device_ms(pkg, prob, eng, reps):
    """CUDA events around classify_edges on the engine's stream: without a level change (no scatter) and with every edge changing
    level (re-inclusion after all levels were set to 1: the mask scatter runs too)"""
    import torch
    stream = torch.cuda.ExternalStream(eng.stream_ptr())
    set_kernel(eng, HUBER); eng.initialize(prob); eng.optimize(5)
    out = {}
    for name in ("no_change", "with_scatter"):
        tot = 0.0
        for _ in range(reps):
            if name == "with_scatter":
                eng.set_edge_levels(np.ones(prob.nedges, np.uint8))
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            eng.classify_edges(*THR, depth=True, reinclude=name == "with_scatter")
            b.record(stream)
            b.synchronize()
            tot += a.elapsed_time(b)
        out[name] = tot / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--classify-reps", type=int, default=200)
    args = ap.parse_args()
    ge.build()
    pkg = ge.load_package()
    fx = os.path.join(ROOT, "oracle", "_ref", "fixtures", "ba_kitti_00.cubagraph")
    name = "ba_kitti_00" if os.path.exists(fx) else "kitti00_shaped"
    g = pkg.graphio.read_graph(fx) if name == "ba_kitti_00" else pkg.synth.make_config(name)
    prob = pkg.graphio.flatten(g)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    def run(arm):
        # one engine at a time, warmed up on the problem (every allocation, one structure build): each arm's first set_problem
        # reuses the structure, as in repeated local BA on one graph
        e = pkg.Engine(device=0)
        set_kernel(e, HUBER); e.initialize(prob); e.optimize(1)
        r = arm(e)
        e.close()
        return r
    runs = {k: [] for k in "abc"}
    for _ in range(args.reps):
        runs["a"].append(run(lambda e: arm_levels(pkg, prob, e)))
        runs["b"].append(run(lambda e: arm_zero_omega(pkg, prob, e)))
        runs["c"].append(run(lambda e: arm_sub_problem(pkg, g, prob, e)))
    # every repetition: (a) against (b), and each arm against its own first run
    ref = runs["a"][0]
    same = all(r["stats"] == ref["stats"] and all(np.array_equal(x, y) for x, y in zip(r["state"], ref["state"]))
               and np.array_equal(r["levels"], ref["levels"]) for r in runs["a"] + runs["b"])
    dev = run(lambda e: classify_device_ms(pkg, prob, e, args.classify_reps))
    res = dict(workload=name, edges=prob.nedges, card=card,
               step_ms={k: [round(r["step_ms"], 3) for r in v] for k, v in runs.items()},
               total_ms={k: [round(r["total_ms"], 3) for r in v] for k, v in runs.items()},
               classify_device_ms={k: round(v, 4) for k, v in dev.items()},
               excluded_after_round1=int(runs["a"][-1]["levels"].sum()), a_equals_b_bitwise=bool(same))
    for k, lbl in (("a", "levels"), ("b", "zero-omega"), ("c", "sub-problem")):
        print("%-12s inter-round step %8.3f ms (min of %d)   protocol %8.2f ms" % (lbl, min(res["step_ms"][k]), args.reps, min(res["total_ms"][k])))
    print("classify_edges device time: %.4f ms without a level change, %.4f ms with the scatter" % (dev["no_change"], dev["with_scatter"]))
    print("card: %s   (a) == (b) bitwise in all %d repetitions: %s" % (card, args.reps, same))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
