#!/usr/bin/env python3
"""ORB-SLAM2's PoseOptimization (four rounds of optimize(10) with the outlier test and re-inclusion) on every pose of ba_kitti_00
(kitti00_shaped when the fixture is absent) at the fixture's own initial estimates, each pose one frame with all of its edges:

  (a) engine path   per frame: set_problem (one free pose, its points fixed), per round set_robust_kernel + set_state + optimize(10)
                    + classify_edges, then get_state; host clock around the whole, over --engine-frames frames
  (b) batch         Engine.optimize_poses on the first B frames, B = 1, 8, 64 and all: host clock around the whole call (packing,
                    the copies, the launch and the unpacking), and the kernel alone (k_pose_batch's device time from torch.profiler,
                    in a pass of its own)

The arms alternate within each of --reps repetitions.  Prints one JSON line: microseconds per frame and edge-iterations per second
(edges at level 0 times LM iterations, summed over the frames and rounds) per arm, the card and its power limit.
Usage: python tools/pose_batch_timing.py [--reps 3] [--engine-frames 100] [--out path.json]"""
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

BATCHES = (1, 8, 64, None)       # None: every frame


def engine_path(pkg, eng, f, rounds):
    """one frame through the engine; returns edge-iterations"""
    prob = f.flat_problem()
    eng.initialize(prob)
    work = 0
    included = prob.nedges
    for r in rounds:
        for et in (0, 1):
            eng.set_robust_kernels(r.kernel[et], r.delta[et], et)
        if r.restart:
            eng.set_state(prob.q, prob.t, prob.Xw)
        work += included * len(eng.optimize(r.iterations))
        c = eng.classify_edges(r.chi2_mono, r.chi2_stereo, depth=r.depth, reinclude=r.reinclude)
        included = c["included_mono"] + c["included_stereo"]
    eng.state()
    return work


def batch_work(frames, res):
    """edge-iterations of a batch result: per round, the edges at level 0 during the round times its iterations"""
    work = 0
    for f, r in zip(frames, res):
        inc = len(f.omega2) + len(f.omega3)
        for k, st in enumerate(r["stats"]):
            work += inc * len(st)
            inc = int(r["counts"][k][0] + r["counts"][k][1])
    return work


def kernel_ms(eng, frames, rounds, calls):
    """mean device ms of k_pose_batch over `calls` calls, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            eng.optimize_poses(frames, rounds)
        torch.cuda.synchronize()
    tot, n = 0.0, 0
    for ev in prof.events():
        if "k_pose_batch" in ev.name and ev.device_type.name == "CUDA":
            tot += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            n += 1
    if n != calls:
        raise RuntimeError("torch.profiler saw %d k_pose_batch launches, expected %d" % (n, calls))
    return tot / n / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--engine-frames", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pkg = ge.load_package()
    fx = os.path.join(ROOT, "oracle", "_ref", "fixtures", "ba_kitti_00.cubagraph")
    if os.path.exists(fx):
        graph, g = "ba_kitti_00", pkg.graphio.read_graph(fx)
    else:
        graph, g = "kitti00_shaped", pkg.synth.make_config("kitti00_shaped")
    prob = pkg.graphio.flatten(g)
    frames = pkg.graphio.pose_frames(prob, range(prob.Pall))
    rounds = pkg.orbslam2_pose_schedule()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    sel = np.linspace(0, len(frames) - 1, args.engine_frames).astype(int)

    eng = pkg.Engine(device=0)       # the engine path's engine
    beng = pkg.Engine(device=0)      # the batch's engine
    # warm-up: every shape the timed window uses
    for b in sel[:5]:
        engine_path(pkg, eng, frames[b], rounds)
    for B in BATCHES:
        beng.optimize_poses(frames[:B], rounds)

    rec = {"graph": graph, "frames": len(frames), "edges_per_frame": float(np.mean([len(f.omega2) + len(f.omega3) for f in frames])),
           "card": card, "reps": []}
    for _ in range(args.reps):
        rep = {}
        t0 = time.perf_counter()
        work = sum(engine_path(pkg, eng, frames[b], rounds) for b in sel)
        dt = time.perf_counter() - t0
        rep["engine_path"] = dict(frames=len(sel), us_per_frame=1e6 * dt / len(sel), edge_iters_per_s=work / dt)
        for B in BATCHES:
            fr = frames[:B]
            calls = max(1, min(200, 2000 // len(fr)))
            t0 = time.perf_counter()
            for _ in range(calls):
                res = beng.optimize_poses(fr, rounds)
            dt = (time.perf_counter() - t0) / calls
            work = batch_work(fr, res)
            rep["batch_%d" % len(fr)] = dict(calls=calls, us_per_frame=1e6 * dt / len(fr), edge_iters_per_s=work / dt)
        rec["reps"].append(rep)
    # the kernel alone, in a pass of its own (tracing slows the host)
    rec["kernel"] = {}
    for B in BATCHES:
        fr = frames[:B]
        ms = kernel_ms(beng, fr, rounds, max(3, min(50, 500 // len(fr))))
        work = batch_work(fr, beng.optimize_poses(fr, rounds))
        rec["kernel"]["batch_%d" % len(fr)] = dict(ms=ms, us_per_frame=1e3 * ms / len(fr), edge_iters_per_s=work / (ms * 1e-3))
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
