#!/usr/bin/env python3
"""The batched LM entry points on host arrays against the same batches on device-resident arrays:

  pose batch  ORB-SLAM2's PoseOptimization schedule on the poses of ba_kitti_00 (kitti00_shaped when the fixture is absent), every
              pose one frame with all of its edges, B = 1, 8, 64 and all
  Sim3        the OptimizeSim3 problems of tools/sim3_batch_timing.py, B = 1, 8, 64 and all

  host     Engine.optimize_poses_flat / optimize_sim3_flat from numpy arrays (pack, H2D, launch, D2H, synchronise, unpack)
  device   Engine.optimize_poses_device / optimize_sim3_device on tensors already in device memory, outputs and workspace reused
  graph    the device call captured once into a CUDA graph, replayed

Whole-call wall time: a host clock around `calls` calls, ending in a device synchronise, the arms alternating within each of --reps
repetitions.  Kernel time: the device time of every kernel of one device call (the LM kernel and the validate / pack / unpack
kernels), from torch.profiler in a pass of its own.  Prints one JSON line with the card's name and power limit.
Usage: python tools/device_batch_timing.py [--reps 3] [--out path.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import __graft_entry__ as ge  # noqa: E402
import sim3_batch_timing  # noqa: E402

BATCHES = (1, 8, 64, None)       # None: the whole workload


def arms(torch, eng, kind, flat, rounds):
    """(host call, device call, graph replay) of one batch; the device call reuses its outputs and workspace"""
    dev = {k: None if v is None else torch.from_numpy(v).cuda() for k, v in flat.items()}
    if kind == "pose":
        host = lambda: eng.optimize_poses_flat(rounds=rounds, **flat)
        first = eng.optimize_poses_device(rounds=rounds, **dev)
        device = lambda: eng.optimize_poses_device(rounds=rounds, out=first, workspace=first["workspace"], **dev)
    else:
        host = lambda: eng.optimize_sim3_flat(**flat)
        first = eng.optimize_sim3_device(**dev)
        device = lambda: eng.optimize_sim3_device(out=first, workspace=first["workspace"], **dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        device()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        device()
    # the three arms give the same bytes
    ref = host()
    for run in (device, graph.replay):
        run()
        torch.cuda.synchronize()
        for k in ("q", "t", "levels"):
            if not np.array_equal(first[k].cpu().numpy().view(np.uint8), np.ascontiguousarray(ref[k]).view(np.uint8)):
                raise RuntimeError("%s: the device path's %s differs from the host path's" % (kind, k))
    return host, device, graph.replay


def wall_ms(torch, fn, calls):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / calls


def kernel_ms(torch, fn, calls):
    """device ms per call of every kernel the call launches, by kernel name, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and ("k_" in ev.name):
            name = ev.name.split("(")[0].split("::")[-1].replace("void ", "")
            out[name] = out.get(name, 0.0) + (ev.device_time if hasattr(ev, "device_time") else ev.cuda_time) / 1e3 / calls
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    pkg = ge.load_package()
    fx = os.path.join(ROOT, "oracle", "_ref", "fixtures", "ba_kitti_00.cubagraph")
    if os.path.exists(fx):
        graph, g = "ba_kitti_00", pkg.graphio.read_graph(fx)
    else:
        graph, g = "kitti00_shaped", pkg.synth.make_config("kitti00_shaped")
    prob = pkg.graphio.flatten(g)
    frames = pkg.graphio.pose_frames(prob, range(prob.Pall))
    problems = sim3_batch_timing.workload(pkg, prob, 5)
    rounds = pkg.orbslam2_pose_schedule()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    eng = pkg.Engine(device=0)
    cases = {}
    for kind, items in (("pose", frames), ("sim3", problems)):
        for B in BATCHES:
            sel = items[:B]
            flat = pkg.graphio.pose_batch_arrays(sel) if kind == "pose" else pkg.graphio.sim3_batch_arrays(sel)
            cases["%s_%d" % (kind, len(sel))] = (len(sel), arms(torch, eng, kind, flat, rounds))
    rec = {"graph": graph, "frames": len(frames), "sim3_problems": len(problems), "card": card, "reps": []}
    for _ in range(args.reps):
        rep = {}
        for name, (n, (host, device, replay)) in cases.items():
            calls = max(3, min(200, 2000 // n))
            rep[name] = {arm: wall_ms(torch, fn, calls) for arm, fn in (("host", host), ("device", device), ("graph", replay))}
        rec["reps"].append(rep)
    rec["kernels"] = {name: kernel_ms(torch, device, max(3, min(50, 500 // n))) for name, (n, (host, device, replay)) in cases.items()}
    rec["summary_ms"] = {name: {arm: float(np.median([r[name][arm] for r in rec["reps"]])) for arm in ("host", "device", "graph")}
                         for name in cases}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
