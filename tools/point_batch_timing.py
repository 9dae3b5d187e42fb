#!/usr/bin/env python3
"""Structure-only refinement of every landmark of ba_kitti_00 (kitti00_shaped when the fixture is absent): the poses held fixed at the
fixture's estimates, every point perturbed by seeded noise (0.1 per coordinate), under two rounds -- Huber 5 iterations with the
depth test, then no robust kernel 10 iterations with the depth test -- each from the last round's result:

  (a) engine_single  the engine's one landmark-only problem (every pose fixed, every point free): set_problem, per round
                     set_robust_kernel + optimize + classify_edges, then get_state; host clock around the whole (and without set_problem)
  (b) engine_point   the engine per point (set_problem of the point's sub-problem, the rounds, get_state) over --engine-points points
  (c) batch_B        the host entry (Engine.optimize_points_flat on numpy arrays) on the first B points, B = 1, 64, 4096 and all:
                     host clock around the whole call (packing, the copies, the launch and the unpacking)
  (d) device_all     Engine.optimize_points_device on all points, inputs and outputs in GPU memory: host clock to a device synchronise
  (e) kernel         k_point_batch alone on all points: device time from torch.profiler, in a pass of its own

The arms alternate within each of --reps repetitions.  Prints one JSON line: microseconds per point, edge-iterations per second
(edges at level 0 times LM iterations, summed over the points and rounds), each arm's final total chi2 (the robust chi2 after the
last round, summed over the points), the card and its power limit.
Usage: python tools/point_batch_timing.py [--reps 3] [--engine-points 200] [--out path.json]"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

BATCHES = (1, 64, 4096, None)       # None: every point


def schedule(pkg):
    R = pkg.PoseRound
    huber = dict(kernel=(pkg.ROBUST_HUBER, pkg.ROBUST_HUBER), delta=(5.991 ** 0.5, 7.815 ** 0.5))
    return [R(5, restart=False, depth=True, reinclude=False, **huber), R(10, restart=False, depth=True, reinclude=False)]


def engine_rounds(eng, prob, rounds):
    """the rounds on the engine's problem; returns (edge-iterations, robust chi2 after the last round)"""
    work, chi, included = 0, 0.0, prob.nedges
    for r in rounds:
        for et in (0, 1):
            eng.set_robust_kernels(r.kernel[et], r.delta[et], et)
        st = eng.optimize(r.iterations)
        work += included * len(st)
        chi = st[-1]["chi2"] if st else 0.0
        c = eng.classify_edges(r.chi2_mono, r.chi2_stereo, depth=r.depth, reinclude=r.reinclude)
        included = c["included_mono"] + c["included_stereo"]
    eng.state()
    return work, chi


def batch_work(batch, res, rounds):
    """edge-iterations and final robust chi2 of a result of optimize_points_flat (stats and nstats as numpy arrays)"""
    inc = (np.diff(batch.ptr2) + np.diff(batch.ptr3)).astype(np.int64)
    counts, nstats = np.asarray(res["counts"]), np.asarray(res["nstats"])
    work = 0
    for k in range(len(rounds)):
        work += int((inc * nstats[:, k]).sum())
        inc = counts[:, k, 0].astype(np.int64) + counts[:, k, 1]
    last = sum(int(r.iterations) for r in rounds[:-1]) + nstats[:, -1] - 1
    ran = nstats[:, -1] > 0
    chi = np.asarray(res["stats"])["chi2"][np.nonzero(ran)[0], last[ran]].sum() if ran.any() else 0.0
    return work, float(chi)


def first(pkg, batch, B):
    """the first B points of a batch (the whole pose table)"""
    if B is None or B >= batch.B:
        return batch
    m, s = int(batch.ptr2[B]), int(batch.ptr3[B])
    return pkg.graphio.PointBatch(q=batch.q, t=batch.t, cam=batch.cam, Xw=batch.Xw[:B], ptr2=batch.ptr2[:B + 1], iP2=batch.iP2[:m],
                                  meas2=batch.meas2[:m], omega2=batch.omega2[:m], ptr3=batch.ptr3[:B + 1], iP3=batch.iP3[:s],
                                  meas3=batch.meas3[:s], omega3=batch.omega3[:s])


def kernel_ms(eng, d_in, rounds, calls):
    """mean device ms of k_point_batch over `calls` device-entry calls, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            eng.optimize_points_device(rounds=rounds, **d_in)
        torch.cuda.synchronize()
    tot, n = 0.0, 0
    for ev in prof.events():
        if "k_point_batch" in ev.name and ev.device_type.name == "CUDA":
            tot += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            n += 1
    if n != calls:
        raise RuntimeError("torch.profiler saw %d k_point_batch launches, expected %d" % (n, calls))
    return tot / n / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--engine-points", type=int, default=200)
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
    prob.Xw = prob.Xw + np.random.default_rng(7).normal(0, 0.1, prob.Xw.shape)
    single = prob.copy()
    single.numP, single.numL = 0, single.Lall              # every pose fixed, every point free
    batch = pkg.graphio.point_batch(prob, range(prob.Lall))
    rounds = schedule(pkg)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    sel = np.linspace(0, batch.B - 1, args.engine_points).astype(int)

    seng = pkg.Engine(device=0)      # the single problem's engine
    peng = pkg.Engine(device=0)      # the per-point engine
    beng = pkg.Engine(device=0)      # the batches' engine
    d_in = {k: torch.from_numpy(np.ascontiguousarray(v)).to("cuda:0") for k, v in batch.arrays().items()}
    # warm-up: every shape the timed window uses
    seng.initialize(single)
    engine_rounds(seng, single, rounds)
    for b in sel[:5]:
        sub = batch.sub_problem(int(b))
        peng.initialize(sub)
        engine_rounds(peng, sub, rounds)
    for B in BATCHES:
        beng.optimize_points_flat(rounds=rounds, **first(pkg, batch, B).arrays())
    out = beng.optimize_points_device(rounds=rounds, **d_in)
    torch.cuda.synchronize()

    rec = {"graph": graph, "points": batch.B, "poses": len(batch.q), "edges": int(len(batch.omega2) + len(batch.omega3)),
           "edges_per_point": float((len(batch.omega2) + len(batch.omega3)) / batch.B), "card": card, "reps": []}
    for _ in range(args.reps):
        rep = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seng.initialize(single)
        t1 = time.perf_counter()
        work, chi = engine_rounds(seng, single, rounds)
        t2 = time.perf_counter()
        rep["engine_single"] = dict(us_per_point=1e6 * (t2 - t0) / batch.B, us_per_point_without_set_problem=1e6 * (t2 - t1) / batch.B,
                                    edge_iters_per_s=work / (t2 - t0), chi2=chi)
        t0 = time.perf_counter()
        work = 0
        for b in sel:
            sub = batch.sub_problem(int(b))
            peng.initialize(sub)
            work += engine_rounds(peng, sub, rounds)[0]
        dt = time.perf_counter() - t0
        rep["engine_point"] = dict(points=len(sel), us_per_point=1e6 * dt / len(sel), edge_iters_per_s=work / dt)
        for B in BATCHES:
            pb = first(pkg, batch, B)
            arrays = pb.arrays()
            calls = max(3, min(50, 4096 // pb.B))
            res = None
            gc.collect()
            t0 = time.perf_counter()
            for _ in range(calls):
                res = beng.optimize_points_flat(rounds=rounds, **arrays)
            dt = (time.perf_counter() - t0) / calls
            work, chi = batch_work(pb, res, rounds)
            rep["batch_%d" % pb.B] = dict(calls=calls, us_per_point=1e6 * dt / pb.B, edge_iters_per_s=work / dt, chi2=chi)
        calls = 5
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(calls):
            out = beng.optimize_points_device(rounds=rounds, out=out, workspace=out["workspace"], **d_in)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / calls
        rep["device_all"] = dict(calls=calls, us_per_point=1e6 * dt / batch.B, edge_iters_per_s=work / dt, status=int(out["status"].item()))
        rec["reps"].append(rep)
    # the kernel alone, in a pass of its own (tracing slows the host)
    ms = kernel_ms(beng, d_in, rounds, 5)
    rec["kernel"] = dict(ms=ms, us_per_point=1e3 * ms / batch.B, edge_iters_per_s=work / (ms * 1e-3))
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
