#!/usr/bin/env python3
"""Structure-only refinement of every free landmark of ba_kitti_00 (kitti00_shaped when the fixture is absent) held by an engine, in
place: the poses at the fixture's estimates, every point perturbed by seeded noise (0.1 per coordinate), under test_point_batch's
huber_depth schedule (Huber 5 iterations with the depth test, then no robust kernel 10 iterations with the depth test, each from the
last round's result).  Before every timed call the engine gets the perturbed state back and every level at 0 (not timed).

  (a) inplace_host     Engine.optimize_landmarks (every landmark, no per-landmark output): host clock around the call
  (b) inplace_device   Engine.optimize_landmarks_device (every landmark, nstats on the device): host clock to a device synchronise
  (c) kernel           k_refine_landmarks alone: device time from torch.profiler, in a pass of its own
  (d) device_path      what a caller does without the call, on the device: state_device, the points cut from the state with torch
                       (the layout of graphio.point_batch, built once), optimize_points_device, the positions scattered back,
                       set_state_device, the levels scattered into edge-id order, set_edge_levels_device; host clock to a synchronise
  (e) engine_single    the engine's landmark-only problem of tools/point_batch_timing.py (every pose fixed, every point free):
                       set_problem, per round set_robust_kernel + optimize + classify_edges, get_state

The arms alternate within each of --reps repetitions, after a warm-up of each.  The in-place and point-batch results are compared as
in tests/test_landmark_refine.py: the landmarks whose edges are of one type, cut in the stream's order, bit for bit; every landmark
to within `max_rel_dx`.  Prints one JSON line with the card and its power limit.
Usage: python tools/landmark_refine_timing.py [--reps 5] [--out path.json]"""
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
import point_batch_timing as pbt  # noqa: E402


def kernel_ms(eng, rounds, reset, calls):
    """mean device ms of k_refine_landmarks over `calls` device-entry calls, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            reset()
            eng.optimize_landmarks_device(rounds, with_stats=False)
        torch.cuda.synchronize()
    tot, n = 0.0, 0
    for ev in prof.events():
        if "k_refine_landmarks" in ev.name and ev.device_type.name == "CUDA":
            tot += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
            n += 1
    if n != calls:
        raise RuntimeError("torch.profiler saw %d k_refine_landmarks launches, expected %d" % (n, calls))
    return tot / n / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
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
    single.numP, single.numL = 0, single.Lall
    rounds = pbt.schedule(pkg)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    L = np.arange(prob.numL)

    eng = pkg.Engine(device=0)
    eng.initialize(prob)
    q0, t0, X0 = eng.state()
    dq, dt_, dX = (torch.from_numpy(a).to(dev) for a in (q0, t0, X0))

    def reset():
        eng.set_state_device(dq, dt_, dX)
        eng.set_edge_levels_device(None)

    # (d)'s layout, built once: the points of every free landmark and where their edges sit in edge-id order
    batch = pkg.graphio.point_batch(prob, L)
    lay = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in batch.arrays().items()}
    edge_ids = torch.from_numpy(np.concatenate([batch.mono_ids, prob.E2 + batch.stereo_ids]).astype(np.int64)).to(dev)
    Ld = torch.from_numpy(L.astype(np.int64)).to(dev)
    peng = pkg.Engine(device=0)
    lev_full = torch.zeros(prob.nedges, dtype=torch.uint8, device=dev)

    def device_path(out=None):
        q, t, X = eng.state_device()
        lay["q"], lay["t"], lay["Xw"] = q, t, X.index_select(0, Ld)
        out = peng.optimize_points_device(rounds=rounds, with_stats=False, out=out, workspace=None if out is None else out["workspace"], **lay)
        X.index_copy_(0, Ld, out["Xw"])
        eng.set_state_device(q, t, X)
        lev_full.zero_()
        lev_full.index_copy_(0, edge_ids, out["levels"])
        eng.set_edge_levels_device(lev_full)
        return out

    seng = pkg.Engine(device=0)
    # warm-up: every arm once
    reset(); eng.optimize_landmarks(rounds)
    reset(); eng.optimize_landmarks_device(rounds, with_stats=False)
    reset(); pout = device_path()
    seng.initialize(single); pbt.engine_rounds(seng, single, rounds)
    torch.cuda.synchronize()

    # agreement with k_point_batch (test 2 of tests/test_landmark_refine.py)
    reset()
    eng.optimize_landmarks(rounds)
    Xin = eng.state()[2][:prob.numL]
    lev_in = eng.edge_levels()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_landmark_refine as tlr   # noqa: E402
    pure = np.nonzero((np.diff(batch.ptr2) == 0) | (np.diff(batch.ptr3) == 0))[0]
    sel = pure[:: max(1, len(pure) // 20000)]
    sb = tlr.stream_order(pkg, pkg.graphio.point_batch(prob, sel))
    ref = pkg.Engine(device=0).optimize_points_flat(rounds=rounds, **sb.arrays())
    E2s = len(sb.omega2)
    lev_ok = all(np.array_equal(tlr.levels_of(sb, b, lev_in, prob.E2),
                                np.concatenate([ref["levels"][sb.ptr2[b]:sb.ptr2[b + 1]], ref["levels"][E2s + sb.ptr3[b]:E2s + sb.ptr3[b + 1]]]))
                 for b in range(sb.B))
    allb = peng.optimize_points_flat(rounds=rounds, **batch.arrays())
    agree = dict(single_type_checked=int(sb.B), single_type_bitwise=bool(np.array_equal(Xin[sel], ref["Xw"]) and lev_ok),
                 max_rel_dx=float(np.abs(Xin - allb["Xw"]).max() / max(1.0, np.abs(allb["Xw"]).max())),
                 levels_differ=int((np.concatenate([lev_in[batch.mono_ids], lev_in[prob.E2 + batch.stereo_ids]]) != allb["levels"]).sum()))

    rec = {"graph": graph, "landmarks": int(prob.numL), "poses": int(prob.Pall), "edges": int(prob.nedges), "card": card,
           "agreement": agree, "reps": []}
    for _ in range(args.reps):
        rep = {}
        reset(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = eng.optimize_landmarks(rounds)
        rep["inplace_host_ms"] = 1e3 * (time.perf_counter() - t0)
        rep["counts"] = r["counts"].tolist()
        reset(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.optimize_landmarks_device(rounds, with_stats=False)
        torch.cuda.synchronize()
        rep["inplace_device_ms"] = 1e3 * (time.perf_counter() - t0)
        reset(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        pout = device_path(pout)
        torch.cuda.synchronize()
        rep["device_path_ms"] = 1e3 * (time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seng.initialize(single)
        pbt.engine_rounds(seng, single, rounds)
        rep["engine_single_ms"] = 1e3 * (time.perf_counter() - t0)
        rec["reps"].append(rep)
    rec["kernel_ms"] = kernel_ms(eng, rounds, reset, 5)
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
