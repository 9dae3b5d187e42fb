#!/usr/bin/env python3
"""The engine's own problem from host arrays against the same problem on device-resident arrays (Engine.initialize_device and
the other *_device methods), on ba_kitti_00 and ba_kitti_07 (kitti00_shaped / kitti07_shaped when the fixtures are absent):

  fresh       set_problem that builds every structure (structure reuse off)
  changed     set_problem with structure reuse on, the sizes held but one (iP, iL) list changed on every call (two edges swap their
              landmarks): a full build after the comparison; on device arrays, after the refresh queued behind it too
  reuse       set_problem on the held topology (structure reuse: only the values)
  set_state   set_state
  get_state   get_state
  get_chi2    get_chi2
  cycle       a local-BA cycle: initialize + optimize(10) + state, structure reuse on

  host        the host entry point from numpy arrays (results into numpy arrays)
  device      the *_device entry point on torch tensors already in device memory (results into reused tensors)
  torch       a torch caller today: the tensors .cpu()'d, the host entry point, the results copied up with .cuda()

Wall time: a host clock around `calls` calls, ending in a device synchronise, the arms alternating within each of --reps
repetitions; the medians are in "summary_ms".  Before timing, the three arms of get_chi2, of a cycle and of get_state are checked to
give the same bytes.  Prints one JSON line with the card's name and power limit.
Usage: python tools/device_problem_timing.py [--reps 5] [--out path.json]"""
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

FIELDS = ("q", "t", "cam", "Xw", "idx2", "meas2", "omega2", "idx3", "meas3", "omega3")
HUBER = (5.991 ** 0.5, 7.815 ** 0.5)


def workload(pkg, fixture, synthetic):
    fx = os.path.join(ROOT, "oracle", "_ref", "fixtures", fixture + ".cubagraph")
    if os.path.exists(fx):
        return fixture, pkg.graphio.flatten(pkg.graphio.read_graph(fx))
    return synthetic, pkg.graphio.flatten(pkg.synth.make_config(synthetic))


def engine(pkg, reuse):
    eng = pkg.Engine(device=0)
    for et in (0, 1):
        eng.set_robust_kernels(pkg.ROBUST_HUBER, HUBER[et], et)
    eng.set_structure_reuse(reuse)
    return eng


def swapped(prob):
    """the same sizes, idx2 changed: two monocular edges of different poses and landmarks swap their landmarks"""
    p = prob.copy()
    i2 = p.idx2.copy()
    k = next(k for k in range(1, len(i2)) if i2[k, 0] != i2[0, 0] and i2[k, 1] != i2[0, 1])
    i2[[0, k], 1] = i2[[k, 0], 1]
    p.idx2 = i2
    return p


def arms(torch, pkg, prob):
    """{operation: {arm: callable}}; every callable leaves its results where the caller can read them"""
    to_dev = lambda p: dict({k: torch.from_numpy(np.ascontiguousarray(getattr(p, k))).cuda() for k in FIELDS},
                            Pall=p.Pall, numP=p.numP, Lall=p.Lall, numL=p.numL)
    dev = to_dev(prob)
    alt = swapped(prob)
    alt_dev = to_dev(alt)
    host_state = (prob.q, prob.t, prob.Xw)
    dev_state = (dev["q"], dev["t"], dev["Xw"])

    def cpu_problem():
        p = prob.copy()
        for k in FIELDS:
            setattr(p, k, dev[k].cpu().numpy())
        return p

    up = lambda arrays: tuple(torch.from_numpy(a).cuda() for a in arrays)
    fresh = {a: engine(pkg, False) for a in ("host", "device", "torch")}
    flip = {a: engine(pkg, True) for a in ("host", "device", "torch")}
    turn = {a: [0] for a in flip}

    def changed(arm):
        turn[arm][0] ^= 1
        p, d = (alt, alt_dev) if turn[arm][0] else (prob, dev)
        if arm == "device":
            return flip[arm].initialize_device(d)
        if arm == "torch":
            q = p.copy()
            for k in FIELDS:
                setattr(q, k, d[k].cpu().numpy())
            p = q
        return flip[arm].initialize(p)
    held = {a: engine(pkg, True) for a in ("host", "device", "torch")}
    for a, e in held.items():
        e.initialize(prob)
    outs = held["device"].state_device(), held["device"].chi_squared_device()
    ops = {
        "fresh": {"host": lambda: fresh["host"].initialize(prob), "device": lambda: fresh["device"].initialize_device(dev),
                  "torch": lambda: fresh["torch"].initialize(cpu_problem())},
        "changed": {a: (lambda a=a: changed(a)) for a in ("host", "device", "torch")},
        "reuse": {"host": lambda: held["host"].initialize(prob), "device": lambda: held["device"].initialize_device(dev),
                  "torch": lambda: held["torch"].initialize(cpu_problem())},
        "set_state": {"host": lambda: held["host"].set_state(*host_state), "device": lambda: held["device"].set_state_device(*dev_state),
                      "torch": lambda: held["torch"].set_state(*(a.cpu().numpy() for a in dev_state))},
        "get_state": {"host": lambda: held["host"].state(), "device": lambda: held["device"].state_device(out=outs[0]),
                      "torch": lambda: up(held["torch"].state())},
        "get_chi2": {"host": lambda: held["host"].chi_squared(), "device": lambda: held["device"].chi_squared_device(out=outs[1]),
                     "torch": lambda: up((held["torch"].chi_squared(),))},
    }

    def cycle(arm):
        e = held[arm]
        if arm == "host":
            e.initialize(prob); e.optimize(10); return e.state()
        if arm == "device":
            e.initialize_device(dev); e.optimize(10); return e.state_device(out=outs[0])
        e.initialize(cpu_problem()); e.optimize(10); return up(e.state())
    ops["cycle"] = {a: (lambda a=a: cycle(a)) for a in ("host", "device", "torch")}
    # the three arms of the getters and of a cycle give the same bytes
    as_np = lambda r: [np.ascontiguousarray(x.cpu().numpy() if hasattr(x, "cpu") else x) for x in (r if isinstance(r, tuple) else (r,))]
    for op in ("get_chi2", "cycle", "get_state"):
        res = {a: as_np(f()) for a, f in ops[op].items()}
        torch.cuda.synchronize()
        for a in ("device", "torch"):
            if [x.tobytes() for x in res[a]] != [x.tobytes() for x in res["host"]]:
                raise RuntimeError("%s: the %s arm differs from the host arm" % (op, a))
    for a, f in ops["changed"].items():
        f(); f()
        if flip[a].structure_reuses() != 0:
            raise RuntimeError("changed: the %s arm reused the structure" % a)
    return ops


def wall_ms(torch, fn, calls):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / calls


CALLS = {"fresh": 5, "changed": 6, "reuse": 10, "set_state": 20, "get_state": 20, "get_chi2": 20, "cycle": 3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    pkg = ge.load_package()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rec = {"card": card, "workloads": {}}
    for fixture, synthetic in (("ba_kitti_00", "kitti00_shaped"), ("ba_kitti_07", "kitti07_shaped")):
        name, prob = workload(pkg, fixture, synthetic)
        ops = arms(torch, pkg, prob)
        for op in ops.values():          # warm-up: every shape of the timed window
            for f in op.values():
                f()
        reps = []
        for _ in range(args.reps):
            reps.append({op: {a: wall_ms(torch, f, CALLS[op]) for a, f in fns.items()} for op, fns in ops.items()})
        rec["workloads"][name] = {"Pall": prob.Pall, "Lall": prob.Lall, "edges": prob.nedges, "reps": reps,
                                  "summary_ms": {op: {a: float(np.median([r[op][a] for r in reps])) for a in fns} for op, fns in ops.items()}}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
