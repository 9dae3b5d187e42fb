#!/usr/bin/env python3
"""What every reduced-system solver path computes after optimize(10), so that two builds of the library can be compared exactly
(swap the in-tree library between two `dump` runs, as tools/ab_libs.sh does):

  dump OUT.npz        optimize(10) on kitti00_shaped, kitti07_shaped and orbit_600 under every pcg_variant (0, 2..6), the fp32 and
                      mixed-precision engines, CUBA_PCG5_LEGACY=1, the dense solver, every J+H kernel (jh_variant 1..4, 7..9; mixed with
                      8, fp32 with 1 and 7) and the tensor-pipe Schur (schur_variant 5), and on rows_11k (whose automatic block-Jacobi
                      solve is k_pcg2) in fp32 and fp64; then classify_edges and optimize(5) (the level mask rewrites the edge streams),
                      and initialize() of the same problem and optimize(5) (structure reuse refreshes them): the launch count,
                      cuba_debug_get_pcg_info, cuba_debug_get_coarse (when a k_pcg5 coarse level exists), the state, chi2 and the
                      per-iteration statistics after each phase; a path that refuses the problem records its error message
  compare A.npz B.npz the bytes, dtype and shape of every array; prints the arrays that differ and exits 1 if any does

Usage: python tools/pcg_paths_ab.py dump out.npz;  python tools/pcg_paths_ab.py compare a.npz b.npz"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

GRAPHS = ("kitti00_shaped", "kitti07_shaped", "orbit_600")
# (name, Engine keyword arguments, CUBA_PCG5_LEGACY, linear solver)
SETTINGS = [("v%d" % v, dict(pcg_variant=v), False, "pcg") for v in (0, 2, 3, 4, 5, 6)] + [
    ("fp32", dict(use_fp32=True), False, "pcg"),
    ("fp32_v3", dict(use_fp32=True, pcg_variant=3), False, "pcg"),
    ("mixed", dict(use_fp32="mixed"), False, "pcg"),
    ("legacy", dict(), True, "pcg"),
    ("dense", dict(), False, "dense"),
] + [("jh%d" % v, dict(jh_variant=v), False, "pcg") for v in (1, 2, 3, 4, 7, 8, 9)] + [
    ("schur5", dict(schur_variant=5), False, "pcg"),
    ("mixed_jh8", dict(use_fp32="mixed", jh_variant=8), False, "pcg"),
    ("fp32_jh1", dict(use_fp32=True, jh_variant=1), False, "pcg"),
    ("fp32_jh7", dict(use_fp32=True, jh_variant=7), False, "pcg"),
]
RUNS = [(g, s) for g in GRAPHS for s in SETTINGS] + [("rows_11k", s) for s in SETTINGS if s[0] in ("fp32", "fp32_v3", "v0")]


def run(pkg, prob, kw, legacy, solver):
    eng = pkg.Engine(device=0, **kw)
    try:
        if legacy:
            os.environ["CUBA_PCG5_LEGACY"] = "1"      # read by set_problem
        eng.set_linear_solver(solver)
        eng.initialize(prob)
        out = phase(pkg, eng, eng.optimize(10), "")
        out["levels_counts"] = np.array(list(eng.classify_edges(5.991, 7.815).values()), np.int64)
        out.update(phase(pkg, eng, eng.optimize(5), "levels_"))
        eng.initialize(prob)
        out["reuse_structure_reuses"] = np.array([eng.structure_reuses()], np.int64)
        out.update(phase(pkg, eng, eng.optimize(5), "reuse_"))
        return out
    except pkg.CubaError as ex:
        return {"error": np.array([str(ex)])}
    finally:
        eng.close()
        os.environ.pop("CUBA_PCG5_LEGACY", None)


def phase(pkg, eng, stats, pre):
    out = {pre + "launches": np.array([eng.launch_count()], np.int64)}
    info = eng.pcg_info()
    out[pre + "pcg_info"] = np.array([str(info[k]) for k in sorted(info)])
    out[pre + "kernel"] = np.array([info["kernel"]])
    try:
        agg, AcP, AcInv = eng.coarse()
        out.update({pre + "coarse_agg": agg, pre + "coarse_AcP": AcP, pre + "coarse_AcInv": AcInv})
    except pkg.CubaError as ex:
        out[pre + "coarse_error"] = np.array([str(ex)])
    q, t, Xw = eng.state()
    out.update({pre + "q": q, pre + "t": t, pre + "Xw": Xw, pre + "chi2": np.array([eng.chi2()])})
    for f in ("iteration", "trials", "chi2", "lambda_", "pcg_iters", "pcg_failed"):
        out[pre + "stats_" + f] = np.array([s[f] for s in stats])
    return out


def dump(path):
    pkg = ge.load_package()
    arrays, probs = {}, {}
    for graph, (name, kw, legacy, solver) in RUNS:
        if graph not in probs:
            probs[graph] = pkg.graphio.flatten(pkg.synth.make_config(graph))
        res = run(pkg, probs[graph], kw, legacy, solver)
        print("%s %s: %s" % (graph, name, res["error"][0] if "error" in res else "%s, %d launches, chi2 %.10g" % (
            res["kernel"][0], res["launches"][0], res["chi2"][0])), flush=True)
        arrays.update({"%s/%s/%s" % (graph, name, k): v for k, v in res.items()})
    np.savez(path, **arrays)
    print("%s: %d runs, %d arrays" % (path, len(RUNS), len(arrays)))


def compare(a, b):
    A, B = np.load(a), np.load(b)
    same = lambda x, y: x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
    bad = sorted(k for k in set(A.files) | set(B.files) if k not in A.files or k not in B.files or not same(A[k], B[k]))
    for k in bad:
        print("DIFFERENT:", k)
    print("%d arrays, %d different" % (len(set(A.files) | set(B.files)), len(bad)))
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "dump":
        dump(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
