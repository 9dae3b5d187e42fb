"""Time of one rebuild of k_pcg5's coarse inverse (projection Z^T S Z, assembly, inverse) and of one two-level solve, with CUDA
events, for the aggregates per CTA CUBA_PCG5_AGGS_PER_CTA allows (run once per setting; CUBA_PCG_VERBOSE=1 prints the plan):
  CUBA_PCG5_AGGS_PER_CTA=1 python tools/coarse_rebuild_timing.py [ba_kitti_00 ...]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

pkg = ge.load_package()
apc = os.environ.get("CUBA_PCG5_AGGS_PER_CTA", "default")
for workload in sys.argv[1:] or ["ba_kitti_00"]:
    path = os.path.join(ROOT, "oracle", "_ref", "fixtures", workload + ".cubagraph")
    g = pkg.graphio.read_graph(path) if workload.startswith("ba_") else pkg.synth.make_config(workload)
    prob = pkg.graphio.flatten(g)
    eng = pkg.Engine(device=0, pcg_variant=5)          # every solve two-level k_pcg5
    eng.initialize(prob)
    eng.linearize()
    md = eng.max_diagonal()
    out = ["%s aggs/CTA %s" % (workload, apc)]
    for scale in (1e-5, 1e-8):
        lam = scale * md
        it, ok = eng.solve(lam)                          # (also forms the reduced system the rebuild reads)
        rebuild = eng.bench_stage(7, reps=20, flush_l2=False)
        ms = eng.bench_stage(4, reps=5, flush_l2=False, lam=lam)
        out.append("lambda %.0e max_diag: coarse rebuild %.1f us, %d iters, %.1f us/solve, %.2f us/iter" % (scale, 1e3 * rebuild, it, 1e3 * ms, 1e3 * ms / max(it, 1)))
    print("; ".join(out), flush=True)
    eng.close()
