"""PCG kernel comparison: iterations and device time of k_pcg5 (default and 74-aggregate bound) vs k_pcg3 on one linearised system."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

pkg = ge.load_package()
for workload in sys.argv[1:] or ["kitti07_shaped", "kitti00_shaped"]:
    path = os.path.join(ROOT, "oracle", "_ref", "fixtures", workload + ".cubagraph")
    g = pkg.graphio.read_graph(path) if workload.startswith("ba_") else pkg.synth.make_config(workload)
    prob = pkg.graphio.flatten(g)
    for variant, magg in ((5, 0), (5, 74), (4, 0)):
        eng = pkg.Engine(device=0, pcg_variant=variant, max_aggregates=magg)
        eng.initialize(prob)
        eng.linearize()
        md = eng.max_diagonal()
        for lam in (1e-5 * md, 1e-8 * md, 1e-10 * md):
            eng.linearize()
            it, ok = eng.solve(lam)
            ms = eng.bench_stage(4, reps=5, flush_l2=False, lam=lam)
            print("%s variant %d/%d lambda %.3g: iters %d ok %s  %.3f ms/solve  %.2f us/iter" % (workload, variant, magg, lam, it, ok, ms, 1e3 * ms / max(it, 1)), flush=True)
        eng.close()
