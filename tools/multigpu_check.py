"""Landmark-sharded run under torchrun: parity of the N-GPU trajectory with the CPU oracle (rank 0 prints).
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/multigpu_check.py [workload ...]
Environment: PCG_VARIANT (cuba_config.reserved[0]: 0 automatic, 7 replicated PCG, 8 rows always distributed over the ranks),
NO_ORACLE=1 (large graphs: print the trajectory instead of comparing it with the single-threaded CPU oracle), KERNEL=none|huber,
LINEAR_SOLVER=pcg|dense (Engine.set_linear_solver; with RESULT_JSON every rank also reports whether its poses equal rank 0's bit for bit)."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

pkg = ge.load_package()
rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
HUBER = ((1, 1), (5.991 ** 0.5, 7.815 ** 0.5))
NONE = ((0, 0), (0.0, 0.0))
RK = NONE if os.environ.get("KERNEL", "huber") == "none" else HUBER
variant = int(os.environ.get("PCG_VARIANT", "0"))
solver = os.environ.get("LINEAR_SOLVER", "pcg")
for workload in sys.argv[1:] or ["small", "kitti07_shaped"]:
    path = os.path.join(ROOT, "oracle", "_ref", "fixtures", workload + ".cubagraph")
    prob = pkg.graphio.flatten(pkg.graphio.read_graph(path) if workload.startswith("ba_") else pkg.synth.make_config(workload))
    eng = pkg.Engine(device=local, pcg_variant=variant)
    for et in (0, 1):
        eng.set_robust_kernels(RK[0][et], RK[1][et], et)
    if world > 1:
        eng.set_comm(rank, world, pkg.sharding.broadcast_unique_id(pkg.Engine, rank, world))
    eng.set_linear_solver(solver)
    eng.initialize(prob)
    stats = eng.optimize(10)          # warm-up (also the run that is checked)
    q, t, Xw = eng.state()
    eng.reset_state()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    t0 = time.perf_counter()
    stats2 = eng.optimize(10)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    prof = eng.time_profile()
    same_poses = True
    if world > 1:
        # the poses are replicated: every rank solved the same reduced system, so they agree bit for bit
        mine = np.concatenate([q.ravel(), t.ravel()])
        allp = [None] * world
        dist.all_gather_object(allp, mine.tobytes())
        same_poses = all(b == allp[0] for b in allp)
    if rank == 0:
        got = np.array([s["chi2"] for s in stats])
        rep = np.abs(got - np.array([s["chi2"] for s in stats2])).max() / got.max()
        head = "%s world %d variant %d solver %s: optimize(10) %.1f ms; repeat diff %.1e; trials %s; pcg iters %s" % (
            workload, world, variant, solver, 1e3 * dt, rep, [s["trials"] for s in stats], [s["pcg_iters"] for s in stats])
        if os.environ.get("NO_ORACLE"):
            print(head + "; chi2 " + " ".join("%.10e" % c for c in got), flush=True)
        else:
            oracle = ge.load_oracle()
            o = oracle.Oracle(prob, *RK)
            chi, lam, tr = o.optimize(10)
            oq, ot, oX = o.state()
            dq, dt_, dX = np.abs(q - oq).max(), np.abs(t - ot).max() / np.abs(ot).max(), np.abs(Xw - oX).max() / np.abs(oX).max()
            print(head + "; chi2 rel diff vs oracle %.2e; oracle trials %s; state diff q %.1e t %.1e Xw %.1e" % (
                np.abs(got - chi).max() / chi.max(), list(tr), dq, dt_, dX), flush=True)
            if os.environ.get("RESULT_JSON"):
                import json
                print("RESULT " + json.dumps({"workload": workload, "world": world, "chi2_rel_diff_vs_oracle": float(np.abs(got - chi).max() / chi.max()),
                                              "state_diff": float(max(dq, dt_, dX)), "repeat_diff": float(rep), "same_poses_on_every_rank": same_poses, "trials_equal": [int(s["trials"]) for s in stats] == [int(x) for x in tr]}), flush=True)
        print("   profile (s, both runs): " + ", ".join("%s %.4f" % (k[:2] + k[3:12], v) for k, v in prof.items()), flush=True)
    eng.close()
if world > 1:
    dist.destroy_process_group()
