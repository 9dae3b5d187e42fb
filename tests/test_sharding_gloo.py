"""world_size-2 gloo test of the landmark-sharded data path (SURVEY.md 8e), on CPU:
each rank linearises only its landmark shard with the oracle, the per-pose quantities are summed with
torch.distributed all_reduce exactly where libcuba_b200.so calls ncclAllReduce, and the result must equal
the unsharded system."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT, HUBER


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    pkg = ge.load_package(); oracle = ge.load_oracle()
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    prob = pkg.graphio.flatten(pkg.synth.make_config("tiny"))
    iL = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    b = pkg.sharding.shard_bounds(iL, prob.Lall, world)
    s = pkg.build_structure_host(prob, rank, world)
    assert (s["shard"][0], s["shard"][1]) == (b[rank], b[rank + 1])
    o = oracle.Oracle(pkg.sharding.sub_problem(prob, b[rank], b[rank + 1]), *HUBER)
    chi = o.compute_errors(); o.build_system()
    Hpp, bp, Hll, bl, Hpl = o.system()
    t = torch.from_numpy(np.concatenate([Hpp.ravel(), bp.ravel(), [chi]]))
    dist.all_reduce(t)                      # <- Hpp/bp/chi2 all-reduce of cuba_stage_linearize
    # Schur contributions of the local landmarks: Hsc_local = -sum products (diagonal Hpp+lambda added once)
    lam = 3.0
    o.solve(lam)
    Hsc, bsc, inv = o.schur()
    rp, ci = o.hsc_structure()
    full = oracle.Oracle(prob, *HUBER); full.compute_errors(); full.build_system(); full.solve(lam)
    frp, fci = full.hsc_structure()
    # scatter the shard's upper blocks into the global pattern, remove the local Hpp+lambda on the diagonal
    glob = np.zeros((len(fci), 36))
    pos = {(r, int(fci[k])): k for r in range(prob.numP) for k in range(frp[r], frp[r + 1])}
    for r in range(prob.numP):
        for k in range(rp[r], rp[r + 1]):
            blk = Hsc[k].copy()
            if ci[k] == r:
                blk -= Hpp[r] + lam * np.eye(6).ravel()
            glob[pos[(r, int(ci[k]))]] = blk
    bloc = bsc - bp
    t2 = torch.from_numpy(np.concatenate([glob.ravel(), bloc.ravel()]))
    dist.all_reduce(t2)                     # <- Hsc/bsc all-reduce of cuba_stage_solve
    if rank == 0:
        fHpp, fbp, _, _, _ = full.system()
        fchi = full.compute_errors()
        fHsc, fbsc, _ = full.schur()
        n1 = fHpp.size; n2 = fbp.size
        got_Hpp = t[:n1].numpy().reshape(fHpp.shape); got_bp = t[n1:n1 + n2].numpy().reshape(fbp.shape)
        gsc = t2[:glob.size].numpy().reshape(glob.shape).copy(); gb = t2[glob.size:].numpy().reshape(fbp.shape) + got_bp
        for r in range(prob.numP):
            gsc[frp[r]] += got_Hpp[r] + lam * np.eye(6).ravel()
        q.put(dict(hpp=float(np.abs(got_Hpp - fHpp).max() / np.abs(fHpp).max()), bp=float(np.abs(got_bp - fbp).max() / np.abs(fbp).max()),
                   chi=float(abs(t[-1].item() - fchi) / fchi), hsc=float(np.abs(gsc - fHsc).max() / np.abs(fHsc).max()),
                   bsc=float(np.abs(gb - fbsc).max() / np.abs(fbsc).max())))
    dist.barrier()
    dist.destroy_process_group()


def test_landmark_sharded_reduction_equals_unsharded(pkg, oracle):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = q.get(timeout=240)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for k, v in res.items():
        assert v < 1e-12, (k, v)
