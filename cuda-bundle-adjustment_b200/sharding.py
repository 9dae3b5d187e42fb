"""Host-side logic of the landmark-sharded multi-GPU run (SURVEY.md 8e).

One process per GPU.  Every rank flattens the same graph (the generator is seeded / the file is shared),
the engine keeps only the landmarks [lmBeg, lmEnd) of its rank for the numeric work, and the per-pose
quantities are summed with NCCL all-reduces inside libcuba_b200.so:
    per linearisation : Hpp (36*numP) and bp (6*numP), chi2 (1 scalar)
    per LM trial      : Hsc values (36*nblk_full) and bsc (6*numP), trial chi2 and landmark scale (2 scalars)
The PCG then runs replicated (bitwise identical inputs on every rank => identical iterates, no further
communication).  No landmark or Hpl data ever crosses GPUs.

`shard_bounds` restates the partition rule of csrc/cuba_structure.cpp so that host code (and the gloo
CPU tests) can reason about it without a GPU.
"""
import numpy as np


def shard_bounds(iL_of_edges, Lall, world):
    """Landmark ranges per rank: balanced by edge count, snapped to landmark boundaries.
    Returns int array [world+1] with bounds[r] = first landmark of rank r."""
    E = int(len(iL_of_edges))
    cnt = np.bincount(np.asarray(iL_of_edges, dtype=np.int64), minlength=Lall)
    ptr = np.concatenate([[0], np.cumsum(cnt)])
    b = np.zeros(world + 1, dtype=np.int64)
    for r in range(1, world):
        target = (E * r) // world
        b[r] = np.searchsorted(ptr, target, side="left")
    b[world] = Lall
    b = np.minimum(b, Lall)
    for r in range(1, world + 1):
        b[r] = max(b[r], b[r - 1])
    return b


def sub_problem(prob, lo, hi):
    """The problem made of the edges of the landmarks [lo, hi) only; every vertex is kept (the engine replicates the poses and
    keeps the foreign landmarks as uploaded).  Rank 0's share of a sharded run is exactly the LM run of this problem."""
    p = prob.copy()
    m2 = (prob.idx2[:, 1] >= lo) & (prob.idx2[:, 1] < hi); m3 = (prob.idx3[:, 1] >= lo) & (prob.idx3[:, 1] < hi)
    p.idx2, p.meas2, p.omega2 = prob.idx2[m2].copy(), prob.meas2[m2].copy(), prob.omega2[m2].copy()
    p.idx3, p.meas3, p.omega3 = prob.idx3[m3].copy(), prob.meas3[m3].copy(), prob.omega3[m3].copy()
    return p


def allreduce_bytes_per_trial(numP, nblk_full, scalar_bytes=8):
    """bytes each rank contributes per LM trial / per linearisation (for DESIGN.md and the bench report)."""
    return {"per_linearize": (42 * numP + 1) * scalar_bytes, "per_trial": (36 * nblk_full + 6 * numP) * scalar_bytes + 16}


def broadcast_unique_id(engine_cls, rank, world):
    """Rank 0 creates the NCCL unique id, torch.distributed (any backend) broadcasts the 128 bytes."""
    import torch
    import torch.distributed as dist
    if rank == 0:
        uid = engine_cls.comm_unique_id()
        t = torch.tensor(list(uid), dtype=torch.uint8)
    else:
        t = torch.zeros(128, dtype=torch.uint8)
    if dist.get_backend() == "nccl":
        t = t.cuda()
    dist.broadcast(t, src=0)
    return bytes(t.cpu().tolist())
