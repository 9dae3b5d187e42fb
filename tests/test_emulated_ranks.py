"""The multi-GPU exchange of a landmark-sharded run, with W ranks emulated on one GPU.

The peer all-reduce (csrc/cuba_peer_reduce.cuh) and the row-distributed k_pcg5 (csrc/cuba_pcg5.cuh) talk to their peers only
through device memory: signal words, and LL words with tags.  cuba_debug_peer_allreduce and cuba_debug_pcg5_ranks keep the boards
of all W ranks in one GPU's memory and run every rank in ONE cooperative launch of W x G CTAs (k_peer_allreduce_ranks,
k_pcg5_ranks: CTA b is CTA b % G of rank b / G), so all ranks are resident at once.  Should the exchange be wrong, the kernels'
spin limit ends the solve with status 3 instead of hanging.

The emulation runs a W-rank plan on 132 / W SMs per rank, where a W-GPU run gives each rank 132: the code paths are the same, the
partition is smaller.  test_gpu_parity.test_two_gpu_trajectory_matches_oracle still covers the real layout and the NVLink fences
where two GPUs exist.

  * the plan each emulated run uses, on the CPU: it exists, passes cuba_debug_pcg5_plan's invariants and fits 132 SMs;
  * the all-reduce: every rank's result bit-equal to the rank-order sum ((0 + p0) + p1) + ... in numpy, at the slice lengths
    where the kernel's indexing changes, in fp64 and fp32, three calls in a row; and on the dry-shard partial Schur complements;
  * the row-distributed k_pcg5 on the lambda ladder of test_pcg_coarse, two-level and block-Jacobi: every rank reports the same
    status and iteration count, no row of x is left unwritten, x matches the oracle's direct solve, the count matches
    restated_pcg5 fed the emulation's own coarse level, and repeated solves are bitwise identical."""
import time

import numpy as np
import pytest

from conftest import KERNELS, make_engine, relerr

SMS = 132                                    # H100 SXM
WORLDS = (2, 3, 4, 8)
RK = KERNELS["huber"]

# (graph, W) -> rows some other rank needs (halo rows), from build_pcg5_plan with W ranks of 132 // W CTAs
HALO = {
    ("kitti07_shaped", 2): 34, ("kitti07_shaped", 3): 95, ("kitti07_shaped", 4): 117, ("kitti07_shaped", 8): 230,
    ("kitti00_shaped", 2): 51, ("kitti00_shaped", 3): 84, ("kitti00_shaped", 4): 128, ("kitti00_shaped", 8): 290,
    ("rows_11k", 2): 35, ("rows_11k", 3): 52, ("rows_11k", 4): 85,
    ("orbit_600", 2): 599, ("orbit_600", 3): 599, ("orbit_600", 4): 599, ("orbit_600", 8): 599,
    ("local_ba", 2): 30, ("local_ba", 3): 30, ("local_ba", 4): 30, ("local_ba", 8): 30,
    ("two_submaps", 2): 22, ("two_submaps", 3): 50, ("two_submaps", 4): 49, ("two_submaps", 8): 52,
}


def _problem(pkg, problems, name):
    if name == "two_submaps":
        from test_topologies import topology
        return topology(pkg, name)
    return problems(name)


# ---- CPU: the plans ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted({n for n, _ in HALO}))
def test_emulated_plans(pkg, problems, name):
    """the plan of every emulated run exists, passes the plan's invariants (pcg5_plan_host raises otherwise) and its W x G CTAs fit
    one H100; rows_11k (10 999 free poses) has none at W = 8: 128 CTAs of at most 85 rows hold 10 880"""
    prob = _problem(pkg, problems, name)
    for W in WORLDS:
        plan = pkg.pcg5_plan_host(prob, W, SMS // W, 148)
        if (name, W) not in HALO:
            assert name == "rows_11k" and W == 8 and not plan["ok"], plan
            continue
        assert plan["ok"] and W * plan["G"] <= SMS, (W, plan)
        assert plan["halo_rows"] == HALO[name, W], (W, plan)
        if name == "orbit_600":
            assert plan["halo_rows"] == prob.numP          # every pose pair coupled: every row is some other rank's halo


# ---- GPU: the peer all-reduce -------------------------------------------------------------------------------------------

def _rank_order_sum(parts, dtype):
    """((0 + p0) + p1) + ... + p_{W-1} per call, in `dtype` (numpy adds elementwise without FMA or reordering)"""
    s = np.zeros(parts.shape[::2], dtype)
    for r in range(parts.shape[1]):
        s = s + parts[:, r].astype(dtype)
    return s.astype(np.float64)


def _bit_equal(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint64), np.ascontiguousarray(b).view(np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("fp32", [False, True], ids=["fp64", "fp32"])
@pytest.mark.parametrize("world", [2, 3, 5, 7, 8])
def test_peer_allreduce_is_the_rank_order_sum(pkg, world, fp32):
    """every rank's buffer after each of three consecutive calls is the rank-order sum, bit for bit.  The sizes: even slices, empty
    trailing slices (n < W), the scalar tail of an odd slice, and a slice longer than one grid stride (132 / W CTAs x 1024)"""
    eng = pkg.Engine(device=0, use_fp32=fp32)
    dtype = np.float32 if fp32 else np.float64
    rng = np.random.default_rng(world)
    stride = (SMS // world) * 512 * 2
    sizes = sorted({1, 2, 3, world - 1, world, world + 1, 2 * world + 1, 1023, world * stride + 2 * stride + 5})
    assert (sizes[-1] + world - 1) // world > stride
    for n in sizes:
        parts = rng.standard_normal((3, world, n)) * 10.0 ** rng.uniform(-6, 6, (3, world, n))    # sums that depend on the order
        parts = parts.astype(dtype).astype(np.float64)
        out = eng.peer_allreduce(parts)
        ref = _rank_order_sum(parts, dtype)
        for c in range(3):
            for r in range(world):
                assert _bit_equal(out[c, r], ref[c]), (n, c, r, np.flatnonzero(out[c, r] != ref[c])[:8])
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,world", [(n, w) for n in ("kitti07_shaped", "kitti00_shaped") for w in (3, 8)])
def test_peer_allreduce_of_dry_shards(pkg, oracle, problems, name, world):
    """the Hsc | bsc partials of every rank's dry shard (test_dry_shards), each rank's Hpp and bp added to its own: the emulated
    all-reduce is their rank-order sum bit for bit, and that sum is the whole problem's Schur complement from the oracle"""
    from test_dry_shards import LAMS, _full_oracle, dry_shards
    prob = problems(name)
    out = dry_shards(pkg, prob, RK, world)
    _, _, _, fschur = _full_oracle(oracle, prob, RK)
    diag = out[0]["hsc"][0][:-1]
    parts = []
    for lam in LAMS:
        row = []
        for r, res in enumerate(out):
            Hsc, bsc = res["schur"][lam][0].copy(), res["schur"][lam][1].copy()
            if r > 0:                                            # a dry shard keeps Hpp and bp on rank 0's diagonal only
                Hsc[diag] += res["system"][0]; bsc += res["system"][1]
            row.append(np.concatenate([Hsc.ravel(), bsc.ravel()]))
        parts.append(row)
    parts = np.array(parts)
    eng = pkg.Engine(device=0)
    got = eng.peer_allreduce(parts)
    eng.close()
    ref = _rank_order_sum(parts, np.float64)
    nH = out[0]["schur"][LAMS[0]][0].size
    for c, lam in enumerate(LAMS):
        for r in range(world):
            assert _bit_equal(got[c, r], ref[c]), (lam, r)
        Hsc, bsc = ref[c][:nH].reshape(-1, 36), ref[c][nH:].reshape(-1, 6)
        assert relerr(Hsc, fschur[lam][0]) < 1e-11, (lam, relerr(Hsc, fschur[lam][0]))
        assert relerr(bsc, fschur[lam][1]) < 1e-11, (lam, relerr(bsc, fschur[lam][1]))


# ---- GPU: the row-distributed k_pcg5 --------------------------------------------------------------------------------------

PCG5_CASES = ([("kitti07_shaped", w, False) for w in WORLDS] + [("kitti00_shaped", w, False) for w in WORLDS]
              + [("rows_11k", w, False) for w in (2, 4)] + [("orbit_600", w, False) for w in (2, 3)]
              + [("local_ba", w, False) for w in (2, 8)] + [("two_submaps", w, False) for w in (2, 3, 4)]
              + [("kitti07_shaped", w, True) for w in (2, 8)])
_BJ_RESTATED = {}


def _bj_restated(name, lam, S, b):
    """restated_pcg5 without a coarse level (the same for every W): cached per graph and damping"""
    from test_pcg_coarse import restated_pcg5
    if (name, lam) not in _BJ_RESTATED:
        _BJ_RESTATED[(name, lam)] = restated_pcg5(S, b, None, None, None)
    return _BJ_RESTATED[(name, lam)]


def _fp32_residual(eng, x, label):
    """test_fp32_stages.check_pcg's bound on the true residual of x against the engine's own Hsc / bsc, in the block-Jacobi norm"""
    import scipy.sparse as sp
    from test_fp32_stages import U
    from test_pcg_coarse import _full_system
    Hsc, bsc, _ = eng.schur()
    rp, ci = eng.hsc_structure()
    P = len(rp) - 1
    S = _full_system(Hsc, rp, ci, P)
    b = bsc.reshape(-1)
    x = x.reshape(-1)
    D = Hsc[rp[:-1]].reshape(-1, 6, 6).transpose(0, 2, 1)
    Li = sp.block_diag(list(np.linalg.inv(np.linalg.cholesky(D))), format="csr")
    nr = np.linalg.norm(Li @ (b - S @ x)); nb = np.linalg.norm(Li @ b); nm = np.linalg.norm(Li @ (abs(S) @ np.abs(x)))
    nnzr = int(np.diff(S.indptr).max())
    bound = 10 * 1e-6 * nb + (8 + nnzr) * U * nm
    print("%s: BJ residual %.2e, bound %.2e" % (label, nr, bound))
    assert nr <= bound, (label, nr, bound)


@pytest.mark.gpu
@pytest.mark.parametrize("name,world,fp32", PCG5_CASES, ids=["%s-w%d%s" % (n, w, "-fp32" if f else "") for n, w, f in PCG5_CASES])
def test_row_distributed_pcg5(pkg, oracle, problems, name, world, fp32):
    """per damping of the ladder, two-level and block-Jacobi, two calls of three solves each on the same boards:
    a. every rank of every solve reports status 0 and the same iteration count;  b. every row of x was written;  c. the solves are
    bitwise identical;  d. x against the oracle's direct solve (fp32: test_fp32_stages.check_pcg's residual bound);  e. the count
    against restated_pcg5 fed the emulation's aggregates and fp32 coarse inverse: within one (two-level), two (block-Jacobi), or 0.3 %
    of a count above a thousand"""
    from test_pcg_coarse import LADDER, _oracle_ladder, coarse_basis, restated_pcg5
    t0 = time.time()
    prob = _problem(pkg, problems, name)
    P = prob.numP
    ladder = None if fp32 else _oracle_ladder(oracle, prob, name)
    Z = coarse_basis(prob, P)
    eng = make_engine(pkg, prob, RK, use_fp32=fp32)
    eng.linearize()
    for lam, tol in LADDER:
        if name == "kitti00_shaped" and lam == 1e3:
            tol = 5e-10                  # the stopping rule leaves 1.1e-10 .. 1.7e-10 in exact arithmetic (test_gpu_parity)
        eng.bench_stage(3, reps=1, flush_l2=False, lam=lam)
        for two in (True, False):
            label = "%s w%d lambda %g %s" % (name, world, lam, "two-level" if two else "block-Jacobi")
            runs = [eng.pcg5_ranks(world, two, 3) for _ in range(2)]
            res = runs[0]
            plan = res["plan"]
            assert plan["halo"] == HALO[name, world] and plan["cinfo"] == 0 and world * plan["G"] <= SMS, (label, plan)
            if name == "rows_11k":
                assert plan["big"] and plan["maxRows"] == 85, (label, plan)     # the BIG shape: blocks streamed from the global copy
            for rr in runs:
                # a. identical scalars on every rank -> identical exits
                assert np.all(rr["status"] == 0), (label, rr["status"])
                assert np.all(rr["iters"] == res["iters"][0, 0]), (label, rr["iters"])
                # b. every row written by its owner
                assert not np.isnan(rr["x"]).any(), (label, np.unique(np.nonzero(np.isnan(rr["x"]))[1]))
                # c. bit-reproducible
                for x in rr["x"]:
                    assert np.array_equal(x, res["x"][0]), label
            iters = int(res["iters"][0, 0])
            x = res["x"][0]
            if fp32:
                _fp32_residual(eng, x, label)
                continue
            S, b, xp, _, _ = ladder[lam]
            if two:
                agg = np.repeat(np.arange(plan["A"]), np.diff(res["aggRow"]))
                assert len(agg) == P
                x_r, it_r = restated_pcg5(S, b.reshape(-1), agg, Z, res["AcInv"])
                bound = 1
            else:
                x_r, it_r = _bj_restated(name, lam, S, b.reshape(-1))
                bound = 2
            # d. x against the direct solve, to the ladder's tolerance or -- where the stopping rule itself leaves more than that
            #    (rows_11k at lambda 1e3: 1.8e-10, as the restatement) -- to what the restatement reaches (test_pcg_coarse)
            d, d_r = relerr(x, xp), relerr(x_r.reshape(-1, 6), xp)
            print("%s: %s G %d A %d halo %d big %d | %d iterations, restated %d | x %.1e (restated %.1e)"
                  % (label, "fp32" if fp32 else "fp64", plan["G"], plan["A"], plan["halo"], plan["big"], iters, it_r, d, d_r))
            assert d < max(tol, 3 * d_r), (label, d, d_r)
            # e. the count against the restatement.  The restatement runs on the oracle's system, which differs from the engine's in
            #    the last bits, and over a thousand iterations that moves the count by a few: rows_11k's block-Jacobi solve at lambda 0.1
            #    takes 1 095 iterations at W = 2 and 4, the restatement 1 098 (H100); every other solve is within one.  So 0.3 % of
            #    the count is allowed where that is more.
            assert abs(iters - it_r) <= max(bound, int(0.003 * it_r)), (label, iters, it_r)
    eng.close()
    print("%s w%d: %.1f s" % (name, world, time.time() - t0))
