"""The direct solver of the reduced camera system (Engine.set_linear_solver("dense"), include/cuba_b200.h:
cuba_engine_set_linear_solver; the kernel k_dense_chol, csrc/cuba_dense_chol.cuh): S xp = bsc by a dense fp64 Cholesky factorisation.

  CPU   the block -> tile layout against numpy, the cap of 2730 free poses, the order of the argument checks
  GPU   the kernel on random SPD matrices (backward error against Cholesky's bound, x against scipy, an indefinite matrix, bitwise
        repeatability); cuba_stage_solve on the lambda ladder against the oracle's direct solve; covis_2000, which the PCG refuses;
        the cap on the device; optimize() against the oracle; structure reuse, a change of solver, edge levels, fp32 and mixed
        precision
"""
import types

import numpy as np
import pytest

from conftest import KERNELS, make_engine, relerr
from test_pcg_coarse import LADDER, _full_system, _oracle_ladder

sp = pytest.importorskip("scipy.sparse")
sla = pytest.importorskip("scipy.linalg")

U = 2.0 ** -53
MAX_POSES = 2730


def _graph(pkg, problems, name):
    if name in ("two_submaps", "unanchored"):
        from test_topologies import topology
        return topology(pkg, name)
    return problems(name)


def _chain_problem(numP, seed=5):
    """numP free poses and one fixed, on a line; every pose sees the 24 landmarks nearest to it in stereo (a banded, well-posed S)"""
    rng = np.random.default_rng(seed)
    Pall = numP + 1
    q = np.zeros((Pall, 4)); q[:, 3] = 1.0
    t = np.zeros((Pall, 3)); t[:, 2] = -0.5 * np.arange(Pall)
    cam = np.tile([700.0, 700.0, 600.0, 180.0, 380.0], (Pall, 1))
    L = 4 * Pall + 20                                       # pose p sees landmarks 4p .. 4p + 23: every landmark has an edge
    Xw = np.stack([rng.uniform(-6, 6, L), rng.uniform(-2, 2, L), 0.125 * np.arange(L) + 6.0], axis=1)
    idx = []
    for p in range(Pall):
        first = 4 * p
        idx += [(p if p < numP else numP, first + k) for k in range(24)]
    idx = np.array(idx, np.int32)
    iP, iL = idx[:, 0], idx[:, 1]
    Xc = Xw[iL] + t[iP]
    u = 700.0 * Xc[:, 0] / Xc[:, 2] + 600.0; v = 700.0 * Xc[:, 1] / Xc[:, 2] + 180.0; ur = u - 380.0 / Xc[:, 2]
    meas3 = np.stack([u, v, ur], axis=1) + rng.normal(0, 0.5, (len(idx), 3))
    return types.SimpleNamespace(Pall=Pall, numP=numP, Lall=L, numL=L, q=q, t=t, cam=cam, Xw=Xw + rng.normal(0, 0.05, Xw.shape),
                                 E2=0, idx2=np.zeros((0, 2), np.int32), meas2=np.zeros((0, 2)), omega2=np.zeros(0),
                                 E3=len(idx), idx3=idx, meas3=meas3, omega3=np.ones(len(idx)))


# ---- CPU ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["tiny", "local_ba", "orbit_600", "small"])
def test_block_map_against_numpy(pkg, problems, name):
    """the packed lower block triangle of S -> block of the full BSR, and the tile counts; tiny (n = 72), local_ba (180) and small
    (354) are not multiples of 32"""
    prob = problems(name)
    s = pkg.build_structure_host(prob)
    lay = pkg.binding.dense_layout_host(prob)
    P = prob.numP
    rp, ci = s["fullRowPtr"], s["fullColInd"]
    want = np.full(P * (P + 1) // 2, -1, np.int32)
    rows = np.repeat(np.arange(P), np.diff(rp))
    low = ci <= rows
    want[rows[low] * (rows[low] + 1) // 2 + ci[low]] = np.arange(len(ci))[low]
    assert np.array_equal(lay["map"], want)
    n = 6 * P; nt = -(-n // 32)
    assert (lay["numP"], lay["n"], lay["nt"], lay["tiles"]) == (P, n, nt, nt * (nt + 1) // 2)
    assert lay["tile_mb"] == (nt * (nt + 1) // 2 * 1024 * 8) >> 20
    # every block present in the upper BSR of S appears once in the map, and no absent block does
    assert (lay["map"] >= 0).sum() == s["nblk"]


def test_cap_arithmetic(pkg):
    """2730 free poses: n = 16380, 512 tile rows, 1.05 GB of tiles; 2731 are refused with the message set_problem gives"""
    lay = pkg.binding.dense_layout_host(_chain_problem(MAX_POSES))
    assert (lay["n"], lay["nt"], lay["tiles"]) == (16380, 512, 512 * 513 // 2)
    assert lay["tile_mb"] == (512 * 513 // 2 * 8192) >> 20 == 1026
    with pytest.raises(pkg.CubaError, match=r"at most 2730 free poses, this problem has numP = 2731"):
        pkg.binding.dense_layout_host(_chain_problem(MAX_POSES + 1))
    assert pkg.binding.DENSE_MAX_POSES == MAX_POSES


def test_set_linear_solver_checks_the_value_first(pkg):
    """a value that names no solver is refused before the engine is looked at (here: no engine, so no device is touched)"""
    for bad in (-1, 2, 9):
        rc, msg = pkg.binding.set_linear_solver_raw(bad)
        assert rc == -1 and "names no solver" in msg, (bad, rc, msg)
    for good in (0, 1):
        rc, msg = pkg.binding.set_linear_solver_raw(good)
        assert rc == -1 and msg == "null engine", (good, rc, msg)


def test_binding_names_the_kernel(pkg):
    assert pkg.binding.PCG_KERNELS[8] == "k_dense_chol"
    assert pkg.binding.LINEAR_SOLVERS == {"pcg": 0, "dense": 1}
    for n in ("cuba_engine_set_linear_solver", "cuba_debug_dense_solve", "cuba_debug_dense_layout"):
        assert n in pkg.binding.exported_symbols()


# ---- GPU: the kernel on random matrices ----------------------------------------------------------------------------------

def _spd(n, kappa, seed):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    ev = np.logspace(0, -np.log10(kappa), n) if n > 1 else np.ones(1)
    S = (Q * ev) @ Q.T
    return 0.5 * (S + S.T), rng.standard_normal(n)


def _backward_error(S, x, b):
    """||S x - b|| / (||S|| ||x|| + ||b||) in 2-norms, the residual in extended precision"""
    r = S.astype(np.longdouble) @ x.astype(np.longdouble) - b.astype(np.longdouble)
    return float(np.linalg.norm(r.astype(np.float64))) / (np.linalg.norm(S, 2) * np.linalg.norm(x) + np.linalg.norm(b))


def _cholesky_bound(n):
    """Cholesky's backward-error theorem (Higham, Accuracy and Stability, Thm 10.4 with 10.3): the computed x solves (S + dS) x = b
    with |dS| <= gamma_{3n+1} |L||L^T|, and || |L||L^T| ||_2 <= n ||S||_2 (up to a factor 1 + O(nu)).  So the normwise backward
    error is at most n gamma_{3n+1}.  The kernel works on the padded order np = 32 ceil(n / 32) (the padding is a decoupled unit
    block) and multiplies by reciprocals of the diagonal of L instead of dividing, one more rounding per solve step: n_p gamma_{3n_p+2}."""
    npad = 32 * (-(-n // 32))
    k = 3 * npad + 2
    return npad * k * U / (1 - k * U)


SIZES = (1, 6, 31, 32, 33, 180, 1482, 3594)
KAPPAS = (1.0, 1e4, 1e8, 1e12)


@pytest.mark.gpu
def test_debug_dense_solve_random_spd(pkg):
    """n x kappa: backward error within Cholesky's bound, x against scipy's cho_solve within what both backward errors allow (the
    forward error of each is at most kappa eta / (1 - kappa eta)), bitwise repeatable.  The largest backward error / bound ratio
    is printed (DESIGN.md 4.7 records it)."""
    eng = pkg.Engine(device=0)
    worst = 0.0
    for n in SIZES:
        for kappa in KAPPAS:
            S, b = _spd(n, kappa, seed=n * 13 + int(np.log10(kappa)))
            x, info = eng.debug_dense_solve(S, b)
            assert info == 0, (n, kappa)
            eta = _backward_error(S, x, b)
            bound = _cholesky_bound(n)
            assert eta <= bound, (n, kappa, eta, bound)
            worst = max(worst, eta / bound)
            xr = sla.cho_solve(sla.cho_factor(S, lower=True), b)
            eta_r = _backward_error(S, xr, b)
            fwd = lambda e: kappa * e / max(1 - kappa * e, 1e-300)
            allow = fwd(eta) + fwd(eta_r) if kappa * max(eta, eta_r) < 0.5 else np.inf
            assert np.linalg.norm(x - xr) <= 2 * allow * np.linalg.norm(xr) + 1e-300, (n, kappa, np.linalg.norm(x - xr) / np.linalg.norm(xr), allow)
            if n in (33, 1482):
                x2, _ = eng.debug_dense_solve(S, b)
                assert np.array_equal(x, x2), (n, kappa)
    print("largest backward error / Cholesky bound: %.3g" % worst)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [6, 33, 180])
def test_debug_dense_solve_indefinite(pkg, n):
    """one negative eigenvalue: info 1 and x = 0"""
    S, b = _spd(n, 1e3, seed=n)
    w, V = np.linalg.eigh(S)
    w[n // 2] = -1.0
    S = (V * w) @ V.T
    eng = pkg.Engine(device=0)
    x, info = eng.debug_dense_solve(0.5 * (S + S.T), b)
    assert info == 1 and not np.any(x), (n, info)
    eng.close()


# ---- GPU: the stage on the engine's systems ------------------------------------------------------------------------------

STAGE_GRAPHS = ("tiny", "small", "kitti07_shaped", "local_ba", "unanchored", "two_submaps", "orbit_600", "covis_1000", "kitti00_shaped")


def _dense_engine(pkg, prob, rk, **kw):
    eng = pkg.Engine(device=0, **kw)
    for et in (0, 1):
        eng.set_robust_kernels(rk[0][et], rk[1][et], et)
    eng.set_linear_solver("dense")
    eng.initialize(prob)
    return eng


@pytest.mark.gpu
@pytest.mark.parametrize("name", STAGE_GRAPHS)
def test_stage_solve_against_oracle(pkg, oracle, problems, name):
    """cuba_stage_solve on the lambda ladder: xp and xl against the oracle's direct solve at LADDER's tolerances (those of the PCG),
    the kernel id and status; then lambda = -2 max diagonal, an indefinite S: ok = 0, status 2, xp = 0, and an ordinary optimize()
    on the same engine gives what a fresh dense engine gives"""
    prob = _graph(pkg, problems, name)
    ladder = _oracle_ladder(oracle, prob, name)
    rk = KERNELS["huber"]
    eng = _dense_engine(pkg, prob, rk)
    eng.linearize()
    worst = 0.0
    for lam, tol in LADDER:
        iters, ok = eng.solve(lam)
        info = eng.pcg_info()
        assert ok and iters == 0, (name, lam)
        assert (info["kernel"], info["status"], info["iters"], info["two_level"], info["coarse_kernel"]) == ("k_dense_chol", 0, 0, False, "none"), info
        assert (info["G"], info["A"], info["aggs_per_cta"]) == (0, 0, 0), info
        xp, xl = eng.delta()
        _, _, oxp, oxl, _ = ladder[lam]
        e = max(relerr(xp.reshape(-1), oxp.reshape(-1)), relerr(xl.reshape(-1), oxl.reshape(-1)))
        assert e < tol, (name, lam, e)
        worst = max(worst, e)
    md = eng.max_diagonal()
    iters, ok = eng.solve(-2.0 * md)
    info = eng.pcg_info()
    assert not ok and info["status"] == 2 and info["kernel"] == "k_dense_chol", info
    assert not np.any(eng.delta()[0])
    if name in ("small", "local_ba"):
        stats = eng.optimize(5)
        fresh = _dense_engine(pkg, prob, rk)
        ref = fresh.optimize(5)
        assert [s["chi2"] for s in stats] == [s["chi2"] for s in ref]
        for a, b in zip(eng.state(), fresh.state()):
            assert np.array_equal(a, b)
        fresh.close()
    print("%s: largest error of x against the oracle's direct solve %.3g" % (name, worst))
    eng.close()


def _own_system(eng, P, lam):
    """S and bsc of the engine's own Schur stage at lam (scipy sparse, symmetric)"""
    eng.solve(lam)
    Hsc, bsc, _ = eng.schur()
    rp, ci = eng.hsc_structure()
    return _full_system(Hsc, rp, ci, P), bsc.reshape(-1)


@pytest.mark.gpu
def test_covis_2000_is_solved(pkg, problems):
    """covis_2000: the PCG refuses it (its need lists do not fit k_pcg3's shared memory); the dense solver accepts it.  One solve
    against scipy's Cholesky of the engine's own S (dense, n = 11 994), and optimize(2) lowers chi2 below its initial value at every
    iteration, with no failed trial.
    The oracle's run on this graph (a direct solve of the 11 994 x 11 994 system per trial on the CPU) is not part of the test:
    it takes minutes."""
    prob = problems("covis_2000")
    eng = _dense_engine(pkg, prob, KERNELS["huber"])
    chi0 = eng.linearize()                         # the initial estimate: solves without a commit leave it in place
    lam = 10.0
    S, b = _own_system(eng, prob.numP, lam)
    xp, _ = eng.delta()
    xr = sla.cho_solve(sla.cho_factor(S.toarray(), lower=True), b)
    assert relerr(xp.reshape(-1), xr) < 1e-9
    assert eng.pcg_info()["kernel"] == "k_dense_chol"
    stats = eng.optimize(2)
    assert len(stats) == 2 and all(s["pcg_failed"] == 0 and s["pcg_iters"] == 0 for s in stats)
    assert stats[0]["chi2"] < chi0 and stats[1]["chi2"] <= stats[0]["chi2"], (chi0, [s["chi2"] for s in stats])
    print("covis_2000 optimize(2): chi2 %.6e -> %s" % (chi0, ["%.6e" % s["chi2"] for s in stats]))
    eng.close()


@pytest.mark.gpu
def test_cap_on_the_device(pkg, problems):
    """2731 free poses are refused before anything changes, and the engine then runs `small` as a fresh one does; 2730 free poses
    solve with status 0 and a backward error (sparse S x on the host) within Cholesky's bound"""
    rk = KERNELS["huber"]
    eng = _dense_engine(pkg, problems("small"), rk)
    with pytest.raises(pkg.CubaError, match=r"at most 2730 free poses, this problem has numP = 2731"):
        eng.initialize(_chain_problem(MAX_POSES + 1))
    eng.initialize(problems("small"))
    stats = eng.optimize(5)
    fresh = _dense_engine(pkg, problems("small"), rk)
    ref = fresh.optimize(5)
    assert [s["chi2"] for s in stats] == [s["chi2"] for s in ref]
    fresh.close()
    prob = _chain_problem(MAX_POSES)
    eng.initialize(prob)
    eng.linearize()
    S, b = _own_system(eng, prob.numP, 1.0)
    info = eng.pcg_info()
    assert (info["kernel"], info["status"]) == ("k_dense_chol", 0), info
    xp = eng.delta()[0].reshape(-1)
    r = S @ xp - b
    eta = np.linalg.norm(r) / (_spectral_norm(S) * np.linalg.norm(xp) + np.linalg.norm(b))
    assert eta <= _cholesky_bound(S.shape[0]), eta
    print("2730 free poses: backward error %.3g, bound %.3g" % (eta, _cholesky_bound(S.shape[0])))
    # no free landmark: the poses are solved block by block whichever solver is chosen, so neither the cap nor the tiles apply
    po = _chain_problem(MAX_POSES + 1)
    keep = po.idx3[:, 0] < po.numP                            # edges of the fixed pose would have both ends fixed
    po.idx3, po.meas3, po.omega3 = po.idx3[keep], po.meas3[keep], po.omega3[keep]
    po.E3, po.numL = int(keep.sum()), 0
    eng.initialize(po)
    stats = eng.optimize(2)
    assert len(stats) >= 1 and all(s["pcg_failed"] == 0 for s in stats)
    assert eng.pcg_info()["kernel"] == "none"
    eng.close()


def _spectral_norm(S):
    return float(sp.linalg.eigsh(S, k=1, which="LA", return_eigenvectors=False)[0])


# ---- GPU: optimize() -----------------------------------------------------------------------------------------------------

OPTIMIZE_CASES = [("tiny", "none", 10), ("small", "huber", 10), ("tiny", "tukey", 10), ("small", "tukey", 10), ("kitti07_shaped", "huber", 10),
                  ("local_ba", "huber", 10), ("unanchored", "huber", 10), ("orbit_600", "huber", 3), ("covis_1000", "huber", 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,kernel,iters", OPTIMIZE_CASES)
def test_optimize_matches_oracle(pkg, oracle, problems, name, kernel, iters):
    """chi2 per iteration, lambda, trials and the final estimate against the oracle (whose solve is a direct one too)"""
    from test_gpu_parity import _trajectory_check
    prob = _graph(pkg, problems, name); rk = KERNELS[kernel]
    eng = _dense_engine(pkg, prob, rk)
    stats = eng.optimize(iters)
    o = oracle.Oracle(prob, *rk)
    chi, lam, tr = o.optimize(iters)
    _trajectory_check(stats, chi, lam, tr)
    assert all(s["pcg_iters"] == 0 for s in stats)
    for nme, a, b in zip(("q", "t", "Xw"), eng.state(), o.state()):
        assert relerr(a, b) < 1e-10, (name, nme, relerr(a, b))
    assert eng.pcg_info()["kernel"] == "k_dense_chol"
    eng.close()


@pytest.mark.gpu
def test_fixed_vertex_cases_match_oracle(pkg, oracle):
    """the fixed-vertex topologies (fixed landmarks seen by free poses, fixed poses seeing free landmarks), at 1e-10"""
    from test_gpu_parity import _trajectory_check
    from test_topologies import topology
    for name in ("pose_fixed_lms", "lm_fixed_poses"):
        prob = topology(pkg, name); rk = KERNELS["huber"]
        eng = _dense_engine(pkg, prob, rk)
        stats = eng.optimize(10)
        o = oracle.Oracle(prob, *rk)
        chi, lam, tr = o.optimize(10)
        _trajectory_check(stats, chi, lam, tr)
        for nme, a, b in zip(("q", "t", "Xw"), eng.state(), o.state()):
            assert relerr(a, b) < 1e-10, (name, nme, relerr(a, b))
            print("%s %s: %.2e against the oracle" % (name, nme, relerr(a, b)))
        eng.close()


# ---- GPU: composition ----------------------------------------------------------------------------------------------------

def _run(eng, n=5):
    stats = eng.optimize(n)
    return [s["chi2"] for s in stats], eng.state()


def _same(a, b):
    assert a[0] == b[0]
    for x, y in zip(a[1], b[1]):
        assert np.array_equal(x, y)


@pytest.mark.gpu
def test_structure_reuse_and_solver_change_are_a_fresh_engine(pkg, problems):
    """a structure-reuse set_problem, and a change of solver followed by set_problem, give bit for bit what a fresh engine gives"""
    prob = problems("kitti07_shaped"); rk = KERNELS["huber"]
    ref_dense = _run(_dense_engine(pkg, prob, rk))
    ref_pcg = _run(make_engine(pkg, prob, rk))
    eng = _dense_engine(pkg, prob, rk)
    _run(eng)
    eng.initialize(prob)                                   # same topology: structure reuse
    assert eng.structure_reuses() == 1
    _same(_run(eng), ref_dense)
    eng.set_linear_solver("pcg"); eng.initialize(prob)     # same topology, other solver: rebuilt
    assert eng.structure_reuses() == 1
    _same(_run(eng), ref_pcg)
    eng.set_linear_solver("dense"); eng.initialize(prob)
    _same(_run(eng), ref_dense)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["none", "huber"])
def test_edge_levels_with_the_dense_solver(pkg, problems, kernel):
    """edges at level 1 give bit for bit what a problem whose omega is 0 on those edges gives"""
    prob = problems("kitti07_shaped"); rk = KERNELS[kernel]
    E = prob.E2 + prob.E3
    lev = (np.random.default_rng(3).random(E) < 0.1).astype(np.uint8)
    eng = _dense_engine(pkg, prob, rk)
    eng.set_edge_levels(lev)
    got = _run(eng, 10)
    masked = types.SimpleNamespace(**{k: getattr(prob, k) for k in ("Pall", "numP", "Lall", "numL", "q", "t", "cam", "Xw", "E2", "idx2",
                                                                        "meas2", "E3", "idx3", "meas3")})
    masked.omega2 = np.where(lev[:prob.E2] != 0, 0.0, prob.omega2)
    masked.omega3 = np.where(lev[prob.E2:] != 0, 0.0, prob.omega3)
    ref = _run(_dense_engine(pkg, masked, rk), 10)
    _same(got, ref)
    eng.close()


@pytest.mark.gpu
def test_fp32_and_mixed_precision(pkg, problems):
    """fp32 engine: xp is the fp64 Cholesky solution of its own widened S, rounded to fp32 (the factorisation is fp64; only the
    summation order differs from scipy's, so a few fp32 units); mixed precision: optimize() within 1e-7 of fp64"""
    prob = problems("kitti07_shaped"); rk = KERNELS["huber"]
    e32 = _dense_engine(pkg, prob, rk, use_fp32=True)
    e32.linearize()
    for lam in (1e3, 10.0):
        S, b = _own_system(e32, prob.numP, lam)
        xr = sla.cho_solve(sla.cho_factor(S.toarray(), lower=True), b).astype(np.float32).astype(np.float64)
        xp = e32.delta()[0].reshape(-1)
        assert relerr(xp, xr) < 4 * 2.0 ** -24, (lam, relerr(xp, xr))
        assert e32.pcg_info()["kernel"] == "k_dense_chol"
    e32.close()
    e64 = _dense_engine(pkg, prob, rk)
    emx = _dense_engine(pkg, prob, rk, use_fp32="mixed")
    a = _run(e64, 10); m = _run(emx, 10)
    assert relerr(m[0], a[0]) < 1e-7
    for x, y in zip(m[1], a[1]):
        assert relerr(x, y) < 1e-7
    e64.close(); emx.close()


# ---- GPU: sharded runs, the compiled reference, the reference's fixtures ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "kitti07_shaped"])
def test_dry_shard_rank0_follows_the_sub_problem(pkg, oracle, problems, name):
    """rank 0 of a three-rank landmark-sharded run (CUBA_DRY_SHARD: its own shard, no collective) with the dense solver: optimize(10)
    is the LM run of the sub-problem of rank 0's landmarks.  The reduced system is the rank's partial S (upper blocks expanded as a
    sharded run expands the all-reduced ones), and the direct solve is not distributed."""
    from test_dry_shards import _edge_landmarks
    from test_gpu_parity import _trajectory_check
    world = 3
    prob = problems(name); rk = KERNELS["huber"]
    b = pkg.sharding.shard_bounds(_edge_landmarks(prob), prob.Lall, world)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("CUBA_DRY_SHARD", "1")
        eng = pkg.Engine(device=0)
        eng.set_comm(0, world, b"\0" * 128)
    for et in (0, 1):
        eng.set_robust_kernels(rk[0][et], rk[1][et], et)
    eng.set_linear_solver("dense")
    eng.initialize(prob)
    stats = eng.optimize(10)
    o = oracle.Oracle(pkg.sharding.sub_problem(prob, b[0], b[1]), *rk)
    chi, lam, tr = o.optimize(10)
    _trajectory_check(stats, chi, lam, tr)
    assert eng.pcg_info()["kernel"] == "k_dense_chol"
    q, t, Xw = eng.state()
    oq, ot, oX = o.state()
    own = np.zeros(prob.Lall, bool); own[b[0]:min(b[1], prob.numL)] = True
    assert relerr(q, oq) < 1e-10 and relerr(t, ot) < 1e-10 and relerr(Xw[own], oX[own]) < 1e-10
    assert np.array_equal(Xw[~own], prob.Xw[~own])
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,kernel,how", [("small", "huber", None), ("kitti07_shaped", "none", None), ("tiny", "tukey", None),
                                             ("small", "tukey", None), ("tiny", "huber", "mixed"), ("tiny", "huber", "pose_only"),
                                             ("tiny", "huber", "landmark_only"), ("ba_kitti_07", "none", "protocol"),
                                             ("ba_kitti_07", "huber", "protocol"), ("ba_kitti_00", "none", "protocol"),
                                             ("ba_kitti_00", "huber", "protocol")])
def test_dense_against_compiled_reference(pkg, problems, name, kernel, how):
    """the reference's own optimize() (its Cholesky solver) on the identical flat problem, as test_gpu_parity checks the default
    engine: live where oracle/_ref/ holds the compiled reference, otherwise tests/golden/reference_runs.npz for the synthetic cases;
    the real fixtures under the reference's protocol (warm-up optimize(1) written back, then initialize() + optimize(10))"""
    from test_gpu_parity import REF_VARIANTS, TOL, _reference, _reference_result, _relerr_vs_reference, _variant
    from conftest import have_fixture
    reference = _reference()
    if name.startswith("ba_") and not (reference.available() and have_fixture(name)):
        pytest.skip("needs the reference's fixture and its compiled build in oracle/_ref/")
    prob = problems(name); rk = KERNELS[kernel]
    if how in REF_VARIANTS:
        prob = _variant(pkg, prob, **REF_VARIANTS[how](prob))
    eng = _dense_engine(pkg, prob, rk)
    pr = prob
    if how == "protocol":
        w = reference.run(prob, 1, *rk)
        assert w is not None
        pr = prob.copy(); pr.q, pr.t, pr.Xw = w["q"], w["t"], w["Xw"]
        mine = eng.optimize(1)
        assert mine[0]["chi2"] == pytest.approx(w["chi2"][0], rel=TOL)
        q, t, Xw = eng.state()
        po = prob.copy(); po.q, po.t, po.Xw = q, t, Xw
        eng.initialize(po)
    r, rows = _reference_result(pr, name, kernel, how)
    stats = eng.optimize(10)
    got = np.array([s["chi2"] for s in stats])
    assert len(got) == len(r["chi2"]), (got, r["chi2"])
    assert np.abs(got - r["chi2"]).max() / got.max() < TOL
    for nme, a in zip(("q", "t", "Xw"), eng.state()):
        assert _relerr_vs_reference(a, r[nme], rows, nme, TOL) < TOL, nme
    assert _relerr_vs_reference(eng.chi_squared(), r["chisq"], rows, "chisq", 1e-8) < 1e-8
    if prob.numP and prob.numL:
        assert eng.pcg_info()["kernel"] == "k_dense_chol"
    eng.close()


@pytest.mark.gpu
def test_dense_kitti00_readme_table(pkg, problems, golden):
    """README.md:141-150 of the reference (ba_kitti_00, NONE, after the sample's warm-up optimize(1)) with the dense solver, to the
    printed 0.1, and the committed oracle trajectory at 1e-10"""
    from conftest import have_fixture
    if not have_fixture("ba_kitti_00"):
        pytest.skip("reference fixture absent")
    prob = problems("ba_kitti_00")
    eng = _dense_engine(pkg, prob, KERNELS["none"])
    eng.optimize(1)
    q, t, Xw = eng.state()
    p2 = prob.copy(); p2.q, p2.t, p2.Xw = q, t, Xw
    eng.initialize(p2)
    stats = eng.optimize(10)
    chi = np.array([s["chi2"] for s in stats])
    assert np.all(np.abs(np.round(chi, 1) - np.array(golden["readme_chi2_kitti00_none"])) < 0.051)
    assert np.allclose(chi, golden["ba_kitti_00_none"]["chi2"], rtol=1e-10)
    assert eng.pcg_info()["kernel"] == "k_dense_chol"
    eng.close()


@pytest.mark.gpu
def test_two_gpu_dense_trajectory_matches_oracle():
    """a landmark-sharded run on two GPUs (NCCL) with the dense solver against the CPU oracle: every rank factors the same
    all-reduced S, so every rank's poses are the same bit for bit; skipped where fewer than two GPUs exist"""
    import json
    import os
    import subprocess
    import sys
    import torch
    from conftest import ROOT
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    env = dict(os.environ, LINEAR_SOLVER="dense", RESULT_JSON="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29537",
           os.path.join(ROOT, "tools", "multigpu_check.py"), "small", "kitti07_shaped"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stderr[-2000:]
    res = [json.loads(l[len("RESULT "):]) for l in out.stdout.splitlines() if l.startswith("RESULT ")]
    assert len(res) == 2
    for r in res:
        assert r["chi2_rel_diff_vs_oracle"] < 1e-10 and r["state_diff"] < 1e-9 and r["repeat_diff"] == 0.0, r
        assert r["same_poses_on_every_rank"] and r["trials_equal"], r
