"""The reduced-system solvers on densely covisible camera graphs (synth.COVISIBLE_CONFIGS), the shape of structure-from-motion
collections and of ORB-SLAM's local-BA windows: hundreds of cameras see the same points, so a row of the reduced camera system S
couples to hundreds of poses.  The odometry-shaped graphs of the other tests never reach the size-dependent paths this takes:
  * a CTA owns thousands of blocks of S: after the registers and the shared-memory cache the rest is read from the global copy
    every pass (k_pcg3 and k_pcg5<BIG>);
  * a CTA's need list holds hundreds of columns: k_pcg3 polls more than PCG3_WPT words per round, and k_pcg5 polls more w entries
    than its block-product staging has columns (PCG5_CHUNK = 512), so the staging is sized by the need list;
  * covis_2000's need lists do not fit k_pcg3's shared memory at all, which set_problem reports as an error.

  graph        free poses  blocks of S        landmark degree   what it reaches
  orbit_600    599         all 358 801        40                k_pcg5<BIG> with needMax 599 > 512; k_pcg3's global blocks
  covis_1000   999         ~30 % of pairs     8                 needMax 970 in k_pcg5's plan: k_pcg5 no longer fits, k_pcg3 solves
  covis_2000   1999        ~30 % of pairs     8                 k_pcg3's need lists beyond shared memory: CubaError
  local_ba     30 (+70 fixed)  all            2 .. 100          jh4's split landmarks, fixed poses on most edges
"""
import numpy as np
import pytest

from conftest import KERNELS, make_engine, relerr
from test_pcg_coarse import LADDER, _full_system, _oracle_ladder, coarse_basis, count_bound, restated_pcg5

sp = pytest.importorskip("scipy.sparse")
sla = pytest.importorskip("scipy.linalg")

DENSE = ("orbit_600", "covis_1000", "covis_2000", "local_ba")
H100_SMS = 132
H100_SMEM_OPTIN = 232448                      # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
PCG3_BUDGET = H100_SMEM_OPTIN - 6144          # Engine::pcg3_budget: the opt-in limit less k_pcg3's static arrays
STAGE_TOL = 1e-11
TOL = 1e-10

# (free poses, k_pcg5 plan on one H100: G, needMax, blkMax; k_pcg3's partition over 132 CTAs: needMax, blkMax)
PINNED = {
    "orbit_600": (599, 75, 599, 4792, 599, 2995),
    "covis_1000": (999, 125, 970, 2709, 956, 2571),
    "covis_2000": (1999, 132, 1996, 9685, 1996, 9685),
    "local_ba": (30, 4, 30, 240, 30, 30),
}


# ---- CPU ------------------------------------------------------------------------------------------------------------------

def test_dense_graphs_have_the_intended_shape(pkg, problems):
    """orbit_600: every pose pair coupled in S; local_ba: 30 free and 70 fixed keyframes, all free pairs coupled; landmark degrees
    above 32, so that the warp tiles of the J+H pass cut landmarks into pieces"""
    for name in ("orbit_600", "local_ba"):
        prob = problems(name)
        s = pkg.build_structure_host(prob)
        assert s["nblk_full"] == prob.numP ** 2, (name, s["nblk_full"])
    lb = problems("local_ba")
    assert (lb.numP, lb.Pall) == (30, 100)
    for name, lo, hi in (("orbit_600", 40, 40), ("local_ba", 33, 100)):
        prob = problems(name)
        deg = np.bincount(np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]]), minlength=prob.Lall)
        assert deg.max() >= lo and deg.max() <= hi, (name, deg.max())


@pytest.mark.parametrize("name", DENSE)
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_pcg5_w_staging_holds_the_need_list(pkg, problems, name, world):
    """k_pcg5 and k_pcg5t poll the w entries of a CTA's needed columns into their block-product staging: it must hold needMax
    columns in both launch shapes' layouts (with 512 columns, k_pcg5 overran it into the coarse residual, the partial sums and the
    board offsets on orbit_600 and covis_1000)"""
    prob = problems(name)
    plan = pkg.pcg5_plan_host(prob, world, H100_SMS, 148)
    if not plan["ok"]:
        return
    assert plan["needMax"] <= plan["w_cols_legacy"], plan
    assert plan["needMax"] <= plan["w_cols_tuned"], plan
    assert plan["w_cols_legacy"] >= 512 and plan["blkMax"] >= plan["needMax"], plan


@pytest.mark.parametrize("name", DENSE)
def test_dense_graph_plans_are_pinned(pkg, problems, name):
    """the need lists and block counts the GPU tests below rely on; k_pcg3 fits orbit_600 and covis_1000 but not covis_2000"""
    nP, G, need5, blk5, need3, blk3 = PINNED[name]
    prob = problems(name)
    assert prob.numP == nP
    plan = pkg.pcg5_plan_host(prob, 1, H100_SMS, 148)
    part = pkg.pcg_partition_host(prob, min(H100_SMS, nP), 148)
    print("%s: k_pcg5 plan %s; k_pcg3 partition %s" % (name, plan, part))
    assert (plan["ok"], plan["G"], plan["needMax"], plan["blkMax"]) == (1, G, need5, blk5), plan
    assert (part["needMax"], part["blkMax"]) == (need3, blk3), part
    assert (part["pcg3_fixed_bytes"] > PCG3_BUDGET) == (name == "covis_2000"), part
    assert plan["needMax"] > 512 or name == "local_ba"


# ---- GPU: stages ---------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["orbit_600", "local_ba"])
def test_dense_stages_match_oracle(pkg, oracle, problems, name):
    """J+H (jh4 with split landmarks), k_inv_hll and the Schur complement (k_schur3 and the tensor-pipe kernel) against the
    oracle, and the host structure builder against the device one"""
    prob = problems(name); rk = KERNELS["huber"]
    o = oracle.Oracle(prob, *rk)
    ochi = o.compute_errors(); o.build_system()
    osys = o.system()
    engs = {v: make_engine(pkg, prob, rk, schur_variant=v) for v in (3, 5)}
    host = make_engine(pkg, prob, rk, structure_on_host=True)
    for x, y in zip(host.hpl_structure() + host.hsc_structure(), engs[3].hpl_structure() + engs[3].hsc_structure()):
        assert np.array_equal(x, y)
    for a, b in zip(engs[3].hpl_structure() + engs[3].hsc_structure(), o.hpl_structure() + o.hsc_structure()):
        assert np.array_equal(a, b)
    for eng in list(engs.values()) + [host]:
        chi = eng.linearize()
        assert abs(chi - ochi) <= STAGE_TOL * ochi
        for nme, a, b in zip(("Hpp", "bp", "Hll", "bl", "Hpl"), eng.system(), osys):
            assert relerr(a, b) < STAGE_TOL, (name, nme)
    for lam in (1e3, 1.0):
        assert o.solve(lam)
        ref = o.schur()
        for v, eng in list(engs.items()) + [("host", host)]:
            assert eng.solve(lam)[1]
            for nme, a, b in zip(("Hsc", "bsc", "invHll"), eng.schur(), ref):
                d = relerr(a, b)
                assert d < STAGE_TOL, (name, v, lam, nme, d)
    for eng in list(engs.values()) + [host]:
        eng.close()


# ---- GPU: every solver path on orbit_600 ---------------------------------------------------------------------------------

# pcg_variant -> the kernel that runs on orbit_600 and whether it is two-level.  The tuned k_pcg5t does not fit (it would cache
# 4 280 blocks), so k_pcg5 takes its BIG shape with the need list of 599 columns; automatic runs k_pcg3 for quick block-Jacobi
# solves and two-level k_pcg5 afterwards.
PATHS = {
    "0": (0, {}, None),
    "2": (2, {}, ("k_pcg2", False)),
    "3": (3, {}, ("k_pcg4", True)),
    "4": (4, {}, ("k_pcg3", False)),
    "5": (5, {}, ("k_pcg5_big", True)),
    "6": (6, {}, ("k_pcg5_big", False)),
    "5-legacy": (5, {"CUBA_PCG5_LEGACY": "1"}, ("k_pcg5_big", True)),
    "6-legacy": (6, {"CUBA_PCG5_LEGACY": "1"}, ("k_pcg5_big", False)),
}


def _direct(S, b):
    """dense fp64 Cholesky of the reduced system"""
    return sla.cho_solve(sla.cho_factor(S.toarray()), b)


def _check_solve(eng, prob, label, lam, tol, S, b, xl_ref, plan, iters, ok, Z):
    info = eng.pcg_info()
    assert ok and info["status"] == 0 and info["iters"] == iters and info["bj_retries"] == 0, (label, lam, info)
    if info["kernel"].startswith("k_pcg5"):
        assert info["G"] == plan["G"], (label, info)
        assert info["capBlocks"] < plan["blkMax"] - 512, (label, info, plan)        # blocks past registers + cache: global copy
    x = _direct(S, b)
    xp, xl = eng.delta()
    dp, dl = relerr(xp.reshape(-1), x), relerr(xl, xl_ref)
    restated = ""
    if info["kernel"] == "k_pcg5_big" and info["two_level"]:
        agg, _, AcInv = eng.coarse()
        x_r, it_r = restated_pcg5(S, b, agg, Z, AcInv)
        restated = " restated %d (%+d)" % (it_r, iters - it_r)
        assert abs(iters - it_r) <= count_bound(it_r), (label, lam, iters, it_r)
    print("dense path %-10s lambda %-6g %-10s two-level %d needMax %4d capBlocks %4d global blocks %5d | iterations %4d%s | "
          "xp %.1e xl %.1e (tol %.0e)" % (label, lam, info["kernel"], info["two_level"], plan["needMax"], info["capBlocks"],
                                          max(plan["blkMax"] - 512 - info["capBlocks"], 0) if info["kernel"].startswith("k_pcg5") else -1,
                                          iters, restated, dp, dl, tol))
    assert dp < tol and dl < tol, (label, lam, dp, dl)
    return info


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(PATHS))
def test_dense_solver_paths(pkg, oracle, problems, monkeypatch, case):
    """every solver path on orbit_600, lambda ladder 1e3 / 10 / 0.1: the kernel, blocks read from the global copy, x against a dense
    Cholesky of the oracle's reduced system (xl against the oracle's back-substitution), and for two-level k_pcg5<BIG> the
    iteration count against restated_pcg5 fed the engine's own coarse inverse"""
    variant, env, want = PATHS[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    name = "orbit_600"
    prob = problems(name)
    plan = pkg.pcg5_plan_host(prob, 1, H100_SMS, 148)
    ladder = _oracle_ladder(oracle, prob, name)
    Z = coarse_basis(prob, prob.numP)
    eng = make_engine(pkg, prob, KERNELS["huber"], pcg_variant=variant)
    eng.linearize()
    for lam, tol in LADDER:
        S, b, xp_o, xl_o, _ = ladder[lam]
        assert relerr(_direct(S, b), xp_o.reshape(-1)) < 0.1 * tol             # the two direct solves agree well inside the tolerance
        iters, ok = eng.solve(lam)
        info = _check_solve(eng, prob, case, lam, tol, S, b, xl_o, plan, iters, ok, Z)
        if want is None:
            assert (info["kernel"], info["two_level"]) in (("k_pcg3", False), ("k_pcg5_big", True)), info
        else:
            assert (info["kernel"], info["two_level"]) == want, info
    eng.close()


@pytest.mark.gpu
def test_covis_1000_automatic_policy(pkg, problems):
    """covis_1000 (k_pcg5 plan with needMax 970) under the automatic policy and with k_pcg5 asked for: with its staging sized for
    970 columns of w, k_pcg5's fp64 layout no longer fits in shared memory, so every solve is block-Jacobi k_pcg3 (with the old
    512-column staging k_pcg5 ran and overran it).  x against a dense Cholesky of the engine's own reduced system (whose Schur
    complement test_dense_stages_match_oracle checks on the other dense graphs)"""
    name = "covis_1000"
    prob = problems(name)
    plan = pkg.pcg5_plan_host(prob, 1, H100_SMS, 148)
    Z = coarse_basis(prob, prob.numP)
    for variant in (0, 5, 6):
        eng = make_engine(pkg, prob, KERNELS["huber"], pcg_variant=variant)
        eng.linearize()
        rp, ci = eng.hsc_structure()
        for lam, tol in LADDER:
            iters, ok = eng.solve(lam)
            Hsc, bsc, _ = eng.schur()
            S = _full_system(Hsc, rp, ci, prob.numP)
            xl_ref = eng.delta()[1].copy()
            info = _check_solve(eng, prob, "c1000-%d" % variant, lam, tol, S, bsc.reshape(-1), xl_ref, plan, iters, ok, Z)
            assert (info["kernel"], info["two_level"]) == ("k_pcg3", False), info
        eng.close()


# ---- GPU: trajectories ---------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name,iters", [("local_ba", 10), ("orbit_600", 3)])
def test_dense_optimize_matches_oracle(pkg, oracle, problems, name, iters):
    """optimize() against the oracle (orbit_600: 3 iterations, its direct solve of the dense 3 594 x 3 594 system takes seconds)"""
    from test_gpu_parity import _no_hidden_coarse_failure, _trajectory_check
    prob = problems(name); rk = KERNELS["huber"]
    eng = make_engine(pkg, prob, rk)
    stats = eng.optimize(iters)
    o = oracle.Oracle(prob, *rk)
    chi, lam, tr = o.optimize(iters)
    _trajectory_check(stats, chi, lam, tr)
    _no_hidden_coarse_failure(eng)
    for nme, a, b in zip(("q", "t", "Xw"), eng.state(), o.state()):
        assert relerr(a, b) < TOL, (name, nme)
    print("%s optimize(%d): chi2 %s, last solve %s" % (name, iters, [round(s["chi2"], 3) for s in stats], eng.pcg_info()["kernel"]))
    eng.close()


# ---- GPU: covis_2000 is beyond k_pcg3 ------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_need_lists_beyond_shared_memory_are_an_error(pkg, oracle, problems):
    """covis_2000: a CTA of k_pcg3 would need 1 996 columns in shared memory.  initialize() raises CubaError naming the need list
    and the limit, and the same engine then optimises `small` as a fresh one does"""
    eng = make_engine(pkg, problems("small"), KERNELS["huber"])
    with pytest.raises(pkg.CubaError, match=r"needs 1996 columns of the reduced camera system.*available: at most \d+ columns"):
        eng.initialize(problems("covis_2000"))
    eng.initialize(problems("small"))
    stats = eng.optimize(10)
    fresh = make_engine(pkg, problems("small"), KERNELS["huber"])
    ref = fresh.optimize(10)
    assert [s["chi2"] for s in stats] == [s["chi2"] for s in ref]
    for a, b in zip(eng.state(), fresh.state()):
        assert np.array_equal(a, b)
    eng.close(); fresh.close()


# ---- GPU: fp32 engine ----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("variant", [5, 6])
def test_fp32_dense_pcg5(pkg, problems, variant):
    """k_pcg5<float, BIG> shares the layout: on orbit_600 its true residual in the block-Jacobi norm (test_fp32_stages.check_pcg)"""
    from test_fp32_stages import check_pcg
    prob = problems("orbit_600")
    eng = make_engine(pkg, prob, KERNELS["huber"], use_fp32=True, pcg_variant=variant)
    eng.linearize()
    for lam in (1e3, 10.0, 0.1):
        lam32 = float(np.float32(lam))
        iters, ok = eng.solve(lam32)
        Hsc, bsc, _ = eng.schur()
        info, _ = check_pcg(eng, Hsc, bsc, "orbit_600 fp32 pcg %d lambda %g" % (variant, lam), ok)
        print("orbit_600 fp32 pcg_variant %d lambda %g: %s two-level %s status %d, %d iterations" % (variant, lam, info["kernel"], info["two_level"], info["status"], iters))
        assert info["kernel"].startswith("k_pcg5") and info["two_level"] == (variant == 5), info
    eng.close()
