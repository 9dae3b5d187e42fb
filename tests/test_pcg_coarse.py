"""The two-level preconditioner of k_pcg5 / k_pcg5t (csrc/cuba_pcg5.cuh), checked on every path the engine can pick.

CG reaches the same solution with any SPD preconditioner, so comparing x with the oracle cannot see a broken coarse level: it
only costs iterations.  These tests look at the preconditioner itself.  `restated_pcg5` is a numpy restatement of the kernel's
mathematics:
  * hat space A^ = L^-1 S L^-T with L the Cholesky factor of every diagonal block;
  * M^-1 = I + Z^ Ac^-1 Z^^T with Z^_i = L_i^T Z_i, as k_pcg5_prep_rows builds it, and Z_i = Ad(T_i) (k_coarse_basis);
  * Chronopoulos-Gear single-reduction CG, the coarse residual advanced by the same recurrences;
  * stop when r^.r^ <= tol^2 r0^.r0^.
On the GPU, every path of the table in DESIGN.md 6 runs the solve ladder of test_all_pcg_kernels_solve_the_same_system, and each
solve checks the kernel it ran, the coarse matrix against Z^T S Z from the oracle's Schur complement, the fp32 coarse inverse
against fp64, the solution against the direct solve and the iteration count against the restatement fed the engine's own
inverse."""
import time

import numpy as np
import pytest

from conftest import KERNELS, make_engine, relerr
from test_two_level_prototype import _adjoints, _pcg, _system

sp = pytest.importorskip("scipy.sparse")

PCG_TOL = 1e-11
LADDER = ((1e3, 1e-10), (10.0, 1e-9), (0.1, 1e-7))      # (lambda, tolerance of x against the direct solve)
INV_RESIDUAL_FACTOR = 1.5                                # |AcInv Ac - I| over that of the fp64 inverse rounded to fp32 (measured <= 1.0)


# ---- the CPU restatement ------------------------------------------------------------------------------------------------

def coarse_basis(prob, P):
    """Z_i = Ad(T_i) = [[R, 0], [[t]x R, R]] of every free pose, [P][6][6] (row, column) -- k_coarse_basis"""
    return np.stack(_adjoints(prob, P))


def coarse_operator(agg, Z, A):
    """Z as a sparse [6P][6A] matrix: rows of pose i, columns of its aggregate"""
    P = len(agg)
    rr, cc = np.meshgrid(np.arange(6), np.arange(6), indexing="ij")
    I = (6 * np.arange(P)[:, None, None] + rr).ravel()
    J = (6 * agg[:, None, None] + cc).ravel()
    return sp.csr_matrix((Z.reshape(-1), (I, J)), shape=(6 * P, 6 * A))


def coarse_matrix(S, agg, Z, A):
    Zs = coarse_operator(agg, Z, A)
    return (Zs.T @ S @ Zs).toarray()


def packed_to_dense(AcP, A):
    """AcP: lower block triangle, block (ib >= jb) at ib (ib+1)/2 + jb, each column-major 6x6 -> symmetric [6A][6A]"""
    M = np.zeros((6 * A, 6 * A))
    b = 0
    for ib in range(A):
        for jb in range(ib + 1):
            blk = AcP[b].reshape(6, 6).T                # column-major -> [r][c]
            M[6 * ib:6 * ib + 6, 6 * jb:6 * jb + 6] = blk
            M[6 * jb:6 * jb + 6, 6 * ib:6 * ib + 6] = blk.T
            b += 1
    return M


def restated_pcg5(S, b, agg, Z, AcInv, tol=PCG_TOL, maxit=20000):
    """k_pcg5's solve in fp64 on the CPU: returns (x, iterations).  agg[i] is the aggregate of pose i, Z[i] = Z_i (6x6),
    AcInv the coarse inverse the kernel applies (any precision; None: block-Jacobi)."""
    P = len(b) // 6
    S = sp.csr_matrix(S)
    D = np.stack([S[6 * i:6 * i + 6, 6 * i:6 * i + 6].toarray() for i in range(P)])
    L = np.linalg.cholesky(D)                                    # lower, per block
    Li = np.linalg.inv(L)
    Lis = sp.block_diag(list(Li), format="csr")
    Ah = (Lis @ S @ Lis.T).tocsr()
    x_hat_to_x = Lis.T                                           # x = L^-T y
    r = Lis @ b
    coarse = AcInv is not None
    if coarse:
        A = AcInv.shape[0] // 6
        Zh = np.einsum("ikr,ikq->irq", L, Z)                     # Z^_i(r, q) = sum_{k >= r} L_i(k, r) Z_i(k, q)
        Zhs = coarse_operator(agg, Zh, A)
        Ci = np.asarray(AcInv, dtype=np.float64)
        rc = Zhs.T @ r
    u = r + Zhs @ (Ci @ rc) if coarse else r.copy()
    w = Ah @ u
    gamma, delta, rho0 = r @ u, w @ u, r @ r
    if rho0 <= 0:
        return np.zeros_like(b), 0
    alpha, beta = gamma / delta, 0.0
    s = np.zeros_like(b); p = np.zeros_like(b); y = np.zeros_like(b)
    if coarse:
        sc = np.zeros(6 * A)
    it = 0
    for k in range(maxit + 1):
        if k >= 1:
            it = k
            if rnew <= tol * tol * rho0:
                break
            beta = gnew / gamma
            ga = gamma * alpha
            alpha = gnew * ga / (delta * ga - gnew * gnew)
            gamma = gnew
        s = w + beta * s
        r = r - alpha * s
        p = u + beta * p
        y = y + alpha * p
        if coarse:
            sc = Zhs.T @ w + beta * sc
            rc = rc - alpha * sc
            u = r + Zhs @ (Ci @ rc)
        else:
            u = r
        w = Ah @ u
        gnew, delta, rnew = r @ u, w @ u, r @ r
    return x_hat_to_x @ y, it


def contiguous_aggregates(P, m):
    return np.arange(P) // m


def count_bound(n):
    """how far the kernel's iteration count may lie from the restatement's (see test_pcg5_coarse_level_on_every_path)"""
    return max(3, int(np.ceil(0.03 * n)))


# ---- CPU: the yardstick ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def kitti07_system(pkg, oracle, problems):
    prob = problems("kitti07_shaped")
    P = prob.numP
    o = oracle.Oracle(prob, *KERNELS["huber"])
    o.compute_errors(); o.build_system()
    out = {}
    for lam, _ in LADDER:
        out[lam] = _system(o, P, lam)
    return prob, out


def test_restatement_matches_the_prototype_pcg(kitti07_system):
    """with an exact fp64 coarse inverse the restatement and the prototype's textbook PCG (same preconditioner D^-1 + Z Ac^-1 Z^T,
    stopping on r.z instead of r^.r^) agree on x and, to one iteration, on the count"""
    prob, systems = kitti07_system
    P = prob.numP
    agg = contiguous_aggregates(P, 8)
    A = int(agg.max()) + 1
    Z = coarse_basis(prob, P)
    Zs = coarse_operator(agg, Z, A)
    for lam, _ in LADDER:
        S, b = systems[lam]
        Aci = np.linalg.inv(coarse_matrix(S, agg, Z, A))
        x, it = restated_pcg5(S, b, agg, Z, Aci)
        Dinv = sp.block_diag([np.linalg.inv(S[6 * i:6 * i + 6, 6 * i:6 * i + 6].toarray()) for i in range(P)], format="csr")
        x0, it0 = _pcg(S, b, lambda r: Dinv @ r + Zs @ (Aci @ (Zs.T @ r)))
        print("restatement lambda %g: %d iterations, prototype %d, |dx| %.1e" % (lam, it, it0, relerr(x, x0)))
        assert abs(it - it0) <= 1, (lam, it, it0)
        assert relerr(x, x0) < 1e-9, lam
        # and it solves the system
        assert np.abs(S @ x - b).max() <= 1e-8 * np.abs(b).max()


def test_restatement_sees_a_broken_coarse_level(kitti07_system):
    """negative control for the iteration-count check on the GPU: a coarse level that is only partly right moves the count
    further than count_bound allows, though x stays right"""
    prob, systems = kitti07_system
    P = prob.numP
    agg = contiguous_aggregates(P, 8)
    A = int(agg.max()) + 1
    Z = coarse_basis(prob, P)
    S, b = systems[0.1]
    Aci = np.linalg.inv(coarse_matrix(S, agg, Z, A))
    x, it = restated_pcg5(S, b, agg, Z, Aci)
    # (1) the rows and columns of one aggregate of Ac^-1 zeroed (still positive semi-definite: a valid, weaker preconditioner)
    bad = Aci.copy()
    a0 = A // 2
    bad[6 * a0:6 * a0 + 6, :] = 0; bad[:, 6 * a0:6 * a0 + 6] = 0
    x1, it1 = restated_pcg5(S, b, agg, Z, bad)
    # (2) Z built from the wrong pose (each aggregate uses its first pose's Ad(T) for all its rows)
    Zw = Z[agg * 8]
    Aciw = np.linalg.inv(coarse_matrix(S, agg, Zw, A))
    x2, it2 = restated_pcg5(S, b, agg, Zw, Aciw)
    print("negative control: %d iterations; one aggregate zeroed %d; Z from the wrong pose %d" % (it, it1, it2))
    for got, xg in ((it1, x1), (it2, x2)):
        assert abs(got - it) > count_bound(it), (it, got)
        assert relerr(xg, x) < 1e-7


# ---- GPU: every path of the coarse level -------------------------------------------------------------------------------

def _full_system(Hsc, rp, ci, P):
    """symmetric CSR of the reduced system from its upper blocks (column-major), as test_two_level_prototype._system"""
    B = Hsc.reshape(-1, 6, 6).transpose(0, 2, 1)
    rows = np.repeat(np.arange(P), np.diff(rp))
    rr, cc = np.meshgrid(np.arange(6), np.arange(6), indexing="ij")
    I = (6 * rows[:, None, None] + rr).ravel(); J = (6 * ci[:, None, None] + cc).ravel(); V = B.ravel()
    off = np.repeat(rows != ci, 36)
    return sp.csr_matrix((np.concatenate([V, V[off]]), (np.concatenate([I, J[off]]), np.concatenate([J, I[off]]))), shape=(6 * P, 6 * P))


_ORACLE = {}


def _oracle_ladder(oracle, prob, name):
    """per lambda of LADDER: the oracle's reduced system (S, b) and its direct solution (xp, xl), Huber kernels"""
    if name not in _ORACLE:
        o = oracle.Oracle(prob, *KERNELS["huber"])
        o.compute_errors(); o.build_system()
        out = {}
        for lam, _ in LADDER:
            t0 = time.time()
            S, b = _system(o, prob.numP, lam)
            xp, xl = (v.copy() for v in o.delta())
            out[lam] = (S, b, xp, xl, time.time() - t0)
        _ORACLE.clear()                                      # one graph at a time: rows_11k's system alone is ~250 MB
        _ORACLE[name] = out
    return _ORACLE[name]


# The plan sizes follow from the 132 SMs of an H100; `plan` holds what that GPU gives.  Each case checks it, so that a case that
# drifts to another path fails instead of testing something else.  nc = 6A is a multiple of 16 (k_coarse_dense's tile) in
# k00_two_per_cta (1584) and not in k00_gs2 (396), k00_dense / k00_legacy / r11k_* (792, padded) or k07_three_per_cta (558).
PATH_CASES = {
    # id: (graph, Engine kwargs, environment, kernel, coarse kernel, plan)
    "k07_invert": ("kitti07_shaped", {}, {}, "k_pcg5t", "k_coarse_invert", dict(aggs_per_cta=1, G=31, gs=1, A=31)),
    "k00_span_ctas": ("kitti00_shaped", dict(max_aggregates=37), {}, "k_pcg5t", "k_coarse_invert", dict(aggs_per_cta=1, G=132, gs=4, A=33)),
    "k00_dense": ("kitti00_shaped", {}, {}, "k_pcg5t", "k_coarse_dense", dict(aggs_per_cta=1, G=132, gs=1, A=132)),
    "k00_gs2": ("kitti00_shaped", dict(max_aggregates=66), {}, "k_pcg5t", "k_coarse_dense", dict(aggs_per_cta=1, G=132, gs=2, A=66)),
    "k00_two_per_cta": ("kitti00_shaped", {}, {"CUBA_PCG5_AGGS_PER_CTA": "2"}, "k_pcg5t", "k_coarse_dense", dict(aggs_per_cta=2, G=132, gs=1, A=264)),
    "k07_three_per_cta": ("kitti07_shaped", {}, {"CUBA_PCG5_AGGS_PER_CTA": "3"}, "k_pcg5t", "k_coarse_dense", dict(aggs_per_cta=3, G=31, gs=1, A=93)),
    "k00_legacy": ("kitti00_shaped", {}, {"CUBA_PCG5_LEGACY": "1"}, "k_pcg5", "k_coarse_dense", dict(G=132, gs=1, A=132)),
    "r11k_row_capped": ("rows_11k", {}, {}, "k_pcg5_big", "k_coarse_dense", dict(aggs_per_cta=1, G=132, gs=1, A=132, maxRows=85)),
    "r11k_big": ("rows_11k", {}, {"CUBA_PCG5_LEGACY": "1"}, "k_pcg5_big", "k_coarse_dense", dict(G=132, gs=1, A=132, maxRows=85)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(PATH_CASES))
def test_pcg5_coarse_level_on_every_path(pkg, oracle, problems, monkeypatch, case):
    """a. the kernel and the coarse-inverse kernel the case names ran;  b. Ac = Z^T S Z;  c. the fp32 inverse against fp64;
    d. x against the direct solve, no breakdown;  e. the iteration count against restated_pcg5 fed the engine's own inverse.

    Measured on one H100 80GB HBM3 (700 W limit), all nine cases x three dampings:
      b. Ac against Z^T S Z from the engine's own Schur complement <= 1.4e-14, from the oracle's <= 3.1e-12 (rows_11k, lambda 0.1);
      c. Ac^-1 against the fp64 inverse <= 5.2e-8 of its largest entry.  |AcInv Ac - I|_max reaches 7.3 on kitti00_shaped and
         about 1e3 on rows_11k at lambda 0.1: Ac is that ill-conditioned (about 1e11 on kitti00_shaped; the rigid-motion basis
         carries translations of kilometres), and the same residual follows from rounding the fp64 inverse once to fp32.  The
         check is therefore against that floor: measured 0.90 .. 1.00 times it, bound INV_RESIDUAL_FACTOR;
      d. the solution is as close to the direct solve as the restatement's (within a few per cent everywhere);
      e. the kernel's iteration count is within one of the restatement's in all 27 solves (18 .. 589 iterations).  count_bound
         allows max(3, 3 %); the broken coarse levels of test_restatement_sees_a_broken_coarse_level move the count by 9 and 112.
    The nine cases take about 80 s, most of it the CPU restatement on rows_11k (590 iterations on 10.7 M non-zeros).
    """
    name, kw, env, want_kernel, want_coarse, want_plan = PATH_CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    t_case = time.time()
    prob = problems(name)
    P = prob.numP
    ladder = _oracle_ladder(oracle, prob, name)
    Z = coarse_basis(prob, P)
    eng = make_engine(pkg, prob, KERNELS["huber"], pcg_variant=5, **kw)
    eng.linearize()
    rp, ci = eng.hsc_structure()
    own = {}                                                 # the engine's own reduced system per lambda (for check b)
    for lam, tol in LADDER:
        iters, ok = eng.solve(lam)
        info = eng.pcg_info()
        own[lam] = _full_system(eng.schur()[0], rp, ci, P)
        # a. path
        assert info["kernel"] == want_kernel and info["two_level"] and info["coarse_kernel"] == want_coarse, (case, info)
        for k, v in want_plan.items():
            assert info[k] == v, (case, k, info)
        A = info["A"]; nc = 6 * A
        agg, AcP, AcInv = eng.coarse()
        assert agg.min() == 0 and agg.max() == A - 1 and np.all(np.diff(agg) >= 0)
        # b. coarse matrix, rebuilt on the CPU at the damping it was assembled at
        lc = info["coarse_lambda"]
        assert lc in own, (case, lc)
        Ac = packed_to_dense(AcP, A)
        d_own = relerr(Ac, coarse_matrix(own[lc], agg, Z, A))
        d_orc = relerr(Ac, coarse_matrix(ladder[lc][0], agg, Z, A))
        assert d_own < 1e-12, (case, lam, d_own)
        assert d_orc < 1e-10, (case, lam, d_orc)
        # c. coarse inverse
        assert info["cinfo"] == 0 and info["bad_rebuilds"] == 0, (case, info)
        inv64 = np.linalg.inv(Ac)
        d_inv = np.abs(AcInv - inv64).max() / np.abs(inv64).max()
        eye = np.eye(nc)
        resid = np.abs(AcInv.astype(np.float64) @ Ac - eye).max()
        floor = np.abs(inv64.astype(np.float32).astype(np.float64) @ Ac - eye).max()     # the fp64 inverse rounded once to fp32
        assert d_inv < 2e-6, (case, lam, d_inv)
        assert resid <= INV_RESIDUAL_FACTOR * floor, (case, lam, resid, floor)
        # d. solution: against the direct solve, to the ladder's tolerance or -- where the stopping rule itself leaves more than that
        #    (kitti00_shaped at lambda 1e3: 1.1e-10 in exact arithmetic) -- to what the restatement reaches
        assert ok and info["status"] == 0 and info["iters"] == iters and info["bj_retries"] == 0, (case, info)
        S, b, xp, xl, _ = ladder[lam]
        x_r, it_r = restated_pcg5(S, b.reshape(-1), agg, Z, AcInv)
        d_r = relerr(x_r.reshape(-1, 6), xp)
        assert d_r < 10 * tol, (case, lam, d_r)
        dx = [relerr(a, ref) for a, ref in zip(eng.delta(), (xp, xl))]
        for nme, d in zip(("xp", "xl"), dx):
            assert d < max(tol, 3 * d_r), (case, nme, lam, iters, d, d_r)
        # e. iteration count against the restatement fed the engine's own inverse
        print("pcg5 path %-18s lambda %-6g %-10s %-15s A %3d nc %4d gs %d K %d maxRows %2d capBlocks %4d zh %d | Ac %.1e/%.1e inv %.1e "
              "|AcInv Ac - I| %.1e (fp32 floor %.1e) | x %.1e (restated %.1e) | iterations %d restated %d (%+d)"
              % (case, lam, info["kernel"], info["coarse_kernel"], A, nc, info["gs"], info["aggs_per_cta"], info["maxRows"], info["capBlocks"],
                 info["zhInSmem"], d_own, d_orc, d_inv, resid, floor, dx[0], d_r, iters, it_r, iters - it_r))
        assert abs(iters - it_r) <= count_bound(it_r), (case, lam, iters, it_r)
    assert eng.pcg_info()["coarse_rebuilds"] == 2            # 1e3, then reused at 10 (100x), rebuilt at 0.1 (1e4x)
    eng.close()
    print("pcg5 path %s: %.1f s" % (case, time.time() - t_case))



def test_rows_11k_plan_is_row_capped(pkg, problems):
    """rows_11k (10 999 free poses) keeps cases r11k_* on the row-capped plan: balanced by blocks alone a CTA would own more
    than 85 rows (2 x 256 threads / 6 components, the most the row sums take), so the rows are balanced again under that cap.  85
    rows are more than the 42 of the legacy shape's one (row, component) pair per thread: that shape must be BIG."""
    prob = problems("rows_11k")
    assert prob.numP == 10999 and prob.numP <= 85 * 132            # more poses than that and no plan exists on 132 SMs
    by_blocks = pkg.pcg_partition_host(prob, 132, 148)
    plan = pkg.pcg5_plan_host(prob, 1, 132, 148)
    assert by_blocks["G"] == 132 and by_blocks["maxRows"] > 85, by_blocks
    assert plan["ok"] and plan["G"] == 132 and plan["gs"] == 1 and plan["A"] == 132, plan
    assert plan["maxRows"] == 85 and plan["maxRows"] * 6 > 256, plan
