"""The fp32 engine (use_fp32=True, the reference's USE_FLOAT32 build) stage by stage, and the two fp32-operand kernels of the mixed
engine (use_fp32="mixed"), each against an fp64 restatement fed the same stage's inputs as read back from the engine.

A whole-trajectory comparison cannot see a slightly wrong Hessian, Schur block or solve: LM still converges.  So each stage here is
checked on its own, with a forward-error bound |engine - ref| <= K u M: u = 2^-24, M the elementwise sum of the magnitudes of the
terms the stage adds (so cancellation cannot hide an error), K derived next to each use (at most the gamma_n of the longest sum).
Downstream of J+H the bounds sit far below one product's contribution, so a dropped, doubled, mis-indexed or transposed term fails
by far; the J+H bound (gamma_n over a pose's edges, with the residual's and the robust weight's sensitivities) is looser, and prints
how it compares with one edge's term.  Every check prints its largest measured/bound ratio."""
import numpy as np
import pytest

from conftest import KERNELS, have_fixture, make_engine
from test_host_math import jacobian_magnitude, quat_rot, se3_exact
from test_pcg_coarse import coarse_basis, coarse_matrix, packed_to_dense
from test_two_level_prototype import _system

sp = pytest.importorskip("scipy.sparse")
spla = pytest.importorskip("scipy.sparse.linalg")

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F32 = lambda a: np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def report(label, err, bound):
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    ratio = float(np.max(err / np.maximum(bound, 1e-300))) if err.size else 0.0
    print("%-58s max measured/bound %.3g" % (label, ratio))
    return ratio


def rounded(prob):
    """the problem with every number rounded to fp32 (the synthetic graphs already are; the reference's fixtures are not)"""
    p = prob.copy()
    for f in ("q", "t", "cam", "Xw", "meas2", "omega2", "meas3", "omega3"):
        setattr(p, f, F32(getattr(p, f)))
    return p


def problem(problems, pkg, name):
    if name.startswith("ba_") and not have_fixture(name):
        pytest.skip("reference fixture absent")
    if name == "near_origin":
        # small, with the world shifted so that free pose 5 sits at the origin: its translation, and the step's, are then the whole pose
        p = problems("small").copy()
        R = quat_rot(p.q[5:6])[0]
        C = -R.T @ p.t[5]
        p.Xw = F32(p.Xw - C)
        p.t = F32(p.t + np.einsum("nij,j->ni", quat_rot(p.q), C))
        # and free poses 3 .. 8, within a few metres of it, moved (centres scaled by 1e-4) to within a millimetre of the origin
        p.t[3:9] = F32(p.t[3:9] * 1e-4)
        assert (np.linalg.norm(p.t[:p.numP], axis=1) < 1e-3).sum() >= 5
        return p
    return rounded(problems(name))


# ---- per-edge quantities in fp64 ---------------------------------------------------------------------------------------------

class Edges:
    """the edges in the engine's order (mono then stereo) at a state, with their fp64 residuals, weights and the magnitudes of the
    fp32 engine's residual and Jacobians (the M of test_host_math: u M bounds the fp32 error of each entry, before K)"""

    def __init__(self, prob, rk, q, t, Xw):
        E2, E3 = prob.E2, prob.E3
        idx = np.concatenate([prob.idx2.reshape(-1, 2), prob.idx3.reshape(-1, 2)]).astype(np.int64)
        self.iP, self.iL = idx[:, 0], idx[:, 1]
        self.st = np.concatenate([np.zeros(E2, bool), np.ones(E3, bool)])
        m = np.zeros((E2 + E3, 3)); m[:E2, :2] = prob.meas2.reshape(-1, 2); m[E2:] = prob.meas3.reshape(-1, 3)
        self.om = np.concatenate([prob.omega2.reshape(-1), prob.omega3.reshape(-1)])
        qe, te, cam, X = q[self.iP], t[self.iP], prob.cam[self.iP], Xw[self.iL]
        R = quat_rot(qe)
        Xc = np.einsum("nij,nj->ni", R, X) + te
        iz = 1 / Xc[:, 2]
        uu = cam[:, 0] * Xc[:, 0] * iz + cam[:, 2]; vv = cam[:, 1] * Xc[:, 1] * iz + cam[:, 3]
        r = np.stack([uu - m[:, 0], vv - m[:, 1], np.where(self.st, uu - cam[:, 4] * iz - m[:, 2], 0)], axis=1)
        MX = (np.abs(R) @ np.abs(X)[..., None])[..., 0] + np.abs(te)
        xn, yn = np.abs(Xc[:, 0] * iz), np.abs(Xc[:, 1] * iz)
        c = MX.max(1) * np.abs(iz) * (1 + xn + yn)
        f = cam[:, :2].max(1)
        self.Mr = np.abs(np.stack([uu, vv, uu], 1)) + np.abs(m) + (f * (1 + c) + cam[:, 4] * np.abs(iz))[:, None]
        self.Mr[~self.st, 2] = 0
        self.r = r
        MP, ML = jacobian_magnitude(qe, cam, Xc, self.st)
        G = (f * (1 + 2 * xn + 2 * yn) + 3 * cam[:, 4] * np.abs(iz)) * c
        self.MP = MP * (1 + c)[:, None, None] + G[:, None, None]             # |J| plus its fp32 error / u, up to K
        self.ML = ML * (1 + c)[:, None, None] + (f * np.abs(iz) * c)[:, None, None]
        self.MP[~self.st, 2] = 0; self.ML[~self.st, 2] = 0
        # weights w = omega rho'(omega |r|^2) and dw, the change of w per unit of u in the fp32 residual
        s = (r * r).sum(1); e = self.om * s
        kind = np.where(self.st, rk[0][1], rk[0][0]); delta = np.where(self.st, rk[1][1], rk[1][0]); d2 = delta * delta
        drho = np.ones_like(e); dd = np.zeros_like(e)
        hub = (kind == 1) & (e > d2)
        drho[hub] = delta[hub] / np.sqrt(e[hub]); dd[hub] = delta[hub] / (2 * e[hub] ** 1.5)
        tk = kind == 2
        uq = np.where(tk & (e <= d2), 1 - e / np.where(tk, d2, 1), 0)
        drho[tk] = uq[tk] ** 2; dd[tk] = 2 * uq[tk] / d2[tk]
        de = self.om * 2 * (np.abs(r) * self.Mr).sum(1)                      # |d e| / u
        self.w = self.om * drho
        self.dw = self.om * dd * de
        self.e = e


def block_sums(keys, vals, n):
    out = np.zeros((n,) + vals.shape[1:])
    ok = keys >= 0
    np.add.at(out, keys[ok], vals[ok])
    return out


def count(keys, n):
    return np.bincount(keys[keys >= 0], minlength=n) if n else np.zeros(0, int)


# ---- J+H -----------------------------------------------------------------------------------------------------------------

def check_linearize(eng, o, prob, rk, label):
    chi = eng.linearize()
    ochi = o.compute_errors(); o.build_system()
    sysE, sysO = eng.system(), o.system()
    ed = Edges(prob, rk, prob.q, prob.t, prob.Xw)
    numP, numL = prob.numP, prob.numL
    kp = np.where(ed.iP < numP, ed.iP, -1); kl = np.where(ed.iL < numL, ed.iL, -1)
    _, _, e2h = eng.hpl_structure()
    # one edge's term of H is w J^T J: its fp32 error is K1 u (w MJ^T MJ + dw |J|^T |J|) with K1 = 8 (the residual, J and w errors
    # are in MJ, Mr, dw; the 3-term dot product and the product with w round a few more times); the sums over a block's edges add
    # gamma_n with n the block's edge count
    K1 = 8
    wv = K1 * (ed.w + ed.dw)
    P6 = ed.MP; L3 = ed.ML
    tP = np.einsum("e,eki,ekj->eij", wv, P6, P6); tL = np.einsum("e,eki,ekj->eij", wv, L3, L3)
    tPL = np.einsum("e,ekn,ekl->enl", wv, L3, P6)              # Hpl block [n][l] (landmark column n, pose row l)
    tbp = np.einsum("e,eki,ek->ei", wv, P6, ed.Mr + np.abs(ed.r)); tbl = np.einsum("e,eki,ek->ei", wv, L3, ed.Mr + np.abs(ed.r))
    nP, nL, nH = count(kp, numP), count(kl, numL), count(np.where((kp >= 0) & (kl >= 0), e2h, -1), eng.sizes["nhpl"])
    gam = lambda n: (1 + n)[:, None, None]
    bounds = {"Hpp": (block_sums(kp, tP, numP) * gam(nP)).reshape(numP, 36),
              "bp": block_sums(kp, tbp, numP) * (1 + nP)[:, None],
              "Hll": (block_sums(kl, tL, numL) * gam(nL)).reshape(numL, 9),
              "bl": block_sums(kl, tbl, numL) * (1 + nL)[:, None],
              "Hpl": (block_sums(np.where((kp >= 0) & (kl >= 0), e2h, -1), tPL, eng.sizes["nhpl"]) * gam(nH)).reshape(-1, 18)}
    for nme, a, b in zip(("Hpp", "bp", "Hll", "bl", "Hpl"), sysE, sysO):
        assert report("%s %s" % (label, nme), np.abs(a - b), U * bounds[nme]) <= 1, nme
    # single edges: the bound must be far below one edge's own term (else a dropped edge could pass)
    one = np.abs(np.einsum("e,eki,ekj->eij", ed.w, ed.MP, ed.MP))[:, range(6), range(6)].max(1)
    print("%s: median Hpp diagonal bound / one edge's own term %.3g" % (
        label, np.median(U * bounds["Hpp"].reshape(numP, 6, 6)[kp[kp >= 0]][:, range(6), range(6)].max(1) / one[kp >= 0])))
    rho_b = (K1 * U * (ed.w * 2 * (np.abs(ed.r) * ed.Mr).sum(1) + ed.e)).sum() + U * len(ed.e) * ochi
    assert report("%s chi2" % label, abs(chi - ochi), rho_b) <= 1
    return sysE


def check_chi_sqs(eng, o, prob, rk, label):
    q, t, Xw = eng.state()
    o.set_state(q, t, Xw)
    ed = Edges(prob, rk, q, t, Xw)
    got, ref = eng.chi_squared(), o.chi_sqs()
    b = 8 * U * ed.om * ((np.abs(ed.r) * ed.Mr).sum(1) * 2 + (ed.r * ed.r).sum(1))
    assert report("%s chi_squared" % label, np.abs(got - ref), b) <= 1


# ---- Schur, back-substitution --------------------------------------------------------------------------------------------

def schur_restated(eng, sysE, invHll, lam):
    """Hsc (upper blocks, column-major) and bsc from the engine's own Hpp, bp, Hpl, bl and invHll, in fp64, with the magnitudes
    sum |terms| of each entry and the number of products per block"""
    Hpp, bp, Hll, bl, Hpl = sysE
    numP, numL = Hpp.shape[0], Hll.shape[0]
    colPtr, rowInd, _ = eng.hpl_structure()
    rp, ci = eng.hsc_structure()
    A = Hpl.reshape(-1, 3, 6).transpose(0, 2, 1)               # [blk][l(6)][n(3)]
    inv = invHll.reshape(-1, 3, 3).transpose(0, 2, 1)
    lmOf = np.repeat(np.arange(numL), np.diff(colPtr))
    W = np.einsum("kln,knm->klm", A, inv[lmOf]); Wa = np.einsum("kln,knm->klm", np.abs(A), np.abs(inv[lmOf]))
    # pairs (i, j) of Hpl blocks of one landmark with row_i <= row_j
    cnt = np.diff(colPtr)
    starts = colPtr[:-1]
    pi, pj = [], []
    for a in range(int(cnt.max(initial=0))):
        for b in range(a, int(cnt.max(initial=0))):
            m = cnt > b
            pi.append(starts[m] + a); pj.append(starts[m] + b)
    pi = np.concatenate(pi) if pi else np.zeros(0, int); pj = np.concatenate(pj) if pj else np.zeros(0, int)
    ri, rj = rowInd[pi], rowInd[pj]
    sw = ri > rj
    pi[sw], pj[sw] = pj[sw].copy(), pi[sw].copy()
    ri, rj = rowInd[pi], rowInd[pj]
    rows = np.repeat(np.arange(numP), np.diff(rp))
    key = rows.astype(np.int64) * numP + ci
    kb = np.searchsorted(key, ri.astype(np.int64) * numP + rj)
    assert np.array_equal(key[kb], ri.astype(np.int64) * numP + rj)
    prod = np.einsum("klm,kcm->klc", W[pi], A[pj])             # W_i Hpl_j^T  [6][6]
    proda = np.einsum("klm,kcm->klc", Wa[pi], np.abs(A[pj]))
    nb = len(ci)
    Hsc = np.zeros((nb, 6, 6)); Mag = np.zeros((nb, 6, 6))
    np.add.at(Hsc, kb, -prod); np.add.at(Mag, kb, proda)
    diag = rp[:-1]
    Hsc[diag] += Hpp.reshape(-1, 6, 6).transpose(0, 2, 1) + lam * np.eye(6)
    Mag[diag] += np.abs(Hpp.reshape(-1, 6, 6)) + lam * np.eye(6)
    nprod = np.bincount(kb, minlength=nb)
    bsc = bp.copy(); bM = np.abs(bp).copy()
    np.add.at(bsc, rowInd, -np.einsum("klm,km->kl", W, bl[lmOf])); np.add.at(bM, rowInd, np.einsum("klm,km->kl", Wa, np.abs(bl[lmOf])))
    nb_p = np.bincount(rowInd, minlength=numP)
    return (Hsc.transpose(0, 2, 1).reshape(nb, 36), bsc, Mag.transpose(0, 2, 1).reshape(nb, 36), bM, nprod, nb_p)


def backsub_restated(eng, sysE, invHll, xp):
    Hpp, bp, Hll, bl, Hpl = sysE
    numL = Hll.shape[0]
    colPtr, rowInd, _ = eng.hpl_structure()
    lmOf = np.repeat(np.arange(numL), np.diff(colPtr))
    A = Hpl.reshape(-1, 3, 6)                                   # [blk][n][l]
    c = bl.copy(); cM = np.abs(bl).copy()
    np.add.at(c, lmOf, -np.einsum("knl,kl->kn", A, xp[rowInd])); np.add.at(cM, lmOf, np.einsum("knl,kl->kn", np.abs(A), np.abs(xp[rowInd])))
    inv = invHll.reshape(-1, 3, 3)
    return np.einsum("kji,kj->ki", inv, c), np.einsum("kji,kj->ki", np.abs(inv), cM), np.diff(colPtr)


def check_inv_hll(sysE, invHll, lam, label):
    H = sysE[2].reshape(-1, 3, 3) + lam * np.eye(3)
    ref = np.linalg.inv(H)
    a = H
    a00, a01, a02, a11, a12, a22 = a[:, 0, 0], a[:, 0, 1], a[:, 0, 2], a[:, 1, 1], a[:, 1, 2], a[:, 2, 2]
    ab = np.abs
    # the closed-form adjugate: cofactor and determinant magnitudes (test_host_math.test_sym3_inverse)
    Cm = np.stack([ab(a11 * a22) + a12 * a12, ab(a02 * a12) + ab(a01 * a22), ab(a01 * a12) + ab(a02 * a11),
                   ab(a02 * a12) + ab(a01 * a22), ab(a00 * a22) + a02 * a02, ab(a02 * a01) + ab(a00 * a12),
                   ab(a01 * a12) + ab(a02 * a11), ab(a02 * a01) + ab(a00 * a12), ab(a00 * a11) + a01 * a01], axis=1)
    Dm = ab(a00 * a11 * a22) + 2 * ab(a01 * a12 * a02) + ab(a00) * a12 * a12 + ab(a11) * a02 * a02 + ab(a22) * a01 * a01
    det = np.linalg.det(H)
    ev = np.linalg.eigvalsh(H)
    b1 = 16 * U * (Cm / det[:, None] + ab(ref.reshape(-1, 9)) * (Dm / det)[:, None])
    b2 = 16 * U * (ev[:, -1] / ev[:, 0]) / ev[:, 0] * (ev[:, -1] / ev[:, 1])
    assert report("%s invHll" % label, ab(invHll - ref.reshape(-1, 9)), np.minimum(b1, b2[:, None])) <= 1


def check_schur(eng, sysE, lam, label, exact=False):
    Hsc, bsc, invHll = eng.schur()
    if not exact:
        check_inv_hll(sysE, invHll, lam, label)
    Hr, br, HM, bM, npb, npp = schur_restated(eng, sysE, invHll, lam)
    u = 2.0 ** -53 if exact else U
    # each product W Hpl^T: two 3-term dot products (K 8); the sum over a block's products: gamma_n
    K = 8 + npb[:, None]
    assert report("%s Hsc" % label, np.abs(Hsc - Hr), u * K * HM) <= 1
    assert report("%s bsc" % label, np.abs(bsc - br), u * (8 + npp[:, None]) * bM) <= 1
    return Hsc, bsc, invHll


def check_backsub(eng, sysE, invHll, label, exact=False):
    xp, xl = eng.delta()
    ref, M, n = backsub_restated(eng, sysE, invHll, xp)
    u = 2.0 ** -53 if exact else U
    assert report("%s xl" % label, np.abs(xl - ref), u * (8 + n[:, None]) * M) <= 1
    return xp, xl


# ---- PCG --------------------------------------------------------------------------------------------------------------------

EXPECTED_KERNEL = {2: ("k_pcg2", False), 3: ("k_pcg4", True), 4: ("k_pcg3", False), 5: ("k_pcg5t", True),
                   6: ("k_pcg5t", False), "legacy": ("k_pcg5", True), 0: ("k_pcg3", False)}
# rows_11k: beyond k_pcg3's rows per CTA the automatic policy's block-Jacobi solve is k_pcg2, and k_pcg5 takes its BIG shape
EXPECTED_KERNEL_ROWS_CAPPED = {0: ("k_pcg2", False), 5: ("k_pcg5_big", True), "legacy": ("k_pcg5_big", True)}


def check_pcg(eng, Hsc, bsc, label, ok, kappa_check=True):
    """true residual of xp in fp64 against the engine's own Hsc / bsc, in the block-Jacobi norm: <= c tol |b| + K u |(|Hsc| |xp|)|;
    then |L^T (xp - x*)| <= |r|_BJ / lambda_min(L^-1 S L^-T)"""
    rp, ci = eng.hsc_structure()
    P = len(rp) - 1

    class _O:
        def solve(self, lam):
            return True

        def schur(self):
            return Hsc, bsc, None

        def hsc_structure(self):
            return rp, ci
    S, b = _system(_O(), P, 0.0)
    Sa = abs(S)
    xp, _ = eng.delta()
    x = xp.reshape(-1)
    r = b - S @ x
    D = Hsc[rp[:-1]].reshape(-1, 6, 6).transpose(0, 2, 1)
    L = np.linalg.cholesky(D)
    Li = sp.block_diag(list(np.linalg.inv(L)), format="csr")
    nr = np.linalg.norm(Li @ r); nb = np.linalg.norm(Li @ b); nm = np.linalg.norm(Li @ (Sa @ np.abs(x)))
    info = eng.pcg_info()
    tol = 1e-6 if info["status"] == 0 else 1e-3
    nnzr = int(np.diff(sp.csr_matrix(S).indptr).max())
    bound = 10 * tol * nb + (8 + nnzr) * U * nm
    assert ok == (info["status"] == 0)
    if info["status"] == 2:
        # a breakdown: only a two-level solve may report one, and only after it has stagnated (test_fp32_pcg_variants checks why
        # and that the block-Jacobi retry of optimize() converges)
        assert info["two_level"], info
        print("%s PCG breakdown after %d iterations, relative BJ residual %.3g" % (label, info["iters"], nr / nb))
        assert nr <= 1e-3 * nb
        return info, S
    assert info["status"] in (0, 1)
    assert report("%s PCG residual (status %d, %d it)" % (label, info["status"], info["iters"]), nr, bound) <= 1
    if kappa_check:
        xs = spla.spsolve(sp.csc_matrix(S), b)
        Ah = (Li @ S @ Li.T).tocsc()
        lmin = spla.eigsh(Ah, k=1, sigma=0, which="LM", return_eigenvectors=False)[0]      # shift-invert: the smallest eigenvalue
        err = np.linalg.norm(L.transpose(0, 2, 1) @ (x - xs).reshape(P, 6, 1))
        assert report("%s PCG error (kappa_BJ %.3g)" % (label, 1 / lmin), err, 1.01 * nr / lmin + 1e-12 * np.linalg.norm(xs)) <= 1
    return info, S


# ---- update -------------------------------------------------------------------------------------------------------------------

def check_update(eng, o, prob, rk, lam32, sysE, state0, label):
    q0, t0, X0 = state0
    xp, xl = eng.delta()
    chi_t, scale = eng.update(float(lam32))
    eng.commit(True)
    q1, t1, X1 = eng.state()
    nP = prob.numP
    qr, tr, _, _ = se3_exact(xp, q0[:nP], t0[:nP])
    # q: a few roundings of unit-size numbers (K 32, test_host_math); t: K u (|t| + |upsilon|)
    dq = np.minimum(np.abs(q1[:nP] - qr).max(1), np.abs(q1[:nP] + qr).max(1))
    assert report("%s q" % label, dq, 32 * U) <= 1
    bt = 32 * U * (np.linalg.norm(t0[:nP], axis=1) + np.linalg.norm(xp[:, 3:], axis=1))
    assert report("%s t" % label, np.abs(t1[:nP] - tr).max(1), bt) <= 1
    assert np.array_equal(q1[nP:], q0[nP:]) and np.array_equal(t1[nP:], t0[nP:])
    nL = prob.numL
    assert np.array_equal(X1[:nL], F32(X0[:nL] + xl)) and np.array_equal(X1[nL:], X0[nL:])
    o.set_state(q1, t1, X1)
    ochi = o.compute_errors()
    ed = Edges(prob, rk, q1, t1, X1)
    bchi = (8 * U * (ed.w * 2 * (np.abs(ed.r) * ed.Mr).sum(1) + ed.e)).sum() + U * len(ed.e) * ochi
    assert report("%s trial chi2" % label, abs(chi_t - ochi), bchi) <= 1
    bp, bl = sysE[1], sysE[3]
    sref = (xp * (lam32 * xp + bp)).sum() + (xl * (lam32 * xl + bl)).sum()
    sM = (np.abs(xp) * (lam32 * np.abs(xp) + np.abs(bp))).sum() + (np.abs(xl) * (lam32 * np.abs(xl) + np.abs(bl))).sum()
    assert report("%s scale" % label, abs(scale - sref), 16 * U * sM) <= 1


# ---- the tests ----------------------------------------------------------------------------------------------------------------

STAGE_CASES = [("tiny", "huber", {}), ("small", "none", {}), ("small", "huber", {}), ("small", "tukey", {}),
               ("kitti07_shaped", "huber", {}), ("shard_edges", "huber", {}), ("near_origin", "huber", {}),
               ("small", "huber", {"structure_on_host": True}), ("ba_kitti_00", "huber", {})]


@pytest.mark.parametrize("name,kernel,kw", STAGE_CASES, ids=["%s-%s%s" % (n, k, "-host" if kw else "") for n, k, kw in STAGE_CASES])
def test_fp32_stages(pkg, oracle, problems, name, kernel, kw):
    """J+H, invHll, Schur, PCG (automatic policy), back-substitution, update, trial chi2 and scale of one LM step, then the
    per-edge chi2 at the new state"""
    prob = problem(problems, pkg, name); rk = KERNELS[kernel]
    eng = make_engine(pkg, prob, rk, use_fp32=True, **kw)
    o = oracle.Oracle(prob, *rk)
    label = "%s/%s%s" % (name, kernel, "/host" if kw else "")
    sysE = check_linearize(eng, o, prob, rk, label)
    state0 = eng.state()
    check_chi_sqs(eng, o, prob, rk, label)
    lam32 = float(np.float32(1e-5 * eng.max_diagonal()))
    iters, ok = eng.solve(lam32)
    Hsc, bsc, invHll = check_schur(eng, sysE, lam32, label)
    info, _ = check_pcg(eng, Hsc, bsc, label, ok)
    print("%s: automatic policy ran %s (two-level %s, coarse %s)" % (label, info["kernel"], info["two_level"], info["coarse_kernel"]))
    check_backsub(eng, sysE, invHll, label)
    check_update(eng, o, prob, rk, lam32, sysE, state0, label)
    check_chi_sqs(eng, o, prob, rk, label + " after")
    eng.close()


@pytest.mark.parametrize("name", ["small", "kitti07_shaped", "shard_edges"])
def test_fp32_jh_variants_agree(pkg, oracle, problems, name):
    """k_linearize_landmark<float, 128|256, minB> at its four tile shapes (jh_variant 0/4 = 128x6, 1 = 256x2, 2 = 256x3, 3 = 128x4)
    against the oracle within the J+H bound, and with each other"""
    prob = problem(problems, pkg, name); rk = KERNELS["huber"]
    o = oracle.Oracle(prob, *rk)
    outs = []
    for v in (0, 1, 2, 3):
        eng = make_engine(pkg, prob, rk, use_fp32=True, jh_variant=v)
        outs.append(check_linearize(eng, o, prob, rk, "%s jh %d" % (name, v)))
        eng.close()
    for v, s in zip((1, 2, 3), outs[1:]):
        for nme, a, b in zip(("Hpp", "bp", "Hll", "bl", "Hpl"), s, outs[0]):
            assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max(), (v, nme)


@pytest.mark.parametrize("name", ["small", "kitti07_shaped", "shard_edges"])
def test_fp32_schur3(pkg, problems, name):
    """k_schur3<float> against the fp64 Schur complement of the engine's own blocks"""
    prob = problem(problems, pkg, name); rk = KERNELS["huber"]
    eng = make_engine(pkg, prob, rk, use_fp32=True, schur_variant=3)
    eng.linearize()
    sysE = eng.system()
    for lam in (1e3, 1.0):
        lam32 = float(np.float32(lam))
        eng.solve(lam32)
        check_schur(eng, sysE, lam32, "%s schur 3 lambda %g" % (name, lam))
    eng.close()


PCG_VARIANTS = [0, 2, 3, 4, 5, 6, "legacy"]


def check_breakdown(pkg, prob, rk, eng, info, own, lam32, name, variant):
    """A two-level fp32 solve that reports a breakdown.  Why: Z_i = Ad(T_i) carries [t_i]x R_i, so the coarse matrix Z^T S Z scales
    with |t|^2 in some directions and not in others -- kappa(Ac) ~ 3e13 on rows_11k, whose poses lie up to 1e4 m from the origin.
    With u32 kappa(Ac) >> 1 the explicit fp32 coarse inverse has no correct digit, the preconditioned residual stagnates just above
    the fp32 tolerance (1.6e-6 against 1e-6, measured on an H100), the Chronopoulos-Gear recurrences then lose positivity and the
    kernel reports status 2.  optimize() answers that with one block-Jacobi solve.  Checked here: the cause (for k_pcg5, whose coarse
    level can be read back: |Ac^-1 Ac - I| >= 1), the stagnation (in check_pcg) and that the block-Jacobi solve optimize() falls back
    to converges on the same system."""
    if info["kernel"].startswith("k_pcg5"):
        agg, AcP, AcInv = eng.coarse()
        Ac = packed_to_dense(AcP, info["A"])
        dev = np.abs(AcInv.astype(np.float64) @ Ac - np.eye(len(Ac))).max()
        print("%s pcg %s lambda %g: fp32 coarse inverse residual |Ac^-1 Ac - I| = %.3g, kappa(Ac) %.3g" % (name, variant, lam32, dev, np.linalg.cond(Ac)))
        assert dev >= 1
    # the fallback: k_pcg5's block-Jacobi mode after a k_pcg5 breakdown, k_pcg3 after a k_pcg4 one (Engine.launch_pcg)
    bj = make_engine(pkg, prob, rk, use_fp32=True, pcg_variant=6 if info["kernel"].startswith("k_pcg5") else 4)
    bj.linearize()
    it, ok = bj.solve(lam32)
    Hsc, bsc, _ = bj.schur()
    binfo, _ = check_pcg(bj, Hsc, bsc, "%s block-Jacobi retry lambda %g" % (name, lam32), ok)
    assert binfo["status"] == 0 and not binfo["two_level"], binfo
    bj.close()


@pytest.mark.parametrize("name,variant", [pytest.param(n, v, id="%s-%s" % (v, n))
                                          for n in ("kitti07_shaped", "kitti00_shaped", "rows_11k") for v in PCG_VARIANTS])
def test_fp32_pcg_variants(pkg, problems, name, variant, monkeypatch):
    """every PCG path of the fp32 engine on the lambda ladder: the kernel it ran, the true residual of its solution in fp64 against
    its own Hsc / bsc, the error against the direct solve, and for two-level solves the coarse matrix against Z^T S Z"""
    if name == "rows_11k" and variant not in (0, 5, "legacy"):
        pytest.skip("the row-capped plan is exercised by the automatic and the k_pcg5 paths")
    prob = problem(problems, pkg, name); rk = KERNELS["huber"]
    if variant == "legacy":
        monkeypatch.setenv("CUBA_PCG5_LEGACY", "1")
    eng = make_engine(pkg, prob, rk, use_fp32=True, pcg_variant=5 if variant == "legacy" else variant)
    eng.linearize()
    own = {}
    for lam in (1e3, 10.0, 0.1):
        lam32 = float(np.float32(lam))
        iters, ok = eng.solve(lam32)
        Hsc, bsc, _ = eng.schur()
        info, S = check_pcg(eng, Hsc, bsc, "%s pcg %s lambda %g" % (name, variant, lam), ok)
        own[lam32] = S
        if info["status"] == 2:
            check_breakdown(pkg, prob, rk, eng, info, own, lam32, name, variant)
        print("%s pcg_variant %s lambda %g: %s two-level %s coarse %s, %d iterations, A %d G %d" % (
            name, variant, lam, info["kernel"], info["two_level"], info["coarse_kernel"], info["iters"], info["A"], info["G"]))
        k, two = (EXPECTED_KERNEL_ROWS_CAPPED if name == "rows_11k" else EXPECTED_KERNEL)[variant]
        assert (info["kernel"], info["two_level"]) == (k, two), info
        if info["two_level"] and info["kernel"].startswith("k_pcg5"):
            agg, AcP, _ = eng.coarse()
            A = info["A"]
            st = eng.state()
            Z = coarse_basis(type("P", (), {"q": st[0], "t": st[1]}), prob.numP)
            # the coarse matrix is cached: it was assembled at the damping info["coarse_lambda"] (an earlier solve's, or this one's)
            lc = [k for k in own if k == info["coarse_lambda"]]
            assert lc, (info["coarse_lambda"], list(own))
            Ac = coarse_matrix(own[lc[0]], agg, Z, A)
            got = packed_to_dense(AcP, A)
            # Z^T S Z: entry (a, b) sums 36 products per block of S between aggregates a and b: K = 16 + 36 x the most such blocks
            Am = coarse_matrix(abs(S), agg, np.abs(Z), A)
            rp, ci = eng.hsc_structure()
            ra, ca = agg[np.repeat(np.arange(len(rp) - 1), np.diff(rp))], agg[ci]
            npair = np.bincount(np.minimum(ra, ca) * A + np.maximum(ra, ca), minlength=A * A).max() * 2
            assert report("%s coarse Ac" % name, np.abs(got - Ac), (16 + 36 * npair) * U * Am) <= 1
    eng.close()


@pytest.mark.parametrize("how", ["pose_only", "landmark_only"])
def test_fp32_fixed_vertex_solves(pkg, oracle, problems, how):
    """k_solve_poses_only<float> (no free landmark) and k_solve_landmarks_only<float> (no free pose) on tiny"""
    from test_structure import _variant
    base = problems("tiny")
    prob = _variant(pkg, base, **({"fixed_lms": range(base.Lall)} if how == "pose_only" else {"fixed_poses": range(base.Pall)}))
    rk = KERNELS["huber"]
    eng = make_engine(pkg, prob, rk, use_fp32=True)
    o = oracle.Oracle(prob, *rk)
    sysE = check_linearize(eng, o, prob, rk, how)
    lam32 = float(np.float32(1e-5 * eng.max_diagonal()))
    eng.solve(lam32)
    xp, xl = eng.delta()
    if how == "pose_only":
        H = sysE[0].reshape(-1, 6, 6) + lam32 * np.eye(6)
        ref = np.linalg.solve(H, sysE[1][..., None])[..., 0]
        ev = np.linalg.eigvalsh(H)
        b = 64 * U * (ev[:, -1] / ev[:, 0]) * np.linalg.norm(ref, axis=1)
        assert report("pose_only xp", np.abs(xp - ref).max(1), b) <= 1
    else:
        _, _, invHll = eng.schur()
        check_inv_hll(sysE, invHll, lam32, how)
        inv = invHll.reshape(-1, 3, 3)
        ref = np.einsum("kji,kj->ki", inv, sysE[3])
        assert report("landmark_only xl", np.abs(xl - ref), 8 * U * np.einsum("kji,kj->ki", np.abs(inv), np.abs(sysE[3]))) <= 1
    eng.close()


# ---- mixed precision: fp64 arithmetic on fp32 Hpl blocks ---------------------------------------------------------------------

@pytest.mark.parametrize("name", ["small", "kitti07_shaped", "shard_edges", "ba_kitti_00"])
def test_mixed_schur_and_backsub_exact(pkg, problems, name):
    """k_schur3<double, float> and k_backsub<double, float> read the fp32 blocks and do fp64 arithmetic: against numpy on the engine's
    own system (whose Hpl already is the rounded blocks) they agree to fp64 rounding"""
    prob = problem(problems, pkg, name); rk = KERNELS["huber"]
    eng = make_engine(pkg, prob, rk, use_fp32="mixed")
    eng.linearize()
    sysE = eng.system()
    assert np.array_equal(sysE[4], F32(sysE[4]))
    for lam in (1e3, 1e-5 * eng.max_diagonal()):
        iters, ok = eng.solve(lam)
        assert ok
        Hsc, bsc, invHll = check_schur(eng, sysE, lam, "mixed %s lambda %g" % (name, lam), exact=True)
        H = sysE[2].reshape(-1, 3, 3) + lam * np.eye(3)
        assert np.abs(invHll - np.linalg.inv(H).reshape(-1, 9)).max() <= 1e-12 * np.abs(invHll).max()
        check_backsub(eng, sysE, invHll, "mixed %s lambda %g" % (name, lam), exact=True)
    eng.close()
