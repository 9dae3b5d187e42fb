"""Sim(3) alignment of many keyframe pairs in one launch (include/cuba_b200.h: cuba_engine_optimize_sim3, csrc/cuba_sim3_batch.cuh),
its math in csrc/cuba_math.cuh (tests/cpp/sim3_math_driver.cpp), the Python front end (Engine.optimize_sim3, graphio.sim3_problems)
and the drop-in's cuba::optimizeSim3 (include/cuba_b200_sim3.h, tests/cpp/sim3_batch_driver.cpp).

The reference is a numpy restatement of ORB-SLAM2's OptimizeSim3 kept in this file, independent of the kernel's formulas: the
update is scipy.linalg.expm of the 4x4 generator [[sigma I + [w]x, upsilon], [0, 0]], S is carried as a rotation matrix, the
Jacobians follow d Y / d xi = [-[Y]x, I, Y] and d Z / d xi = (1/s) R^T [[X1]x, -I, -X1], and the LM rules are those of
Engine::optimize."""
import json
import os
import subprocess

import numpy as np
import pytest
import scipy.linalg
import scipy.spatial.transform

from conftest import ROOT
from test_pose_batch import check_trajectory

CSRC = os.path.join(ROOT, "cuda-bundle-adjustment_b200", "csrc")
LD = np.longdouble
U = 2.0 ** -53


# ---- the numpy reference ------------------------------------------------------------------------------------------------------
def skew(w):
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], dtype=np.asarray(w).dtype)


def quat_to_R(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def exp_update(xi, R, t, s):
    """S <- Exp(xi) S through the matrix exponential of the Sim(3) generator"""
    G = np.zeros((4, 4))
    G[:3, :3] = xi[6] * np.eye(3) + skew(xi[:3])
    G[:3, 3] = xi[3:6]
    M = scipy.linalg.expm(G)
    sd = np.exp(xi[6])
    return (M[:3, :3] / sd) @ R, M[:3, :3] @ t + M[:3, 3], sd * s


def proj(cam, P):
    return np.stack([cam[0] * P[:, 0] / P[:, 2] + cam[2], cam[1] * P[:, 1] / P[:, 2] + cam[3]], 1)


def proj_jac(cam, P):
    J = np.zeros((len(P), 2, 3))
    J[:, 0, 0] = cam[0] / P[:, 2]
    J[:, 0, 2] = -cam[0] * P[:, 0] / P[:, 2] ** 2
    J[:, 1, 1] = cam[1] / P[:, 2]
    J[:, 1, 2] = -cam[1] * P[:, 1] / P[:, 2] ** 2
    return J


def residuals(p, R, t, s, sel):
    Y = s * p.X2[sel] @ R.T + t
    Z = ((p.X1[sel] - t) @ R) / s
    return Y, Z, proj(p.cam1, Y) - p.obs1[sel], proj(p.cam2, Z) - p.obs2[sel]


def huber(e, delta):
    rho = np.where(e <= delta * delta, e, 2 * np.sqrt(e) * delta - delta * delta)
    drho = np.where(e <= delta * delta, 1.0, delta / np.sqrt(np.maximum(e, 1e-300)))
    return rho, drho


def jacobians(p, R, s, Y, Z, sel):
    n = len(Y)
    D1 = np.zeros((n, 3, 7))
    D2 = np.zeros((n, 3, 7))
    X1 = p.X1[sel]
    for k in range(n):
        D1[k, :, :3] = -skew(Y[k]); D1[k, :, 3:6] = np.eye(3); D1[k, :, 6] = Y[k]
        D2[k, :, :3] = skew(X1[k]); D2[k, :, 3:6] = -np.eye(3); D2[k, :, 6] = -X1[k]
        D2[k] = R.T @ D2[k] / s
    J1 = proj_jac(p.cam1, Y) @ D1
    J2 = proj_jac(p.cam2, Z) @ D2
    if p.fix_scale:
        J1[:, :, 6] = 0
        J2[:, :, 6] = 0
    return J1, J2


def chi2(p, R, t, s, sel, delta):
    _, _, r1, r2 = residuals(p, R, t, s, sel)
    return huber(p.omega1[sel] * (r1 ** 2).sum(1), delta)[0].sum() + huber(p.omega2[sel] * (r2 ** 2).sum(1), delta)[0].sum()


def lm(p, R, t, s, sel, iterations, delta):
    """optimize(iterations) over the pairs `sel` under Engine::optimize's rules; returns (R, t, s, (chi2s, lambdas, trials))"""
    traj = ([], [], [])
    if not sel.any():
        return R, t, s, traj
    nu, lam = 2.0, 0.0
    for it in range(iterations):
        Y, Z, r1, r2 = residuals(p, R, t, s, sel)
        e1, e2 = p.omega1[sel] * (r1 ** 2).sum(1), p.omega2[sel] * (r2 ** 2).sum(1)
        (rho1, d1), (rho2, d2) = huber(e1, delta), huber(e2, delta)
        F = rho1.sum() + rho2.sum()
        J1, J2 = jacobians(p, R, s, Y, Z, sel)
        w1, w2 = p.omega1[sel] * d1, p.omega2[sel] * d2
        H = np.einsum("n,nki,nkj->ij", w1, J1, J1) + np.einsum("n,nki,nkj->ij", w2, J2, J2)
        b = -(np.einsum("n,nki,nk->i", w1, J1, r1) + np.einsum("n,nki,nk->i", w2, J2, r2))
        if it == 0:
            lam = 1e-5 * max(0.0, np.diag(H).max())
        q, trials, rho = 0, 0, -1.0
        while q < 10 and rho < 0:
            trials += 1
            M = H + lam * np.eye(7)
            try:
                np.linalg.cholesky(M)
                x = np.linalg.solve(M, b)
            except np.linalg.LinAlgError:
                x = np.zeros(7)
            Rn, tn, sn = exp_update(x, R, t, s)
            Fh = chi2(p, Rn, tn, sn, sel, delta)
            rho = (F - Fh) / (x @ (lam * x + b) + 1e-3)
            if rho != rho:
                rho = -1.0
            if rho > 0:
                a = 2 * rho - 1
                lam *= min(max(1 - a ** 3, 1 / 3), 2 / 3)
                nu, F = 2.0, Fh
                R, t, s = Rn, tn, sn
                break
            lam *= nu
            nu *= 2
            q += 1
        traj[0].append(F); traj[1].append(lam); traj[2].append(trials)
        if q == 10 or rho <= 0 or not np.isfinite(lam):
            break
    return R, t, s, traj


def pair_test(p, R, t, s, sel, chi2_th):
    """(fail, edges within 1e-9 of the threshold) per pair of sel"""
    _, _, r1, r2 = residuals(p, R, t, s, sel)
    e1, e2 = p.omega1[sel] * (r1 ** 2).sum(1), p.omega2[sel] * (r2 ** 2).sum(1)
    near = (np.abs(e1 - chi2_th) <= 1e-9 * chi2_th) | (np.abs(e2 - chi2_th) <= 1e-9 * chi2_th)
    return (e1 > chi2_th) | (e2 > chi2_th), near


def reference(p, prm):
    """OptimizeSim3 restated: dict of R, t, s, levels, ninliers, stats (two trajectories), near (pairs at a threshold tie)"""
    n = len(p.omega1)
    delta = np.sqrt(prm.chi2)
    R0, t0, s0 = quat_to_R(p.q), np.array(p.t, dtype=np.float64), float(p.s)
    lev = np.zeros(n, np.uint8)
    near = np.zeros(n, bool)
    R, t, s, tr1 = lm(p, R0, t0, s0, lev == 0, prm.iterations, delta)
    fail, nr = pair_test(p, R, t, s, np.ones(n, bool), prm.chi2)
    lev[fail] = 1; near |= nr
    left = int((lev == 0).sum())
    if left < prm.min_pairs:
        return dict(R=R0, t=t0, s=s0, levels=lev, ninliers=0, stats=[tr1, ([], [], [])], near=near)
    R, t, s, tr2 = lm(p, R, t, s, lev == 0, prm.iterations_bad if fail.any() else prm.iterations_good, delta)
    sel = lev == 0
    fail2, nr2 = pair_test(p, R, t, s, sel, prm.chi2)
    idx = np.nonzero(sel)[0]
    lev[idx[fail2]] = 1; near[idx] |= nr2
    return dict(R=R, t=t, s=s, levels=lev, ninliers=int((lev == 0).sum()), stats=[tr1, tr2], near=near)


# ---- problems -------------------------------------------------------------------------------------------------------------------
def shared_pairs(prob, k_max=3, min_shared=20):
    """every pose pair (i, i + k), k <= k_max, with at least min_shared common landmarks"""
    P = np.concatenate([prob.idx2[:, 0], prob.idx3[:, 0]]); L = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    sets = [set(L[P == i].tolist()) for i in range(prob.Pall)]
    return [(i, i + k) for k in range(1, k_max + 1) for i in range(prob.Pall - k) if len(sets[i] & sets[i + k]) >= min_shared]


def perturb(pkg, problems, seed, wrong=(0.1, 0.2), fix_scale=None):
    """initial S12 off the planted one (about 1 degree, 5 % of |t| + 2 cm, scale by up to 3 %), 10-20 % wrong matches (obs1 moved
    30-80 px, or X2 taken from another pair)"""
    rng = np.random.default_rng(seed)
    out = []
    for k, p in enumerate(problems):
        p = pkg.graphio.Sim3Problem(**{f: (np.array(v, copy=True) if isinstance(v, np.ndarray) else v) for f, v in vars(p).items()})
        p.planted = (quat_to_R(p.q), p.t.copy(), p.s)
        dq = np.concatenate([rng.normal(0, 0.01, 3), [1.0]]); dq /= np.linalg.norm(dq)
        R = quat_to_R(dq) @ quat_to_R(p.q)
        p.q = _quat_of(R)
        p.t = p.t + rng.normal(0, 1, 3) * (0.05 * np.linalg.norm(p.t) + 0.02) / np.sqrt(3)
        p.s = p.s * np.exp(rng.uniform(-0.03, 0.03))
        n = len(p.omega1)
        bad = rng.random(n) < rng.uniform(*wrong)
        move = bad & (rng.random(n) < 0.5)
        p.obs1[move] += rng.uniform(30, 80, (int(move.sum()), 2)) * rng.choice([-1, 1], (int(move.sum()), 2))
        swap = np.nonzero(bad & ~move)[0]
        if len(swap) > 1:
            p.X2[swap] = p.X2[np.roll(swap, 1)]
        p.wrong = bad
        if fix_scale is not None:
            p.fix_scale = bool(fix_scale[k % len(fix_scale)])
        out.append(p)
    return out


def _quat_of(R):
    w = np.sqrt(max(0.0, 1 + np.trace(R))) / 2
    if w > 0.1:
        q = np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])
    else:
        q = np.array(scipy.spatial.transform.Rotation.from_matrix(R).as_quat())
    return q / np.linalg.norm(q) * (1 if q[3] >= 0 else -1)


_made = {}


def make_problems(pkg, name, seed=41, fix=(False, True)):
    if (name, seed) not in _made:
        prob = pkg.graphio.flatten(pkg.synth.make_config(name))
        pairs = shared_pairs(prob)
        rng = np.random.default_rng(seed)
        s0 = np.exp(rng.uniform(np.log(0.8), np.log(1.25), len(pairs)))
        _made[(name, seed)] = perturb(pkg, pkg.graphio.sim3_problems(prob, pairs, scale=s0), seed + 1, fix_scale=fix)
    return _made[(name, seed)]


# ---- no GPU: the math through g++ ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cppsim3") / "sim3_math_driver")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-I", CSRC,
                           os.path.join(ROOT, "tests", "cpp", "sim3_math_driver.cpp"), "-o", out])
    return out


def run(driver, fn, rows):
    rows = np.atleast_2d(np.asarray(rows, dtype=np.float64))
    txt = "\n".join(" ".join(repr(float(v)) for v in r) for r in rows) + "\n"
    out = subprocess.run([driver, fn], input=txt, capture_output=True, text=True, check=True).stdout
    res = np.array([[float(v) for v in line.split()] for line in out.splitlines()])
    assert res.shape[0] == rows.shape[0]
    return res


THETAS = [0.0, 1e-9, 1e-6, 1e-4, 1e-3, 1e-2, 0.1, 0.5, 1.0, 2.0, np.pi]
SIGMAS = [0.0] + [sg * v for v in (1e-12, 1e-9, 1e-6, 1e-4, 1e-2, 0.1, 0.5, 0.9, 1.0) for sg in (1, -1)]


def test_sim3_update_against_expm(driver):
    """sim3_update over theta x sigma against the 4x4 matrix exponential.  Bound: W = A I + B [w]x + C [w]x^2 and e^sigma R t are sums
    of a few dozen rounded products of magnitude <= e^|sigma| (|t| + |upsilon|), each term's coefficient within 40 u of exact (the
    series' 20 terms, or the closed forms' cancellation of at most a factor 30 outside |z| <= 1), and expm itself is accurate to a few
    u on these generators: |dt| <= 200 u e^|sigma| (|t| + |upsilon|) = 4.4e-14 e^|sigma| (|t| + |upsilon|), under the required 1e-12
    relative; s = e^sigma s to 4 u; the rotation to 256 u: se3_update's 32 u, plus expm's scaling and squaring, which on generators of
    norm up to 4 is itself off by up to ~40 u."""
    rng = np.random.default_rng(3)
    rows = []
    for th in THETAS:
        for sg in SIGMAS:
            for _ in range(3):
                d = rng.normal(size=3); d /= np.linalg.norm(d)
                q = rng.normal(size=4); q /= np.linalg.norm(q)
                rows.append(np.concatenate([d * th, rng.normal(0, 0.5, 3), [sg], q, rng.normal(0, 5, 3), [np.exp(rng.uniform(-1, 1))]]))
    rows = np.array(rows)
    out = run(driver, "sim3", rows)
    worst_t = worst_R = worst_s = 0.0
    for r, o in zip(rows, out):
        R, t, s = exp_update(r[:7], quat_to_R(r[7:11]), r[11:14], r[14])
        M = np.exp(abs(r[6])) * (np.linalg.norm(r[11:14]) + np.linalg.norm(r[3:6]))
        worst_t = max(worst_t, np.abs(o[4:7] - t).max() / (200 * U * M))
        worst_R = max(worst_R, np.abs(quat_to_R(o[:4]) - R).max() / (256 * U))
        worst_s = max(worst_s, abs(o[7] - s) / (4 * U * s))
        assert np.abs(o[4:7] - t).max() <= 1e-12 * max(1.0, np.abs(t).max())
    print("sim3_update: max measured/bound t %.3g, R %.3g, s %.3g" % (worst_t, worst_R, worst_s))
    assert worst_t <= 1 and worst_R <= 1 and worst_s <= 1
    # sigma = 0 leaves s bit for bit
    z = rows[rows[:, 6] == 0]
    assert np.array_equal(run(driver, "sim3", z)[:, 7], z[:, 14])


def test_sim3_update_with_sigma_zero_is_se3_update(driver):
    """sigma = 0: the rotation is se3_update's bit for bit, t agrees to rounding (W = V summed differently)"""
    rng = np.random.default_rng(4)
    rows = []
    for th in THETAS:
        for _ in range(4):
            d = rng.normal(size=3); d /= np.linalg.norm(d)
            q = rng.normal(size=4); q /= np.linalg.norm(q)
            rows.append(np.concatenate([d * th, rng.normal(0, 0.5, 3), [0.0], q, rng.normal(0, 5, 3), [1.3]]))
    rows = np.array(rows)
    a = run(driver, "sim3", rows)
    b = run(driver, "se3", np.concatenate([rows[:, :6], rows[:, 7:14]], 1))
    assert np.array_equal(a[:, :4], b[:, :4])
    M = np.abs(rows[:, 11:14]).max(1) + np.abs(rows[:, 3:6]).max(1)
    # se3_update's a2 = (1 - cos th) / th^2 costs up to 1.1e-11 |upsilon| near th = 1e-5 (test_host_math); W has no such cancellation
    assert np.all(np.abs(a[:, 4:7] - b[:, 4:7]).max(1) <= 2e-11 * M)
    assert np.array_equal(a[:, 7], rows[:, 14])


def test_sim3_edge_jacobians_against_central_differences(driver):
    """e12 / e21 residuals against a longdouble restatement, and their Jacobians against longdouble central differences of the
    residual under S <- Exp(xi) S (fourth order in h = 1e-4: truncation ~h^4 |r^(5)|, rounding ~1e-19 / h in longdouble)"""
    rng = np.random.default_rng(5)
    rows = []
    for _ in range(40):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        t = rng.normal(0, 2, 3); s = np.exp(rng.uniform(-0.3, 0.3))
        cam = np.array([718.9, 718.9, 607.2, 185.2])
        Y = np.array([rng.uniform(-5, 5), rng.uniform(-2, 2), rng.uniform(3, 40)])
        R = quat_to_R(q)
        X2 = R.T @ (Y - t) / s
        X1 = np.array([rng.uniform(-5, 5), rng.uniform(-2, 2), rng.uniform(3, 40)])
        rows.append(np.concatenate([q, t, [s], cam, cam * [1.01, 0.99, 1, 1], X1, X2, rng.uniform(0, 1000, 2), rng.uniform(0, 400, 2)]))
    rows = np.array(rows)
    out = run(driver, "edge", rows)

    def res_ld(r, xi):
        q, t, s = r[:4], r[4:7].astype(LD), LD(r[7])
        G = np.zeros((4, 4))
        R = quat_to_R(q.astype(LD)).astype(LD)
        # Exp(xi) to second order is enough for a central difference of order h^2: use the exact 4x4 exponential in longdouble series
        Gl = np.zeros((4, 4), dtype=LD)
        Gl[:3, :3] = xi[6] * np.eye(3, dtype=LD) + skew(xi[:3]).astype(LD)
        Gl[:3, 3] = xi[3:6]
        E = np.eye(4, dtype=LD); term = np.eye(4, dtype=LD)
        for k in range(1, 16):
            term = term @ Gl / k
            E = E + term
        del G
        Rn = (E[:3, :3] / np.exp(LD(xi[6]))) @ R
        tn = E[:3, :3] @ t + E[:3, 3]
        sn = np.exp(LD(xi[6])) * s
        c1, c2 = r[8:12].astype(LD), r[12:16].astype(LD)
        X1, X2, o1, o2 = r[16:19].astype(LD), r[19:22].astype(LD), r[22:24].astype(LD), r[24:26].astype(LD)
        Y = sn * Rn @ X2 + tn
        Z = Rn.T @ (X1 - tn) / sn
        p = lambda c, P: np.array([c[0] * P[0] / P[2] + c[2], c[1] * P[1] / P[2] + c[3]])
        return np.concatenate([p(c1, Y) - o1, p(c2, Z) - o2])

    h = LD(1e-4)
    worst = 0.0
    for r, o in zip(rows, out):
        r0 = res_ld(r, np.zeros(7, dtype=LD))
        assert np.allclose(o[:4], r0.astype(np.float64), rtol=0, atol=1e-9)
        J = np.zeros((4, 7))
        for k in range(7):
            e = np.zeros(7, dtype=LD); e[k] = h
            J[:, k] = ((8 * (res_ld(r, e) - res_ld(r, -e)) - (res_ld(r, 2 * e) - res_ld(r, -2 * e))) / (12 * h)).astype(np.float64)
        got = np.concatenate([o[4:18].reshape(2, 7), o[18:32].reshape(2, 7)])
        scale = np.abs(J).max(1, keepdims=True) + 1
        worst = max(worst, float((np.abs(got - J) / scale).max()))
    print("sim3 Jacobians: max |analytic - central difference| / (max |J| + 1) = %.3g" % worst)
    assert worst < 1e-9


def test_spd_inverse_7(driver):
    """spd_inverse<7> against numpy on SPD matrices up to condition 1e10, and its refusal of indefinite and singular matrices"""
    rng = np.random.default_rng(6)
    rows, kinds = [], []
    for cond in (1.0, 1e3, 1e6, 1e10):
        Q, _ = np.linalg.qr(rng.normal(size=(7, 7)))
        A = Q @ np.diag(np.logspace(0, np.log10(cond), 7)) @ Q.T
        rows.append(((A + A.T) / 2).T.ravel()); kinds.append(cond)
    Q, _ = np.linalg.qr(rng.normal(size=(7, 7)))
    rows.append((Q @ np.diag([1, 2, 3, -1, 4, 5, 6.0]) @ Q.T).T.ravel()); kinds.append(-1)
    S = np.diag([1, 2, 3, 4, 5, 6, 0.0])
    rows.append(S.T.ravel()); kinds.append(0)
    out = run(driver, "spd7", np.array(rows))
    for r, o, k in zip(rows, out, kinds):
        if k <= 0:
            assert o[0] == 0, k
            continue
        assert o[0] == 1
        A = r.reshape(7, 7).T
        inv = o[1:].reshape(7, 7).T
        assert np.abs(inv - np.linalg.inv(A)).max() <= 1e3 * U * k * np.abs(np.linalg.inv(A)).max(), k


def test_sim3_problems_against_hand_construction(pkg):
    prob = pkg.graphio.flatten(pkg.synth.make_config("small"))
    pairs = shared_pairs(prob)[:6]
    s0 = [0.8, 1.0, 1.25, 1.1, 0.9, 1.0]
    got = pkg.graphio.sim3_problems(prob, pairs, scale=s0, fix_scale=True)
    for (i, j), s, p in zip(pairs, s0, got):
        obs = {}
        for e, (iP, iL) in enumerate(prob.idx2):
            obs.setdefault((int(iP), int(iL)), (prob.meas2[e][:2], prob.omega2[e]))
        for e, (iP, iL) in enumerate(prob.idx3):
            obs.setdefault((int(iP), int(iL)), (prob.meas3[e][:2], prob.omega3[e]))
        # stereo edges come after every mono edge in edge-id order: a mono observation of the same landmark wins
        common = sorted({l for (pp, l) in obs if pp == i} & {l for (pp, l) in obs if pp == j})
        assert list(p.landmarks) == common and p.fix_scale and p.s == s
        Ri, Rj = quat_to_R(prob.q[i]), quat_to_R(prob.q[j])
        for k, l in enumerate(common):
            X = prob.Xw[l]
            assert np.allclose(p.X1[k], Ri @ X + prob.t[i], rtol=1e-14, atol=1e-12)
            assert np.allclose(p.X2[k], (Rj @ X + prob.t[j]) / s, rtol=1e-14, atol=1e-12)
            assert np.array_equal(p.obs1[k], obs[(i, l)][0]) and p.omega1[k] == obs[(i, l)][1]
            assert np.array_equal(p.obs2[k], obs[(j, l)][0]) and p.omega2[k] == obs[(j, l)][1]
        # the planted S12 maps X2 onto X1
        R = quat_to_R(p.q)
        assert np.allclose(R, Ri @ Rj.T, atol=1e-12)
        assert np.abs(p.s * p.X2 @ R.T + p.t - p.X1).max() <= 1e-9 * (1 + np.abs(p.X1).max())


@pytest.mark.parametrize("fix_scale", [False, True])
def test_reference_recovers_planted_sim3(pkg, fix_scale):
    """the numpy reference on noise-free problems (obs = the exact projections) from a perturbed S12 recovers the planted one to
    1e-9 (with fix_scale, the scale is started at the planted one)"""
    prob = pkg.graphio.flatten(pkg.synth.make_config("small"))
    pairs = shared_pairs(prob)[:4]
    P = pkg.graphio.sim3_problems(prob, pairs, scale=[0.85, 1.2, 1.0, 1.1])
    prm = pkg.Sim3Params(iterations=20, iterations_bad=20, iterations_good=20, min_pairs=3)
    rng = np.random.default_rng(7)
    for p in P:
        R0, t0, s0 = quat_to_R(p.q), p.t.copy(), p.s
        p.obs1 = proj(p.cam1, p.X1); p.obs2 = proj(p.cam2, p.X2)
        p.fix_scale = fix_scale
        dq = np.concatenate([rng.normal(0, 0.005, 3), [1.0]]); dq /= np.linalg.norm(dq)
        p.q = _quat_of(quat_to_R(dq) @ R0)
        p.t = t0 + rng.normal(0, 0.02, 3)
        if not fix_scale:
            p.s = s0 * 1.02
        r = reference(p, prm)
        assert r["ninliers"] == len(p.omega1)
        assert np.abs(r["R"] - R0).max() < 1e-9
        assert np.abs(r["t"] - t0).max() < 1e-9 * max(1, np.abs(t0).max())
        assert abs(r["s"] - s0) < 1e-9 * s0


def _build_batch_driver(tmp_path_factory, pkg):
    out = str(tmp_path_factory.mktemp("cppsim3b") / "sim3_batch_driver")
    libdir = os.path.dirname(pkg.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCUBA_FORCE_EIGEN_COMPAT", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "sim3_batch_driver.cpp"), "-L", libdir, "-lcuba_b200",
                           "-Wl,-rpath," + libdir, "-o", out])
    return out


def test_sim3_driver_compiles_against_dropin_headers(pkg, tmp_path_factory):
    assert os.path.exists(_build_batch_driver(tmp_path_factory, pkg))
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", pkg.library_path()], capture_output=True, text=True).stdout
    assert "cuba::optimizeSim3(" in out
    assert "cuba_engine_optimize_sim3" in pkg.binding.exported_symbols()


def test_default_params(pkg):
    p = pkg.Sim3Params()
    assert (p.chi2, p.iterations, p.iterations_bad, p.iterations_good, p.min_pairs) == (10.0, 5, 10, 5, 10)


# ---- on the GPU --------------------------------------------------------------------------------------------------------------------
def rot_angle(Ra, Rb):
    return float(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1)))


ST_TOL = 5e-8
_worst = [0.0]


def check_problem(got, ref, what, trajectory=True):
    """chi2 per iteration to 1e-10, R to 1e-9, levels and inlier counts identical except pairs at a threshold tie.  t and s to
    ST_TOL: along the optical axis a translation and a scale change move the projections nearly alike (a narrow baseline), so the
    7x7 system is ill-conditioned in that direction, and the kernel's Cholesky inverse and numpy's LU solve round apart there by
    up to 1.4e-8 relative in t and s (kitti07_shaped) while chi2, R and the levels agree."""
    if trajectory:
        for gs, rs in zip(got["stats"], ref["stats"]):
            check_trajectory(gs, rs, what)
    assert np.abs(quat_to_R(got["q"]) - ref["R"]).max() < 1e-9, what
    et = np.abs(got["t"] - ref["t"]).max() / max(1.0, np.abs(ref["t"]).max())
    es = abs(got["s"] - ref["s"]) / ref["s"]
    _worst[0] = max(_worst[0], et, es)
    assert et < ST_TOL and es < ST_TOL, (what, et, es)
    bad = np.nonzero(got["levels"] != ref["levels"])[0]
    assert ref["near"][bad].all(), (what, bad)
    if len(bad) == 0:
        assert got["ninliers"] == ref["ninliers"], what


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "kitti07_shaped"])
def test_sim3_batch_against_reference(pkg, name):
    P = make_problems(pkg, name)
    assert len(P) >= 20
    prm = pkg.Sim3Params()
    res = pkg.Engine(device=0).optimize_sim3(P, prm)
    dropped = kept = nwrong = nright = 0
    for b, (p, got) in enumerate(zip(P, res)):
        ref = reference(p, prm)
        check_problem(got, ref, (name, b))
        assert all(s["pcg_iters"] == 0 and s["pcg_failed"] == 0 for st in got["stats"] for s in st)
        if p.fix_scale:
            assert got["s"] == p.s
        if got["ninliers"] > 0:
            chi = [s["chi2"] for st in got["stats"] for s in st]
            assert chi[-1] <= chi[0], (name, b)
            dropped += int((got["levels"][p.wrong] == 1).sum()); nwrong += int(p.wrong.sum())
            kept += int((got["levels"][~p.wrong] == 0).sum()); nright += int((~p.wrong).sum())
    # the planted wrong matches are the ones the test drops
    assert dropped >= 0.95 * nwrong
    print("%s: %d problems, %.3f of the wrong matches dropped, %.3f of the others kept, largest t / s difference %.3g"
          % (name, len(P), dropped / nwrong, kept / nright, _worst[0]))


@pytest.mark.gpu
def test_sim3_batch_recovers_planted_sim3(pkg):
    """noise-free problems (obs = the exact projections of the planted S12) from a perturbed S12: the planted R to 1e-9, t and s to
    1e-6 (the chi2 floor, below)"""
    prob = pkg.graphio.flatten(pkg.synth.make_config("kitti07_shaped"))
    pairs = shared_pairs(prob)[::7]
    rng = np.random.default_rng(8)
    P = pkg.graphio.sim3_problems(prob, pairs, scale=np.exp(rng.uniform(np.log(0.8), np.log(1.25), len(pairs))))
    planted = []
    for k, p in enumerate(P):
        planted.append((quat_to_R(p.q), p.t.copy(), p.s))
        p.obs1 = proj(p.cam1, p.X1); p.obs2 = proj(p.cam2, p.X2)
        p.fix_scale = k % 3 == 0
        dq = np.concatenate([rng.normal(0, 0.005, 3), [1.0]]); dq /= np.linalg.norm(dq)
        p.q = _quat_of(quat_to_R(dq) @ quat_to_R(p.q))
        p.t = p.t + rng.normal(0, 0.02, 3)
    prm = pkg.Sim3Params(iterations=20, iterations_bad=20, iterations_good=20)
    res = pkg.Engine(device=0).optimize_sim3(P, prm)
    for b, (p, got, (R0, t0, s0)) in enumerate(zip(P, res, planted)):
        # chi2 here is rounding noise around 0 (1e-17): the trajectory is not compared
        check_problem(got, reference(p, prm), ("planted", b), trajectory=False)
        assert got["ninliers"] == len(p.omega1), b
        assert np.abs(quat_to_R(got["q"]) - R0).max() < 1e-9, b
        # t and s to 1e-6: LM stops once chi2 reaches its rounding floor (~1e-17 here), which along the optical axis, where t and
        # s move the projections nearly alike, leaves them up to 1.4e-7 from the planted values (the reference stops at the same S)
        assert np.abs(got["t"] - t0).max() < 1e-6 * max(1, np.abs(t0).max()), b
        assert abs(got["s"] - s0) < 1e-6 * s0, b


@pytest.mark.gpu
def test_sim3_edge_cases(pkg):
    eng = pkg.Engine(device=0)
    prm = pkg.Sim3Params()
    n0 = eng.launch_count()
    assert eng.optimize_sim3([], prm) == []
    assert eng.launch_count() == n0
    p = make_problems(pkg, "small")[0]
    G = pkg.graphio.Sim3Problem

    def sub(p, idx, **kw):
        d = {f: (np.array(v, copy=True) if isinstance(v, np.ndarray) else v) for f, v in vars(p).items() if f in G.__dataclass_fields__}
        for f in ("X1", "X2", "obs1", "obs2", "omega1", "omega2", "landmarks"):
            d[f] = d[f][idx]
        d.update(kw)
        return G(**d)
    empty = sub(p, np.arange(0))
    few = sub(p, np.arange(6))
    allbad = sub(p, np.arange(len(p.omega1)))
    allbad.obs1 = allbad.obs1 + 200.0
    fixed = sub(p, np.arange(len(p.omega1)), fix_scale=True)
    res = eng.optimize_sim3([empty, few, allbad, fixed], prm)
    for r, x in zip(res[:3], (empty, few, allbad)):
        assert r["ninliers"] == 0
        assert np.array_equal(r["q"], x.q) and np.array_equal(r["t"], x.t) and r["s"] == x.s
        assert len(r["stats"][1]) == 0
    assert len(res[0]["stats"][0]) == 0 and len(res[0]["levels"]) == 0
    assert len(res[1]["stats"][0]) > 0
    assert res[2]["levels"].all()
    assert res[3]["s"] == fixed.s and res[3]["ninliers"] > 0
    for x, r in zip((few, allbad, fixed), res[1:]):
        check_problem(r, reference(x, prm), "edge")
    # every pair an outlier with min_pairs = 0: the second optimize has no pair, S is the first one's result
    r0 = eng.optimize_sim3([allbad], pkg.Sim3Params(min_pairs=0))[0]
    ref = reference(allbad, pkg.Sim3Params(min_pairs=0))
    check_problem(r0, ref, "allbad0")
    assert r0["ninliers"] == 0 and len(r0["stats"][1]) == 0


def _same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(x["q"], y["q"]) and np.array_equal(x["t"], y["t"]) and x["s"] == y["s"]
        assert np.array_equal(x["levels"], y["levels"]) and x["ninliers"] == y["ninliers"] and x["stats"] == y["stats"]


@pytest.mark.gpu
def test_sim3_independence_and_reproducibility(pkg):
    P = make_problems(pkg, "small") + make_problems(pkg, "kitti07_shaped")
    big = [P[k % len(P)] for k in range(2000)]
    eng = pkg.Engine(device=0)
    n0 = eng.launch_count()
    r1 = eng.optimize_sim3(big)
    assert eng.launch_count() == n0 + 1
    _same(r1, eng.optimize_sim3(big))
    for b in (0, 7, 999, 1999):
        _same(eng.optimize_sim3([big[b]]), [r1[b]])
    # the same problem at several positions of the batch
    for b in range(len(P), 2000, len(P)):
        _same([r1[b]], [r1[0]])


@pytest.mark.gpu
def test_sim3_leaves_the_engine_alone(pkg):
    from conftest import KERNELS, make_engine
    prob = pkg.graphio.flatten(pkg.synth.make_config("small"))
    a = make_engine(pkg, prob, KERNELS["huber"])
    b = make_engine(pkg, prob, KERNELS["huber"])
    a.optimize_sim3(make_problems(pkg, "small"))
    sa, sb = a.optimize(10), b.optimize(10)
    assert sa == sb
    for x, y in zip(a.state(), b.state()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.edge_levels(), b.edge_levels())
    assert a.pcg_info() == b.pcg_info()


@pytest.mark.gpu
def test_sim3_malformed_input(pkg):
    eng = pkg.Engine(device=0)
    P = make_problems(pkg, "small")[:3]
    good = eng.optimize_sim3(P)
    n1 = eng.launch_count()
    cat = lambda name, w: np.concatenate([np.asarray(getattr(x, name), np.float64).reshape(-1, w) for x in P])
    n = np.array([len(x.omega1) for x in P])
    base = dict(ptr=np.concatenate([[0], np.cumsum(n)]), q=cat("q", 4), t=cat("t", 3), s=np.array([x.s for x in P]), cam1=cat("cam1", 4),
                cam2=cat("cam2", 4), fix_scale=None, X1=cat("X1", 3), X2=cat("X2", 3), obs1=cat("obs1", 2), obs2=cat("obs2", 2),
                omega1=cat("omega1", 1).ravel(), omega2=cat("omega2", 1).ravel())

    def with_(k, i, v):
        d = dict(base); x = np.array(d[k], dtype=np.float64 if k != "ptr" else np.int32); x.flat[i] = v; d[k] = x
        return d
    S = pkg.Sim3Params
    cases = {
        "B<0": (dict(base, B=-1), S()), "ptr[0]": (with_("ptr", 0, 1), S()), "ptr decreasing": (with_("ptr", 1, int(n.sum()) + 1), S()),
        "ptr end": (dict(base, N=int(n.sum()) + 1), S()), "q nan": (with_("q", 2, np.nan), S()), "t inf": (with_("t", 1, np.inf), S()),
        "s = 0": (with_("s", 1, 0.0), S()), "s < 0": (with_("s", 0, -1.0), S()), "cam nan": (with_("cam2", 3, np.nan), S()),
        "X1 inf": (with_("X1", 5, np.inf), S()), "obs2 nan": (with_("obs2", 3, np.nan), S()), "omega nan": (with_("omega1", 2, np.nan), S()),
        "iterations": (base, S(iterations=-1)), "iterations_bad": (base, S(iterations_bad=-1)), "iterations_good": (base, S(iterations_good=-2)),
        "min_pairs": (base, S(min_pairs=-1)), "chi2 0": (base, S(chi2=0.0)), "chi2 nan": (base, S(chi2=np.nan)), "chi2 inf": (base, S(chi2=np.inf)),
    }
    for what, (kw, prm) in cases.items():
        with pytest.raises(pkg.CubaError, match="error -1"):
            eng.optimize_sim3_flat(params=prm, **kw)
        assert eng.launch_count() == n1, what
    _same(eng.optimize_sim3(P), good)


@pytest.mark.gpu
def test_dropin_optimize_sim3(pkg, tmp_path_factory):
    """cuba::optimizeSim3 bit for bit equal to Engine.optimize_sim3; an unrelated graph held by the same object unchanged"""
    P = make_problems(pkg, "small")[:12]
    d = tmp_path_factory.mktemp("sim3")
    ppath, opath = str(d / "problems.txt"), str(d / "other.cubagraph")
    with open(ppath, "w") as f:
        f.write("%d\n" % len(P))
        for p in P:
            f.write(" ".join(repr(float(v)) for v in np.concatenate([p.q, p.t, [p.s], p.cam1, p.cam2, [int(p.fix_scale), len(p.omega1)]])) + "\n")
            for k in range(len(p.omega1)):
                f.write(" ".join(repr(float(v)) for v in np.concatenate([p.X1[k], p.X2[k], p.obs1[k], p.obs2[k], [p.omega1[k], p.omega2[k]]])) + "\n")
    pkg.graphio.write_graph(opath, pkg.synth.make_config("tiny"))
    out = subprocess.run([_build_batch_driver(tmp_path_factory, pkg), ppath, opath], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    res = json.loads(out.stdout)
    assert res["other_before"] == res["other_after"] and len(res["other_before"]) > 0 and res["other_state_equal"]
    assert res["threw_scale"] and res["threw_options"]
    ref = pkg.Engine(device=0).optimize_sim3(P)
    for b, (g, e) in enumerate(zip(res["problems"], ref)):
        assert np.array_equal(np.array(g["q"]), e["q"]) and np.array_equal(np.array(g["t"]), e["t"]) and g["s"] == e["s"], b
        assert np.array_equal(np.array(g["levels"], np.uint8), e["levels"]) and g["inliers"] == e["ninliers"], b
        assert g["rounds"] == [[s["chi2"] for s in st] for st in e["stats"]], b
