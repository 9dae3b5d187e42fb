"""The assembled Gauss-Newton system and one LM step against an independent fp64 reference built from the cost, on graph topologies
the other tests' graphs lack.

The oracle (oracle/ba_oracle.c) restates the reference's algorithm step by step, so where the reference is wrong the oracle is
wrong with it.  The reference here is built from the cost alone: per-edge residuals and Jacobians in longdouble
(test_host_math.residual_ld and the sixth-order central difference jacobians_fd), robust weights from robust_ref, blocks summed by
vertex index, the Schur complement from the summed coupling of every (pose, landmark) pair, and the step from a sparse direct solve
of the UNREDUCED system H + lambda I -- no Schur code and no builder's block order anywhere.

Topologies (each built from synth.make_graph or synth.make_shard_edges_graph and then edited):
  rep_mono_stereo   a mono and a stereo edge on the same (pose, landmark) pair
  rep_two_mono      two mono edges on one pair
  rep_three         three edges on one pair
  rep_warp_pieces   repeats on the 65-observation landmark placed so that the copies fall in different 32-edge pieces
  rep_fixed_ends    repeats whose pose is fixed (no Hpl block) and whose landmark is fixed
  rep_shuffled      repeats, with the caller's edge order shuffled so that the copies are not next to each other
  pose_fixed_lms    a free pose that sees only fixed landmarks (its row of Hsc is the diagonal block alone)
  lm_fixed_poses    free landmarks seen only by fixed poses (Hll and bl, no Hpl)
  single_mono       single-observation mono landmarks: Hll of rank 2, invertible only through lambda
  intrinsics        different intrinsics on every pose
  two_submaps       two disconnected sub-maps, each anchored by its own fixed pose
  unanchored        a second sub-map without a fixed pose: its rigid motions are held by lambda alone

A repeated pair is two terms of the cost on the same two vertices: g2o sums them, and so does the engine (DESIGN.md section 6).
"""
import numpy as np
import pytest

from conftest import KERNELS, make_engine, relerr
from test_host_math import LD, jacobians_fd, residual_ld, robust_ref

sp = pytest.importorskip("scipy.sparse")
spla = pytest.importorskip("scipy.sparse.linalg")

SYSTEM_TOL = 1e-11       # system blocks, Hsc, bsc against the reference
CALIB_TOL = 1e-12        # the oracle against the reference where the oracle is right
TOL = 1e-10              # the step: PCG (tolerance 1e-11) against the direct solve, as in test_gpu_parity.py
RK = KERNELS["huber"]
# optimize(10)'s final state against the oracle, where TOL is too tight for the conditioning (chi2 still agrees to TOL).  The
# shard-edges graphs' reduced systems have kappa ~8e5 at lambda = 1e-5 of the largest diagonal: one PCG step (tolerance 1e-11)
# already differs from the direct solve by 1.2e-10 in xp and 2.2e-10 in xl, and ten steps leave 1.5e-10 (q, rep_warp_pieces) and
# 1.0e-10 (t, rep_fixed_ends).  The sub-map without a fixed pose can move rigidly at no cost: only lambda holds that motion, which
# shrinks as the LM run proceeds, so the two solves part along it (t 3.0e-10).  All measured on an H100 80GB HBM3.
STATE_TOL = {"rep_warp_pieces": 1e-9, "rep_fixed_ends": 1e-9, "unanchored": 1e-8}


# ---- graphs --------------------------------------------------------------------------------------------------------------

def _project(g, prow, lrow, stereo, rng, noise=0.5):
    """measurements of new edges: the projection at the current estimate plus pixel noise"""
    n = len(prow)
    _, r = residual_ld(g["q"][prow], g["t"][prow], g["cam"][prow], g["Xw"][lrow], np.zeros((n, 3)), np.full(n, stereo))
    m = r.astype(np.float64) + rng.normal(0, noise, (n, 3))
    return m if stereo else m[:, :2]


def _add(g, kind, prow, lrow, rng, info=None):
    """append edges of `kind` ("mono" / "stereo") between pose rows and landmark rows of graph g"""
    prow, lrow = np.asarray(prow, np.int64), np.asarray(lrow, np.int64)
    meas = _project(g, prow, lrow, kind == "stereo", rng)
    info = np.full(len(prow), 1.0) if info is None else np.asarray(info, np.float64)
    for k, v in (("vP", g["pose_id"][prow]), ("vL", g["lm_id"][lrow]), ("meas", meas), ("info", info)):
        key = "%s_%s" % (kind, k)
        g[key] = np.concatenate([g[key], v.astype(g[key].dtype)])


def _rows(g, kind, k):
    """pose row and landmark row of edge k of `kind`"""
    prow = np.nonzero(g["pose_id"] == g[kind + "_vP"][k])[0][0]
    lrow = np.nonzero(g["lm_id"] == g[kind + "_vL"][k])[0][0]
    return prow, lrow


def _free_free(g, kind):
    """edges of `kind` whose both ends are free"""
    pf = dict(zip(g["pose_id"].tolist(), g["pose_fixed"].tolist())); lf = dict(zip(g["lm_id"].tolist(), g["lm_fixed"].tolist()))
    return np.array([k for k in range(len(g[kind + "_vP"])) if not pf[int(g[kind + "_vP"][k])] and not lf[int(g[kind + "_vL"][k])]])


def _repeat(g, kind_from, kind_to, edges, rng, copies=1):
    for k in edges:
        p, l = _rows(g, kind_from, k)
        for _ in range(copies):
            _add(g, kind_to, [p], [l], rng, info=[g[kind_from + "_info"][k]])


def _base(pkg, seed=7):
    return pkg.synth.make_graph(12, 300, 400, 900, seed)


def _merge(g1, g2):
    """two graphs side by side, the second's vertex ids shifted past the first's"""
    off = int(max(g1["pose_id"].max(), g1["lm_id"].max())) + 1
    g = {}
    for k in g1:
        b = g2[k] + off if k in ("pose_id", "lm_id", "mono_vP", "mono_vL", "stereo_vP", "stereo_vL") else g2[k]
        g[k] = np.concatenate([g1[k], b.astype(g1[k].dtype)])
    return g


def _graph(pkg, name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "rep_mono_stereo":
        g = _base(pkg)
        _repeat(g, "stereo", "mono", rng.choice(_free_free(g, "stereo"), 12, replace=False), rng)
    elif name == "rep_two_mono":
        g = _base(pkg)
        _repeat(g, "mono", "mono", rng.choice(_free_free(g, "mono"), 12, replace=False), rng)
    elif name == "rep_three":
        g = _base(pkg)
        _repeat(g, "mono", "mono", rng.choice(_free_free(g, "mono"), 6, replace=False), rng, copies=2)
        e = rng.choice(_free_free(g, "stereo"), 6, replace=False)
        _repeat(g, "stereo", "mono", e, rng)
        _repeat(g, "stereo", "stereo", e, rng)
    elif name == "rep_warp_pieces":
        g = pkg.synth.make_shard_edges_graph()
        # landmark 4 has 65 observations on consecutive free poses; repeats on its 32nd and (after that insertion) 63rd pose put
        # original and copy at positions 31 | 32 and 63 | 64 of its run: different 32-edge pieces
        lid = g["lm_id"][4]
        poses = np.sort(np.concatenate([g["mono_vP"][g["mono_vL"] == lid], g["stereo_vP"][g["stereo_vL"] == lid]]))
        assert len(poses) == 65
        for p in (poses[31], poses[62]):
            _add(g, "mono", [int(p)], [4], rng)
        # and on the hot landmark (every pose), near its start and end
        for p in (10, 11, 150, 290):
            _add(g, "stereo", [p], [0], rng)
    elif name == "rep_fixed_ends":
        g = pkg.synth.make_shard_edges_graph()
        # fixed poses 0, 1, 2 on the hot landmark: no Hpl block, Hll and bl take both terms
        _add(g, "mono", [0, 1, 2], [0, 0, 0], rng)
        _add(g, "stereo", [1], [0], rng)
        # free poses on fixed landmarks: Hpp and bp take both terms
        fixed = np.nonzero(g["lm_fixed"])[0]
        ks = [k for k in range(len(g["stereo_vL"])) if g["stereo_vL"][k] in set(g["lm_id"][fixed[:6]].tolist())][:6]
        _repeat(g, "stereo", "mono", ks, rng)
        # and four ordinary repeats
        _repeat(g, "stereo", "mono", rng.choice(_free_free(g, "stereo"), 4, replace=False), rng)
    elif name == "rep_shuffled":
        g = _base(pkg, seed=9)
        _repeat(g, "stereo", "mono", rng.choice(_free_free(g, "stereo"), 8, replace=False), rng)
        _repeat(g, "mono", "mono", rng.choice(_free_free(g, "mono"), 8, replace=False), rng)
        _repeat(g, "stereo", "stereo", rng.choice(_free_free(g, "stereo"), 4, replace=False), rng)
        for kind in ("mono", "stereo"):
            perm = rng.permutation(len(g[kind + "_vP"]))
            for k in ("vP", "vL", "meas", "info"):
                g["%s_%s" % (kind, k)] = g["%s_%s" % (kind, k)][perm]
    elif name == "pose_fixed_lms":
        g = _base(pkg)
        # a new pose at pose 6's estimate; eight landmarks pose 6 sees become fixed, and the new pose sees only them
        src = 6
        seen = np.unique(g["stereo_vL"][g["stereo_vP"] == g["pose_id"][src]])[:8]
        lrows = np.nonzero(np.isin(g["lm_id"], seen))[0]
        g["lm_fixed"][lrows] = 1
        new_id = int(max(g["pose_id"].max(), g["lm_id"].max())) + 1
        for k, v in (("pose_id", [new_id]), ("pose_fixed", [0]), ("q", g["q"][src:src + 1]), ("t", g["t"][src:src + 1] + 0.01),
                     ("cam", g["cam"][src:src + 1])):
            g[k] = np.concatenate([g[k], np.asarray(v, dtype=g[k].dtype)])
        _add(g, "stereo", np.full(len(lrows), len(g["pose_id"]) - 1), lrows, rng)
    elif name == "lm_fixed_poses":
        g = _base(pkg)
        g["pose_fixed"][1] = 1
        # new landmarks next to ones poses 0 and 1 both see, observed by those two fixed poses only
        both = np.intersect1d(g["stereo_vL"][g["stereo_vP"] == g["pose_id"][0]], g["mono_vL"][g["mono_vP"] == g["pose_id"][1]])
        both = np.union1d(both, np.intersect1d(g["stereo_vL"][g["stereo_vP"] == g["pose_id"][0]], g["stereo_vL"][g["stereo_vP"] == g["pose_id"][1]]))[:4]
        assert len(both) >= 2
        src = np.nonzero(np.isin(g["lm_id"], both))[0]
        base_id = int(max(g["pose_id"].max(), g["lm_id"].max())) + 1
        L0 = len(g["lm_id"])
        g["lm_id"] = np.concatenate([g["lm_id"], np.arange(base_id, base_id + len(src), dtype=g["lm_id"].dtype)])
        g["lm_fixed"] = np.concatenate([g["lm_fixed"], np.zeros(len(src), g["lm_fixed"].dtype)])
        g["Xw"] = np.concatenate([g["Xw"], g["Xw"][src] + np.array([0.3, -0.2, 0.5])])
        new = np.arange(L0, L0 + len(src))
        _add(g, "stereo", np.zeros(len(new)), new, rng)
        _add(g, "mono", np.ones(len(new)), new, rng)
    elif name == "single_mono":
        g = _base(pkg)
        # ten new landmarks, each seen by one mono edge of a free pose, next to a landmark that pose sees
        ks = rng.choice(_free_free(g, "mono"), 10, replace=False)
        base_id = int(max(g["pose_id"].max(), g["lm_id"].max())) + 1
        prows, lsrc = zip(*[_rows(g, "mono", k) for k in ks])
        L0 = len(g["lm_id"])
        g["lm_id"] = np.concatenate([g["lm_id"], np.arange(base_id, base_id + 10, dtype=g["lm_id"].dtype)])
        g["lm_fixed"] = np.concatenate([g["lm_fixed"], np.zeros(10, g["lm_fixed"].dtype)])
        g["Xw"] = np.concatenate([g["Xw"], g["Xw"][list(lsrc)] + rng.normal(0, 0.5, (10, 3))])
        _add(g, "mono", prows, np.arange(L0, L0 + 10), rng)
    elif name == "intrinsics":
        g = _base(pkg)
        g["cam"] = g["cam"] * (1.0 + 0.01 * rng.standard_normal(g["cam"].shape))
    elif name in ("two_submaps", "unanchored"):
        g1 = pkg.synth.make_graph(30, 500, 700, 1100, 21)
        g2 = pkg.synth.make_graph(24, 400, 500, 900, 22)
        if name == "unanchored":
            g2["pose_fixed"][:] = 0
        g = _merge(g1, g2)
    else:
        raise KeyError(name)
    return g


TOPOLOGIES = ["rep_mono_stereo", "rep_two_mono", "rep_three", "rep_warp_pieces", "rep_fixed_ends", "rep_shuffled", "pose_fixed_lms",
              "lm_fixed_poses", "single_mono", "intrinsics", "two_submaps", "unanchored"]
REPEATED = [t for t in TOPOLOGIES if t.startswith("rep_")]
LAMBDAS = {"single_mono": (1e-5, 1e-8)}       # lambda / max diagonal of H; 1e-5 everywhere else

_CACHE = {}


def topology(pkg, name):
    if name not in _CACHE:
        _CACHE[name] = pkg.graphio.flatten(_graph(pkg, name))
    return _CACHE[name]


# ---- the reference ---------------------------------------------------------------------------------------------------------

def _edges(prob):
    idx = np.concatenate([prob.idx2, prob.idx3]).astype(np.int64)
    stereo = np.r_[np.zeros(prob.E2, bool), np.ones(prob.E3, bool)]
    meas = np.zeros((prob.nedges, 3)); meas[:prob.E2, :2] = prob.meas2; meas[prob.E2:] = prob.meas3
    return idx[:, 0], idx[:, 1], stereo, meas, np.r_[prob.omega2, prob.omega3]


def _inv3(A):
    """exact inverse of symmetric 3x3 blocks (adjugate over the determinant, longdouble)"""
    a0, a1, a2 = A[:, :, 0], A[:, :, 1], A[:, :, 2]
    adj = np.stack([np.cross(a1, a2), np.cross(a2, a0), np.cross(a0, a1)], axis=1)       # rows of the adjugate
    det = (a0 * adj[:, 0]).sum(1)
    return adj / det[:, None, None]


class Reference:
    """Gauss-Newton system of the robust cost at prob's estimate, and one LM step, keyed by vertex index only"""

    # b = SIGN * w J^T r with J = jacobians_fd (= -dr/d(delta)): fixed once by test_reference_calibration
    SIGN = 1.0

    def __init__(self, prob, rk):
        self.prob = prob
        P, L = prob.numP, prob.numL
        iP, iL, stereo, meas, om = _edges(prob)
        Xc, r = residual_ld(prob.q[iP], prob.t[iP], prob.cam[iP], prob.Xw[iL], meas, stereo)
        JP, _ = jacobians_fd(prob.q[iP], prob.t[iP], prob.cam[iP], prob.Xw[iL], meas, stereo)
        # d r / d Xw by the same sixth-order difference, of the residual itself: the graphs' quaternions are unit to fp32 only,
        # and the cost rotates with q as given, not with q / |q| as jacobians_fd's landmark Jacobian assumes
        JL = np.zeros((len(iP), 3, 3))
        for k in range(3):
            h = LD(1e-3) * np.abs(Xc[:, 2])

            def f(s):
                X = np.asarray(prob.Xw[iL], LD).copy(); X[:, k] += s * h
                return residual_ld(prob.q[iP], prob.t[iP], prob.cam[iP], X, meas, stereo)[1]
            df = 45 * (f(1) - f(-1)) - 9 * (f(2) - f(-2)) + (f(3) - f(-3))
            JL[:, :, k] = -(df / (60 * h)[:, None]).astype(np.float64)
        e = np.asarray(om, LD) * (r * r).sum(1)
        w = np.empty(len(e), LD)
        for k in range(len(e)):
            ty = int(stereo[k])
            delta = rk[1][ty]
            w[k] = LD(om[k]) * robust_ref(rk[0][ty], delta, float(delta) * float(delta), e[k])[1]
        JP, JL = JP.astype(LD), JL.astype(LD)
        pf, lf = iP < P, iL < L
        self.Hpp = np.zeros((P, 6, 6), LD); self.bp = np.zeros((P, 6), LD)
        self.Hll = np.zeros((L, 3, 3), LD); self.bl = np.zeros((L, 3), LD)
        np.add.at(self.Hpp, iP[pf], w[pf, None, None] * np.einsum("nki,nkj->nij", JP[pf], JP[pf]))
        np.add.at(self.bp, iP[pf], self.SIGN * w[pf, None] * np.einsum("nki,nk->ni", JP[pf], r[pf]))
        np.add.at(self.Hll, iL[lf], w[lf, None, None] * np.einsum("nki,nkj->nij", JL[lf], JL[lf]))
        np.add.at(self.bl, iL[lf], self.SIGN * w[lf, None] * np.einsum("nki,nk->ni", JL[lf], r[lf]))
        self.ff = np.nonzero(pf & lf)[0]
        self.Hpl_edge = w[self.ff, None, None] * np.einsum("nki,nkj->nij", JP[self.ff], JL[self.ff])     # [ff edges][6][3]
        # the coupling of every (pose, landmark) pair: the sum over its edges
        key = iL[self.ff] * max(P, 1) + iP[self.ff]
        self.pairs, inv = np.unique(key, return_inverse=True)
        self.C = np.zeros((len(self.pairs), 6, 3), LD)
        np.add.at(self.C, inv, self.Hpl_edge)
        self.pa, self.pl = self.pairs % max(P, 1), self.pairs // max(P, 1)
        self.max_diagonal = float(max(np.diagonal(self.Hpp, axis1=1, axis2=2).max(initial=0), np.diagonal(self.Hll, axis1=1, axis2=2).max(initial=0)))

    def system(self, e2h, nhpl):
        """(Hpp, bp, Hll, bl, Hpl) in the engine's layouts: blocks column-major, Hpl by the engine's edge -> block map"""
        Hpl = np.zeros((nhpl, 18))
        Hpl[e2h[self.ff]] = self.Hpl_edge.transpose(0, 2, 1).reshape(-1, 18).astype(np.float64)
        assert np.all(e2h[self.ff] >= 0) and len(np.unique(e2h[self.ff])) == len(self.ff) == nhpl
        f = lambda a, n: a.transpose(0, 2, 1).reshape(-1, n * n).astype(np.float64)
        return f(self.Hpp, 6), self.bp.astype(np.float64), f(self.Hll, 3), self.bl.astype(np.float64), Hpl

    def schur(self, lam):
        """upper pattern (rows, cols), Hsc blocks [nblk][36] column-major, bsc [P][6], from the summed pair couplings"""
        P, L = self.prob.numP, self.prob.numL
        inv = _inv3(self.Hll + LD(lam) * np.eye(3, dtype=LD))
        W = np.einsum("nij,njk->nik", self.C, inv[self.pl])                       # C_al inv_l
        bsc = self.bp.copy()
        np.add.at(bsc, self.pa, -np.einsum("nij,nj->ni", W, self.bl[self.pl]))
        # every pair of pairs of one landmark (pairs are sorted by landmark, then pose)
        start = np.searchsorted(self.pl, np.arange(L + 1))
        pi, pj = [], []
        for l in range(L):
            a, b = np.triu_indices(start[l + 1] - start[l])
            pi.append(start[l] + a); pj.append(start[l] + b)
        pi = np.concatenate(pi) if pi else np.zeros(0, int); pj = np.concatenate(pj) if pj else np.zeros(0, int)
        dest = np.concatenate([np.arange(P) * (P + 1), self.pa[pi] * P + self.pa[pj]])
        blocks, dinv = np.unique(dest, return_inverse=True)
        H = np.zeros((len(blocks), 6, 6), LD)
        np.add.at(H, dinv[:P], self.Hpp + LD(lam) * np.eye(6, dtype=LD))
        np.add.at(H, dinv[P:], -np.einsum("nik,njk->nij", W[pi], self.C[pj]))
        return (blocks // P, blocks % P), H.transpose(0, 2, 1).reshape(-1, 36).astype(np.float64), bsc.astype(np.float64), inv

    def step(self, lam):
        """(xp, xl) of (H + lambda I) x = b by a sparse direct solve of the unreduced system, and the 1-norm condition estimate"""
        P, L = self.prob.numP, self.prob.numL
        def blocks(first_row, first_col, B):          # triplets of blocks B[k] at (first_row[k], first_col[k])
            rr, cc = np.meshgrid(np.arange(B.shape[1]), np.arange(B.shape[2]), indexing="ij")
            return ((first_row[:, None, None] + rr).ravel(), (first_col[:, None, None] + cc).ravel(), B.astype(np.float64).ravel())
        dp, dl = 6 * np.arange(P), 6 * P + 3 * np.arange(L)
        parts = [blocks(dp, dp, self.Hpp + LD(lam) * np.eye(6, dtype=LD)), blocks(dl, dl, self.Hll + LD(lam) * np.eye(3, dtype=LD)),
                 blocks(6 * self.pa, 6 * P + 3 * self.pl, self.C), blocks(6 * P + 3 * self.pl, 6 * self.pa, self.C.transpose(0, 2, 1))]
        n = 6 * P + 3 * L
        I, J, V = (np.concatenate(x) for x in zip(*parts))
        H = sp.csc_matrix((V, (I, J)), shape=(n, n))
        b = np.concatenate([self.bp.astype(np.float64).ravel(), self.bl.astype(np.float64).ravel()])
        lu = spla.splu(H)
        x = lu.solve(b)
        op = spla.LinearOperator(H.shape, matvec=lu.solve, rmatvec=lambda v: lu.solve(v, trans="T"), dtype=np.float64)
        kappa = spla.norm(H, 1) * spla.onenormest(op)
        return x[:6 * P].reshape(P, 6), x[6 * P:].reshape(L, 3), kappa


_REF = {}


def reference(pkg, name):
    if name not in _REF:
        _REF[name] = Reference(topology(pkg, name), RK)
    return _REF[name]


def step_tol(kappa):
    """x of an iterative solve with relative residual 1e-11 against the direct solve: TOL on well-conditioned systems, otherwise
    kappa times the residual tolerance (and the direct solve's own kappa u)"""
    return max(TOL, 1e-11 * kappa)


def expected_products(prob):
    """product list of the Schur complement from the edge list: per landmark, (i, j) for blocks on poses row_i < row_j and every
    ordered pair (i, j) of blocks on one pose -> the number of products and the upper pattern"""
    idx = np.concatenate([prob.idx2, prob.idx3])
    ff = idx[(idx[:, 0] < prob.numP) & (idx[:, 1] < prob.numL)]
    n, pattern = 0, set((p, p) for p in range(prob.numP))
    for l in np.unique(ff[:, 1]):
        poses = np.sort(ff[ff[:, 1] == l, 0])
        u, m = np.unique(poses, return_counts=True)
        n += (len(poses) * (len(poses) - 1)) // 2 - int((m * (m - 1) // 2).sum()) + int((m * m).sum())
        pattern.update((int(a), int(b)) for k, a in enumerate(u) for b in u[k:])
    return n, pattern


# ---- CPU: the reference itself, the structure builders, the oracle ----------------------------------------------------------

@pytest.mark.parametrize("name", ["tiny", "small"])
def test_reference_calibration(pkg, oracle, problems, name):
    """on graphs without repeated pairs the oracle is right: the reference's system, Schur complement and step agree with it"""
    prob = problems(name)
    ref = Reference(prob, RK)
    o = oracle.Oracle(prob, *RK)
    o.compute_errors(); o.build_system()
    e2h = o.hpl_structure()[2]
    for nme, a, b in zip(("Hpp", "bp", "Hll", "bl", "Hpl"), ref.system(e2h, o.nhpl), o.system()):
        assert relerr(a, b) < CALIB_TOL, (nme, relerr(a, b))
    assert ref.max_diagonal == pytest.approx(o.max_diagonal(), rel=1e-13)
    lam = 1e-5 * ref.max_diagonal
    assert o.solve(lam)
    (rows, cols), Hsc, bsc, inv = ref.schur(lam)
    rp, ci = o.hsc_structure()
    assert np.array_equal(np.repeat(np.arange(prob.numP), np.diff(rp)), rows) and np.array_equal(ci, cols)
    oH, ob, oinv = o.schur()
    assert relerr(Hsc, oH) < CALIB_TOL and relerr(bsc, ob) < CALIB_TOL
    assert relerr(inv.transpose(0, 2, 1).reshape(-1, 9).astype(np.float64), oinv) < CALIB_TOL
    xp, xl, kappa = ref.step(lam)
    oxp, oxl = o.delta()
    print("%s: kappa_1 %.3g, xp %.2g xl %.2g" % (name, kappa, relerr(oxp, xp), relerr(oxl, xl)))
    assert relerr(oxp, xp) < max(CALIB_TOL, 16 * kappa * 2.0 ** -53) and relerr(oxl, xl) < max(CALIB_TOL, 16 * kappa * 2.0 ** -53)


def test_topologies_have_the_intended_shape(pkg):
    """each edited graph has what its name promises"""
    for name in TOPOLOGIES:
        prob = topology(pkg, name)
        idx = np.concatenate([prob.idx2, prob.idx3]).astype(np.int64)
        key = idx[:, 0] * prob.Lall + idx[:, 1]
        _, cnt = np.unique(key, return_counts=True)
        assert (cnt.max() > 1) == name.startswith("rep_"), name
        ff = (idx[:, 0] < prob.numP) & (idx[:, 1] < prob.numL)
        _, cff = np.unique(key[ff], return_counts=True)
        if name in ("rep_mono_stereo", "rep_two_mono", "rep_warp_pieces", "rep_shuffled", "rep_fixed_ends"):
            assert cff.max() == 2, name
        if name == "rep_three":
            assert cff.max() == 3
        if name == "rep_fixed_ends":
            assert np.any((cnt > 1) & np.isin(np.unique(key), key[idx[:, 0] >= prob.numP]))
            assert np.any((cnt > 1) & np.isin(np.unique(key), key[idx[:, 1] >= prob.numL]))
        if name == "rep_shuffled":
            k2 = key[:prob.E2]
            assert not any(k2[i] == k2[i + 1] for i in range(len(k2) - 1))
        if name == "pose_fixed_lms":
            lone = [p for p in range(prob.numP) if np.all(idx[idx[:, 0] == p, 1] >= prob.numL)]
            assert len(lone) == 1
        if name == "lm_fixed_poses":
            assert any(np.all(idx[idx[:, 1] == l, 0] >= prob.numP) for l in range(prob.numL))
        if name == "single_mono":
            deg = np.bincount(idx[:, 1], minlength=prob.Lall)
            assert np.sum((deg[:prob.numL] == 1) & np.isin(np.arange(prob.numL), prob.idx2[:, 1]) & ~np.isin(np.arange(prob.numL), prob.idx3[:, 1])) >= 10
        if name == "intrinsics":
            assert len(np.unique(prob.cam[:, 0])) == prob.Pall
        if name in ("two_submaps", "unanchored"):
            assert prob.Pall - prob.numP == (2 if name == "two_submaps" else 1)


@pytest.mark.parametrize("name", TOPOLOGIES)
def test_host_structure_products(pkg, oracle, name):
    """the host builder's product count and upper pattern against the list built from the edge list here, for the whole graph
    and summed over the shards of a three-rank run; the oracle's count likewise; the builder's self-check passes"""
    prob = topology(pkg, name)
    n, pattern = expected_products(prob)
    s = pkg.build_structure_host(prob)
    rows = np.repeat(np.arange(prob.numP), np.diff(s["hscRowPtr"]))
    assert set(zip(rows.tolist(), s["hscColInd"].tolist())) == pattern
    assert s["nmul"] == n, (s["nmul"], n)
    assert sum(pkg.build_structure_host(prob, r, 3)["shard"][3] for r in range(3)) == n
    assert oracle.Oracle(prob).nmul == n


@pytest.mark.parametrize("name", TOPOLOGIES)
def test_oracle_against_reference(pkg, oracle, name):
    """the oracle on every topology: system, Schur complement (Hsc, its diagonal blocks' symmetry, bsc) and the step"""
    prob = topology(pkg, name); ref = reference(pkg, name)
    o = oracle.Oracle(prob, *RK)
    o.compute_errors(); o.build_system()
    for nme, a, b in zip(("Hpp", "bp", "Hll", "bl", "Hpl"), o.system(), ref.system(o.hpl_structure()[2], o.nhpl)):
        assert relerr(a, b) < SYSTEM_TOL, (nme, relerr(a, b))
    for f in LAMBDAS.get(name, (1e-5,)):
        lam = f * ref.max_diagonal
        assert o.solve(lam)
        (rows, cols), Hsc, bsc, _ = ref.schur(lam)
        oH, ob, _ = o.schur()
        check_schur(prob, o.hsc_structure(), oH, ob, rows, cols, Hsc, bsc, "oracle %s lambda %g" % (name, f))
        xp, xl, kappa = ref.step(lam)
        oxp, oxl = o.delta()
        tol = max(CALIB_TOL, 16 * kappa * 2.0 ** -53)
        print("oracle %s lambda %g: kappa_1 %.3g xp %.2g xl %.2g (tol %.1g)" % (name, f, kappa, relerr(oxp, xp), relerr(oxl, xl), tol))
        assert relerr(oxp, xp) < tol and relerr(oxl, xl) < tol


def check_schur(prob, structure, Hsc, bsc, rows, cols, Hr, br, label, tol=SYSTEM_TOL):
    rp, ci = structure
    assert np.array_equal(np.repeat(np.arange(prob.numP), np.diff(rp)), rows) and np.array_equal(ci, cols), label
    D = Hsc[rp[:-1]].reshape(-1, 6, 6)
    asym = np.abs(D - D.transpose(0, 2, 1)).max() / np.abs(D).max()
    dH, db = relerr(Hsc, Hr), relerr(bsc, br)
    print("%s: Hsc %.2g bsc %.2g, diagonal asymmetry %.2g" % (label, dH, db, asym))
    assert asym < 1e-14, (label, asym)
    assert dH < tol and db < tol, (label, dH, db)


# ---- GPU: stage outputs on every path --------------------------------------------------------------------------------------

# id: (Engine keyword arguments, environment)
PATHS = {
    "default": ({}, {}),
    "host_structure": (dict(structure_on_host=True), {}),
    "jh1": (dict(jh_variant=1), {}),
    "jh7": (dict(jh_variant=7), {}),
    "jh8": (dict(jh_variant=8), {}),
    "jh9": (dict(jh_variant=9), {}),
    "schur3": (dict(schur_variant=3), {}),
    "schur5": (dict(schur_variant=5), {}),
    "pcg2": (dict(pcg_variant=2), {}),
    "pcg3": (dict(pcg_variant=3), {}),
    "pcg4": (dict(pcg_variant=4), {}),
    "pcg5": (dict(pcg_variant=5), {}),
    "pcg6": (dict(pcg_variant=6), {}),
    "pcg5_legacy": (dict(pcg_variant=5), {"CUBA_PCG5_LEGACY": "1"}),
}


@pytest.mark.gpu
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("name", TOPOLOGIES)
def test_stages_against_reference(pkg, name, path, monkeypatch):
    """linearize, system, solve(lambda), Schur complement and step of the engine against the reference: blocks to 1e-11, every
    diagonal block of Hsc symmetric to rounding, xp / xl to the PCG tolerance (scaled by the condition estimate where it is large)"""
    kw, env = PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    prob = topology(pkg, name); ref = reference(pkg, name)
    eng = make_engine(pkg, prob, RK, **kw)
    eng.linearize()
    _, _, e2h = eng.hpl_structure()
    for nme, a, b in zip(("Hpp", "bp", "Hll", "bl", "Hpl"), eng.system(), ref.system(e2h, eng.sizes["nhpl"])):
        assert relerr(a, b) < SYSTEM_TOL, (name, path, nme, relerr(a, b))
    md = eng.max_diagonal()
    assert md == pytest.approx(ref.max_diagonal, rel=1e-12)
    for f in LAMBDAS.get(name, (1e-5,)):
        lam = f * ref.max_diagonal
        iters, ok = eng.solve(lam)
        info = eng.pcg_info()
        (rows, cols), Hr, br, _ = ref.schur(lam)
        Hsc, bsc, _ = eng.schur()
        label = "%s %s lambda %g" % (name, path, f)
        check_schur(prob, eng.hsc_structure(), Hsc, bsc, rows, cols, Hr, br, label)
        xp_r, xl_r, kappa = ref.step(lam)
        xp, xl = eng.delta()
        tol = step_tol(kappa)
        print("%s: %s two-level %s status %d, %d iterations, kappa_1 %.3g: xp %.2g xl %.2g (tol %.2g)" % (
            label, info["kernel"], info["two_level"], info["status"], iters, kappa, relerr(xp, xp_r), relerr(xl, xl_r), tol))
        # a solve that did not converge must say so; one that says it did must be right
        if ok:
            assert relerr(xp, xp_r) < tol and relerr(xl, xl_r) < tol, (label, relerr(xp, xp_r), relerr(xl, xl_r), tol)
        else:
            assert info["status"] != 0, (label, info)
            assert name == "unanchored", (label, info)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", TOPOLOGIES)
def test_fp32_and_mixed_engines(pkg, name):
    """the fp32 engine (Schur complement, PCG residual and error, back-substitution) and the mixed engine (Schur complement and
    back-substitution in fp64 on fp32 Hpl) against fp64 restatements of their own inputs, to the bounds of test_fp32_stages.py"""
    from test_fp32_stages import check_backsub, check_pcg
    from test_fp32_stages import check_schur as check_schur_fp32
    prob = topology(pkg, name)
    eng = make_engine(pkg, prob, RK, use_fp32=True)
    eng.linearize()
    sysE = eng.system()
    for f in LAMBDAS.get(name, (1e-5,)):
        lam32 = float(np.float32(f * eng.max_diagonal()))
        iters, ok = eng.solve(lam32)
        Hsc, bsc, invHll = check_schur_fp32(eng, sysE, lam32, "fp32 %s lambda %g" % (name, f))
        info, _ = check_pcg(eng, Hsc, bsc, "fp32 %s lambda %g" % (name, f), ok)
        check_backsub(eng, sysE, invHll, "fp32 %s lambda %g" % (name, f))
    eng.close()
    eng = make_engine(pkg, prob, RK, use_fp32="mixed")
    eng.linearize()
    sysE = eng.system()
    for f in LAMBDAS.get(name, (1e-5,)):
        lam = f * eng.max_diagonal()
        iters, ok = eng.solve(lam)
        Hsc, bsc, invHll = check_schur_fp32(eng, sysE, lam, "mixed %s lambda %g" % (name, f), exact=True)
        check_backsub(eng, sysE, invHll, "mixed %s lambda %g" % (name, f), exact=True)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", TOPOLOGIES)
def test_optimize_against_oracle(pkg, oracle, name):
    """optimize(10): chi2, lambda and trial count per iteration and the final state against the oracle, with no hidden coarse
    failure; on the sub-map without a fixed pose a failed solve must be reported, never taken silently"""
    from test_gpu_parity import _no_hidden_coarse_failure, _trajectory_check
    prob = topology(pkg, name)
    eng = make_engine(pkg, prob, RK)
    stats = eng.optimize(10)
    o = oracle.Oracle(prob, *RK)
    chi, lam, tr = o.optimize(10)
    print("%s optimize(10): chi2 %s, last solve %s" % (name, [round(s["chi2"], 3) for s in stats], eng.pcg_info()["kernel"]))
    _trajectory_check(stats, chi, lam, tr)
    _no_hidden_coarse_failure(eng)
    for nme, a, b in zip(("q", "t", "Xw"), eng.state(), o.state()):
        assert relerr(a, b) < STATE_TOL.get(name, TOL), (name, nme, relerr(a, b))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rep_mono_stereo", "rep_shuffled"])
def test_dry_shard_repeated_pairs(pkg, name):
    """the ranks' partial Schur complements of a three-rank landmark-sharded run, each computed on one GPU (CUBA_DRY_SHARD), sum
    to the reference's"""
    from test_dry_shards import LAMS, dry_shards
    prob = topology(pkg, name); ref = reference(pkg, name)
    out = dry_shards(pkg, prob, RK, 3)
    rp, ci = out[0]["hsc"]
    for lam in LAMS:
        Hsc = sum(res["schur"][lam][0] for res in out); bsc = sum(res["schur"][lam][1] for res in out)
        for res in out[1:]:                 # the diagonal's Hpp + lambda I and bp are on rank 0 only
            Hsc[rp[:-1]] += res["system"][0]; bsc += res["system"][1]
        (rows, cols), Hr, br, _ = ref.schur(lam)
        check_schur(prob, (rp, ci), Hsc, bsc, rows, cols, Hr, br, "dry shards %s lambda %g" % (name, lam))


@pytest.mark.gpu
def test_drop_in_class_repeated_pair(tmp_path_factory, pkg, oracle):
    """the drop-in C++ class keys edges by object: a mono and a stereo edge object on one (pose, landmark) pair both reach the
    engine, and optimize() follows the oracle of the summed cost"""
    from test_dynamic_graph import _run
    g = _graph(pkg, "rep_mono_stereo")
    _run(pkg, oracle, tmp_path_factory, g, ["init", "opt:5", "rmedge:m:%d" % (len(g["mono_vP"]) - 1), "init", "opt:2"])
