"""Every rank's share of a landmark-sharded run, on one GPU.

With CUBA_DRY_SHARD set, set_comm(r, W, ...) keeps rank r's landmark shard [lmBeg, lmEnd) and skips every collective, so every
stage output is rank r's partial result: the Hll / bl / Hpl blocks and edges of its own landmarks, its own block products in the
Schur complement, and Hpp + lambda I and bp on the diagonal of rank 0 only.  Each rank is checked against the CPU oracle run on the
sub-problem made of the shard's edges (sharding.sub_problem).  Rank 0's partial reduced system is the Schur complement of that
sub-problem, so rank 0's solve, update and whole optimize() are the sub-problem's LM run; the other ranks never solve (their
partial Hsc has no Hpp and is not SPD).  The peer all-reduce and the row-distributed k_pcg5 run with the ranks emulated on one GPU
in test_emulated_ranks.py; what one GPU cannot show is the NCCL landmark gather."""
import numpy as np
import pytest

from conftest import KERNELS, have_fixture, relerr
from test_gpu_parity import REF_VARIANTS, STAGE_TOL, TOL, _no_hidden_coarse_failure, _trajectory_check, _variant

LAMS = (1e3, 1.0)
# ba_kitti_00 (real data): the sums of bl cancel more, and the engine and the oracle add them in another order.  Measured on an
# H100 80GB HBM3: 1.7e-11 on one rank, up to 7.3e-11 on a shard of four (relative to the shard's largest |bl|); every other
# output stays below 1e-11
GRAPH_TOL = {"ba_kitti_00": {"bl": 1e-9}}


def _problem(pkg, problems, name):
    """`tiny-mixed` etc.: the fixed-vertex variants of test_gpu_parity on tiny"""
    base, _, how = name.partition("-")
    prob = problems(base)
    return _variant(pkg, prob, **REF_VARIANTS[how](prob)) if how else prob


def _edge_landmarks(prob):
    return np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])


def dry_engine(pkg, prob, rk, rank, world, **engine_kw):
    """an engine that keeps rank `rank`'s shard of a `world`-rank run and skips every collective"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("CUBA_DRY_SHARD", "1")
        eng = pkg.Engine(device=0, **engine_kw)
        eng.set_comm(rank, world, b"\0" * 128)
    for et in (0, 1):
        eng.set_robust_kernels(rk[0][et], rk[1][et], et)
    eng.initialize(prob)
    return eng


def dry_shards(pkg, prob, rk, world, **engine_kw):
    """the partial outputs of every rank: linearize (chi2, system, per-edge chi2) and the Schur stage alone at each of LAMS"""
    bounds = pkg.sharding.shard_bounds(_edge_landmarks(prob), prob.Lall, world)
    out = []
    for r in range(world):
        shard = pkg.build_structure_host(prob, r, world)["shard"]
        assert (shard[0], shard[1]) == (bounds[r], bounds[r + 1])
        eng = dry_engine(pkg, prob, rk, r, world, **engine_kw)
        res = dict(lo=int(bounds[r]), hi=int(bounds[r + 1]), sizes=dict(eng.sizes), hpl=eng.hpl_structure(), hsc=eng.hsc_structure())
        res["chi"] = eng.linearize()
        res["system"] = eng.system()
        res["chisq"] = eng.chi_squared()
        res["schur"] = {}
        for lam in LAMS:
            eng.bench_stage(3, reps=1, flush_l2=False, lam=lam)
            res["schur"][lam] = eng.schur()
        eng.close()
        out.append(res)
    return out


class Layout:
    """global index structures of the whole problem (the oracle's), and the maps of a sub-problem onto them"""

    def __init__(self, full, prob):
        self.prob = prob
        self.hpl = full.hpl_structure()
        self.rp, self.ci = full.hsc_structure()
        self.nblk, self.nhpl = len(self.ci), len(self.hpl[1])
        rows = np.repeat(np.arange(prob.numP), np.diff(self.rp))
        self.keys = rows.astype(np.int64) * max(prob.numP, 1) + self.ci
        self.diag = self.rp[:-1] if prob.numP else np.zeros(0, np.int64)

    def edges(self, lo, hi):
        """global ids of the sub-problem's edges, in its order"""
        p = self.prob
        m2 = (p.idx2[:, 1] >= lo) & (p.idx2[:, 1] < hi); m3 = (p.idx3[:, 1] >= lo) & (p.idx3[:, 1] < hi)
        return np.concatenate([np.nonzero(m2)[0], p.E2 + np.nonzero(m3)[0]])

    def blocks(self, rp, ci):
        """global position of every upper block of a sub-problem's Hsc pattern"""
        rows = np.repeat(np.arange(self.prob.numP), np.diff(rp))
        k = np.searchsorted(self.keys, rows.astype(np.int64) * max(self.prob.numP, 1) + ci)
        assert np.array_equal(self.keys[k], rows.astype(np.int64) * max(self.prob.numP, 1) + ci)
        return k


def sub_reference(pkg, oracle, prob, rk, lay, lo, hi, rank):
    """the oracle's outputs of the sub-problem of landmarks [lo, hi), in the global layout and as rank `rank` holds them"""
    p = prob
    E = p.nedges
    z = dict(chi=0.0, system=(np.zeros((p.numP, 36)), np.zeros((p.numP, 6)), np.zeros((p.numL, 9)), np.zeros((p.numL, 3)),
                              np.zeros((lay.nhpl, 18))), chisq=np.zeros(E), schur={}, own_hpl=np.zeros(lay.nhpl, bool), own_e=np.zeros(E, bool))
    if hi == lo:
        assert rank != 0
        for lam in LAMS:
            z["schur"][lam] = (np.zeros((lay.nblk, 36)), np.zeros((p.numP, 6)), np.zeros((p.numL, 9)))
        return z
    sub = pkg.sharding.sub_problem(p, lo, hi)
    o = oracle.Oracle(sub, *rk)
    z["chi"] = o.compute_errors(); o.build_system()
    Hpp, bp, Hll, bl, Hpl_s = o.system()
    g = lay.edges(lo, hi)
    e2h_s = o.hpl_structure()[2]
    Hpl = np.zeros((lay.nhpl, 18))
    has = e2h_s >= 0
    gb = lay.hpl[2][g[has]]
    assert np.all(gb >= 0)
    Hpl[gb] = Hpl_s[e2h_s[has]]
    z["own_hpl"][gb] = True
    z["system"] = (Hpp, bp, Hll, bl, Hpl)
    z["chisq"][g] = o.chi_sqs(); z["own_e"][g] = True
    if p.numP and p.numL:
        k = lay.blocks(*o.hsc_structure())
        for lam in LAMS:
            assert o.solve(lam)
            Hsc_s, bsc, inv = o.schur()
            Hsc = np.zeros((lay.nblk, 36))
            Hsc[k] = Hsc_s
            if rank != 0:
                Hsc[lay.diag] -= Hpp + lam * np.eye(6).ravel()
                bsc = bsc - bp
            z["schur"][lam] = (Hsc, bsc, inv)
    return z


def _check_rank(res, ref, prob, r, hpl64=None, tols=None):
    """rank r's outputs against the oracle's sub-problem; with `hpl64` (mixed precision) the Hpl blocks must be those fp64 blocks
    rounded once to fp32"""
    tol = dict.fromkeys(("Hpp", "bp", "Hll", "bl", "Hpl", "chisq", "Hsc", "bsc", "invHll"), STAGE_TOL)
    tol.update(tols or {})
    mixed = hpl64 is not None
    lo, hi = res["lo"], res["hi"]
    own_l = np.zeros(prob.numL, bool); own_l[min(lo, prob.numL):min(hi, prob.numL)] = True
    assert abs(res["chi"] - ref["chi"]) <= STAGE_TOL * ref["chi"], (r, res["chi"], ref["chi"])
    Hpp, bp, Hll, bl, Hpl = res["system"]
    for nme, a, b in zip(("Hpp", "bp", "Hll", "bl"), res["system"][:4], ref["system"][:4]):
        assert relerr(a, b) < tol[nme], (r, nme, relerr(a, b))
    assert not Hll[~own_l].any() and not bl[~own_l].any(), r
    if mixed:       # the stored blocks are the fp64 blocks rounded once to fp32
        assert np.array_equal(Hpl, hpl64.astype(np.float32).astype(np.float64)), r
    else:
        assert relerr(Hpl, ref["system"][4]) < tol["Hpl"], (r, "Hpl", relerr(Hpl, ref["system"][4]))
    assert not Hpl[~ref["own_hpl"]].any(), r
    own_e = ref["own_e"]
    assert relerr(res["chisq"][own_e], ref["chisq"][own_e]) < tol["chisq"] and not res["chisq"][~own_e].any(), r
    if not (prob.numP and prob.numL) or mixed:
        return
    for lam in LAMS:
        for nme, a, b in zip(("Hsc", "bsc"), res["schur"][lam][:2], ref["schur"][lam][:2]):
            assert relerr(a, b) < tol[nme], (r, lam, nme, relerr(a, b))
        assert relerr(res["schur"][lam][2][own_l], ref["schur"][lam][2][own_l]) < tol["invHll"], (r, lam, "invHll")


def _check_sums(out, prob, lay, full_sys, full_chi, full_schur, mixed=False, tols=None):
    """the partials sum to the whole system; every landmark row, Hpl block and edge is non-zero on one rank only (and on one rank
    exactly where the whole system's is: Tukey's weight is zero on large residuals)"""
    tols = tols or {}
    assert abs(sum(res["chi"] for res in out) - full_chi) <= STAGE_TOL * full_chi
    for i, nme in enumerate(("Hpp", "bp", "Hll", "bl", "Hpl")):
        if mixed and nme == "Hpl":
            continue
        s = sum(res["system"][i] for res in out)
        assert relerr(s, full_sys[i]) < tols.get(nme, STAGE_TOL), (nme, relerr(s, full_sys[i]))
    for i in (2, 4):
        cnt = sum(np.any(res["system"][i] != 0, axis=1).astype(int) for res in out)
        assert np.array_equal(cnt, np.any(full_sys[i] != 0, axis=1).astype(int)), i
    cnt = sum((res["chisq"] != 0).astype(int) for res in out)
    assert np.array_equal(cnt, np.ones(prob.nedges, int))
    if not (prob.numP and prob.numL):
        return
    for lam in LAMS:
        Hsc = sum(res["schur"][lam][0] for res in out); bsc = sum(res["schur"][lam][1] for res in out)
        for res in out[1:]:
            Hsc[lay.diag] += res["system"][0]; bsc += res["system"][1]
        tol = 1e-12 if mixed else STAGE_TOL
        assert relerr(Hsc, full_schur[lam][0]) < tol, (lam, relerr(Hsc, full_schur[lam][0]))
        assert relerr(bsc, full_schur[lam][1]) < tol, (lam, relerr(bsc, full_schur[lam][1]))


def _full_oracle(oracle, prob, rk):
    full = oracle.Oracle(prob, *rk)
    chi = full.compute_errors(); full.build_system()
    schur = {}
    if prob.numP and prob.numL:
        for lam in LAMS:
            assert full.solve(lam)
            schur[lam] = full.schur()
    return full, chi, full.system(), schur


def _world1_schur(pkg, prob, rk, **engine_kw):
    eng = dry_engine(pkg, prob, rk, 0, 1, **engine_kw)
    eng.linearize()
    out = {}
    for lam in LAMS:
        eng.bench_stage(3, reps=1, flush_l2=False, lam=lam)
        out[lam] = eng.schur()
    eng.close()
    return out


PATHS = {"default": {}, "schur5": dict(schur_variant=5), "jh1": dict(jh_variant=1), "jh2": dict(jh_variant=2), "jh3": dict(jh_variant=3),
         "jh4": dict(jh_variant=4), "jh7": dict(jh_variant=7), "jh8": dict(jh_variant=8), "jh9": dict(jh_variant=9),
         "mixed": dict(use_fp32="mixed")}
SMALL_PATHS = ("default", "schur5", "jh4", "mixed")
SHARD_EDGE_PATHS = ("default", "jh7", "jh8", "jh9", "jh4")
CASES = ([(n, w, "default", "huber") for n in ("tiny", "tiny-mixed", "tiny-pose_only", "tiny-landmark_only") for w in (2, 3, 8)]
         + [("small", w, p, "huber") for w in (2, 3) for p in SMALL_PATHS] + [("small", 2, "default", "none"), ("small", 3, "default", "tukey")]
         + [("kitti07_shaped", w, p, "huber") for w in (2, 8) for p in ("default", "schur5", "mixed")]
         + [("kitti00_shaped", 8, "default", "huber")]
         + [("shard_edges", w, p, "huber") for w in (1, 3) for p in SHARD_EDGE_PATHS]
         + [("shard_edges", 1, p, "huber") for p in ("jh1", "jh2", "jh3")] + [("shard_edges", 8, "default", "huber")]
         + [("ba_kitti_00", 4, "default", "huber")])


@pytest.mark.gpu
@pytest.mark.parametrize("name,world,path,kernel", [pytest.param(*c, id="%s-w%d-%s-%s" % c) for c in CASES])
def test_dry_shards_match_sub_problem_oracle(pkg, oracle, problems, name, world, path, kernel):
    """each rank's linearisation and Schur stage against the oracle's sub-problem of its shard; the ranks' partials sum to the
    whole system"""
    if name.startswith("ba_") and not have_fixture(name):
        pytest.skip("reference fixture absent")
    prob = _problem(pkg, problems, name); rk = KERNELS[kernel]
    mixed = path == "mixed"
    out = dry_shards(pkg, prob, rk, world, **PATHS[path])
    out64 = dry_shards(pkg, prob, rk, world) if mixed else None
    tols = GRAPH_TOL.get(name)
    full, fchi, fsys, fschur = _full_oracle(oracle, prob, rk)
    lay = Layout(full, prob)
    for r, res in enumerate(out):
        assert res["sizes"]["nhpl"] == lay.nhpl and res["sizes"]["nblk"] == lay.nblk
        for a, b in zip(res["hpl"] + res["hsc"], lay.hpl + (lay.rp, lay.ci)):
            assert np.array_equal(a, b), r                    # a shard keeps the global numbering
        _check_rank(res, sub_reference(pkg, oracle, prob, rk, lay, res["lo"], res["hi"], r), prob, r,
                    out64[r]["system"][4] if mixed else None, tols)
    _check_sums(out, prob, lay, fsys, fchi, _world1_schur(pkg, prob, rk, **PATHS[path]) if mixed else fschur, mixed, tols)


@pytest.mark.gpu
def test_dry_shards_fp32(pkg, problems):
    """the fp32 engine (generation-1 J+H, fp32 partial all-reduce layout): the summed partials of two ranks against one rank.
    Measured on an H100: at most 1.3e-7 relative (fp32 rounding of the partial sums, added in another order); checked at 1.3e-6."""
    prob = problems("small"); rk = KERNELS["huber"]
    out = dry_shards(pkg, prob, rk, 2, use_fp32=True)
    one = dry_shards(pkg, prob, rk, 1, use_fp32=True)[0]
    tol = 1.3e-6
    dev = {"chi": abs(out[0]["chi"] + out[1]["chi"] - one["chi"]) / one["chi"]}
    for i, nme in enumerate(("Hpp", "bp", "Hll", "bl", "Hpl")):
        dev[nme] = relerr(out[0]["system"][i] + out[1]["system"][i], one["system"][i])
    diag = one["hsc"][0][:-1]
    for lam in LAMS:
        Hsc = out[0]["schur"][lam][0] + out[1]["schur"][lam][0]; Hsc[diag] += out[1]["system"][0]
        bsc = out[0]["schur"][lam][1] + out[1]["schur"][lam][1] + out[1]["system"][1]
        dev["Hsc%g" % lam] = relerr(Hsc, one["schur"][lam][0]); dev["bsc%g" % lam] = relerr(bsc, one["schur"][lam][1])
    print("fp32 dry shards vs one rank:", {k: "%.1e" % v for k, v in dev.items()})
    assert max(dev.values()) < tol, dev


RANK0_CASES = [("tiny", 3), ("small", 2), ("kitti07_shaped", 2), ("shard_edges", 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,world", RANK0_CASES, ids=["%s-w%d" % c for c in RANK0_CASES])
def test_dry_rank0_stages_match_sub_problem(pkg, oracle, problems, name, world):
    """rank 0's solve / update / commit / state are the sub-problem's; landmarks of the other shards come back as uploaded"""
    prob = problems(name); rk = KERNELS["huber"]
    b = pkg.sharding.shard_bounds(_edge_landmarks(prob), prob.Lall, world)
    eng = dry_engine(pkg, prob, rk, 0, world)
    o = oracle.Oracle(pkg.sharding.sub_problem(prob, b[0], b[1]), *rk)
    chi = eng.linearize(); ochi = o.compute_errors(); o.build_system()
    assert abs(chi - ochi) <= STAGE_TOL * ochi
    md = eng.max_diagonal(); assert md == pytest.approx(o.max_diagonal(), rel=1e-12)
    lam = 1e-5 * md
    iters, ok = eng.solve(lam); assert ok and o.solve(lam)
    for nme, a, c in zip(("xp", "xl"), eng.delta(), o.delta()):
        assert relerr(a, c) < TOL, (nme, relerr(a, c))
    fh, sc = eng.update(lam); o.update()
    assert abs(fh - o.compute_errors()) <= TOL * fh
    assert abs(sc - o.compute_scale(lam)) <= TOL * abs(sc)
    eng.commit(True)
    q, t, Xw = eng.state()
    oq, ot, oX = o.state()
    assert relerr(q, oq) < TOL and relerr(t, ot) < TOL
    own = np.zeros(prob.Lall, bool); own[b[0]:min(b[1], prob.numL)] = True
    assert relerr(Xw[own], oX[own]) < TOL
    assert np.array_equal(Xw[~own], prob.Xw[~own])
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,world", [("kitti07_shaped", 2), ("kitti00_shaped", 8)], ids=["kitti07_shaped-w2", "kitti00_shaped-w8"])
def test_dry_rank0_optimize_matches_sub_problem(pkg, oracle, problems, name, world):
    """a fresh rank-0 engine's optimize(10) is the sub-problem's LM run.  kitti00_shaped (1 321 free poses) moves to the two-level
    k_pcg5t on the sharded engine."""
    prob = problems(name); rk = KERNELS["huber"]
    b = pkg.sharding.shard_bounds(_edge_landmarks(prob), prob.Lall, world)
    eng = dry_engine(pkg, prob, rk, 0, world)
    stats = eng.optimize(10)
    o = oracle.Oracle(pkg.sharding.sub_problem(prob, b[0], b[1]), *rk)
    chi, lam, tr = o.optimize(10)
    _trajectory_check(stats, chi, lam, tr)
    _no_hidden_coarse_failure(eng)
    info = eng.pcg_info()
    assert info["kernel"] in ("k_pcg3", "k_pcg5t"), info
    if name == "kitti00_shaped":
        assert info["coarse_rebuilds"] > 0, info                 # a two-level k_pcg5t solve ran
    q, t, Xw = eng.state()
    oq, ot, oX = o.state()
    own = np.zeros(prob.Lall, bool); own[b[0]:min(b[1], prob.numL)] = True
    assert relerr(q, oq) < TOL and relerr(t, ot) < TOL and relerr(Xw[own], oX[own]) < TOL
    assert np.array_equal(Xw[~own], prob.Xw[~own])
    eng.close()


def _stage_outputs(eng, lo, hi):
    """linearize, then the Schur stage at each of LAMS (invHll on the shard's own landmarks: the others are never written)"""
    chi = eng.linearize()
    out = [np.array([chi]), *eng.system()]
    for lam in LAMS:
        eng.bench_stage(3, reps=1, flush_l2=False, lam=lam)
        Hsc, bsc, inv = eng.schur()
        out += [Hsc, bsc, inv[lo:hi]]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,world", [("small", 3), ("shard_edges", 3)], ids=["small-w3", "shard_edges-w3"])
def test_dry_shard_structure_reuse(pkg, problems, name, world):
    """a second initialize() on the same topology keeps the shard's structures (refresh_values with non-zero edge and Hpl offsets):
    bitwise the same linearisation and Schur stage as a fresh engine"""
    prob = problems(name); rk = KERNELS["huber"]
    p2 = prob.copy()
    rng = np.random.default_rng(5)
    p2.meas2 = p2.meas2 + 0.25; p2.meas3 = p2.meas3 - 0.125; p2.omega3 = p2.omega3 * 0.5
    p2.t = p2.t + rng.normal(0, 0.01, p2.t.shape); p2.Xw = p2.Xw + rng.normal(0, 0.05, p2.Xw.shape)
    b = pkg.sharding.shard_bounds(_edge_landmarks(prob), prob.Lall, world)
    for r in range(world):
        lo, hi = min(b[r], prob.numL), min(b[r + 1], prob.numL)
        eng = dry_engine(pkg, prob, rk, r, world)
        eng.linearize()
        eng.initialize(p2)
        assert eng.structure_reuses() == 1
        fresh = dry_engine(pkg, p2, rk, r, world)
        for i, (a, c) in enumerate(zip(_stage_outputs(eng, lo, hi), _stage_outputs(fresh, lo, hi))):
            assert np.array_equal(a, c), (r, i)
        eng.close(); fresh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,world", [("small", 3), ("shard_edges", 3)], ids=["small-w3", "shard_edges-w3"])
def test_dry_shard_host_and_device_structure_builders_agree(pkg, problems, name, world):
    """cuba_structure.cpp and the device builder cut the same shard: identical structures, numbers to rounding"""
    prob = problems(name); rk = KERNELS["huber"]
    b = pkg.sharding.shard_bounds(_edge_landmarks(prob), prob.Lall, world)
    for r in range(world):
        lo, hi = min(b[r], prob.numL), min(b[r + 1], prob.numL)
        a = dry_engine(pkg, prob, rk, r, world); h = dry_engine(pkg, prob, rk, r, world, structure_on_host=True)
        assert a.sizes == h.sizes
        for x, y in zip(a.hpl_structure() + a.hsc_structure(), h.hpl_structure() + h.hsc_structure()):
            assert np.array_equal(x, y), r
        sa, sh = _stage_outputs(a, lo, hi), _stage_outputs(h, lo, hi)
        for i, (x, y) in enumerate(zip(sa, sh)):
            assert relerr(x, y) < (1e-13 if i < 6 else 1e-12), (r, i, relerr(x, y))
        a.close(); h.close()


def _greedy_tiles(counts, cap=32):
    """numpy restatement of the warp-tile packing (jh4::k_next): from landmark j, the most landmarks with at most `cap` edges
    together, at most `cap` landmarks; a landmark with more edges is a tile of its own (cut into pieces of `cap`)"""
    p = np.concatenate([[0], np.cumsum(counts)])
    N, j, tiles = len(counts), 0, []
    while j < N:
        m = j
        while m < min(N, j + cap) and p[m + 1] - p[j] <= cap:
            m += 1
        nxt = m if m > j else j + 1
        tiles.append((j, nxt))
        j = nxt
    return tiles, p


def test_shard_edges_graph(pkg, problems):
    """the properties the shard_edges graph is built for, asserted on its flat arrays"""
    prob = problems("shard_edges")
    iL = _edge_landmarks(prob); iP = np.concatenate([prob.idx2[:, 0], prob.idx3[:, 0]])
    E = len(iL)
    stereo = np.arange(E) >= prob.E2
    cnt = np.bincount(iL, minlength=prob.Lall)
    # hot landmark: over a quarter of the edges, over 128 poses (>= 5 pieces of 32), mono and stereo, fixed observers
    hot = int(np.argmax(cnt))
    assert hot < prob.numL and cnt[hot] * 4 > E and len(np.unique(iP[iL == hot])) > 128 and -(-cnt[hot] // 32) >= 5
    assert stereo[iL == hot].any() and (~stereo[iL == hot]).any() and (iP[iL == hot] >= prob.numP).any()
    b8 = pkg.sharding.shard_bounds(iL, prob.Lall, 8)
    assert np.any(np.diff(b8) == 0)                                     # an empty shard
    # landmarks cut into two and three pieces, and one filling a tile exactly
    for n in (32, 33, 64, 65):
        assert np.any(cnt[:prob.numL] == n), n
    # the fixed tail: the last third of the landmarks; at three ranks the last shard holds fixed landmarks only
    assert prob.Lall - prob.numL >= prob.Lall / 3
    b3 = pkg.sharding.shard_bounds(iL, prob.Lall, 3)
    assert b3[2] >= prob.numL and b3[3] > b3[2]
    # single-observation landmarks are stereo (full-rank Hll)
    single = np.nonzero(cnt[:prob.numL] == 1)[0]
    assert len(single) >= 64 and np.all(stereo[np.isin(iL, single)])
    # some warp tile holds more than 24 landmarks on more than 23 distinct poses: over the staged windows of jh_variant 8, 9, 7
    # (XW 24 / 16 landmarks, PC 23 / 19 poses), so those take the global-memory overflow path; at one rank and at three
    order = np.lexsort((np.arange(E), iP, iL))
    for world in (1, 3):
        b = pkg.sharding.shard_bounds(iL, prob.Lall, world)
        found = False
        for r in range(world):
            tiles, p = _greedy_tiles(cnt[b[r]:b[r + 1]])
            base = cnt[:b[r]].sum()
            for j, nxt in tiles:
                poses = iP[order[base + p[j]:base + p[nxt]]]
                found |= nxt - j > 24 and len(np.unique(poses)) > 23
        assert found, world
    # the host structure builder cuts the same shards
    for world, bb in ((3, b3), (8, b8)):
        for r in range(world):
            s = pkg.build_structure_host(prob, r, world)["shard"]
            assert (s[0], s[1]) == (bb[r], bb[r + 1])
