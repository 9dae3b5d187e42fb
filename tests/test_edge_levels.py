"""Edge levels (g2o Edge::setLevel + initializeOptimization(0)): include/cuba_b200.h cuba_engine_set_edge_levels /
_get_edge_levels / _classify_edges, the drop-in's include/cuba_b200_levels.h, and ORB-SLAM2's outlier rounds built on them.

The synthetic graphs carry 1 px noise only, so every test plants its own outliers with a seeded rng: measurements pushed by
20-50 px, a few landmarks moved behind one of their observing cameras, and masks that leave one free pose and one free landmark
without an included edge."""
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import KERNELS, ROOT, make_engine, relerr

STAGE_TOL = 1e-11
CHI2_MONO, CHI2_STEREO = 5.991, 7.815


# ---- planted outliers and masks ------------------------------------------------------------------------
def _conj(q):
    c = np.array(q, copy=True); c[..., :3] *= -1
    return c


def plant_outliers(pkg, g, seed=1, frac=0.02, behind=3):
    """a copy of g with measurements pushed by 20-50 px and `behind` landmarks moved behind one of their observing cameras;
    returns (graph, planted mono rows, planted stereo rows)"""
    rng = np.random.default_rng(seed)
    g = {k: np.array(v, copy=True) for k, v in g.items()}
    out = []
    for kind, w in (("mono", 2), ("stereo", 3)):
        n = len(g[kind + "_vP"])
        rows = rng.choice(n, max(1, int(frac * n)), replace=False) if n else np.zeros(0, np.int64)
        push = rng.uniform(20, 50, (len(rows), w)) * rng.choice([-1.0, 1.0], (len(rows), w))
        g[kind + "_meas"][rows] += push
        out.append(np.sort(rows))
    lrow = {int(v): i for i, v in enumerate(g["lm_id"])}
    prow = {int(v): i for i, v in enumerate(g["pose_id"])}
    cand = [int(l) for l in rng.permutation(np.unique(g["stereo_vL"]))[:behind]]
    for lid in cand:
        e = int(np.nonzero(g["stereo_vL"] == lid)[0][0])
        p = prow[int(g["stereo_vP"][e])]; r = lrow[lid]
        q, t = g["q"][p], g["t"][p]
        Xc = pkg.synth._rotate(q[None], g["Xw"][r][None])[0] + t
        Xc[2] = -Xc[2]
        g["Xw"][r] = pkg.synth._rotate(_conj(q)[None], (Xc - t)[None])[0]
    return g, out[0], out[1]


def make_mask(prob, seed=2, frac=0.1, planted=None):
    """random levels in edge-id order + the planted edges + every edge of one free pose and of one free landmark"""
    rng = np.random.default_rng(seed)
    E2, E = prob.E2, prob.nedges
    mask = rng.random(E) < frac
    if planted is not None:
        pm, ps = planted
        mask[np.nonzero(np.isin(prob.mono_rows, pm))[0]] = True
        mask[E2 + np.nonzero(np.isin(prob.stereo_rows, ps))[0]] = True
    ip = np.concatenate([prob.idx2[:, 0], prob.idx3[:, 0]]); il = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    p_free = prob.numP // 2 if prob.numP > 1 else None
    l_free = prob.numL // 2 if prob.numL > 0 else None
    if p_free is not None:
        mask[ip == p_free] = True
    if l_free is not None:
        mask[il == l_free] = True
    return mask.astype(np.uint8), p_free, l_free


def zeroed(prob, mask):
    p = prob.copy()
    p.omega2 = np.where(mask[:prob.E2] != 0, 0.0, prob.omega2)
    p.omega3 = np.where(mask[prob.E2:] != 0, 0.0, prob.omega3)
    return p


def sub_graph(g, prob, mask):
    """the graph without the edges at level 1 (flatten() then drops the vertices left without an edge)"""
    s = dict(g)
    km = np.ones(len(g["mono_vP"]), bool); ks = np.ones(len(g["stereo_vP"]), bool)
    km[prob.mono_rows[mask[:prob.E2] != 0]] = False
    ks[prob.stereo_rows[mask[prob.E2:] != 0]] = False
    for k in ("mono_vP", "mono_vL", "mono_meas", "mono_info"):
        s[k] = g[k][km]
    for k in ("stereo_vP", "stereo_vL", "stereo_meas", "stereo_info"):
        s[k] = g[k][ks]
    return s


_graphs = {}


def planted_problem(pkg, name):
    if name not in _graphs:
        g, pm, ps = plant_outliers(pkg, pkg.synth.make_config(name))
        _graphs[name] = (g, pkg.graphio.flatten(g), (pm, ps))
    return _graphs[name]


def depth_of(pkg, prob, q, t, Xw):
    ip = np.concatenate([prob.idx2[:, 0], prob.idx3[:, 0]]); il = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    return (pkg.synth._rotate(q[ip], Xw[il]) + t[ip])[:, 2]


def restate_levels(prob, chi, depth, old, depth_test, reinclude):
    thr = np.where(np.arange(prob.nedges) < prob.E2, CHI2_MONO, CHI2_STEREO)
    fail = (chi > thr) | ((depth <= 0) if depth_test else False)
    new = fail if reinclude else (old.astype(bool) | fail)
    return new.astype(np.uint8), thr


# ---- the drop-in's bookkeeping (no GPU) ------------------------------------------------------------------
def _build_driver(tmp_path_factory, pkg):
    out = str(tmp_path_factory.mktemp("cpplv") / "levels_driver")
    libdir = os.path.dirname(pkg.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCUBA_FORCE_EIGEN_COMPAT", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "levels_driver.cpp"), "-L", libdir, "-lcuba_b200",
                           "-Wl,-rpath," + libdir, "-o", out])
    return out


def _drive(tmp_path_factory, pkg, g, ops):
    exe = _build_driver(tmp_path_factory, pkg)
    d = tmp_path_factory.mktemp("lv")
    path = str(d / "g.cubagraph"); dump = str(d / "state.bin")
    pkg.graphio.write_graph(path, g)
    out = subprocess.run([exe, path, ";".join(ops), dump], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    nP, nL = len(g["pose_id"]), len(g["lm_id"])
    raw = np.fromfile(dump, dtype=np.float64)
    state = (raw[:4 * nP].reshape(nP, 4), raw[4 * nP:7 * nP].reshape(nP, 3), raw[7 * nP:].reshape(nL, 3))
    return json.loads(out.stdout)["steps"], state


def test_levels_symbols_and_header(pkg, tmp_path_factory):
    import ctypes
    lib = ctypes.CDLL(pkg.library_path())
    for n in ("cuba_engine_set_edge_levels", "cuba_engine_get_edge_levels", "cuba_engine_classify_edges", "cuba_debug_dropin_levels"):
        assert hasattr(lib, n) and n in pkg.binding.exported_symbols(), n
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", pkg.library_path()], capture_output=True, text=True).stdout
    for s in ("cuba::setEdgeLevel(", "cuba::edgeLevel(", "cuba::classifyEdges("):
        assert s in out, s
    assert os.path.exists(_build_driver(tmp_path_factory, pkg))    # cuba_b200_levels.h with -DCUBA_FORCE_EIGEN_COMPAT


class ListMirror:
    """the drop-in's edge lists (insertion order, tombstones compacted at initialize()) and their levels, by graph row"""

    def __init__(self, g):
        self.g = {k: np.array(v, copy=True) for k, v in g.items()}
        self.lists = {"m": list(range(len(g["mono_vP"]))), "s": list(range(len(g["stereo_vP"])))}
        self.level = {"m": {r: 0 for r in self.lists["m"]}, "s": {r: 0 for r in self.lists["s"]}}

    def both_fixed(self, kind, r):
        key = "mono" if kind == "m" else "stereo"
        pid = self.g[key + "_vP"][r]; lid = self.g[key + "_vL"][r]
        return bool(self.g["pose_fixed"][self.g["pose_id"] == pid][0]) and bool(self.g["lm_fixed"][self.g["lm_id"] == lid][0])

    def flat(self):
        return [self.level[k][r] for k in ("m", "s") for r in self.lists[k] if not self.both_fixed(k, r)]

    def apply(self, op):
        f = op.split(":")
        if f[0] == "level":
            held = int(f[2]) in self.lists[f[1]]
            if held:
                self.level[f[1]][int(f[2])] = int(int(f[3]) != 0)
            return {"threw": not held}
        if f[0] == "rmedge":
            self.lists[f[1]].remove(int(f[2])); self.level[f[1]].pop(int(f[2]))
        elif f[0] == "addedge":
            self.lists[f[1]].append(int(f[2])); self.level[f[1]][int(f[2])] = 0
        elif f[0] in ("fixp", "unfixp"):
            self.g["pose_fixed"][self.g["pose_id"] == int(f[1])] = int(f[0] == "fixp")
        elif f[0] in ("fixl", "unfixl"):
            self.g["lm_fixed"][self.g["lm_id"] == int(f[1])] = int(f[0] == "fixl")
        return {}


def test_dropin_level_bookkeeping(pkg, tmp_path_factory):
    """setEdgeLevel, removeEdge + re-add (level back to 0), an edge made both-fixed and unfixed again, the value-only initialize()
    path and tombstone compaction, followed through cuba_debug_dropin_levels against a mirror of the edge lists.  (Between an edge
    list edit and the next initialize() the flat array is still the last initialize()'s: "flat" is read only where they agree.)"""
    g = pkg.synth.make_config("tiny")
    p = int(g["stereo_vP"][4]); l = int(g["stereo_vL"][4])
    ops = ["init", "flat", "level:m:3:1", "level:s:4:7", "level:s:9:1", "flat", "init", "flat",          # value-only initialize()
           "rmedge:m:3", "level:m:3:1", "addedge:m:3", "init", "flat",                                   # re-added: level 0, at the end
           "level:m:3:1", "rmedge:s:2", "rmedge:m:0", "init", "flat",                                    # tombstone compaction
           "fixp:%d" % p, "fixl:%d" % l, "init", "flat", "level:m:5:1", "level:s:9:0", "flat",            # both-fixed edge dropped
           "unfixp:%d" % p, "unfixl:%d" % l, "init", "flat", "level:s:4:0", "init", "flat"]              # ... and back with its level
    steps, _ = _drive(tmp_path_factory, pkg, g, ops)
    m = ListMirror(g)
    nflat = 0
    for st, op in zip(steps, ops):
        exp = m.apply(op)
        if "threw" in exp:
            assert st["threw"] == exp["threw"], op
        if op == "flat":
            assert st["flat"] == m.flat(), (op, len(st["flat"]), len(m.flat()))
            nflat += 1
    assert nflat == ops.count("flat")
    assert sum(m.flat()) >= 2


# ---- the engine, on the GPU -------------------------------------------------------------------------------
def _engines(pkg, prob, mask, rk, host, **kw):
    """(engine with levels, engine given omega = 0 on the masked edges through set_problem -- structure reuse with the device
    builder, a rebuild with the host builder)"""
    a = make_engine(pkg, prob, rk, structure_on_host=host, **kw)
    a.set_edge_levels(mask)
    b = make_engine(pkg, prob, rk, structure_on_host=host, **kw)
    n0 = b.structure_reuses()
    b.initialize(zeroed(prob, mask))
    assert b.structure_reuses() == n0 + (0 if host else 1)
    return a, b


def _bitwise(a, b, what):
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(np.asarray(x), np.asarray(y)), (what, k, relerr(x, y))


def _check_equivalent(a, b):
    assert a.linearize() == b.linearize()
    _bitwise(a.system(), b.system(), "system")
    assert a.max_diagonal() == b.max_diagonal()
    for lam in (1e3, 1.0):
        assert a.solve(lam) == b.solve(lam)
        _bitwise(a.schur(), b.schur(), "schur")
        _bitwise(a.delta(), b.delta(), "delta")
    sa, sb = a.optimize(10), b.optimize(10)
    assert sa == sb
    _bitwise(a.state(), b.state(), "state")


EQUIV = [(n, k, "default") for n in ("tiny", "small", "kitti07_shaped", "kitti00_shaped", "shard_edges") for k in ("none", "huber", "tukey")] + \
        [("small", "huber", v) for v in ("jh1", "host", "fp32", "mixed", "pcg5", "pcg6", "clean")] + \
        [("kitti00_shaped", "huber", "pcg5")]
VARIANT = {"default": {}, "jh1": dict(jh_variant=1), "host": {},
           "fp32": dict(use_fp32=True), "mixed": dict(use_fp32="mixed"), "pcg5": dict(pcg_variant=5), "pcg6": dict(pcg_variant=6),
           "clean": {}}


@pytest.mark.gpu
@pytest.mark.parametrize("name,kernel,variant", EQUIV)
def test_levels_equal_zeroed_omega(pkg, problems, name, kernel, variant):
    """bit for bit: levels == set_problem with omega 0 on the same edges (stages at lambda 1e3 and 1, optimize(10), state)"""
    if variant == "clean":
        prob = problems(name); mask, _, _ = make_mask(prob, seed=7)
    else:
        g, prob, planted = planted_problem(pkg, name)
        mask, _, _ = make_mask(prob, seed=3, planted=planted)
    a, b = _engines(pkg, prob, mask, KERNELS[kernel], variant == "host", **VARIANT[variant])
    _check_equivalent(a, b)
    # set_state keeps the levels; a second mask on the same engine equals a fresh zeroed-omega engine again
    mask2, _, _ = make_mask(prob, seed=11, planted=None)
    q, t, Xw = a.state()
    a.set_edge_levels(mask2)
    p2 = zeroed(prob, mask2); p2.q, p2.t, p2.Xw = q, t, Xw
    c = make_engine(pkg, prob, KERNELS[kernel], structure_on_host=variant == "host", **VARIANT[variant])
    c.initialize(p2)
    _check_equivalent(a, c)
    assert np.array_equal(a.edge_levels(), mask2)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny", "small", "kitti07_shaped"])
def test_levels_follow_sub_problem_oracle(pkg, oracle, name):
    """g2o semantics: optimize() with levels follows the CPU oracle on the graph without the excluded edges; landmarks without an
    included edge stay bitwise where they were; the oracle given omega = 0 in place has the same system and Schur complement"""
    g, prob, planted = planted_problem(pkg, name)
    mask, p_free, l_free = make_mask(prob, seed=4, planted=planted)
    rk = KERNELS["huber"]
    eng = make_engine(pkg, prob, rk)
    eng.set_edge_levels(mask)
    # stage-wise against the oracle with omega zeroed in place
    o0 = oracle.Oracle(zeroed(prob, mask), *rk)
    chi = eng.linearize(); ochi = o0.compute_errors(); o0.build_system()
    assert abs(chi - ochi) <= STAGE_TOL * ochi
    for nme, a, b in zip(("Hpp", "bp", "Hll", "bl", "Hpl"), eng.system(), o0.system()):
        assert relerr(a, b) < STAGE_TOL, nme
    lam = 1e-5 * eng.max_diagonal()
    assert eng.solve(lam)[1] and o0.solve(lam)
    for nme, a, b in zip(("Hsc", "bsc", "invHll"), eng.schur(), o0.schur()):
        assert relerr(a, b) < STAGE_TOL, nme
    # the trajectory against the sub-problem
    sub = pkg.graphio.flatten(sub_graph(g, prob, mask))
    assert sub.nedges == prob.nedges - int(mask.sum())
    chi_o, _, _ = oracle.Oracle(sub, *rk).optimize(10)
    o = oracle.Oracle(sub, *rk); o.optimize(10)
    st = eng.optimize(10)
    got = np.array([s["chi2"] for s in st])
    assert len(got) == len(chi_o) and np.allclose(got, chi_o, rtol=1e-10, atol=0), (got, chi_o)
    q, t, Xw = eng.state(); oq, ot, oX = o.state()
    pr = {int(r): i for i, r in enumerate(prob.pose_rows)}; lr = {int(r): i for i, r in enumerate(prob.lm_rows)}
    pi = np.array([pr[int(r)] for r in sub.pose_rows]); li = np.array([lr[int(r)] for r in sub.lm_rows])
    assert np.abs(q[pi] - oq).max() < 1e-9
    assert np.abs(t[pi] - ot).max() < 1e-8 * max(1.0, np.abs(ot).max())
    assert np.abs(Xw[li] - oX).max() < 1e-8 * max(1.0, np.abs(oX).max())
    # vertices left without an included edge
    il = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    alone = np.setdiff1d(np.arange(prob.numL), il[mask == 0])
    assert l_free in alone
    assert np.array_equal(Xw[alone], prob.Xw[alone])
    # a pose without an included edge: its rows decouple (lambda I, zero right-hand side).  The update re-normalises q (the synthetic
    # quaternions are unit to fp32 only), and under the two-level PCG the coarse correction moves it at the solver's tolerance.
    qn = prob.q[p_free] / np.linalg.norm(prob.q[p_free])
    assert np.abs(q[p_free] - qn).max() < 1e-9 and np.abs(t[p_free] - prob.t[p_free]).max() < 1e-9 * max(1.0, np.abs(prob.t).max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "kitti07_shaped"])
def test_chi2_reports_excluded_edges(pkg, oracle, problems, name):
    g, prob, planted = planted_problem(pkg, name)
    rk = KERNELS["huber"]
    plain = make_engine(pkg, prob, rk); plain.optimize(3)
    ref = plain.chi_squared()
    # all levels 0 set explicitly: today's output, bit for bit
    eng = make_engine(pkg, prob, rk); eng.set_edge_levels(None); eng.optimize(3)
    assert np.array_equal(eng.chi_squared(), ref)
    # with levels: omega |r|^2 with the caller's omega for every edge, excluded ones too
    mask, _, _ = make_mask(prob, seed=5, planted=planted)
    eng.set_edge_levels(mask); eng.optimize(3)
    q, t, Xw = eng.state()
    o = oracle.Oracle(prob, *rk); o.set_state(q, t, Xw)
    cs, ocs = eng.chi_squared(), o.chi_sqs()
    assert relerr(cs, ocs) < 1e-12
    assert (cs[mask != 0] > 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "kitti07_shaped", "shard_edges"])
@pytest.mark.parametrize("depth", [True, False])
@pytest.mark.parametrize("reinclude", [False, True])
def test_classify_matches_restatement(pkg, oracle, name, depth, reinclude):
    g, prob, planted = planted_problem(pkg, name)
    rk = KERNELS["huber"]
    start, _, _ = make_mask(prob, seed=6, frac=0.05)
    runs = []
    for _ in range(2):
        eng = make_engine(pkg, prob, rk)
        eng.optimize(2)
        eng.set_edge_levels(start)
        assert np.array_equal(eng.edge_levels(), start)
        counts = eng.classify_edges(CHI2_MONO, CHI2_STEREO, depth=depth, reinclude=reinclude)
        runs.append((counts, eng.edge_levels(), eng))
    assert runs[0][0] == runs[1][0] and np.array_equal(runs[0][1], runs[1][1])     # bit-reproducible
    counts, lv, eng = runs[0]
    q, t, Xw = eng.state()
    o = oracle.Oracle(prob, *rk); o.set_state(q, t, Xw)
    chi = o.chi_sqs()
    want, thr = restate_levels(prob, chi, depth_of(pkg, prob, q, t, Xw), start, depth, reinclude)
    bad = np.nonzero(lv != want)[0]
    near = np.abs(chi - thr) <= 1e-9 * thr
    assert near[bad].all(), (len(bad), bad[:10])
    print("%s: %d edges at level 1, %d threshold ties" % (name, int(lv.sum()), len(bad)))
    mono = np.arange(prob.nedges) < prob.E2
    assert counts["included_mono"] == int(((lv == 0) & mono).sum()) and counts["included_stereo"] == int(((lv == 0) & ~mono).sum())
    assert counts["excluded"] == int(((start == 0) & (lv != 0)).sum()) and counts["reincluded"] == int(((start != 0) & (lv == 0)).sum())
    if depth:
        assert lv[depth_of(pkg, prob, q, t, Xw) <= 0].all()
    if not reinclude:
        assert lv[start != 0].all()
    # the classified engine equals one given the same levels
    ref = make_engine(pkg, prob, rk); ref.set_state(q, t, Xw); ref.set_edge_levels(lv)
    _check_equivalent(eng, ref)


@pytest.mark.gpu
def test_level_change_rebuilds_coarse_matrix(pkg, oracle, problems):
    """two-level k_pcg5 on kitti00_shaped: a new mask between two solves at the same lambda rebuilds the coarse matrix once"""
    prob = problems("kitti00_shaped")
    rk = KERNELS["huber"]
    eng = make_engine(pkg, prob, rk, pcg_variant=5)
    eng.linearize()
    lam = 1e-3 * eng.max_diagonal()
    assert eng.solve(lam)[1]
    i1 = eng.pcg_info()
    assert i1["two_level"] and i1["coarse_rebuilds"] >= 1
    mask, _, _ = make_mask(prob, seed=8)
    eng.set_edge_levels(mask)
    eng.linearize()
    assert eng.solve(lam)[1]
    i2 = eng.pcg_info()
    assert i2["coarse_rebuilds"] == i1["coarse_rebuilds"] + 1 and i2["bj_retries"] == 0 and i2["bad_rebuilds"] == 0, (i1, i2)
    assert i2["coarse_lambda"] == lam
    o = oracle.Oracle(zeroed(prob, mask), *rk)
    o.compute_errors(); o.build_system(); assert o.solve(lam)
    for nme, a, b in zip(("xp", "xl"), eng.delta(), o.delta()):
        assert relerr(a, b) < 1e-8, nme
    # every edge excluded: no iteration, the estimate stays
    before = eng.state()
    eng.set_edge_levels(np.ones(prob.nedges, np.uint8))
    assert eng.optimize(10) == []
    _bitwise(eng.state(), before, "state")
    eng.set_edge_levels(None)
    assert len(eng.optimize(1)) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("name,world", [("small", 3), ("shard_edges", 3)])
def test_levels_on_dry_shards(pkg, oracle, name, world, monkeypatch):
    """landmark sharding on one GPU (CUBA_DRY_SHARD): with a mask, every rank's partial system is the oracle's sub-problem system on
    the rank's edges; classify counts and get_edge_levels cover exactly the rank's own edges"""
    monkeypatch.setenv("CUBA_DRY_SHARD", "1")
    g, prob, planted = planted_problem(pkg, name)
    mask, _, _ = make_mask(prob, seed=9, planted=planted)
    rk = KERNELS["huber"]
    total = None
    own_all = np.zeros(prob.nedges, np.int64)
    for r in range(world):
        eng = pkg.Engine(device=0)
        for et in (0, 1):
            eng.set_robust_kernels(rk[0][et], rk[1][et], et)
        eng.set_comm(r, world)
        eng.initialize(prob)
        eng.linearize()
        own = np.zeros(prob.nedges, bool)
        own[eng.chi_squared() != 0] = True           # a rank reports the chi2 of its own edges only
        own_all += own
        eng.set_edge_levels(mask)
        lv = eng.edge_levels()
        assert np.array_equal(lv[own], mask[own]) and not lv[~own].any()
        eng.linearize()
        sysm = eng.system()
        total = sysm if total is None else tuple(a + b for a, b in zip(total, sysm))
        counts = eng.classify_edges(CHI2_MONO, CHI2_STEREO)
        lv2 = eng.edge_levels()
        assert not lv2[~own].any()
        mono = np.arange(prob.nedges) < prob.E2
        assert counts["included_mono"] == int(((lv2 == 0) & own & mono).sum())
        assert counts["included_stereo"] == int(((lv2 == 0) & own & ~mono).sum())
        assert counts["excluded"] == int((own & (mask == 0) & (lv2 != 0)).sum())
        # a dry rank judges "no edge included" on its own edges, whether the levels came from set_edge_levels or classify_edges
        eng.set_edge_levels(own.astype(np.uint8))
        assert eng.optimize(3) == []
        eng.set_edge_levels(own.astype(np.uint8))
        eng.classify_edges(CHI2_MONO, CHI2_STEREO)
        assert eng.optimize(3) == []
    assert (own_all == 1).all()
    o = oracle.Oracle(zeroed(prob, mask), *rk)
    o.compute_errors(); o.build_system()
    for nme, a, b in zip(("Hpp", "bp", "Hll", "bl", "Hpl"), total, o.system()):
        assert relerr(a, b) < 1e-10, nme


# ---- ORB-SLAM2's rounds through the drop-in class ---------------------------------------------------------
def _levels_from(st, prob):
    lm = np.array(st["mono_levels"]); ls = np.array(st["stereo_levels"])
    return np.concatenate([lm[prob.mono_rows], ls[prob.stereo_rows]]).astype(np.uint8)


def _run_protocol(pkg, oracle, tmp_path_factory, g, ops):
    """every opt step against the oracle on the sub-problem of the engine's own levels, from the written-back estimate"""
    steps, state = _drive(tmp_path_factory, pkg, g, ops)
    cur = {k: np.array(v, copy=True) for k, v in g.items()}
    prob = pkg.graphio.flatten(cur)
    mask = np.zeros(prob.nedges, np.uint8)
    rk = KERNELS["huber"]
    for st, op in zip(steps, ops):
        f = op.split(":")
        if f[0] == "kernel":
            rk = KERNELS[f[1]]
        elif f[0] == "classify":
            mask = _levels_from(st, prob)
            assert st["counts"][0] + st["counts"][1] == int((mask == 0).sum())
        elif f[0] == "level":
            rows = prob.mono_rows if f[1] == "m" else prob.stereo_rows
            k = int(np.nonzero(rows == int(f[2]))[0][0]) + (0 if f[1] == "m" else prob.E2)
            mask = mask.copy(); mask[k] = int(int(f[3]) != 0)
            assert not st["threw"], op
        elif f[0] == "levels":
            assert np.array_equal(_levels_from(st, prob), mask), op
        elif f[0] == "opt":
            sub = pkg.graphio.flatten(sub_graph(cur, prob, mask))
            o = oracle.Oracle(sub, *rk)
            chi, _, _ = o.optimize(int(f[1]))
            # once converged, whether an LM iteration still finds rho > 0 turns on last-bit differences between engine and oracle,
            # so the runs may stop a few iterations apart: the longer run's extra iterations must sit on the converged value
            n = min(len(st["chi2"]), len(chi))
            assert n >= 1 and np.allclose(st["chi2"][:n], chi[:n], rtol=1e-10, atol=0), (op, st["chi2"], chi)
            tail = list(st["chi2"][n:]) + list(chi[n:])
            assert all(abs(v - chi[n - 1]) <= 1e-12 * chi[n - 1] for v in tail), (op, st["chi2"], chi)
            q, t, Xw = o.state()
            pkg.graphio.write_back(cur, sub, q, t, Xw)
            prob = pkg.graphio.flatten(cur)
            # chiSquared(e) of every edge, excluded ones too, at the new estimate
            ocs = oracle.Oracle(prob, *rk).chi_sqs()
            cs = np.concatenate([np.array(st["mono_chi2"])[prob.mono_rows], np.array(st["stereo_chi2"])[prob.stereo_rows]])
            assert relerr(cs, ocs) < 1e-8, op
            assert (cs[mask != 0] > 0).all()
    q, t, Xw = state
    assert np.abs(q - cur["q"]).max() < 1e-9
    assert np.abs(t - cur["t"]).max() < 1e-8 * max(1.0, np.abs(cur["t"]).max())
    assert np.abs(Xw - cur["Xw"]).max() < 1e-8 * max(1.0, np.abs(cur["Xw"]).max())
    return steps


@pytest.mark.gpu
def test_levels_set_between_initialize_and_optimize(pkg, oracle, tmp_path_factory):
    """g2o's order: initialize(), setEdgeLevel(), optimize() -- the levels set after initialize() reach the engine; so do those set
    between two optimize() calls and those carried through a second (value-only) initialize()"""
    g, pm, ps = plant_outliers(pkg, pkg.synth.make_config("small"), seed=13)
    ops = ["kernel:huber", "init"] + ["level:m:%d:1" % r for r in pm[:20]] + ["level:s:%d:1" % r for r in ps[:20]] + \
          ["opt:5", "levels", "level:m:%d:0" % pm[0], "level:s:%d:1" % ps[20], "opt:3", "levels", "init", "opt:2", "levels"]
    steps = _run_protocol(pkg, oracle, tmp_path_factory, g, ops)
    assert sum(steps[-1]["mono_levels"]) == 19 and sum(steps[-1]["stereo_levels"]) == 21


@pytest.mark.gpu
def test_orbslam_local_ba(pkg, oracle, tmp_path_factory):
    g, _, _ = plant_outliers(pkg, pkg.synth.make_config("small"), seed=12)
    ops = ["kernel:huber", "init", "opt:5", "classify:5.991:7.815:1:0", "kernel:none", "opt:10", "classify:5.991:7.815:1:0", "levels"]
    steps = _run_protocol(pkg, oracle, tmp_path_factory, g, ops)
    assert steps[3]["counts"][2] > 0


@pytest.mark.gpu
def test_orbslam_pose_optimization(pkg, oracle, tmp_path_factory):
    """one free pose, every landmark fixed (the engine's pose-only path): four rounds with re-inclusion, NONE from round 3"""
    g = pkg.synth.make_config("small")
    g["lm_fixed"][:] = 1
    g["pose_fixed"][:] = 1
    p = len(g["pose_id"]) // 2
    g["pose_fixed"][p] = 0
    g["t"][p] += np.array([0.05, -0.03, 0.08])
    rows = np.nonzero(g["mono_vP"] == g["pose_id"][p])[0]
    g["mono_meas"][rows[::4]] += 30.0
    ops = ["kernel:huber", "init"]
    for r in range(4):
        if r == 2:
            ops.append("kernel:none")
        ops += ["opt:10", "classify:5.991:7.815:1:1"]
    steps = _run_protocol(pkg, oracle, tmp_path_factory, g, ops)
    assert any(s["counts"][2] > 0 for s in steps if s["op"].startswith("classify"))
