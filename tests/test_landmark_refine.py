"""Structure-only refinement of the engine's own landmarks in place (include/cuba_b200.h: cuba_engine_optimize_landmarks, _device;
csrc/cuba_landmark_refine.cuh), the Python front end (Engine.optimize_landmarks, optimize_landmarks_device) and the drop-in's
cuba::optimizeLandmarks (include/cuba_b200_points.h).

The problems are the planted synthetic graphs of test_edge_levels (measurements pushed 20-50 px, points moved behind a camera), every
landmark perturbed.  A refined landmark's reference is its point cut from the engine's state (get_state) and levels: the CPU oracle
round by round (test_point_batch.oracle_reference), and k_point_batch on the same point, which gives bitwise the same result when the
point's edges are listed in the order of the engine's stream."""
import json
import os
import subprocess

import numpy as np
import pytest

import test_edge_levels as tel
import test_point_batch as tpb
from conftest import KERNELS, ROOT, have_fixture, fixture_path
from test_dry_shards import dry_engine
from test_pose_batch import RTOL

CHI2_MONO, CHI2_STEREO = 5.991, 7.815
STEP = {"small": 13, "kitti07_shaped": 97}


def planted(pkg, name, seed=41):
    """the planted graph `name` as a flat problem, every landmark moved by 0.1 per coordinate (seeded)"""
    g, _, _ = tel.plant_outliers(pkg, pkg.synth.make_config(name), seed=seed)
    prob = pkg.graphio.flatten(g)
    prob.Xw = prob.Xw + np.random.default_rng(seed + 1).normal(0, 0.1, prob.Xw.shape)
    return prob


def engine(pkg, prob, kernel="none", solver="pcg", **kw):
    eng = pkg.Engine(device=0, **kw)
    eng.set_linear_solver(solver)
    rk = KERNELS[kernel]
    for et in (0, 1):
        eng.set_robust_kernels(rk[0][et], rk[1][et], et)
    eng.initialize(prob)
    return eng


def cut(pkg, eng, prob, landmarks):
    """the landmarks as a point batch at the engine's current state"""
    q, t, X = eng.state()
    p = prob.copy()
    p.q, p.t, p.Xw = q, t, X
    return pkg.graphio.point_batch(p, landmarks)


def stream_order(pkg, batch):
    """the batch with each point's edges in the order of the engine's stream: ascending pose, then edge id (mono edges before stereo
    ones only matters for a mixed point, whose order this cannot match)"""
    pts = []
    for b in range(batch.B):
        m = np.arange(batch.ptr2[b], batch.ptr2[b + 1])
        s = np.arange(batch.ptr3[b], batch.ptr3[b + 1])
        m = m[np.lexsort((batch.mono_ids[m], batch.iP2[m]))] - batch.ptr2[b]
        s = s[np.lexsort((batch.stereo_ids[s], batch.iP3[s]))] - batch.ptr3[b]
        pts.append(tpb.one_point(pkg, batch, b, m, s))
    out = tpb.concat(pkg, pts)
    perm = lambda ptr, ids, ip: np.concatenate([ids[ptr[b]:ptr[b + 1]][np.lexsort((ids[ptr[b]:ptr[b + 1]], ip[ptr[b]:ptr[b + 1]]))]
                                                for b in range(batch.B)] + [np.zeros(0, np.int64)])
    out.mono_ids = perm(batch.ptr2, batch.mono_ids, batch.iP2)
    out.stereo_ids = perm(batch.ptr3, batch.stereo_ids, batch.iP3)
    return out


def levels_of(batch, b, lev, E2):
    """point b's edges' levels from the engine's edge-id-ordered levels, in the batch's edge order (mono, then stereo)"""
    return np.concatenate([lev[batch.mono_ids[batch.ptr2[b]:batch.ptr2[b + 1]]], lev[E2 + batch.stereo_ids[batch.ptr3[b]:batch.ptr3[b + 1]]]])


def snapshot(eng):
    q, t, X = eng.state()
    return dict(q=q, t=t, Xw=X, levels=eng.edge_levels(), chi2=eng.chi_squared())


def same_snapshot(a, b, what=""):
    for k in a:
        assert np.array_equal(a[k], b[k]), (what, k)


# ---- no GPU ------------------------------------------------------------------------------------------------------------------
def test_symbols_declared_and_exported(pkg):
    with open(os.path.join(ROOT, "include", "cuba_b200.h")) as f:
        header = f.read()
    with open(os.path.join(ROOT, "include", "cuba_b200_points.h")) as f:
        points = f.read()
    L = pkg.load_library()
    for s in ("cuba_engine_optimize_landmarks", "cuba_engine_optimize_landmarks_device"):
        assert "int %s(" % s in header
        assert s in pkg.binding.exported_symbols()
        assert getattr(L, s) is not None
    assert "optimizeLandmarks(CudaBundleAdjustment& ba, const std::vector<PoseRound>& schedule);" in points


def test_refusals_without_gpu(pkg):
    """a NULL engine, and the schedule / n checks that run before the engine's problem is looked at"""
    L = pkg.load_library()
    rs = pkg.Engine._rounds_struct(tpb.schedules(pkg)["huber"])
    assert L.cuba_engine_optimize_landmarks(None, None, 0, 2, rs, None, None, None) == -1
    assert L.cuba_engine_optimize_landmarks_device(None, None, 0, 2, rs, None, None, None, None) == -1


def _build_driver(tmp_path_factory, pkg):
    out = str(tmp_path_factory.mktemp("cpplandmark") / "landmark_refine_driver")
    libdir = os.path.dirname(pkg.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCUBA_FORCE_EIGEN_COMPAT", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "landmark_refine_driver.cpp"), "-L", libdir, "-lcuba_b200",
                           "-Wl,-rpath," + libdir, "-o", out])
    return out


def test_driver_compiles_against_dropin_headers(pkg, tmp_path_factory):
    assert os.path.exists(_build_driver(tmp_path_factory, pkg))
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", pkg.library_path()], capture_output=True, text=True).stdout
    assert "cuba::optimizeLandmarks(" in out


# ---- on the GPU: 1. against the CPU oracle ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "kitti07_shaped"])
@pytest.mark.parametrize("sched", ["huber_depth", "none", "huber", "tukey"])
def test_against_oracle(pkg, oracle, name, sched):
    """one call per sampled landmark (its own counts), each against the oracle on its point cut before the calls"""
    prob = planted(pkg, name)
    L = np.arange(0, prob.numL, STEP[name])
    rounds = tpb.schedules(pkg)[sched]
    eng = engine(pkg, prob)
    batch = cut(pkg, eng, prob, L)
    runs = [eng.optimize_landmarks(rounds, [l], with_stats=True) for l in L]
    X, lev = eng.state()[2], eng.edge_levels()
    ties = via_engine = excluded = 0
    for b, (l, r) in enumerate(zip(L, runs)):
        got = dict(Xw=X[l], levels=levels_of(batch, b, lev, prob.E2), counts=r["counts"],
                   stats=pkg.Engine._round_stats(r["stats"][0], r["nstats"][0], rounds))
        nt, ve = tpb.check_against_oracle(pkg, oracle, batch, b, got, rounds, (name, sched, int(l)))
        ties += nt; via_engine += ve
        excluded += int(got["levels"].sum())
    assert excluded > 0 and via_engine <= len(L) // 10
    # the whole list in one call: the same engine state, and the per-landmark counts summed
    one = engine(pkg, prob)
    r = one.optimize_landmarks(rounds, L)
    assert np.array_equal(r["counts"], sum(x["counts"] for x in runs))
    same_snapshot(snapshot(one), snapshot(eng), (name, sched))


# ---- 2. against k_point_batch ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "kitti07_shaped"])
@pytest.mark.parametrize("sched", ["huber_depth", "tukey"])
def test_against_point_batch(pkg, oracle, name, sched):
    prob = planted(pkg, name)
    rounds = tpb.schedules(pkg)[sched]
    L = np.arange(0, prob.numL, 3 if name == "small" else 29)
    eng = engine(pkg, prob)
    batch = stream_order(pkg, cut(pkg, eng, prob, L))
    ref = pkg.Engine(device=0).optimize_points_flat(rounds=rounds, **batch.arrays())
    got = eng.optimize_landmarks(rounds, L, with_stats=True)
    X, lev = eng.state()[2], eng.edge_levels()
    nm, ns = np.diff(batch.ptr2), np.diff(batch.ptr3)
    pure = (nm == 0) | (ns == 0)
    assert pure.sum() > 0 and (~pure).sum() > 0
    written = lambda st, n: tpb._written(st[None], n[None], rounds)
    E2 = len(batch.omega2)
    same_levels = True
    for b in range(batch.B):
        mine = levels_of(batch, b, lev, prob.E2)
        theirs = np.concatenate([ref["levels"][batch.ptr2[b]:batch.ptr2[b + 1]], ref["levels"][E2 + batch.ptr3[b]:E2 + batch.ptr3[b + 1]]])
        if pure[b]:
            assert np.array_equal(X[L[b]], ref["Xw"][b]), b
            assert np.array_equal(mine, theirs), b
            assert np.array_equal(got["nstats"][b], ref["nstats"][b]), b
            assert written(got["stats"][b], got["nstats"][b]) == written(ref["stats"][b], ref["nstats"][b]), b
        else:
            # the same problem summed in another order: the point batch's tolerances against the point batch's result
            # (a landmark's own counts are not an output of the in-place call: the totals are checked below)
            same_levels &= bool(np.array_equal(mine, theirs))
            r = dict(Xw=ref["Xw"][b], levels=theirs, counts=[], near=np.ones(len(theirs), bool),
                     stats=[([s["chi2"] for s in st], [s["lambda_"] for s in st], [s["trials"] for s in st])
                            for st in pkg.Engine._round_stats(ref["stats"][b], ref["nstats"][b], rounds)])
            g = dict(Xw=X[L[b]], levels=mine, counts=[],
                     stats=pkg.Engine._round_stats(got["stats"][b], got["nstats"][b], rounds))
            tpb.check_point(g, r, (name, sched, b), H=tpb.hessian(oracle, batch, b, g["Xw"]), scale=tpb.start_chi2(oracle, batch, b, rounds))
    if same_levels:
        assert np.array_equal(got["counts"], ref["counts"].sum(0))


# ---- 3. the engine afterwards ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["none", "huber", "tukey"])
@pytest.mark.parametrize("solver", ["pcg", "dense"])
@pytest.mark.parametrize("precision", ["fp64", "mixed"])
def test_engine_afterwards(pkg, kernel, solver, precision):
    """an engine after the call against one given set_state / set_edge_levels with its results: optimize(10), get_state, get_chi2
    and classify_edges bitwise"""
    prob = planted(pkg, "small")
    kw = dict(use_fp32="mixed") if precision == "mixed" else {}
    a, b = engine(pkg, prob, kernel, solver, **kw), engine(pkg, prob, kernel, solver, **kw)
    for e in (a, b):
        e.optimize(3)
        e.classify_edges(CHI2_MONO, CHI2_STEREO)
    a.optimize_landmarks(tpb.schedules(pkg)["huber_depth"])
    q, t, X = a.state()
    b.set_state(q, t, X)
    b.set_edge_levels(a.edge_levels())
    same_snapshot(snapshot(a), snapshot(b))
    assert a.optimize(10) == b.optimize(10)
    same_snapshot(snapshot(a), snapshot(b))
    assert a.classify_edges(CHI2_MONO, CHI2_STEREO, reinclude=True) == b.classify_edges(CHI2_MONO, CHI2_STEREO, reinclude=True)
    assert a.optimize(5) == b.optimize(5)
    same_snapshot(snapshot(a), snapshot(b))


# ---- 4. levels carried in ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_levels_carried_in(pkg):
    R = pkg.PoseRound
    prob = planted(pkg, "small")
    eng = engine(pkg, prob)
    rng = np.random.default_rng(3)
    mask = (rng.random(prob.nedges) < 0.1).astype(np.uint8)
    # edges of landmark 0 all at level 1: bitwise where it was, no iteration
    l0 = 0
    il = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    mask[il == l0] = 1
    eng.set_edge_levels(mask)
    X0 = eng.state()[2]
    r = eng.optimize_landmarks([R(10, restart=False, reinclude=False), R(5, restart=False, reinclude=False)], with_stats=True)
    lev = eng.edge_levels()
    assert np.all(lev[mask == 1] == 1)                       # no re-inclusion: excluded edges stay excluded
    assert np.array_equal(eng.state()[2][l0], X0[l0]) and not r["nstats"][l0].any()
    assert r["counts"][0][0] + r["counts"][0][1] == int((lev[il < prob.numL] == 0).sum()) + r["counts"][1][2] - r["counts"][1][3]
    # with re-inclusion they come back where the test passes
    r = eng.optimize_landmarks([R(10, restart=False, reinclude=True)])
    back = (lev == 1) & (eng.edge_levels() == 0)
    assert r["counts"][0][3] == int(back.sum()) > 0
    # every edge of the listed landmarks excluded, the others already out: a following optimize() runs no iteration
    eng.set_edge_levels(np.where(np.isin(il, [1, 2, 3]), 0, 1).astype(np.uint8))
    r = eng.optimize_landmarks([R(3, chi2_mono=-1.0, chi2_stereo=-1.0)], [1, 2, 3])
    assert r["counts"][0][0] + r["counts"][0][1] == 0 and r["counts"][0][2] == int(np.isin(il, [1, 2, 3]).sum())
    assert eng.optimize(5) == []


# ---- 5. lists ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_lists(pkg):
    rounds = tpb.schedules(pkg)["huber"]
    prob = planted(pkg, "small")
    il = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    rng = np.random.default_rng(5)
    sub = np.sort(rng.choice(prob.numL, prob.numL // 5, replace=False))
    full = engine(pkg, prob)
    rf = full.optimize_landmarks(rounds, with_stats=True)
    a = engine(pkg, prob)
    before = snapshot(a)
    ra = a.optimize_landmarks(rounds, sub, with_stats=True)
    after = snapshot(a)
    other = np.setdiff1d(np.arange(prob.Lall), sub)
    assert np.array_equal(after["Xw"][other], before["Xw"][other]) and np.array_equal(after["q"], before["q"])
    assert np.array_equal(after["levels"][~np.isin(il, sub)], before["levels"][~np.isin(il, sub)])
    f = snapshot(full)
    assert np.array_equal(after["Xw"][sub], f["Xw"][sub])
    assert np.array_equal(after["levels"][np.isin(il, sub)], f["levels"][np.isin(il, sub)])
    assert np.array_equal(ra["nstats"], rf["nstats"][sub])
    assert tpb._written(ra["stats"], ra["nstats"], rounds) == tpb._written(rf["stats"][sub], rf["nstats"][sub], rounds)
    # a permuted list: permuted outputs, the same engine
    perm = rng.permutation(len(sub))
    p = engine(pkg, prob)
    rp = p.optimize_landmarks(rounds, sub[perm], with_stats=True)
    same_snapshot(snapshot(p), after)
    assert np.array_equal(rp["counts"], ra["counts"]) and np.array_equal(rp["nstats"], ra["nstats"][perm])
    assert tpb._written(rp["stats"], rp["nstats"], rounds) == tpb._written(ra["stats"][perm], ra["nstats"][perm], rounds)
    # an empty list: nothing launched, zero counts
    n0 = p.launch_count()
    r0 = p.optimize_landmarks(rounds, np.zeros(0, np.int32))
    assert p.launch_count() == n0 and not r0["counts"].any() and r0["counts"].shape == (2, 4)
    same_snapshot(snapshot(p), after)


# ---- 6. refusals ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals(pkg):
    import torch
    R = pkg.PoseRound
    rounds = tpb.schedules(pkg)["huber"]
    prob = planted(pkg, "small")
    eng = engine(pkg, prob)
    eng.optimize(2)
    eng.classify_edges(CHI2_MONO, CHI2_STEREO)
    good = snapshot(eng)
    L = pkg.load_library()
    rs = pkg.Engine._rounds_struct(rounds)
    fixed = prob.numL if prob.Lall > prob.numL else prob.numL + 5
    cases = {
        "no rounds": ([], None), "nine rounds": ([R()] * 9, None), "negative iterations": ([R(-1)], None),
        "kernel type": ([R(kernel=(0, 3))], None), "fixed": (rounds, [0, fixed]), "negative": (rounds, [4, -1]), "repeated": (rounds, [3, 7, 3]),
    }
    for what, (rd, lst) in cases.items():
        with pytest.raises(pkg.CubaError, match="error -1"):
            eng.optimize_landmarks(rd, lst)
        msg = L.cuba_last_error().decode()
        assert ("optimize_points" if lst is None else "optimize_landmarks") in msg, (what, msg)
        same_snapshot(snapshot(eng), good, what)
        if lst is not None:
            nst = torch.full((len(lst), 2), 7, dtype=torch.int32, device="cuda:0")
            st = torch.full((len(lst), 20, 4), 7.0, dtype=torch.float64, device="cuda:0")
            out = dict(nstats=nst.clone(), stats=st.clone())
            with pytest.raises(pkg.CubaError, match="error -1"):
                eng.optimize_landmarks_device(rd, torch.tensor(lst, dtype=torch.int32, device="cuda:0"), out=out)
            assert torch.equal(out["nstats"], nst) and torch.equal(out["stats"], st), what
            same_snapshot(snapshot(eng), good, what + " (device)")
    # n < 0, and NULL with n != numL, through the C ABI
    assert L.cuba_engine_optimize_landmarks(eng.h, None, -1, 2, rs, None, None, None) == -1
    assert L.cuba_engine_optimize_landmarks(eng.h, None, prob.numL - 1, 2, rs, None, None, None) == -1
    assert L.cuba_engine_optimize_landmarks_device(eng.h, None, prob.numL + 1, 2, rs, None, None, None, None) == -1
    same_snapshot(snapshot(eng), good)
    # the fp32 engine, and a call before set_problem
    f32 = engine(pkg, prob, use_fp32=True)
    with pytest.raises(pkg.CubaError, match="fp32"):
        f32.optimize_landmarks(rounds)
    fresh = pkg.Engine(device=0)
    assert L.cuba_engine_optimize_landmarks(fresh.h, None, 0, 2, rs, None, None, None) == -3


# ---- 7. the device entry ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_entry(pkg):
    import torch
    rounds = tpb.schedules(pkg)["huber_depth"]
    R = len(rounds)
    prob = planted(pkg, "small")
    L = np.arange(1, prob.numL, 2)[::-1].copy()
    h = engine(pkg, prob)
    rh = h.optimize_landmarks(rounds, L, with_stats=True)
    d = engine(pkg, prob)
    dl = torch.tensor(L, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    h2d0, d2h0 = pkg.transfer_bytes()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        dl2 = torch.empty_like(dl)
        dl2.copy_(dl)                  # written on the side stream right before the call
        rd = d.optimize_landmarks_device(rounds, dl2)
        nst = rd["nstats"].clone()     # read on it right after
    side.synchronize()
    h2d1, d2h1 = pkg.transfer_bytes()
    assert (h2d1 - h2d0, d2h1 - d2h0) == (0, 8 * (4 * R + 1))
    assert np.array_equal(rd["counts"], rh["counts"]) and np.array_equal(nst.cpu().numpy(), rh["nstats"])
    assert tpb._written(pkg.binding.stats_view(rd["stats"]), rh["nstats"], rounds) == tpb._written(rh["stats"], rh["nstats"], rounds)
    same_snapshot(snapshot(d), snapshot(h))
    # NULL list: every free landmark, without stats
    a, b = engine(pkg, prob), engine(pkg, prob)
    ra = a.optimize_landmarks(rounds)
    rb = b.optimize_landmarks_device(rounds, with_stats=False)
    assert rb["stats"] is None and np.array_equal(rb["nstats"].cpu().numpy(), ra["nstats"]) and np.array_equal(rb["counts"], ra["counts"])
    same_snapshot(snapshot(a), snapshot(b))
    # the Python checks fire before any library call
    n0 = d.launch_count()
    bad = {"dtype": dl.to(torch.int64), "device": dl.cpu(), "shape": dl.reshape(-1, 1), "contiguity": torch.stack([dl, dl], 1)[:, 0]}
    for what, t in bad.items():
        with pytest.raises((TypeError, ValueError)):
            d.optimize_landmarks_device(rounds, t)
    with pytest.raises(ValueError):
        d.optimize_landmarks_device(rounds, dl, out=dict(nstats=torch.zeros((len(L), R + 1), dtype=torch.int32, device="cuda:0"),
                                                          stats=rd["stats"]))
    assert d.launch_count() == n0


# ---- 8. landmark-sharded runs -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_dry_shards(pkg, world):
    rounds = tpb.schedules(pkg)["huber_depth"]
    prob = planted(pkg, "small")
    one = engine(pkg, prob)
    r1 = one.optimize_landmarks(rounds, with_stats=True)
    X1, lev1 = one.state()[2], one.edge_levels()
    il = np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]])
    tot = np.zeros_like(r1["counts"])
    for r in range(world):
        eng = dry_engine(pkg, prob, KERNELS["none"], r, world)
        lo, hi = (int(v) for v in pkg.build_structure_host(prob, r, world)["shard"][:2])
        rr = eng.optimize_landmarks(rounds, with_stats=True)
        tot += rr["counts"]
        own = np.arange(prob.numL)
        own = own[(own >= lo) & (own < hi)]
        others = np.setdiff1d(np.arange(prob.numL), own)
        assert np.array_equal(eng.state()[2][own], X1[own])
        assert np.array_equal(eng.edge_levels()[np.isin(il, own)], lev1[np.isin(il, own)])
        assert np.array_equal(rr["nstats"][own], r1["nstats"][own]) and not rr["nstats"][others].any()
        assert tpb._written(rr["stats"][own], rr["nstats"][own], rounds) == tpb._written(r1["stats"][own], r1["nstats"][own], rounds)
        assert not rr["stats"][others].view(np.uint8).any()
    assert np.array_equal(tot, r1["counts"])


# ---- 9. the drop-in -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dropin_optimize_landmarks(pkg, tmp_path_factory):
    g, _, _ = tel.plant_outliers(pkg, pkg.synth.make_config("tiny"), seed=43)
    g["Xw"] = g["Xw"] + np.random.default_rng(44).normal(0, 0.1, g["Xw"].shape)
    path = str(tmp_path_factory.mktemp("landmarks") / "graph.cubagraph")
    pkg.graphio.write_graph(path, g)
    out = subprocess.run([_build_driver(tmp_path_factory, pkg), path], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    res = json.loads(out.stdout)
    assert res["threw_state"] and (res["threw_fixed"] or not res["has_fixed"])
    assert [r["all"] for r in res["runs"]] == [False, True]
    for run in res["runs"]:
        assert len(run["points"]) > 0 and len(run["counts"]) == 2
        ties = 0
        for pt in run["points"]:
            x, ref = np.array(pt["Xw"]), np.array(pt["ref"])
            assert np.abs(x - ref).max() <= 1e-7 * max(1.0, np.abs(ref).max()), pt
            lv = np.array(pt["levels"]).reshape(-1, 2)
            ties += int((lv[:, 0] != lv[:, 1]).sum())
            if np.abs(x - ref).max() <= RTOL * max(1.0, np.abs(ref).max()):
                assert np.array_equal(lv[:, 0], lv[:, 1]), pt
        assert ties <= 2, ties
        inl = sum(int((np.array(pt["levels"]).reshape(-1, 2)[:, 0] == 0).sum()) for pt in run["points"])
        assert run["counts"][-1][0] + run["counts"][-1][1] == inl


# ---- ba_kitti_00 ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.skipif(not have_fixture("ba_kitti_00"), reason="oracle/_ref/fixtures/ba_kitti_00.cubagraph not built")
def test_kitti_against_point_batch(pkg):
    """every landmark of ba_kitti_00 in one call against k_point_batch on the points in stream order: bitwise for single-type
    landmarks, within 1e-6 for the others"""
    prob = pkg.graphio.flatten(pkg.graphio.read_graph(fixture_path("ba_kitti_00")))
    rounds = tpb.schedules(pkg)["huber_depth"]
    L = np.arange(0, prob.numL, 7)
    eng = engine(pkg, prob)
    batch = stream_order(pkg, cut(pkg, eng, prob, L))
    ref = pkg.Engine(device=0).optimize_points_flat(rounds=rounds, **batch.arrays())
    eng.optimize_landmarks(rounds, L)
    X = eng.state()[2][L]
    pure = (np.diff(batch.ptr2) == 0) | (np.diff(batch.ptr3) == 0)
    assert np.array_equal(X[pure], ref["Xw"][pure])
    assert np.abs(X - ref["Xw"]).max() <= 1e-6 * max(1.0, np.abs(ref["Xw"]).max())
