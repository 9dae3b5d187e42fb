"""Structure-only refinement of many map points in one launch (include/cuba_b200.h: cuba_engine_optimize_points, _points_device,
csrc/cuba_point_batch.cuh), the Python front end (Engine.optimize_points, graphio.point_batch) and the drop-in's cuba::optimizePoints
(include/cuba_b200_points.h).

Points are cut from the synthetic graphs with outliers planted as in test_edge_levels (measurements pushed 20-50 px, points moved
behind a camera), every point perturbed.  The reference for a point is the CPU oracle on the point's sub-problem (its landmark-only
branch) without its edges at level 1, round by round, with the outlier test restated in numpy; the engine's own per-point path
(set_problem + set_robust_kernel / set_state / optimize / classify_edges per round) is a second reference."""
import json
import os
import subprocess

import numpy as np
import pytest

import test_edge_levels as tel
from conftest import KERNELS, ROOT, make_engine
from test_pose_batch import RTOL

CHI2_MONO, CHI2_STEREO = 5.991, 7.815
# The floor of a chi2 comparison: 1e-12 of the point's chi2 at its input position (`scale`), at least CHI2_FLOOR px^2.  A point with
# few edges (one stereo edge, one or two mono edges) fits them almost exactly; its chi2 after a step is then a small remainder of
# residuals taken from pixel coordinates of ~1e3, through a 3x3 solve whose condition grows with depth over baseline, and two
# solves of the same system leave remainders that differ far above 1e-10 of themselves, though not of where the point started.
CHI2_FLOOR = 1e-14


# ---- points and schedules ---------------------------------------------------------------------------------
_cut = {}


def cut_points(pkg, name, step=1, seed=41):
    """every step-th landmark of the planted graph `name` as a point against the graph's pose table, perturbed by 0.1 per
    coordinate (cached: callers must not modify it)"""
    if (name, step, seed) not in _cut:
        g, _, _ = tel.plant_outliers(pkg, pkg.synth.make_config(name), seed=seed)
        prob = pkg.graphio.flatten(g)
        batch = pkg.graphio.point_batch(prob, np.arange(0, prob.Lall, step))
        batch.Xw = batch.Xw + np.random.default_rng(seed + 1).normal(0, 0.1, batch.Xw.shape)
        _cut[(name, step, seed)] = batch
    return _cut[(name, step, seed)]


def schedules(pkg):
    R = pkg.PoseRound
    hub = dict(kernel=KERNELS["huber"][0], delta=KERNELS["huber"][1])
    tuk = dict(kernel=KERNELS["tukey"][0], delta=KERNELS["tukey"][1])
    return {
        # local-BA-like: depth test, no re-inclusion, each round from the last one's result (the timing tool's schedule)
        "huber_depth": [R(5, restart=False, depth=True, reinclude=False, **hub), R(10, restart=False, depth=True, reinclude=False)],
        "none": [R(10, restart=False), R(10, depth=True)],
        "huber": [R(10, restart=False, **hub), R(10, **hub)],
        "tukey": [R(10, restart=False, **tuk), R(10, depth=True, reinclude=False, **tuk)],
    }


def one_point(pkg, batch, b, mono=None, stereo=None, Xw=None):
    """point b of batch (against the same pose table) with its mono / stereo edges (indices within the point; default all)"""
    m0, s0 = batch.ptr2[b], batch.ptr3[b]
    m = m0 + (np.arange(batch.ptr2[b + 1] - m0) if mono is None else np.asarray(mono, np.int64))
    s = s0 + (np.arange(batch.ptr3[b + 1] - s0) if stereo is None else np.asarray(stereo, np.int64))
    return pkg.graphio.PointBatch(
        q=batch.q, t=batch.t, cam=batch.cam, Xw=np.array(batch.Xw[b] if Xw is None else Xw, dtype=np.float64).reshape(1, 3),
        ptr2=np.array([0, len(m)], np.int32), iP2=batch.iP2[m], meas2=batch.meas2[m].reshape(-1, 2), omega2=batch.omega2[m],
        ptr3=np.array([0, len(s)], np.int32), iP3=batch.iP3[s], meas3=batch.meas3[s].reshape(-1, 3), omega3=batch.omega3[s])


def concat(pkg, batches):
    """one PointBatch of the points of several, their pose tables stacked"""
    P = np.cumsum([0] + [len(x.q) for x in batches])
    cat = lambda k: np.concatenate([getattr(x, k) for x in batches])
    ptr = lambda k: np.concatenate([[0], np.cumsum(np.concatenate([np.diff(getattr(x, k)) for x in batches]))]).astype(np.int32)
    return pkg.graphio.PointBatch(
        q=cat("q"), t=cat("t"), cam=cat("cam"), Xw=cat("Xw").reshape(-1, 3), ptr2=ptr("ptr2"),
        iP2=np.concatenate([x.iP2 + p for x, p in zip(batches, P)]).astype(np.int32), meas2=cat("meas2").reshape(-1, 2),
        omega2=cat("omega2"), ptr3=ptr("ptr3"), iP3=np.concatenate([x.iP3 + p for x, p in zip(batches, P)]).astype(np.int32),
        meas3=cat("meas3").reshape(-1, 3), omega3=cat("omega3"))


def select(pkg, batch, rows):
    return concat(pkg, [one_point(pkg, batch, b) for b in rows])


# ---- the references -------------------------------------------------------------------------------------------
def classify(pkg, oracle, batch, b, X, lev, r):
    """the outlier test of classify_edges restated on point b at X: (new levels, counts, edges within 1e-9 of a threshold)"""
    E2 = int(batch.ptr2[b + 1] - batch.ptr2[b])
    E = E2 + int(batch.ptr3[b + 1] - batch.ptr3[b])
    if E == 0:
        return lev, [0, 0, 0, 0], np.zeros(0, bool)
    full = batch.sub_problem(b, X)
    chi = oracle.Oracle(full).chi_sqs()
    ip = np.concatenate([full.idx2[:, 0], full.idx3[:, 0]])
    depth = (pkg.synth._rotate(full.q[ip], np.repeat(full.Xw, E, 0)) + full.t[ip])[:, 2]
    mono = np.arange(E) < E2
    thr = np.where(mono, r.chi2_mono, r.chi2_stereo)
    fail = (chi > thr) | ((depth <= 0) if r.depth else False)
    new = (fail if r.reinclude else (lev.astype(bool) | fail)).astype(np.uint8)
    counts = [int(((new == 0) & mono).sum()), int(((new == 0) & ~mono).sum()), int(((lev == 0) & (new != 0)).sum()),
              int(((lev != 0) & (new == 0)).sum())]
    return new, counts, np.abs(chi - thr) <= 1e-9 * np.abs(thr)


def oracle_reference(pkg, oracle, batch, b, rounds):
    """round by round: the oracle on the sub-problem without the edges at level 1, then the restated test"""
    E = int(batch.ptr2[b + 1] - batch.ptr2[b] + batch.ptr3[b + 1] - batch.ptr3[b])
    X = batch.Xw[b].copy()
    lev = np.zeros(E, np.uint8)
    out = dict(stats=[], counts=[], near=np.zeros(E, bool))
    for r in rounds:
        if r.restart:
            X = batch.Xw[b].copy()
        keep = lev == 0
        traj = ([], [], [])
        if keep.any() and r.iterations > 0:
            o = oracle.Oracle(batch.sub_problem(b, X, keep), tuple(r.kernel), tuple(r.delta))
            traj = o.optimize(r.iterations)
            X = o.state()[2][0].copy()
        out["stats"].append(traj)
        lev, c, near = classify(pkg, oracle, batch, b, X, lev, r)
        out["counts"].append(c)
        out["near"] |= near
    out.update(Xw=X, levels=lev)
    return out


def engine_reference(pkg, batch, b, rounds):
    """the engine's own path for one point: set_problem, then per round set_robust_kernel, set_state on restart, optimize, classify"""
    full = batch.sub_problem(b)
    out = dict(stats=[], counts=[])
    if full.nedges == 0:
        out.update(Xw=batch.Xw[b].copy(), levels=np.zeros(0, np.uint8), stats=[([], [], [])] * len(rounds), counts=[[0] * 4] * len(rounds))
        return out
    eng = pkg.Engine(device=0)
    eng.initialize(full)
    for r in rounds:
        for et in (0, 1):
            eng.set_robust_kernels(r.kernel[et], r.delta[et], et)
        if r.restart:
            eng.set_state(full.q, full.t, full.Xw)
        st = eng.optimize(r.iterations)
        out["stats"].append(([s["chi2"] for s in st], [s["lambda_"] for s in st], [s["trials"] for s in st]))
        c = eng.classify_edges(r.chi2_mono, r.chi2_stereo, depth=r.depth, reinclude=r.reinclude)
        out["counts"].append([c["included_mono"], c["included_stereo"], c["excluded"], c["reincluded"]])
    out.update(Xw=eng.state()[2][0], levels=eng.edge_levels())
    eng.close()
    return out


def check_trajectory(got, ref, what, rtol=RTOL, scale=0.0):
    """test_pose_batch.check_trajectory with the floor of `scale` (see CHI2_FLOOR) besides the relative one: chi2 per iteration to rtol;
    runs that stop a few iterations apart once converged must sit on the converged value; trial counts, and lambda to 1e-6, over
    the leading iterations whose decrease is far above rounding.  Returns whether the two runs made the same number of iterations."""
    chi, lam, tr = (np.asarray(v, dtype=np.float64) for v in ref)
    g = np.array([s["chi2"] for s in got])
    if len(chi) == 0 or len(g) == 0:
        assert len(chi) == len(g), (what, g, chi)
        return True
    floor = max((1e-12 if rtol <= RTOL else rtol) * max(abs(chi[0]), abs(g[0]), scale), CHI2_FLOOR)
    n = min(len(g), len(chi))
    assert np.all(np.abs(g[:n] - chi[:n]) <= rtol * np.abs(chi[:n]) + floor), (what, g, chi)
    tail = list(g[n:]) + list(chi[n:])
    assert all(abs(v - chi[n - 1]) <= max(1e-12, rtol) * abs(chi[n - 1]) + floor for v in tail), (what, g, chi)
    k = 1
    while k < n and chi[k - 1] - chi[k] > 1e-6 * abs(chi[k - 1]) + floor:
        k += 1
    if k > 1 and rtol <= RTOL:
        assert [s["trials"] for s in got[:k]] == [int(x) for x in tr[:k]], (what, got[:k], tr[:k])
        gl = np.array([s["lambda_"] for s in got[:k]])
        assert np.allclose(gl, lam[:k], rtol=1e-6, atol=0), (what, gl, lam[:k])
    return len(g) == len(chi)


def hessian(oracle, batch, b, X):
    """Hll of point b's sub-problem at X, every edge, no robust kernel (the oracle's build_system)"""
    o = oracle.Oracle(batch.sub_problem(b, X))
    o.compute_errors()
    o.build_system()
    return o.system()[2][0].reshape(3, 3)


def start_chi2(oracle, batch, b, rounds):
    """the robust chi2 of point b at its input position under the first round's kernels: the `scale` of check_trajectory"""
    if batch.ptr2[b + 1] - batch.ptr2[b] + batch.ptr3[b + 1] - batch.ptr3[b] == 0:
        return 0.0
    return oracle.Oracle(batch.sub_problem(b), tuple(rounds[0].kernel), tuple(rounds[0].delta)).compute_errors()


def check_point(got, ref, what, exact_levels=False, rtol=RTOL, H=None, scale=0.0):
    """chi2 trajectories (check_trajectory); Xw to rtol relative to max(1, |Xw|) when every round ran as many iterations as the
    reference (1e-7 otherwise: a converged plateau leaves the point free to ~sqrt(eps)) or, given H (the point's Hll), where the two
    positions differ by less than (1e-9 of the chi2, at least 1e-9) in the metric of H: along a direction that the edges barely
    constrain (a short baseline, a rank-2 single mono edge) the solves of the same system land apart by far more than rounding
    without a difference in chi2; levels exact except at threshold ties, or exact with counts"""
    same = all([check_trajectory(gs, rs, (what, r), rtol, scale) for r, (gs, rs) in enumerate(zip(got["stats"], ref["stats"]))])
    xtol = (RTOL if same and rtol <= RTOL else 1e-7) * max(1.0, np.abs(ref["Xw"]).max())
    d = np.asarray(got["Xw"]) - np.asarray(ref["Xw"])
    if H is not None and np.abs(d).max() > xtol:
        final = [st[-1]["chi2"] for st in got["stats"] if st]
        assert d @ H @ d <= 1e-9 * max(1.0, final[-1] if final else 0.0), (what, got["Xw"], ref["Xw"], d @ H @ d)
    else:
        assert np.abs(d).max() <= xtol, (what, got["Xw"], ref["Xw"])
    bad = np.nonzero(got["levels"] != ref["levels"])[0]
    if exact_levels:
        assert len(bad) == 0, (what, bad)
        assert [list(c) for c in got["counts"]] == [list(c) for c in ref["counts"]], (what, got["counts"], ref["counts"])
        return 0
    assert ref["near"][bad].all(), (what, bad)
    if len(bad) == 0:
        assert [list(c) for c in got["counts"]] == [list(c) for c in ref["counts"]], (what, got["counts"], ref["counts"])
    return len(bad)


def check_against_oracle(pkg, oracle, batch, b, got, rounds, what):
    """the oracle to RTOL; where an ill-conditioned point rounds apart by more than that, it must equal the engine's own path to RTOL
    with identical levels, and the oracle to 1e-7.  Returns (threshold ties, 1 if the point needed the engine path)"""
    ref = oracle_reference(pkg, oracle, batch, b, rounds)
    H = hessian(oracle, batch, b, got["Xw"]) if len(got["levels"]) else None
    F0 = start_chi2(oracle, batch, b, rounds)
    try:
        return check_point(got, ref, what, H=H, scale=F0), 0
    except AssertionError:
        check_point(got, engine_reference(pkg, batch, b, rounds), what, exact_levels=True, H=H, scale=F0)
        return check_point(got, ref, what, rtol=1e-7, H=H, scale=F0), 1


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(x["Xw"], y["Xw"]) and np.array_equal(x["levels"], y["levels"])
        assert np.array_equal(x["counts"], y["counts"]) and x["stats"] == y["stats"]


# ---- no GPU ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny", "small"])
def test_point_batch_matches_one_landmark_subgraphs(pkg, name):
    """graphio.point_batch / PointBatch.sub_problem against flatten() of the graph of one landmark, free, with its edges and their
    poses, fixed (pose order aside: flatten orders the poses by id, sub_problem by table index)"""
    g = pkg.synth.make_config(name)
    prob = pkg.graphio.flatten(g)
    rows = np.arange(0, prob.Lall, 7)
    batch = pkg.graphio.point_batch(prob, rows)
    assert batch.B == len(rows) and np.array_equal(batch.landmarks, rows)
    for b, l in enumerate(rows):
        lid = g["lm_id"][prob.lm_rows[l]]
        s = {k: np.array(v, copy=True) for k, v in g.items()}
        s["pose_fixed"][:] = 1
        s["lm_fixed"][:] = 1
        s["lm_fixed"][prob.lm_rows[l]] = 0
        for kind in ("mono", "stereo"):
            keep = s[kind + "_vL"] == lid
            for k in ("_vP", "_vL", "_meas", "_info"):
                s[kind + k] = s[kind + k][keep]
        sub = pkg.graphio.flatten(s)
        got = batch.sub_problem(b)
        assert (got.Pall, got.numP, got.Lall, got.numL) == (sub.Pall, 0, 1, 1)
        assert np.array_equal(got.Xw, sub.Xw) and np.array_equal(batch.Xw[b], prob.Xw[l])
        for idx, gi, meas, gm, om, go in ((sub.idx2, got.idx2, sub.meas2, got.meas2, sub.omega2, got.omega2),
                                          (sub.idx3, got.idx3, sub.meas3, got.meas3, sub.omega3, got.omega3)):
            assert np.array_equal(meas, gm) and np.array_equal(om, go) and np.all(gi[:, 1] == 0)
            for a in ("q", "t", "cam"):
                assert np.array_equal(getattr(sub, a)[idx[:, 0]], getattr(got, a)[gi[:, 0]])
        # the point's edges name the flat problem's poses
        assert np.array_equal(batch.iP2[batch.ptr2[b]:batch.ptr2[b + 1]], prob.idx2[batch.mono_ids[batch.ptr2[b]:batch.ptr2[b + 1]], 0])
        assert np.all(prob.idx3[batch.stereo_ids[batch.ptr3[b]:batch.ptr3[b + 1]], 1] == l)
    # every edge belongs to exactly one point
    every = pkg.graphio.point_batch(prob, range(prob.Lall))
    assert np.array_equal(np.sort(every.mono_ids), np.arange(prob.E2)) and np.array_equal(np.sort(every.stereo_ids), np.arange(prob.E3))
    # keep: the kept edges only, and the poses they name
    k = every.sub_problem(0, keep=np.arange(every.ptr2[1] + every.ptr3[1]) % 2 == 0)
    assert k.nedges == (every.ptr2[1] + every.ptr3[1] + 1) // 2


def test_point_workspace_bytes(pkg):
    L = pkg.load_library()
    rs = pkg.Engine._rounds_struct(schedules(pkg)["huber_depth"])
    for B, P, E2, E3, ws in ((1, 1, 1, 0, 1), (5, 3, 17, 4, 0), (1000, 40, 4000, 300, 1)):
        R, S = 2, 15
        E = E2 + E3
        nIn = 4 * B + 16 * P + 4 * E + (E + 2 * (B + 1) + 1) // 2
        nOut = 4 * B + 4 * (B * S if ws else 0) + (5 * B * R + 1) // 2 + (E + 7) // 8
        assert L.cuba_point_batch_workspace_bytes(B, P, E2, E3, 2, rs, ws) == 8 * (nIn + nOut), (B, P, E2, E3, ws)
    bad = pkg.Engine._rounds_struct([pkg.PoseRound(-1)])
    for args in ((0, 1, 1, 1, 2, rs, 1), (-1, 1, 1, 1, 2, rs, 1), (1, -1, 1, 1, 2, rs, 1), (1, 1, -1, 1, 2, rs, 1), (1, 1, 1, -1, 2, rs, 1),
                 (1, 1, 1, 1, 0, rs, 1), (1, 1, 1, 1, 9, rs, 1), (1, 1, 1, 1, 1, bad, 1), (1, 1, 1, 1, 2, None, 1)):
        assert L.cuba_point_batch_workspace_bytes(*args) == 0, args
    for s in ("cuba_engine_optimize_points", "cuba_engine_optimize_points_device", "cuba_point_batch_workspace_bytes"):
        assert s in pkg.binding.exported_symbols()
    assert pkg.binding.batch_status_message(64) == "iP outside [0, P)"


def _build_driver(tmp_path_factory, pkg):
    out = str(tmp_path_factory.mktemp("cpppoint") / "point_batch_driver")
    libdir = os.path.dirname(pkg.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCUBA_FORCE_EIGEN_COMPAT", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "point_batch_driver.cpp"), "-L", libdir, "-lcuba_b200",
                           "-Wl,-rpath," + libdir, "-o", out])
    return out


def test_point_driver_compiles_against_dropin_headers(pkg, tmp_path_factory):
    assert os.path.exists(_build_driver(tmp_path_factory, pkg))
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", pkg.library_path()], capture_output=True, text=True).stdout
    assert "cuba::optimizePoints(" in out


# ---- on the GPU: against the oracle and the engine's own path ---------------------------------------------------
def _sample(pkg, name):
    return cut_points(pkg, "small", 13) if name == "small" else cut_points(pkg, "kitti07_shaped", 97)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "kitti07_shaped"])
@pytest.mark.parametrize("sched", ["huber_depth", "none", "huber", "tukey"])
def test_point_batch_against_oracle(pkg, oracle, name, sched):
    batch = _sample(pkg, name)
    rounds = schedules(pkg)[sched]
    res = pkg.Engine(device=0).optimize_points(batch, rounds)
    ties = excluded = via_engine = 0
    for b, got in enumerate(res):
        nt, ve = check_against_oracle(pkg, oracle, batch, b, got, rounds, (name, sched, b))
        ties += nt; via_engine += ve
        excluded += int(got["levels"].sum())
        assert all(s["pcg_iters"] == 0 and s["pcg_failed"] == 0 for st in got["stats"] for s in st)
    assert excluded > 0 and via_engine <= batch.B // 10
    print("%s / %s: %d points, %d edges at level 1, %d threshold ties, %d points checked through the engine's path"
          % (name, sched, batch.B, excluded, ties, via_engine))


@pytest.mark.gpu
@pytest.mark.parametrize("sched", ["huber_depth", "tukey"])
def test_point_batch_against_engine_path(pkg, oracle, sched):
    """about 20 points against the engine's per-point set_problem + rounds: identical levels and counts"""
    batch = concat(pkg, [select(pkg, cut_points(pkg, "small", 13), range(10)), select(pkg, cut_points(pkg, "kitti07_shaped", 97), range(0, 200, 20))])
    rounds = schedules(pkg)[sched]
    res = pkg.Engine(device=0).optimize_points(batch, rounds)
    for b, got in enumerate(res):
        check_point(got, engine_reference(pkg, batch, b, rounds), (sched, b), exact_levels=True, H=hessian(oracle, batch, b, got["Xw"]),
                    scale=start_chi2(oracle, batch, b, rounds))


def _synthetic_point(pkg, n2, n3, seed, behind=False):
    """one point seen by n2 + n3 poses of a forward-moving camera (1 px noise, 3 % outliers), perturbed; behind: the point behind
    every camera, its measurements those of its mirror image in front"""
    rng = np.random.default_rng(seed)
    n = n2 + n3
    cam = np.tile([718.856, 718.856, 607.19, 185.22, 386.14], (n, 1))
    q = np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)) + np.concatenate([rng.normal(0, 0.01, (n, 3)), np.zeros((n, 1))], 1)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    t = np.stack([rng.normal(0, 0.5, n), rng.normal(0, 0.2, n), -rng.uniform(0, 10, n)], 1)
    X = np.array([1.0, -0.5, 30.0])
    Xc = pkg.synth._rotate(q, np.repeat(X[None], n, 0)) + t
    u = cam[:, 0] * Xc[:, 0] / Xc[:, 2] + cam[:, 2]
    v = cam[:, 1] * Xc[:, 1] / Xc[:, 2] + cam[:, 3]
    meas = np.stack([u, v, u - cam[:, 4] / Xc[:, 2]], 1) + rng.normal(0, 1, (n, 3))
    out = rng.random(n) < 0.03
    meas[out] += rng.uniform(20, 50, (int(out.sum()), 3))
    X0 = X + rng.normal(0, 0.3, 3)
    if behind:
        X0 = np.array([X[0], X[1], -40.0])
    return pkg.graphio.PointBatch(q=q, t=t, cam=cam, Xw=X0.reshape(1, 3), ptr2=np.array([0, n2], np.int32), iP2=np.arange(n2, dtype=np.int32),
                                  meas2=meas[:n2, :2].copy(), omega2=np.ones(n2), ptr3=np.array([0, n3], np.int32),
                                  iP3=np.arange(n2, n, dtype=np.int32), meas3=meas[n2:].copy(), omega3=np.ones(n3))


@pytest.mark.gpu
def test_point_batch_edge_cases(pkg, oracle):
    rounds = schedules(pkg)["huber_depth"]
    eng = pkg.Engine(device=0)
    src = cut_points(pkg, "small", 13)
    b0 = int(np.nonzero((np.diff(src.ptr2) >= 2) & (np.diff(src.ptr3) >= 2))[0][0])
    # B = 0: nothing launched
    n0 = eng.launch_count()
    zero = pkg.graphio.PointBatch(q=src.q, t=src.t, cam=src.cam, Xw=np.zeros((0, 3)), ptr2=np.zeros(1, np.int32), iP2=np.zeros(0, np.int32),
                                  meas2=np.zeros((0, 2)), omega2=np.zeros(0), ptr3=np.zeros(1, np.int32), iP3=np.zeros(0, np.int32),
                                  meas3=np.zeros((0, 3)), omega3=np.zeros(0))
    assert eng.optimize_points(zero, rounds) == []
    assert eng.launch_count() == n0
    # a point without edges: its position bitwise, no iteration, zero counts
    empty = one_point(pkg, src, b0, [], [])
    r = eng.optimize_points(empty, rounds)[0]
    assert np.array_equal(r["Xw"], empty.Xw[0]) and all(len(s) == 0 for s in r["stats"]) and not r["counts"].any() and len(r["levels"]) == 0
    # a repeated (pose, point) pair, mono + stereo: the stereo edge's pose and (u, v) once more as a mono edge
    p = one_point(pkg, src, b0)
    rep = concat(pkg, [p])
    rep.iP2 = np.concatenate([rep.iP2, rep.iP3[:1]]).astype(np.int32)
    rep.meas2 = np.concatenate([rep.meas2, rep.meas3[:1, :2]])
    rep.omega2 = np.concatenate([rep.omega2, rep.omega3[:1]])
    rep.ptr2 = np.array([0, len(rep.omega2)], np.int32)
    cases = {"one_mono": one_point(pkg, src, b0, [0], []), "one_stereo": one_point(pkg, src, b0, [], [1]), "mono": one_point(pkg, src, b0, None, []),
             "repeated_pair": rep, "over_32": _synthetic_point(pkg, 30, 15, 3), "over_1000": _synthetic_point(pkg, 900, 600, 4)}
    batch = concat(pkg, list(cases.values()))
    res = eng.optimize_points(batch, rounds)
    for b, (what, got) in enumerate(zip(cases, res)):
        check_against_oracle(pkg, oracle, batch, b, got, rounds, what)
        check_point(got, engine_reference(pkg, batch, b, rounds), what, exact_levels=True, H=hessian(oracle, batch, b, got["Xw"]),
                    scale=start_chi2(oracle, batch, b, rounds))
    assert res[-1]["levels"].sum() > 0 and len(res[-1]["stats"][0]) > 0
    # a point behind every camera: the depth test excludes every edge, with or without iterations
    behind = _synthetic_point(pkg, 20, 20, 5, behind=True)
    R = pkg.PoseRound
    for sched in ([R(0, depth=True)], [R(3, depth=True, restart=False), R(5, depth=True, reinclude=False)]):
        got = eng.optimize_points(behind, sched)[0]
        check_point(got, engine_reference(pkg, behind, 0, sched), "behind", exact_levels=True, H=hessian(oracle, behind, 0, got["Xw"]),
                    scale=start_chi2(oracle, behind, 0, sched))
    got = eng.optimize_points(behind, [R(0, depth=True)])[0]
    assert list(got["counts"][0]) == [0, 0, 40, 0] and np.array_equal(got["Xw"], behind.Xw[0])


@pytest.mark.gpu
def test_all_edges_excluded_then_reincluded(pkg, oracle):
    """round 0 excludes every edge (threshold below 0): round 1 runs no iteration and leaves the point alone; round 1's test, at the
    normal thresholds, re-includes them and round 2 optimises again"""
    R = pkg.PoseRound
    hub = dict(kernel=KERNELS["huber"][0], delta=KERNELS["huber"][1])
    src = cut_points(pkg, "kitti07_shaped", 97)
    b = int(np.argmax(np.diff(src.ptr2) + np.diff(src.ptr3)))
    p = one_point(pkg, src, b)
    sched = [R(10, chi2_mono=-1.0, chi2_stereo=-1.0, **hub), R(10, restart=False, **hub), R(10, restart=False)]
    eng = pkg.Engine(device=0)
    got = eng.optimize_points(p, sched)[0]
    check_against_oracle(pkg, oracle, p, 0, got, sched, "excluded")
    check_point(got, engine_reference(pkg, p, 0, sched), "excluded", exact_levels=True, H=hessian(oracle, p, 0, got["Xw"]),
                scale=start_chi2(oracle, p, 0, sched))
    E = len(p.omega2) + len(p.omega3)
    assert list(got["counts"][0]) == [0, 0, E, 0]
    assert len(got["stats"][1]) == 0 and got["counts"][1][3] > 0 and len(got["stats"][2]) > 0
    a = eng.optimize_points(p, sched[:1])[0]
    c = eng.optimize_points(p, [sched[0], R(10, restart=False, chi2_mono=-1.0, chi2_stereo=-1.0)])[0]
    assert np.array_equal(a["Xw"], c["Xw"]) and len(c["stats"][1]) == 0


@pytest.mark.gpu
def test_reproducible_and_independent(pkg):
    """a point alone, in the full batch, at another position and on a repeat gives bitwise the same result; one launch per call"""
    rounds = schedules(pkg)["huber"]
    batch = cut_points(pkg, "kitti07_shaped")
    eng = pkg.Engine(device=0)
    n0 = eng.launch_count()
    r1 = eng.optimize_points(batch, rounds)
    assert eng.launch_count() == n0 + 1
    _same(eng.optimize_points(batch, rounds), r1)
    rng = np.random.default_rng(7)
    for b in (0, 1, 5, 4097, batch.B - 1):
        _same(eng.optimize_points(one_point(pkg, batch, b), rounds), [r1[b]])
    sel = rng.choice(batch.B, 301, replace=False)
    _same(eng.optimize_points(select(pkg, batch, sel), rounds), [r1[i] for i in sel])


def _flat(batch, **kw):
    a = batch.arrays()
    a.update(kw)
    return a


@pytest.mark.gpu
def test_empty_batch_and_malformed_input(pkg):
    eng = pkg.Engine(device=0)
    rounds = schedules(pkg)["huber_depth"]
    batch = select(pkg, cut_points(pkg, "small", 13), range(3))
    good = eng.optimize_points(batch, rounds)
    n1 = eng.launch_count()
    R = pkg.PoseRound

    def with_(k, i, v):
        a = np.array(getattr(batch, k), copy=True); a[i] = v
        return {k: a}

    E2 = len(batch.omega2)
    cases = {
        "B<0": (dict(B=-1), rounds), "P<0": (dict(P=-1), rounds), "E2<0": (dict(E2=-1), rounds), "E3<0": (dict(E3=-1), rounds),
        "ptr2[0]": (with_("ptr2", 0, 1), rounds), "ptr3 decreasing": (with_("ptr3", 1, batch.ptr3[2] + 1), rounds),
        "ptr2 end": (dict(E2=E2 + 1), rounds), "iP2 >= P": (with_("iP2", 1, len(batch.q)), rounds), "iP3 < 0": (with_("iP3", 0, -1), rounds),
        "omega nan": (with_("omega2", 0, np.nan), rounds), "omega inf": (with_("omega3", 2, np.inf), rounds),
        "no rounds": ({}, []), "nine rounds": ({}, [R()] * 9), "negative iterations": ({}, [R(-1)]), "kernel type": ({}, [R(kernel=(0, 3))]),
        "delta nan": ({}, [R(kernel=(1, 1), delta=(1.0, np.nan))]),
    }
    for what, (kw, rs) in cases.items():
        with pytest.raises(pkg.CubaError, match="error -1"):
            eng.optimize_points_flat(rounds=rs, **_flat(batch, **kw))
        assert eng.launch_count() == n1, what
        _same(eng.optimize_points(batch, rounds), good)
        n1 = eng.launch_count()
    msg = pkg.load_library().cuba_last_error().decode()
    assert "optimize_points" in msg


@pytest.mark.gpu
def test_batch_leaves_the_engine_alone(pkg):
    """an engine that runs optimize_points between set_problem and optimize(10), and between classify_edges and optimize, has the
    trajectory, state, levels, chi2 and launch count (less the batch's own launches) of one that never did; fp64 on an fp32 engine"""
    g, prob, planted = tel.planted_problem(pkg, "small")
    rk = KERNELS["huber"]
    batch = cut_points(pkg, "small", 13)
    rounds = schedules(pkg)["huber_depth"]
    a = make_engine(pkg, prob, rk)
    b = make_engine(pkg, prob, rk)
    ra = a.optimize_points(batch, rounds)
    for e in (a, b):
        e.classify_edges(CHI2_MONO, CHI2_STEREO)
    a.optimize_points(batch, rounds)
    assert a.launch_count() - 2 == b.launch_count()
    assert a.optimize(10) == b.optimize(10)
    for x, y in zip(a.state(), b.state()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.edge_levels(), b.edge_levels()) and np.array_equal(a.chi_squared(), b.chi_squared())
    assert a.launch_count() - 2 == b.launch_count()
    _same(pkg.Engine(device=0, use_fp32=True).optimize_points(batch, rounds), ra)


# ---- device-resident batches ---------------------------------------------------------------------------------------
def _dev(torch, batch):
    dev = torch.device("cuda", 0)
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in batch.arrays().items()}


def _host_flat(eng, batch, rounds):
    return eng.optimize_points_flat(rounds=rounds, **batch.arrays())


def _written(stats, nstats, rounds):
    """the stat slots a call wrote (the others are undefined): per point, per round, the first nstats"""
    off = np.concatenate([[0], np.cumsum([int(r.iterations) for r in rounds])])
    return [stats[b, off[k]:off[k] + nstats[b, k]].tobytes() for b in range(len(nstats)) for k in range(len(rounds))]


def _equal_dev(pkg, d, h, rounds):
    assert int(d["status"].item()) == 0
    assert np.array_equal(d["Xw"].cpu().numpy(), h["Xw"]) and np.array_equal(d["levels"].cpu().numpy(), h["levels"])
    assert np.array_equal(d["counts"].cpu().numpy(), h["counts"]) and np.array_equal(d["nstats"].cpu().numpy(), h["nstats"])
    assert _written(pkg.binding.stats_view(d["stats"]), h["nstats"], rounds) == _written(h["stats"], h["nstats"], rounds)


@pytest.mark.gpu
@pytest.mark.parametrize("sched", ["huber_depth", "tukey"])
def test_device_entry_bit_identical(pkg, sched):
    """the device entry against the host entry on every point of the planted small graph and a mixed batch: bit for bit; no
    transfer bytes, no engine launches"""
    import torch
    rounds = schedules(pkg)[sched]
    eng = pkg.Engine(device=0)
    for batch in (cut_points(pkg, "small"), concat(pkg, [select(pkg, cut_points(pkg, "small", 13), range(50)), _synthetic_point(pkg, 900, 600, 4),
                                                         one_point(pkg, cut_points(pkg, "small", 13), 3, [], [])])):
        h = _host_flat(eng, batch, rounds)
        d_in = _dev(torch, batch)
        torch.cuda.synchronize()
        n0 = eng.launch_count()
        t0 = pkg.transfer_bytes()
        d = eng.optimize_points_device(rounds=rounds, **d_in)
        torch.cuda.synchronize()
        assert pkg.transfer_bytes() == t0 and eng.launch_count() == n0
        _equal_dev(pkg, d, h, rounds)
        # without stats, into the same tensors
        d2 = eng.optimize_points_device(rounds=rounds, with_stats=False, **d_in)
        assert d2["stats"] is None
        assert np.array_equal(d2["Xw"].cpu().numpy(), h["Xw"]) and np.array_equal(d2["levels"].cpu().numpy(), h["levels"])


@pytest.mark.gpu
def test_device_status_bits(pkg):
    """every data check sets its bit, and with a non-zero status no output is written"""
    import torch
    rounds = schedules(pkg)["huber_depth"]
    batch = select(pkg, cut_points(pkg, "small", 13), range(5))
    eng = pkg.Engine(device=0)
    good = eng.optimize_points_device(rounds=rounds, **_dev(torch, batch))
    assert int(good["status"].item()) == 0

    def run(bit, k, i, v):
        d_in = _dev(torch, batch)
        d_in[k][i] = v
        out = {k2: (t.fill_(7) if t is not None and k2 not in ("status", "workspace") else t) for k2, t in good.items()}
        before = {k2: t.clone() for k2, t in out.items() if t is not None and k2 not in ("status", "workspace")}
        r = eng.optimize_points_device(rounds=rounds, out=out, workspace=good["workspace"], **d_in)
        assert int(r["status"].item()) == bit, (k, int(r["status"].item()))
        for k2, t in before.items():
            assert torch.equal(r[k2], t), (k, k2)
        assert pkg.binding.batch_status_message(bit) != "ok"

    run(1, "ptr2", 0, -1)
    run(2, "ptr3", 2, 0)
    run(4, "ptr2", 5, int(batch.ptr2[5]) + 1)
    run(8, "omega3", 0, float("nan"))
    run(64, "iP2", 0, len(batch.q))
    run(64, "iP3", 1, -3)


@pytest.mark.gpu
def test_device_graph_capture_and_stream_order(pkg):
    """a CUDA graph of the call replays to the same results into the same tensors; on a side stream the call is ordered after the
    inputs' upload and the reader after the call"""
    import torch
    rounds = schedules(pkg)["huber_depth"]
    batch = cut_points(pkg, "small", 3)
    eng = pkg.Engine(device=0)
    h = _host_flat(eng, batch, rounds)
    d_in = _dev(torch, batch)
    first = eng.optimize_points_device(rounds=rounds, **d_in)
    torch.cuda.synchronize()
    _equal_dev(pkg, first, h, rounds)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        first["Xw"].zero_()
        with torch.cuda.graph(g, stream=side):
            eng.optimize_points_device(rounds=rounds, out=first, workspace=first["workspace"], **d_in)
    torch.cuda.synchronize()
    first["Xw"].zero_(); first["levels"].fill_(9)
    g.replay()
    torch.cuda.synchronize()
    _equal_dev(pkg, first, h, rounds)
    # stream order: inputs written on the side stream right before the call, results read on it right after
    with torch.cuda.stream(side):
        d_in2 = {k: torch.empty_like(v) for k, v in d_in.items()}
        for k in d_in:
            d_in2[k].copy_(d_in[k])
        r = eng.optimize_points_device(rounds=rounds, **d_in2)
        xw = r["Xw"].clone()
    side.synchronize()
    assert np.array_equal(xw.cpu().numpy(), h["Xw"])


# ---- the drop-in ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dropin_optimize_points(pkg, tmp_path_factory):
    """cuba::optimizePoints on points built from LandmarkVertex / PoseVertex / edges: Xw written into the vertices bit for bit what
    Engine.optimize_points gives, levels in the points' edge order, the inlier count, and an unrelated graph held by the same object
    unchanged"""
    g, _, _ = tel.plant_outliers(pkg, pkg.synth.make_config("tiny"), seed=43)
    rng = np.random.default_rng(44)
    g["Xw"] = g["Xw"] + rng.normal(0, 0.1, g["Xw"].shape)
    d = tmp_path_factory.mktemp("points")
    fpath, opath = str(d / "points.cubagraph"), str(d / "other.cubagraph")
    pkg.graphio.write_graph(fpath, g)
    pkg.graphio.write_graph(opath, pkg.synth.make_config("tiny"))
    out = subprocess.run([_build_driver(tmp_path_factory, pkg), fpath, opath], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    res = json.loads(out.stdout)
    assert res["other_before"] == res["other_after"] and len(res["other_before"]) > 0 and res["other_state_equal"]
    assert res["threw_landmark"] and res["threw_schedule"]
    R = pkg.PoseRound
    hub = dict(kernel=KERNELS["huber"][0], delta=KERNELS["huber"][1])
    rounds = [R(5, restart=False, depth=True, reinclude=False, **hub), R(10, restart=False, depth=True, reinclude=True)]
    row = {int(v): i for i, v in enumerate(g["pose_id"])}
    pts = []
    for pt in res["points"]:
        lrow = int(np.nonzero(g["lm_id"] == pt["id"])[0][0])
        edges = np.array(pt["edges"], dtype=np.int64).reshape(-1, 3)
        st, ms = edges[edges[:, 0] == 1, 1], edges[edges[:, 0] == 0, 1]
        pts.append(pkg.graphio.PointBatch(
            q=g["q"], t=g["t"], cam=g["cam"], Xw=g["Xw"][lrow].reshape(1, 3), ptr2=np.array([0, len(ms)], np.int32),
            iP2=np.array([row[int(v)] for v in g["mono_vP"][ms]], np.int32), meas2=g["mono_meas"][ms].reshape(-1, 2), omega2=g["mono_info"][ms],
            ptr3=np.array([0, len(st)], np.int32), iP3=np.array([row[int(v)] for v in g["stereo_vP"][st]], np.int32),
            meas3=g["stereo_meas"][st].reshape(-1, 3), omega3=g["stereo_info"][st]))
    ref = pkg.Engine(device=0).optimize_points(concat(pkg, pts), rounds)
    assert len(ref) == len(res["points"]) > 0
    for b, (pt, e) in enumerate(zip(res["points"], ref)):
        edges = np.array(pt["edges"], dtype=np.int64).reshape(-1, 3)
        assert np.array_equal(np.array(pt["Xw"]), e["Xw"]), b
        assert np.array_equal(np.concatenate([edges[edges[:, 0] == 0, 2], edges[edges[:, 0] == 1, 2]]).astype(np.uint8), e["levels"]), b
        assert pt["rounds"] == [[s["chi2"] for s in st] for st in e["stats"]], b
        assert pt["inliers"] == int((e["levels"] == 0).sum()), b
