"""Pose optimisation of many frames in one launch (include/cuba_b200.h: cuba_engine_optimize_poses, csrc/cuba_pose_batch.cuh), the
Python front end (Engine.optimize_poses, graphio.pose_frames) and the drop-in's cuba::optimizePoses (include/cuba_b200_pose.h).

Frames are cut from the synthetic graphs with outliers planted as in test_edge_levels (measurements pushed 20-50 px, points moved
behind a camera), every pose perturbed.  The reference for a frame is the CPU oracle on the frame's sub-problem without its edges at
level 1, round by round, with the outlier test restated in numpy; the engine's own per-frame path (set_problem + set_robust_kernel /
set_state / optimize / classify_edges per round) is a second reference."""
import json
import os
import subprocess

import numpy as np
import pytest

import test_edge_levels as tel
from conftest import KERNELS, ROOT, make_engine

CHI2_MONO, CHI2_STEREO = 5.991, 7.815
RTOL = 1e-10


# ---- frames and schedules ---------------------------------------------------------------------------------
def _perturb(frames, seed):
    rng = np.random.default_rng(seed)
    for f in frames:
        q = f.q + rng.normal(0, 0.01, 4)
        f.q = q / np.linalg.norm(q)
        f.t = f.t + rng.normal(0, 0.05, 3)
    return frames


_cut = {}


def cut_frames(pkg, name, seed=21):
    """every pose of the planted graph `name` as a frame, perturbed (cached: callers must not modify them)"""
    if (name, seed) not in _cut:
        g, _, _ = tel.plant_outliers(pkg, pkg.synth.make_config(name), seed=seed)
        prob = pkg.graphio.flatten(g)
        _cut[(name, seed)] = _perturb(pkg.graphio.pose_frames(prob, range(prob.Pall)), seed + 1)
    return _cut[(name, seed)]


def schedules(pkg):
    R = pkg.PoseRound
    hub = dict(kernel=KERNELS["huber"][0], delta=KERNELS["huber"][1])
    return {
        "orbslam2": pkg.orbslam2_pose_schedule(),
        # local-BA-like: depth test, no re-inclusion, each round from the last one's result
        "local_ba": [R(5, restart=False, depth=True, reinclude=False, **hub), R(10, restart=False, depth=True, reinclude=False)],
        "none": [R(10, restart=False), R(10, depth=True)],
        "huber": [R(10, restart=False, **hub), R(10, depth=True, **hub)],
        "tukey": [R(10, kernel=KERNELS["tukey"][0], delta=KERNELS["tukey"][1], restart=False),
                  R(10, kernel=KERNELS["tukey"][0], delta=KERNELS["tukey"][1], depth=True)],
    }


def frame_problem(pkg, f, q, t, keep):
    """the flat problem of one frame: its pose the only vertex, free; one fixed landmark per kept edge"""
    return f.flat_problem(q, t, keep)


def classify(pkg, oracle, f, q, t, lev, r):
    """the outlier test of classify_edges restated: (new levels, counts, edges within 1e-9 of a threshold)"""
    E2, E = len(f.omega2), len(f.omega2) + len(f.omega3)
    if E == 0:
        return lev, [0, 0, 0, 0], np.zeros(0, bool)
    full = frame_problem(pkg, f, q, t, np.ones(E, bool))
    o = oracle.Oracle(full)
    chi = o.chi_sqs()
    depth = (pkg.synth._rotate(np.repeat(full.q, E, 0), full.Xw) + full.t)[:, 2]
    thr = np.where(np.arange(E) < E2, r.chi2_mono, r.chi2_stereo)
    fail = (chi > thr) | ((depth <= 0) if r.depth else False)
    new = (fail if r.reinclude else (lev.astype(bool) | fail)).astype(np.uint8)
    mono = np.arange(E) < E2
    counts = [int(((new == 0) & mono).sum()), int(((new == 0) & ~mono).sum()), int(((lev == 0) & (new != 0)).sum()),
              int(((lev != 0) & (new == 0)).sum())]
    return new, counts, np.abs(chi - thr) <= 1e-9 * np.abs(thr)


def oracle_reference(pkg, oracle, f, rounds):
    """round by round: the oracle on the sub-problem without the edges at level 1, then the restated test"""
    E = len(f.omega2) + len(f.omega3)
    q, t = f.q.copy(), f.t.copy()
    lev = np.zeros(E, np.uint8)
    out = dict(stats=[], counts=[], near=np.zeros(E, bool))
    for r in rounds:
        if r.restart:
            q, t = f.q.copy(), f.t.copy()
        keep = lev == 0
        traj = ([], [], [])
        if keep.any() and r.iterations > 0:
            o = oracle.Oracle(frame_problem(pkg, f, q, t, keep), tuple(r.kernel), tuple(r.delta))
            traj = o.optimize(r.iterations)
            oq, ot, _ = o.state()
            q, t = oq[0].copy(), ot[0].copy()
        out["stats"].append(traj)
        lev, c, near = classify(pkg, oracle, f, q, t, lev, r)
        out["counts"].append(c)
        out["near"] |= near
    out.update(q=q, t=t, levels=lev)
    return out


def engine_reference(pkg, f, rounds):
    """the engine's own path for one frame: set_problem, then per round set_robust_kernel, set_state on restart, optimize, classify"""
    E = len(f.omega2) + len(f.omega3)
    full = frame_problem(pkg, f, f.q, f.t, np.ones(E, bool))
    eng = pkg.Engine(device=0)
    eng.initialize(full)
    out = dict(stats=[], counts=[])
    for r in rounds:
        for et in (0, 1):
            eng.set_robust_kernels(r.kernel[et], r.delta[et], et)
        if r.restart:
            eng.set_state(full.q, full.t, full.Xw)
        st = eng.optimize(r.iterations)
        out["stats"].append(([s["chi2"] for s in st], [s["lambda_"] for s in st], [s["trials"] for s in st]))
        c = eng.classify_edges(r.chi2_mono, r.chi2_stereo, depth=r.depth, reinclude=r.reinclude)
        out["counts"].append([c["included_mono"], c["included_stereo"], c["excluded"], c["reincluded"]])
    q, t, _ = eng.state()
    out.update(q=q[0], t=t[0], levels=eng.edge_levels())
    eng.close()
    return out


def check_trajectory(got, ref, what, rtol=RTOL):
    """chi2 per iteration to rtol relative (absolute floor: 1e-12 of the round's first value, for frames that converge to ~0); runs
    that stop a few iterations apart once converged must sit on the converged value (the allowance of test_edge_levels'
    _run_protocol); trial counts, and lambda to 1e-6, over the leading iterations whose decrease is far above rounding (lambda's
    update follows rho = (F - Fhat) / scale, a difference of two sums in different orders).  Returns whether the two runs made the
    same number of iterations."""
    chi, lam, tr = (np.asarray(v, dtype=np.float64) for v in ref)
    g = np.array([s["chi2"] for s in got])
    if len(chi) == 0 or len(g) == 0:
        assert len(chi) == len(g), (what, g, chi)
        return True
    floor = (1e-12 if rtol <= RTOL else rtol) * max(abs(chi[0]), abs(g[0]))
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


def check_frame(got, ref, what, exact_levels=False, rtol=RTOL):
    """q / t to 1e-9 (t relative to max(1, |t|)) when every round ran as many iterations as the reference; a run that stopped a few
    converged iterations apart sits on a chi2 plateau that leaves the pose free to ~sqrt(eps): 1e-7 then"""
    same = all([check_trajectory(gs, rs, (what, r), rtol) for r, (gs, rs) in enumerate(zip(got["stats"], ref["stats"]))])
    ptol = 1e-9 if same and rtol <= RTOL else 1e-7
    assert np.abs(got["q"] - ref["q"]).max() < ptol, (what, got["q"], ref["q"])
    assert np.abs(got["t"] - ref["t"]).max() < ptol * max(1.0, np.abs(ref["t"]).max()), (what, got["t"], ref["t"])
    bad = np.nonzero(got["levels"] != ref["levels"])[0]
    if exact_levels:
        assert len(bad) == 0, (what, bad)
        assert [list(c) for c in got["counts"]] == [list(c) for c in ref["counts"]], (what, got["counts"], ref["counts"])
        return 0
    assert ref["near"][bad].all(), (what, bad)
    if len(bad) == 0:
        assert [list(c) for c in got["counts"]] == [list(c) for c in ref["counts"]], (what, got["counts"], ref["counts"])
    return len(bad)


def check_against_oracle(pkg, oracle, f, got, rounds, what):
    """the oracle to RTOL; where the oracle's 6x6 solve (the reference's 3 + 3 Schur split) and the engine's Cholesky round apart by
    more than that on an ill-conditioned system, the frame must instead equal the engine's own path to RTOL with identical levels,
    and the oracle to 1e-7.  Returns (threshold ties, 1 if the frame needed the engine path)"""
    ref = oracle_reference(pkg, oracle, f, rounds)
    try:
        return check_frame(got, ref, what), 0
    except AssertionError:
        check_frame(got, engine_reference(pkg, f, rounds), what, exact_levels=True)
        return check_frame(got, ref, what, rtol=1e-7), 1


# ---- no GPU ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny", "small"])
def test_pose_frames_match_one_pose_subgraphs(pkg, name):
    """graphio.pose_frames against flatten() of the graph of one pose, free, with its edges and their landmarks, fixed"""
    g = pkg.synth.make_config(name)
    prob = pkg.graphio.flatten(g)
    rows = list(range(0, prob.Pall, 3))
    frames = pkg.graphio.pose_frames(prob, rows)
    assert len(frames) == len(rows)
    for p, f in zip(rows, frames):
        pid = g["pose_id"][prob.pose_rows[p]]
        s = {k: np.array(v, copy=True) for k, v in g.items()}
        s["pose_fixed"][:] = 1
        s["pose_fixed"][prob.pose_rows[p]] = 0
        s["lm_fixed"][:] = 1
        for kind in ("mono", "stereo"):
            keep = s[kind + "_vP"] == pid
            for k in ("_vP", "_vL", "_meas", "_info"):
                s[kind + k] = s[kind + k][keep]
        sub = pkg.graphio.flatten(s)
        assert sub.Pall == 1 and sub.numP == 1 and sub.numL == 0
        assert np.array_equal(f.q, sub.q[0]) and np.array_equal(f.t, sub.t[0]) and np.array_equal(f.cam, sub.cam[0])
        assert np.array_equal(f.X2, sub.Xw[sub.idx2[:, 1]]) and np.array_equal(f.meas2, sub.meas2) and np.array_equal(f.omega2, sub.omega2)
        assert np.array_equal(f.X3, sub.Xw[sub.idx3[:, 1]]) and np.array_equal(f.meas3, sub.meas3) and np.array_equal(f.omega3, sub.omega3)
        assert np.array_equal(prob.idx2[f.mono_ids, 0], np.full(len(f.mono_ids), p))
        assert np.array_equal(prob.idx3[f.stereo_ids, 0], np.full(len(f.stereo_ids), p))
    # every edge belongs to exactly one frame
    all_frames = pkg.graphio.pose_frames(prob, range(prob.Pall))
    assert np.array_equal(np.sort(np.concatenate([f.mono_ids for f in all_frames])), np.arange(prob.E2))
    assert np.array_equal(np.sort(np.concatenate([f.stereo_ids for f in all_frames])), np.arange(prob.E3))


def _build_driver(tmp_path_factory, pkg):
    out = str(tmp_path_factory.mktemp("cpppose") / "pose_batch_driver")
    libdir = os.path.dirname(pkg.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCUBA_FORCE_EIGEN_COMPAT", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "pose_batch_driver.cpp"), "-L", libdir, "-lcuba_b200",
                           "-Wl,-rpath," + libdir, "-o", out])
    return out


def test_pose_driver_compiles_against_dropin_headers(pkg, tmp_path_factory):
    assert os.path.exists(_build_driver(tmp_path_factory, pkg))
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", pkg.library_path()], capture_output=True, text=True).stdout
    for s in ("cuba::optimizePoses(", "cuba::orbSlam2PoseSchedule("):
        assert s in out, s
    assert "cuba_engine_optimize_poses" in pkg.binding.exported_symbols()


def test_orbslam2_schedule_in_python(pkg):
    s = pkg.orbslam2_pose_schedule()
    assert len(s) == 4 and all(r.iterations == 10 and r.restart and r.reinclude and not r.depth for r in s)
    assert [tuple(r.kernel) for r in s] == [(1, 1), (1, 1), (0, 0), (0, 0)]
    assert s[0].delta == (5.991 ** 0.5, 7.815 ** 0.5)
    assert all((r.chi2_mono, r.chi2_stereo) == (CHI2_MONO, CHI2_STEREO) for r in s)


# ---- on the GPU: against the oracle and the engine's own path ---------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "kitti07_shaped"])
@pytest.mark.parametrize("sched", ["orbslam2", "local_ba", "none", "huber", "tukey"])
def test_pose_batch_against_oracle(pkg, oracle, name, sched):
    frames = cut_frames(pkg, name)
    rounds = schedules(pkg)[sched]
    eng = pkg.Engine(device=0)
    res = eng.optimize_poses(frames, rounds)
    ties = excluded = via_engine = 0
    for b, (f, got) in enumerate(zip(frames, res)):
        nt, ve = check_against_oracle(pkg, oracle, f, got, rounds, (name, sched, b))
        ties += nt; via_engine += ve
        excluded += int(got["levels"].sum())
        assert all(s["pcg_iters"] == 0 and s["pcg_failed"] == 0 for st in got["stats"] for s in st)
    assert excluded > 0 and via_engine <= len(frames) // 4
    print("%s / %s: %d frames, %d edges at level 1, %d threshold ties, %d frames checked through the engine's path"
          % (name, sched, len(frames), excluded, ties, via_engine))


@pytest.mark.gpu
@pytest.mark.parametrize("sched", ["orbslam2", "local_ba", "tukey"])
def test_pose_batch_against_engine_path(pkg, sched):
    """about 20 frames against the engine's per-frame set_problem + rounds: same tolerances, identical levels and counts"""
    frames = cut_frames(pkg, "small")[:10] + cut_frames(pkg, "kitti07_shaped")[::25]
    rounds = schedules(pkg)[sched]
    res = pkg.Engine(device=0).optimize_poses(frames, rounds)
    for b, (f, got) in enumerate(zip(frames, res)):
        check_frame(got, engine_reference(pkg, f, rounds), (sched, b), exact_levels=True)


def _frame(pkg, f, mono=None, stereo=None):
    m = np.arange(len(f.omega2)) if mono is None else np.asarray(mono, np.int64)
    s = np.arange(len(f.omega3)) if stereo is None else np.asarray(stereo, np.int64)
    return pkg.graphio.PoseFrame(q=f.q, t=f.t, cam=f.cam, X2=f.X2[m], meas2=f.meas2[m], omega2=f.omega2[m],
                                 X3=f.X3[s], meas3=f.meas3[s], omega3=f.omega3[s])


def _big_frame(pkg, n2=20000, n3=2000, seed=5):
    """one synthetic frame with n2 + n3 edges (1 px noise, 3 % outliers), pose perturbed"""
    rng = np.random.default_rng(seed)
    cam = np.array([718.856, 718.856, 607.19, 185.22, 386.14])
    n = n2 + n3
    Xc = np.stack([rng.uniform(-20, 20, n), rng.uniform(-5, 5, n), rng.uniform(4, 60, n)], 1)
    q = np.array([0.02, -0.1, 0.01, 1.0]); q /= np.linalg.norm(q)
    t = np.array([0.3, -0.2, 1.5])
    conj = q * np.array([-1, -1, -1, 1])
    Xw = pkg.synth._rotate(np.repeat(conj[None], n, 0), Xc - t)
    u = cam[0] * Xc[:, 0] / Xc[:, 2] + cam[2]
    v = cam[1] * Xc[:, 1] / Xc[:, 2] + cam[3]
    ur = u - cam[4] / Xc[:, 2]
    meas = np.stack([u, v, ur], 1) + rng.normal(0, 1, (n, 3))
    out = rng.random(n) < 0.03
    meas[out] += rng.uniform(20, 50, (int(out.sum()), 3))
    f = pkg.graphio.PoseFrame(q=q, t=t, cam=cam, X2=Xw[:n2], meas2=meas[:n2, :2].copy(), omega2=np.ones(n2),
                              X3=Xw[n2:], meas3=meas[n2:].copy(), omega3=np.ones(n3))
    return _perturb([f], seed + 1)[0]


@pytest.mark.gpu
def test_pose_batch_edge_cases(pkg, oracle):
    rounds = pkg.orbslam2_pose_schedule()
    eng = pkg.Engine(device=0)
    f0 = cut_frames(pkg, "small")[7]
    # a frame without edges: its pose bitwise, no iteration, zero counts
    empty = _frame(pkg, f0, mono=[], stereo=[])
    r = eng.optimize_poses([empty], rounds)[0]
    assert np.array_equal(r["q"], empty.q) and np.array_equal(r["t"], empty.t)
    assert all(len(s) == 0 for s in r["stats"]) and not r["counts"].any() and len(r["levels"]) == 0
    # mono-only, stereo-only, one edge (the singular Hpp + lambda I path), >= 20 000 edges: against the oracle
    cases = {"mono": _frame(pkg, f0, stereo=[]), "stereo": _frame(pkg, f0, mono=[]), "one_mono": _frame(pkg, f0, mono=[3], stereo=[]),
             "one_stereo": _frame(pkg, f0, mono=[], stereo=[5]), "big": _big_frame(pkg)}
    res = eng.optimize_poses(list(cases.values()), rounds)
    for (what, f), got in zip(cases.items(), res):
        check_against_oracle(pkg, oracle, f, got, rounds, what)
        check_frame(got, engine_reference(pkg, f, rounds), what, exact_levels=True)
    assert sum(len(s) for s in res[-1]["stats"]) > 0 and res[-1]["levels"].sum() > 0


@pytest.mark.gpu
def test_all_edges_excluded_then_reincluded(pkg, oracle):
    """round 0 excludes every edge (threshold below 0): round 1 runs no iteration and leaves the pose alone; round 1's test, at the
    normal thresholds, re-includes them and round 2 optimises again"""
    R = pkg.PoseRound
    hub = dict(kernel=KERNELS["huber"][0], delta=KERNELS["huber"][1])
    f = cut_frames(pkg, "kitti07_shaped")[11]
    sched = [R(10, chi2_mono=-1.0, chi2_stereo=-1.0, **hub), R(10, restart=False, **hub), R(10, restart=False)]
    eng = pkg.Engine(device=0)
    got = eng.optimize_poses([f], sched)[0]
    check_against_oracle(pkg, oracle, f, got, sched, "excluded")
    check_frame(got, engine_reference(pkg, f, sched), "excluded", exact_levels=True)
    E = len(f.omega2) + len(f.omega3)
    assert list(got["counts"][0]) == [0, 0, E, 0]
    assert len(got["stats"][1]) == 0 and got["counts"][1][3] > 0 and len(got["stats"][2]) > 0
    # the pose after round 1 is the pose after round 0: a run of rounds 0-1 ends where a run of round 0 alone does
    a = eng.optimize_poses([f], sched[:1])[0]
    b = eng.optimize_poses([f], [sched[0], R(10, restart=False, chi2_mono=-1.0, chi2_stereo=-1.0)])[0]
    assert np.array_equal(a["q"], b["q"]) and np.array_equal(a["t"], b["t"])
    assert len(b["stats"][1]) == 0


def _same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(x["q"], y["q"]) and np.array_equal(x["t"], y["t"]) and np.array_equal(x["levels"], y["levels"])
        assert np.array_equal(x["counts"], y["counts"]) and x["stats"] == y["stats"]


@pytest.mark.gpu
def test_large_mixed_batch_and_independence(pkg, oracle):
    """B = 4096 frames of mixed sizes (0 to ~20 000 edges); two calls bitwise equal; a frame run alone, inside a batch of 257 and at a
    permuted position gives bitwise the same output; a sample against the oracle"""
    rounds = pkg.orbslam2_pose_schedule()
    pool = cut_frames(pkg, "small") + cut_frames(pkg, "kitti07_shaped") + cut_frames(pkg, "kitti07_shaped", seed=31)
    rng = np.random.default_rng(3)
    frames = []
    for k in range(4096):
        f = pool[k % len(pool)]
        n2, n3 = len(f.omega2), len(f.omega3)
        kind = k % 7
        if kind == 0:
            frames.append(_frame(pkg, f, mono=[], stereo=[]) if k % 14 == 0 else _frame(pkg, f, mono=[0], stereo=[]))
        elif kind == 1:
            frames.append(_frame(pkg, f, mono=np.sort(rng.choice(n2, n2 // 3, replace=False)), stereo=[]))
        else:
            frames.append(f)
    frames[1000] = _big_frame(pkg)
    eng = pkg.Engine(device=0)
    n0 = eng.launch_count()
    r1 = eng.optimize_poses(frames, rounds)
    assert eng.launch_count() == n0 + 1
    r2 = eng.optimize_poses(frames, rounds)
    _same(r1, r2)
    for b in (0, 1, 2, 5, 1000, 4095):
        _same(eng.optimize_poses([frames[b]], rounds), [r1[b]])
    sel = list(range(100, 357))
    perm = rng.permutation(len(sel))
    rb = eng.optimize_poses([frames[i] for i in sel], rounds)
    rp = eng.optimize_poses([frames[sel[i]] for i in perm], rounds)
    _same(rb, [r1[i] for i in sel])
    _same(rp, [r1[sel[i]] for i in perm])
    for b in (3, 8, 700, 1000, 2500, 4094):
        check_against_oracle(pkg, oracle, frames[b], r1[b], rounds, ("mixed", b))


@pytest.mark.gpu
def test_empty_batch_and_malformed_input(pkg):
    eng = pkg.Engine(device=0)
    rounds = pkg.orbslam2_pose_schedule()
    n0 = eng.launch_count()
    assert eng.optimize_poses([], rounds) == []
    assert eng.launch_count() == n0
    f = cut_frames(pkg, "small")[:3]
    good = eng.optimize_poses(f, rounds)
    n1 = eng.launch_count()
    cat = lambda name, w: np.concatenate([np.asarray(getattr(x, name)).reshape(-1, w) for x in f])
    n2 = np.array([len(x.omega2) for x in f]); n3 = np.array([len(x.omega3) for x in f])
    base = dict(q=cat("q", 4), t=cat("t", 3), cam=cat("cam", 5), ptr2=np.concatenate([[0], np.cumsum(n2)]), X2=cat("X2", 3),
                meas2=cat("meas2", 2), omega2=cat("omega2", 1).ravel(), ptr3=np.concatenate([[0], np.cumsum(n3)]), X3=cat("X3", 3),
                meas3=cat("meas3", 3), omega3=cat("omega3", 1).ravel())
    R = pkg.PoseRound

    def bad_ptr(k, fn):
        def mod(a):
            a = dict(a); p = np.array(a[k]); fn(p); a[k] = p
            return a
        return mod

    def set_at(k, i, v):
        def mod(a):
            a = dict(a); x = np.array(a[k], dtype=np.float64); x[i] = v; a[k] = x
            return a
        return mod

    cases = {
        "B<0": (dict(B=-1), lambda a: a, rounds),
        "ptr2[0]": ({}, bad_ptr("ptr2", lambda p: p.__setitem__(0, 1)), rounds),
        "ptr3 decreasing": ({}, bad_ptr("ptr3", lambda p: p.__setitem__(1, p[2] + 1)), rounds),
        "ptr2 end": (dict(E2=int(n2.sum()) + 1), lambda a: a, rounds),
        "ptr3 end": (dict(E3=int(n3.sum()) - 1), lambda a: a, rounds),
        "no rounds": ({}, lambda a: a, []),
        "nine rounds": ({}, lambda a: a, [R()] * 9),
        "negative iterations": ({}, lambda a: a, [R(-1)]),
        "kernel type": ({}, lambda a: a, [R(kernel=(0, 3))]),
        "omega nan": ({}, set_at("omega2", 5, np.nan), rounds),
        "omega inf": ({}, set_at("omega3", 2, np.inf), rounds),
        "delta inf": ({}, lambda a: a, [R(kernel=(1, 1), delta=(np.inf, 1.0))]),
        "delta nan": ({}, lambda a: a, [R(kernel=(1, 1), delta=(1.0, np.nan))]),
    }
    for what, (kw, mod, rs) in cases.items():
        with pytest.raises(pkg.CubaError, match="error -1"):
            eng.optimize_poses_flat(rounds=rs, **mod(base), **kw)
        assert eng.launch_count() == n1, what
        _same(eng.optimize_poses(f, rounds), good)      # a following valid call succeeds, with the same result
        n1 = eng.launch_count()
    # an unknown flag bit, through the C ABI itself (the schedule is checked before the batch, so an empty batch serves)
    import ctypes
    rs = pkg.Engine._rounds_struct([R()])
    rs[0].flags = 4
    batch = pkg.binding._PoseBatch()
    assert eng.L.cuba_engine_optimize_poses(eng.h, ctypes.byref(batch), 1, rs, None, None, None, None, None, None) == -1
    assert eng.launch_count() == n1
    _same(eng.optimize_poses(f, rounds), good)


@pytest.mark.gpu
def test_batch_leaves_the_engine_alone(pkg):
    """an engine that runs optimize_poses between set_problem and optimize(10) -- and between classify_edges and optimize -- has the
    trajectory, state, levels and PCG info of one that never did; the batch is fp64 on an fp32 engine too"""
    g, prob, planted = tel.planted_problem(pkg, "small")
    rk = KERNELS["huber"]
    frames = cut_frames(pkg, "kitti07_shaped")[:40]
    rounds = pkg.orbslam2_pose_schedule()
    a = make_engine(pkg, prob, rk)
    b = make_engine(pkg, prob, rk)
    n0 = a.launch_count()
    ra = a.optimize_poses(frames, rounds)
    assert a.launch_count() == n0 + 1
    for e in (a, b):
        e.classify_edges(CHI2_MONO, CHI2_STEREO)
    a.optimize_poses(frames, rounds)
    sa, sb = a.optimize(10), b.optimize(10)
    assert sa == sb
    for x, y in zip(a.state(), b.state()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.edge_levels(), b.edge_levels())
    assert a.pcg_info() == b.pcg_info()
    assert np.array_equal(a.chi_squared(), b.chi_squared())
    c = pkg.Engine(device=0, use_fp32=True)
    _same(c.optimize_poses(frames, rounds), ra)


# ---- the drop-in ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dropin_optimize_poses(pkg, oracle, tmp_path_factory):
    """cuba::optimizePoses with the default schedule on frames built from PoseVertex / LandmarkVertex / edges: q / t written into the
    vertices and levels against the oracle, the inlier count, and an unrelated graph held by the same object unchanged"""
    g, _, _ = tel.plant_outliers(pkg, pkg.synth.make_config("small"), seed=23)
    rng = np.random.default_rng(24)
    g["t"] = g["t"] + rng.normal(0, 0.05, g["t"].shape)
    d = tmp_path_factory.mktemp("pose")
    fpath, opath = str(d / "frames.cubagraph"), str(d / "other.cubagraph")
    pkg.graphio.write_graph(fpath, g)
    pkg.graphio.write_graph(opath, pkg.synth.make_config("tiny"))
    out = subprocess.run([_build_driver(tmp_path_factory, pkg), fpath, opath], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    res = json.loads(out.stdout)
    assert res["other_before"] == res["other_after"] and len(res["other_before"]) > 0 and res["other_state_equal"]
    assert res["threw_pose"] and res["threw_schedule"]
    rounds = pkg.orbslam2_pose_schedule()
    assert np.all(np.diff(g["lm_id"]) > 0)
    frames, got = [], []
    for fr in res["frames"]:
        row = int(np.nonzero(g["pose_id"] == fr["id"])[0][0])
        edges = np.array(fr["edges"], dtype=np.int64).reshape(-1, 3)
        st, ms = edges[edges[:, 0] == 1, 1], edges[edges[:, 0] == 0, 1]
        frames.append(pkg.graphio.PoseFrame(
            q=g["q"][row].copy(), t=g["t"][row].copy(), cam=g["cam"][row].copy(),
            X2=g["Xw"][np.searchsorted(g["lm_id"], g["mono_vL"][ms])].reshape(-1, 3), meas2=g["mono_meas"][ms].reshape(-1, 2),
            omega2=g["mono_info"][ms], X3=g["Xw"][np.searchsorted(g["lm_id"], g["stereo_vL"][st])].reshape(-1, 3),
            meas3=g["stereo_meas"][st].reshape(-1, 3), omega3=g["stereo_info"][st]))
        got.append(dict(q=np.array(fr["q"]), t=np.array(fr["t"]), inliers=fr["inliers"], rounds=fr["rounds"],
                        levels=np.concatenate([edges[edges[:, 0] == 0, 2], edges[edges[:, 0] == 1, 2]]).astype(np.uint8)))
    # the drop-in is the C ABI's batch: bit for bit what Engine.optimize_poses gives for the same frames
    ref = pkg.Engine(device=0).optimize_poses(frames, rounds)
    ties = via_engine = 0
    for b, (f, d, e) in enumerate(zip(frames, got, ref)):
        assert np.array_equal(d["q"], e["q"]) and np.array_equal(d["t"], e["t"]), b
        assert np.array_equal(d["levels"], e["levels"]), b
        assert d["rounds"] == [[s["chi2"] for s in st] for st in e["stats"]], b
        assert d["inliers"] == int((e["levels"] == 0).sum()) == int(e["counts"][-1][0] + e["counts"][-1][1]), b
        # ... and that result against the oracle, as every other frame of this file
        nt, ve = check_against_oracle(pkg, oracle, f, e, rounds, ("drop-in", b))
        ties += nt; via_engine += ve
    assert via_engine <= len(frames) // 4
    print("drop-in: %d frames, %d threshold ties, %d frames checked through the engine's path" % (len(frames), ties, via_engine))
