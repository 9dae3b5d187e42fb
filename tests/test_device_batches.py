"""Pose optimisation and Sim3 alignment on device-resident batches (include/cuba_b200.h: cuba_engine_optimize_poses_device /
_optimize_sim3_device, csrc/cuba_batch_io.cuh; Engine.optimize_poses_device / optimize_sim3_device).

Without a GPU: the exported symbols, the workspace sizes against a restatement of the packed layout, the host-side checks on no
engine, and the Python wrappers' refusals before any library call.  On the GPU: every output bit for bit equal to the host entry
points', no host<->device copy, capture into a CUDA graph, stream order, the device-side checks and the engine left alone."""
import ctypes
import subprocess

import numpy as np
import pytest

import __graft_entry__ as ge
import test_edge_levels as tel
from conftest import KERNELS, make_engine
from test_pose_batch import _big_frame, _frame, cut_frames
from test_sim3_batch import make_problems

POSE_KEYS = ("q", "t", "levels", "counts", "nstats")
SIM3_KEYS = ("q", "t", "s", "levels", "ninliers", "nstats")
graphio = ge.load_package().graphio


# ---- the packed layout, restated (csrc/cuba_batch_io.cuh: PoseLayout, Sim3Layout) -------------------------------------------------
def pose_bytes(B, E2, E3, iterations, with_stats):
    if B <= 0:
        return 0
    E, R, n_stat = E2 + E3, len(iterations), B * sum(iterations) if with_stats else 0
    n_in = 16 * B + 8 * E + (B + 1)
    n_out = 8 * B + 4 * n_stat + (5 * B * R + 1) // 2 + (E + 7) // 8
    return 8 * (n_in + n_out)


def sim3_bytes(B, N, prm, with_stats):
    if B <= 0:
        return 0
    n_stat = B * (prm.iterations + max(prm.iterations_bad, prm.iterations_good)) if with_stats else 0
    n_in = 20 * B + 12 * N + (B + 2) // 2
    n_out = 8 * B + 4 * n_stat + (3 * B + 1) // 2 + (N + 7) // 8
    return 8 * (n_in + n_out)


# ---- flat batches -------------------------------------------------------------------------------------------------------------------
pose_flat = graphio.pose_batch_arrays


def sim3_flat(problems, fix):
    """fix: None (scale free everywhere), "on" (held everywhere) or "per" (each problem's own)"""
    d = graphio.sim3_batch_arrays(problems)
    d["fix_scale"] = None if fix is None else np.ones(len(problems), np.int32) if fix == "on" else d["fix_scale"]
    return d


def to_dev(d):
    import torch
    return {k: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).to("cuda:0") for k, v in d.items()}


def written_stats(stats, nstats, offsets):
    """the stat slots a call wrote: per problem and optimize / round, the first nstats of its slots (the rest is not written)"""
    return [stats[b, o:o + int(n)].tobytes() for b in range(len(stats)) for o, n in zip(offsets, nstats[b])]


def same_bytes(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def check_pose_equal(pkg, host, dev, rounds, what):
    got = {k: dev[k].cpu().numpy() for k in POSE_KEYS}
    assert int(dev["status"].cpu()[0]) == 0, what
    for k in POSE_KEYS:
        assert same_bytes(got[k], host[k]), (what, k)
    off = np.concatenate([[0], np.cumsum([int(r.iterations) for r in rounds])])[:-1]
    assert written_stats(pkg.stats_view(dev["stats"]), got["nstats"], off) == written_stats(host["stats"], host["nstats"], off), what


def check_sim3_equal(pkg, host, dev, prm, what):
    got = {k: dev[k].cpu().numpy() for k in SIM3_KEYS}
    assert int(dev["status"].cpu()[0]) == 0, what
    for k in SIM3_KEYS:
        assert same_bytes(got[k], host[k]), (what, k)
    off = (0, prm.iterations)
    assert written_stats(pkg.stats_view(dev["stats"]), got["nstats"], off) == written_stats(host["stats"], host["nstats"], off), what


def restart_off_reinclude(pkg):
    R = pkg.PoseRound
    hub = dict(kernel=KERNELS["huber"][0], delta=KERNELS["huber"][1])
    return [R(10, restart=False, reinclude=True, **hub), R(10, restart=False, reinclude=True, **hub), R(10, restart=False, reinclude=True)]


# ---- no GPU --------------------------------------------------------------------------------------------------------------------------
NEW_SYMBOLS = ("cuba_pose_batch_workspace_bytes", "cuba_engine_optimize_poses_device", "cuba_sim3_batch_workspace_bytes",
               "cuba_engine_optimize_sim3_device")


def test_symbols_exported(pkg):
    out = subprocess.run(["nm", "-D", "--defined-only", pkg.library_path()], capture_output=True, text=True).stdout
    for s in NEW_SYMBOLS:
        assert s in pkg.binding.exported_symbols(), s
        assert " T " + s + "\n" in out, s


@pytest.mark.parametrize("with_stats", [0, 1])
def test_workspace_bytes_against_the_layout(pkg, with_stats):
    L = pkg.load_library()
    R = pkg.PoseRound
    for B, E2, E3, its in [(0, 0, 0, [10]), (1, 0, 0, [10]), (1, 7, 0, [3, 4]), (3, 0, 11, [10] * 4), (1322, 400000, 90000, [10] * 4),
                           (5, 12, 13, [0, 1, 2, 3, 4, 5, 6, 7]), (2, 1, 1, [0])]:
        rs = pkg.Engine._rounds_struct([R(k) for k in its])
        assert L.cuba_pose_batch_workspace_bytes(B, E2, E3, len(its), rs, with_stats) == pose_bytes(B, E2, E3, its, with_stats), (B, E2, E3, its)
    S = pkg.Sim3Params
    for B, N, prm in [(0, 0, S()), (1, 0, S()), (1, 25, S()), (6382, 500000, S()), (7, 100, S(iterations=3, iterations_bad=0, iterations_good=9)),
                      (2, 5, S(iterations=0, iterations_bad=0, iterations_good=0))]:
        p = pkg.binding._Sim3Params(prm.chi2, prm.iterations, prm.iterations_bad, prm.iterations_good, prm.min_pairs)
        assert L.cuba_sim3_batch_workspace_bytes(B, N, ctypes.byref(p), with_stats) == sim3_bytes(B, N, prm, with_stats), (B, N, prm)
    # what the calls refuse sizes to 0
    assert L.cuba_pose_batch_workspace_bytes(-1, 0, 0, 1, pkg.Engine._rounds_struct([R()]), with_stats) == 0
    assert L.cuba_pose_batch_workspace_bytes(1, 0, 0, 0, pkg.Engine._rounds_struct([R()]), with_stats) == 0
    assert L.cuba_pose_batch_workspace_bytes(1, -1, 0, 1, pkg.Engine._rounds_struct([R()]), with_stats) == 0
    assert L.cuba_pose_batch_workspace_bytes(1, 0, 0, 1, pkg.Engine._rounds_struct([R(-1)]), with_stats) == 0
    bad = pkg.binding._Sim3Params(0.0, 5, 10, 5, 10)
    assert L.cuba_sim3_batch_workspace_bytes(1, 5, ctypes.byref(bad), with_stats) == 0
    assert L.cuba_sim3_batch_workspace_bytes(1, 5, None, with_stats) == 0


class _Buf:
    """fake, never dereferenced: the host-side checks only look at whether a pointer is NULL"""
    def __init__(self):
        self.b = (ctypes.c_double * 4)()

    def p(self):
        return ctypes.cast(self.b, ctypes.c_void_p)


def test_host_side_checks_on_no_engine(pkg):
    """every host-side check fails with CUBA_ERR_INVALID and the host entry point's message, on a NULL engine: no device is touched"""
    L = pkg.load_library()
    B = pkg.binding
    buf = _Buf()
    P = buf.p()
    R = pkg.PoseRound
    good_rounds = pkg.Engine._rounds_struct(pkg.orbslam2_pose_schedule())
    ws_ok = pose_bytes(2, 3, 4, [10] * 4, True)

    def pose(batch=True, rounds=(good_rounds, 4), ws=ws_ok, wsp=P, out=P, status=P, **kw):
        f = dict(B=2, E2=3, E3=4, q=P, t=P, cam=P, ptr2=P, X2=P, meas2=P, omega2=P, ptr3=P, X3=P, meas3=P, omega3=P)
        f.update(kw)
        bt = B._PoseBatch(*[f[n] for n, _ in B._PoseBatch._fields_])
        rc = L.cuba_engine_optimize_poses_device(None, ctypes.byref(bt) if batch else None, rounds[1], rounds[0], wsp, ws, out, P, P, P, P, P,
                                                 status, None)
        return rc, L.cuba_last_error().decode()

    assert pose() == (-1, "null engine")
    cases = [
        (dict(batch=False), "optimize_poses: null batch"),
        (dict(B=-1), "optimize_poses: B < 0"),
        (dict(rounds=(good_rounds, 0)), "optimize_poses: nrounds outside 1..CUBA_POSE_MAX_ROUNDS"),
        (dict(rounds=(pkg.Engine._rounds_struct([R()] * 9), 9)), "optimize_poses: nrounds outside 1..CUBA_POSE_MAX_ROUNDS"),
        (dict(rounds=(pkg.Engine._rounds_struct([R(-1)]), 1)), "optimize_poses: negative iterations"),
        (dict(rounds=(pkg.Engine._rounds_struct([R(kernel=(0, 3))]), 1)), "optimize_poses: unknown kernel type"),
        (dict(rounds=(pkg.Engine._rounds_struct([R(kernel=(1, 1), delta=(np.inf, 1.0))]), 1)), "optimize_poses: non-finite delta"),
        (dict(status=None), "optimize_poses_device: null status"),
        (dict(q=None), "optimize_poses: null pose array"),
        (dict(out=None), "optimize_poses: null pose array"),
        (dict(E2=2 ** 31 - 1, E3=1), "optimize_poses: too many edges"),
        (dict(ptr3=None), "optimize_poses: ptr3: null"),
        (dict(E2=-1), "optimize_poses: ptr2[B] is not the item count"),
        (dict(omega2=None), "optimize_poses: ptr2: null item array"),
        (dict(ws=ws_ok - 1), "optimize_poses_device: workspace of %d bytes, %d needed" % (ws_ok - 1, ws_ok)),
        (dict(wsp=None), "optimize_poses_device: workspace of %d bytes, %d needed" % (ws_ok, ws_ok)),
        (dict(wsp=ctypes.c_void_p(P.value + 4)), "optimize_poses_device: workspace not 8-byte aligned"),
    ]
    for kw, msg in cases:
        assert pose(**kw) == (-1, msg), kw
    # an unknown flag bit
    rs = pkg.Engine._rounds_struct([R()])
    rs[0].flags = 4
    assert pose(rounds=(rs, 1)) == (-1, "optimize_poses: unknown flag")
    # B = 0 needs no arrays and no workspace, only the status word and the engine
    assert pose(B=0, E2=0, E3=0, q=None, ptr2=None, ws=0, wsp=None, out=None) == (-1, "null engine")

    S = pkg.Sim3Params
    ws3 = sim3_bytes(2, 5, S(), True)

    def sim3(batch=True, prm=S(), ws=ws3, wsp=P, out=P, status=P, params=True, **kw):
        f = dict(B=2, N=5, ptr=P, q=P, t=P, s=P, cam1=P, cam2=P, fix_scale=None, X1=P, X2=P, obs1=P, obs2=P, omega1=P, omega2=P)
        f.update(kw)
        bt = B._Sim3Batch(*[f[n] for n, _ in B._Sim3Batch._fields_])
        p = B._Sim3Params(prm.chi2, prm.iterations, prm.iterations_bad, prm.iterations_good, prm.min_pairs)
        rc = L.cuba_engine_optimize_sim3_device(None, ctypes.byref(bt) if batch else None, ctypes.byref(p) if params else None, wsp, ws, out,
                                                P, P, P, P, P, P, status, None)
        return rc, L.cuba_last_error().decode()

    assert sim3() == (-1, "null engine")
    cases = [
        (dict(batch=False), "optimize_sim3: null batch or params"),
        (dict(params=False), "optimize_sim3: null batch or params"),
        (dict(prm=S(chi2=0.0)), "optimize_sim3: chi2 not finite and positive"),
        (dict(prm=S(chi2=np.nan)), "optimize_sim3: chi2 not finite and positive"),
        (dict(prm=S(iterations_bad=-1)), "optimize_sim3: negative iterations"),
        (dict(prm=S(min_pairs=-1)), "optimize_sim3: negative min_pairs"),
        (dict(prm=S(iterations=2 ** 31 - 1, iterations_good=1)), "optimize_sim3: too many iterations"),
        (dict(B=-1), "optimize_sim3: B < 0"),
        (dict(N=-1), "optimize_sim3: N < 0"),
        (dict(status=None), "optimize_sim3_device: null status"),
        (dict(ptr=None), "optimize_sim3: ptr: null"),
        (dict(obs2=None), "optimize_sim3: ptr: null item array"),
        (dict(s=None), "optimize_sim3: null problem array"),
        (dict(out=None), "optimize_sim3: null problem array"),
        (dict(ws=ws3 - 8), "optimize_sim3_device: workspace of %d bytes, %d needed" % (ws3 - 8, ws3)),
    ]
    for kw, msg in cases:
        assert sim3(**kw) == (-1, msg), kw
    # no pairs: the pair arrays may be NULL
    assert sim3(N=0, X1=None, X2=None, obs1=None, obs2=None, omega1=None, omega2=None, ws=sim3_bytes(2, 0, S(), True)) == (-1, "null engine")


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError("the library was called: " + name)


def test_wrappers_refuse_before_the_library(pkg):
    """CPU tensors, wrong dtypes, non-contiguous tensors and inconsistent shapes raise before any library call"""
    torch = pytest.importorskip("torch")
    eng = object.__new__(pkg.Engine)
    eng.L, eng.h, eng._device = _NoLibrary(), None, 0
    f = [pkg.graphio.PoseFrame(q=np.array([0, 0, 0, 1.0]), t=np.zeros(3), cam=np.ones(5), X2=np.ones((2, 3)), meas2=np.ones((2, 2)),
                               omega2=np.ones(2), X3=np.ones((1, 3)), meas3=np.ones((1, 3)), omega3=np.ones(1))] * 2
    base = {k: torch.from_numpy(v) for k, v in pose_flat(f).items()}
    rounds = pkg.orbslam2_pose_schedule()
    with pytest.raises(ValueError, match="is on cpu"):
        eng.optimize_poses_device(rounds=rounds, **base)
    with pytest.raises(ValueError, match="is on meta"):
        eng.optimize_poses_device(rounds=rounds, **{k: v.to("meta") for k, v in base.items()})
    with pytest.raises(TypeError, match="must be a torch tensor"):
        eng.optimize_poses_device(rounds=rounds, **dict(base, q=base["q"].numpy()))
    # a reused out / workspace that does not fit the batch, or is not a float64 tensor on the engine's device
    B, E, R, S = 2, 6, len(rounds), sum(r.iterations for r in rounds)
    good = dict(q=torch.zeros(B, 4, dtype=torch.float64), t=torch.zeros(B, 3, dtype=torch.float64), levels=torch.zeros(E, dtype=torch.uint8),
                counts=torch.zeros(B, R, 4, dtype=torch.int32), stats=torch.zeros(B, S, 4, dtype=torch.float64),
                nstats=torch.zeros(B, R, dtype=torch.int32), status=torch.zeros(1, dtype=torch.int32))
    bad_out = {
        "has shape \\(5,\\), must be \\(6,\\)": dict(good, levels=torch.zeros(E - 1, dtype=torch.uint8)),
        "has shape \\(1, 4\\), must be \\(2, 4\\)": dict(good, q=torch.zeros(1, 4, dtype=torch.float64)),
        "has shape \\(2, 3, 4\\)": dict(good, counts=torch.zeros(B, R - 1, 4, dtype=torch.int32)),
        "is torch.float32": dict(good, t=torch.zeros(B, 3, dtype=torch.float32)),
        "is not contiguous": dict(good, nstats=torch.zeros(R, B, dtype=torch.int32).t()),
        "out has no stats": dict(good, stats=None),
        "out lacks status": {k: v for k, v in good.items() if k != "status"},
        "must be the dict": [good],
    }
    for msg, o in bad_out.items():
        with pytest.raises((ValueError, TypeError), match=msg):
            eng.optimize_poses_device(rounds=rounds, out=o, **base)
    with pytest.raises(ValueError, match="out has stats, with_stats is False"):
        eng.optimize_poses_device(rounds=rounds, out=good, with_stats=False, **base)
    with pytest.raises(TypeError, match="workspace is torch.int32"):
        eng.optimize_poses_device(rounds=rounds, out=good, workspace=torch.zeros(100, dtype=torch.int32), **base)
    with pytest.raises(ValueError, match="workspace must be one-dimensional"):
        eng.optimize_poses_device(rounds=rounds, out=good, workspace=torch.zeros(10, 10, dtype=torch.float64), **base)
    # a well-formed out and workspace, still on the CPU: refused for their device
    with pytest.raises(ValueError, match="is on cpu"):
        eng.optimize_poses_device(rounds=rounds, out=good, workspace=torch.zeros(100, dtype=torch.float64), **base)
    with pytest.raises(TypeError, match="omega2 is torch.float32"):
        eng.optimize_poses_device(rounds=rounds, **dict(base, omega2=base["omega2"].float()))
    with pytest.raises(TypeError, match="ptr2 is torch.int64"):
        eng.optimize_poses_device(rounds=rounds, **dict(base, ptr2=base["ptr2"].long()))
    with pytest.raises(ValueError, match="X2 is not contiguous"):
        eng.optimize_poses_device(rounds=rounds, **dict(base, X2=base["X2"].t().contiguous().t()))
    b3 = {k: None if v is None else torch.from_numpy(v) for k, v in sim3_flat(make_problems_cpu(pkg), "per").items()}
    with pytest.raises(ValueError, match="is on cpu"):
        eng.optimize_sim3_device(**b3)
    with pytest.raises(TypeError, match="fix_scale is torch.uint8"):
        eng.optimize_sim3_device(**dict(b3, fix_scale=b3["fix_scale"].to(torch.uint8)))
    with pytest.raises(TypeError, match="s is torch.float32"):
        eng.optimize_sim3_device(**dict(b3, s=b3["s"].float()))
    with pytest.raises(ValueError, match="obs1 is not contiguous"):
        eng.optimize_sim3_device(**dict(b3, obs1=b3["obs1"].t().contiguous().t()))
    B3, N3 = len(b3["s"]), len(b3["omega1"])
    g3 = dict(q=torch.zeros(B3, 4, dtype=torch.float64), t=torch.zeros(B3, 3, dtype=torch.float64), s=torch.zeros(B3, dtype=torch.float64),
              levels=torch.zeros(N3, dtype=torch.uint8), ninliers=torch.zeros(B3, dtype=torch.int32), stats=None,
              nstats=torch.zeros(B3, 2, dtype=torch.int32), status=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(ValueError, match="out\\['levels'\\] has shape"):
        eng.optimize_sim3_device(with_stats=False, out=dict(g3, levels=torch.zeros(N3 + 1, dtype=torch.uint8)), **b3)
    with pytest.raises(ValueError, match="out\\['ninliers'\\] has shape"):
        eng.optimize_sim3_device(with_stats=False, out=dict(g3, ninliers=torch.zeros(B3 - 1, dtype=torch.int32)), **b3)
    with pytest.raises(TypeError, match="workspace is torch.float32"):
        eng.optimize_sim3_device(with_stats=False, out=g3, workspace=torch.zeros(64, dtype=torch.float32), **b3)
    with pytest.raises(ValueError, match="workspace is on cpu"):
        eng.optimize_sim3_device(with_stats=False, out=g3, workspace=torch.zeros(64, dtype=torch.float64), **b3)


def make_problems_cpu(pkg):
    prob = pkg.graphio.flatten(pkg.synth.make_config("tiny"))
    from test_sim3_batch import shared_pairs
    pairs = shared_pairs(prob, min_shared=5)[:3]
    P = pkg.graphio.sim3_problems(prob, pairs, scale=[1.0] * len(pairs))
    assert len(P) >= 2
    return P


# ---- on the GPU -------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    torch.cuda.init()
    return torch


@pytest.fixture(scope="module")
def engine(pkg, torch_cuda):
    return pkg.Engine(device=0)


def pose_cases(pkg):
    kitti = cut_frames(pkg, "kitti07_shaped")
    f0 = cut_frames(pkg, "small")[7]
    mixed = [_frame(pkg, f0, stereo=[]), _frame(pkg, f0, mono=[]), _frame(pkg, f0, mono=[], stereo=[]), kitti[3],
             _frame(pkg, f0, mono=[], stereo=[]), _big_frame(pkg), _frame(pkg, f0, mono=[2], stereo=[])]
    return {"kitti07": kitti, "mixed": mixed, "one": [kitti[5]], "big": [_big_frame(pkg)], "all_empty": [_frame(pkg, f0, mono=[], stereo=[])] * 3,
            "mono_only": [_frame(pkg, f, stereo=[]) for f in kitti[:20]], "stereo_only": [_frame(pkg, f, mono=[]) for f in kitti[:20]]}


@pytest.mark.gpu
@pytest.mark.parametrize("sched", ["orbslam2", "restart_off_reinclude"])
def test_poses_device_bit_identical_to_host(pkg, engine, sched):
    rounds = pkg.orbslam2_pose_schedule() if sched == "orbslam2" else restart_off_reinclude(pkg)
    for what, frames in pose_cases(pkg).items():
        flat = pose_flat(frames)
        host = engine.optimize_poses_flat(rounds=rounds, **flat)
        dev = engine.optimize_poses_device(rounds=rounds, **to_dev(flat))
        check_pose_equal(pkg, host, dev, rounds, (sched, what))
        if what == "kitti07":
            assert host["levels"].sum() > 0
    # without stats: the same arrays
    flat = pose_flat(pose_cases(pkg)["kitti07"])
    host = engine.optimize_poses_flat(rounds=rounds, **flat)
    dev = engine.optimize_poses_device(rounds=rounds, with_stats=False, **to_dev(flat))
    assert dev["stats"] is None and int(dev["status"].cpu()[0]) == 0
    for k in POSE_KEYS:
        assert same_bytes(dev[k].cpu().numpy(), host[k]), k


@pytest.mark.gpu
def test_poses_device_empty_batch(pkg, engine, torch_cuda):
    torch = torch_cuda
    flat = {k: torch.zeros(0, dtype=torch.float64, device="cuda:0") for k in ("q", "t", "cam", "X2", "meas2", "omega2", "X3", "meas3", "omega3")}
    flat["ptr2"] = torch.zeros(1, dtype=torch.int32, device="cuda:0"); flat["ptr3"] = flat["ptr2"].clone()
    dev = engine.optimize_poses_device(rounds=pkg.orbslam2_pose_schedule(), **flat)
    assert dev["q"].shape == (0, 4) and int(dev["status"].cpu()[0]) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("fix", [None, "on", "per"])
def test_sim3_device_bit_identical_to_host(pkg, engine, fix):
    prm = pkg.Sim3Params()
    for name in ("small", "kitti07_shaped"):
        P = make_problems(pkg, name)
        flat = sim3_flat(P, fix)
        host = engine.optimize_sim3_flat(params=prm, **flat)
        dev = engine.optimize_sim3_device(params=prm, **to_dev(flat))
        check_sim3_equal(pkg, host, dev, prm, (name, fix))
        assert (host["ninliers"] > 0).any()
    # one problem, a problem without pairs, and min_pairs 0
    P = make_problems(pkg, "small")
    G = pkg.graphio.Sim3Problem
    d = {f: v for f, v in vars(P[0]).items() if f in G.__dataclass_fields__}
    for f in ("X1", "X2", "obs1", "obs2", "omega1", "omega2", "landmarks"):
        d[f] = d[f][:0]
    for batch, prm in (([P[1]], prm), ([P[2], G(**d), P[3]], pkg.Sim3Params(min_pairs=0))):
        flat = sim3_flat(batch, fix)
        check_sim3_equal(pkg, engine.optimize_sim3_flat(params=prm, **flat), engine.optimize_sim3_device(params=prm, **to_dev(flat)), prm, fix)


@pytest.mark.gpu
def test_no_transfers_and_no_engine_launches(pkg, engine, torch_cuda):
    torch = torch_cuda
    frames = cut_frames(pkg, "kitti07_shaped")
    rounds = pkg.orbslam2_pose_schedule()
    pd = to_dev(pose_flat(frames))
    sd = to_dev(sim3_flat(make_problems(pkg, "small"), "per"))
    torch.cuda.synchronize()
    h2d, d2h = pkg.transfer_bytes()
    n = engine.launch_count()
    a = engine.optimize_poses_device(rounds=rounds, **pd)
    b = engine.optimize_sim3_device(**sd)
    torch.cuda.synchronize()
    assert pkg.transfer_bytes() == (h2d, d2h)
    assert engine.launch_count() == n
    assert int(a["status"].cpu()[0]) == 0 and int(b["status"].cpu()[0]) == 0


@pytest.mark.gpu
def test_capture_into_a_cuda_graph(pkg, engine, torch_cuda):
    """both calls captured in global mode (which refuses a synchronisation or an allocation), replayed twice on fresh inputs copied
    into the captured tensors: each replay equals an eager call"""
    torch = torch_cuda
    rounds = pkg.orbslam2_pose_schedule()
    kitti = cut_frames(pkg, "kitti07_shaped")
    # three pose batches of one shape: the same frame sizes, other poses and measurements
    shapes = [pose_flat(kitti[:40])]
    rng = np.random.default_rng(9)
    for _ in range(2):
        f = dict(shapes[0])
        f["t"] = f["t"] + rng.normal(0, 0.03, f["t"].shape)
        f["meas2"] = f["meas2"] + rng.normal(0, 0.5, f["meas2"].shape)
        shapes.append(f)
    P = make_problems(pkg, "kitti07_shaped")
    s3 = [sim3_flat(P, "per")]
    for _ in range(2):
        f = dict(s3[0])
        f["t"] = f["t"] + rng.normal(0, 0.01, f["t"].shape)
        f["obs1"] = f["obs1"] + rng.normal(0, 0.5, f["obs1"].shape)
        s3.append(f)
    pin, sin = to_dev(shapes[0]), to_dev(s3[0])
    # warm-up on a side stream (torch's rule before capture), outputs and workspaces allocated there
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        pout = engine.optimize_poses_device(rounds=rounds, **pin)
        sout = engine.optimize_sim3_device(**sin)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.graph
    graph = torch.cuda.CUDAGraph()
    with g(graph, capture_error_mode="global"):
        engine.optimize_poses_device(rounds=rounds, out=pout, workspace=pout["workspace"], **pin)
        engine.optimize_sim3_device(out=sout, workspace=sout["workspace"], **sin)
    for k in (1, 2):
        for d, src in ((pin, shapes[k]), (sin, s3[k])):
            for name, v in src.items():
                if v is not None:
                    d[name].copy_(torch.from_numpy(np.ascontiguousarray(v)))
        for o in (pout, sout):
            for name, v in o.items():
                if name != "workspace" and v is not None:
                    v.fill_(-7)
        graph.replay()
        torch.cuda.synchronize()
        check_pose_equal(pkg, engine.optimize_poses_flat(rounds=rounds, **shapes[k]), pout, rounds, ("replay", k))
        check_sim3_equal(pkg, engine.optimize_sim3_flat(**s3[k]), sout, pkg.Sim3Params(), ("replay", k))
        eager = engine.optimize_poses_device(rounds=rounds, **to_dev(shapes[k]))
        for name in POSE_KEYS:
            assert torch.equal(eager[name], pout[name]), name


@pytest.mark.gpu
def test_stream_order(pkg, engine, torch_cuda):
    """inputs written by a torch kernel on a side stream, behind a long sleep, and the call made on that stream with no synchronise in
    between: the host path's result"""
    torch = torch_cuda
    rounds = pkg.orbslam2_pose_schedule()
    flat = pose_flat(cut_frames(pkg, "kitti07_shaped"))
    s3 = sim3_flat(make_problems(pkg, "small"), "per")
    src_p, src_s = to_dev(flat), to_dev(s3)
    dst_p = {k: torch.full_like(v, float("nan")) if v.dtype == torch.float64 else torch.full_like(v, -5) for k, v in src_p.items()}
    dst_s = {k: None if v is None else (torch.full_like(v, float("nan")) if v.dtype == torch.float64 else torch.full_like(v, -5))
             for k, v in src_s.items()}
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        for k in dst_p:
            dst_p[k].copy_(src_p[k])
        dp = engine.optimize_poses_device(rounds=rounds, **dst_p)
        torch.cuda._sleep(200_000_000)
        for k in dst_s:
            if dst_s[k] is not None:
                dst_s[k].copy_(src_s[k])
        ds = engine.optimize_sim3_device(**dst_s)
    side.synchronize()
    check_pose_equal(pkg, engine.optimize_poses_flat(rounds=rounds, **flat), dp, rounds, "stream")
    check_sim3_equal(pkg, engine.optimize_sim3_flat(**s3), ds, pkg.Sim3Params(), "stream")


def _sentinel(out, torch):
    for k, v in out.items():
        if k != "workspace" and v is not None:
            v.fill_(-3)
    return {k: v.clone() for k, v in out.items() if k not in ("workspace", "status") and v is not None}


@pytest.mark.gpu
def test_device_validation(pkg, engine, torch_cuda):
    """each malformed batch: status holds the named code, every output keeps its sentinel, and the same engine and workspace then
    give the host path's result on the valid batch"""
    torch = torch_cuda
    rounds = pkg.orbslam2_pose_schedule()
    frames = cut_frames(pkg, "kitti07_shaped")[:30]
    flat = pose_flat(frames)
    host = engine.optimize_poses_flat(rounds=rounds, **flat)
    good = to_dev(flat)
    first = engine.optimize_poses_device(rounds=rounds, **good)
    out, ws = {k: v for k, v in first.items() if k != "workspace"}, first["workspace"]
    E2, E3 = int(flat["ptr2"][-1]), int(flat["ptr3"][-1])

    def mod(name, i, v):
        a = np.array(flat[name]); a[i] = v
        return dict(good, **{name: torch.from_numpy(a).cuda()})
    cases = {
        "ptr2 start": (mod("ptr2", 0, 1), 1),
        "ptr3 start": (mod("ptr3", 0, -1), 1),
        "ptr2 decreases": (mod("ptr2", 5, int(flat["ptr2"][6]) + 1), 2),
        "ptr3 decreases": (mod("ptr3", 1, int(flat["ptr3"][2]) + 1), 2),
        "ptr2 end": (mod("ptr2", len(frames), E2 - 1), 4),
        "ptr3 end": (mod("ptr3", len(frames), E3 + 1), 4),
        "omega2 nan": (mod("omega2", 17, np.nan), 8),
        "omega3 inf": (mod("omega3", 3, -np.inf), 8),
    }
    for what, (bad, code) in cases.items():
        keep = _sentinel(out, torch)
        r = engine.optimize_poses_device(rounds=rounds, out=out, workspace=ws, **bad)
        assert int(r["status"].cpu()[0]) == code, (what, int(r["status"].cpu()[0]))
        assert pkg.batch_status_message(code) == pkg.BATCH_STATUS[code]
        for k, v in keep.items():
            assert torch.equal(out[k], v), (what, k)
        check_pose_equal(pkg, host, engine.optimize_poses_device(rounds=rounds, out=out, workspace=ws, **good), rounds, what)

    prm = pkg.Sim3Params()
    P = make_problems(pkg, "small")
    s3 = sim3_flat(P, "per")
    host3 = engine.optimize_sim3_flat(params=prm, **s3)
    g3 = to_dev(s3)
    first = engine.optimize_sim3_device(params=prm, **g3)
    out3, ws3 = {k: v for k, v in first.items() if k != "workspace"}, first["workspace"]
    N = int(s3["ptr"][-1])

    def mod3(name, i, v):
        a = np.array(s3[name]); a.flat[i] = v
        return dict(g3, **{name: torch.from_numpy(a).cuda()})
    cases = {
        "ptr start": (mod3("ptr", 0, 2), 1), "ptr decreases": (mod3("ptr", 2, int(s3["ptr"][3]) + 1), 2), "ptr end": (mod3("ptr", len(P), N + 1), 4),
        "X1 nan": (mod3("X1", 7, np.nan), 8), "omega2 nan": (mod3("omega2", 1, np.nan), 8), "obs2 inf": (mod3("obs2", 4, np.inf), 8),
        "q nan": (mod3("q", 2, np.nan), 16), "cam1 nan": (mod3("cam1", 1, np.nan), 16), "s nan": (mod3("s", 3, np.nan), 16),
        "s = 0": (mod3("s", 1, 0.0), 32), "s < 0": (mod3("s", 0, -1.0), 32), "s = -0": (mod3("s", 2, -0.0), 32),
        "two at once": (dict(mod3("t", 0, np.inf), omega1=mod3("omega1", 5, np.nan)["omega1"]), 8 | 16),
    }
    for what, (bad, code) in cases.items():
        keep = _sentinel(out3, torch)
        r = engine.optimize_sim3_device(params=prm, out=out3, workspace=ws3, **bad)
        assert int(r["status"].cpu()[0]) == code, (what, int(r["status"].cpu()[0]))
        for k, v in keep.items():
            assert torch.equal(out3[k], v), (what, k)
        check_sim3_equal(pkg, host3, engine.optimize_sim3_device(params=prm, out=out3, workspace=ws3, **g3), prm, what)


@pytest.mark.gpu
def test_device_batches_leave_the_engine_alone(pkg, torch_cuda):
    """an engine that runs both device batches between set_problem and optimize(10), and between classify_edges and optimize, has
    the trajectory, state, levels, PCG info and launch count of one that never did"""
    g, prob, planted = tel.planted_problem(pkg, "small")
    rk = KERNELS["huber"]
    rounds = pkg.orbslam2_pose_schedule()
    pd = to_dev(pose_flat(cut_frames(pkg, "kitti07_shaped")[:40]))
    sd = to_dev(sim3_flat(make_problems(pkg, "small"), "per"))
    a = make_engine(pkg, prob, rk)
    b = make_engine(pkg, prob, rk)
    na, nb = a.launch_count(), b.launch_count()
    a.optimize_poses_device(rounds=rounds, **pd); a.optimize_sim3_device(**sd)
    for e in (a, b):
        e.classify_edges(5.991, 7.815)
    a.optimize_poses_device(rounds=rounds, **pd); a.optimize_sim3_device(**sd)
    assert a.launch_count() - na == b.launch_count() - nb
    sa, sb = a.optimize(10), b.optimize(10)
    assert sa == sb
    for x, y in zip(a.state(), b.state()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.edge_levels(), b.edge_levels())
    assert a.pcg_info() == b.pcg_info()
    assert np.array_equal(a.chi_squared(), b.chi_squared())


@pytest.mark.gpu
def test_default_device_engine(pkg, torch_cuda):
    """Engine() (device -1, the current device at creation) runs the device batches on that device"""
    torch = torch_cuda
    eng = pkg.Engine()
    assert eng._device == torch.cuda.current_device()
    rounds = pkg.orbslam2_pose_schedule()
    flat = pose_flat(cut_frames(pkg, "small")[:5])
    check_pose_equal(pkg, eng.optimize_poses_flat(rounds=rounds, **flat), eng.optimize_poses_device(rounds=rounds, **to_dev(flat)), rounds,
                     "default device")
