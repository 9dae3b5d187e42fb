"""The engine's own problem on device-resident arrays (include/cuba_b200.h: cuba_engine_set_problem_device and the other *_device
entry points of the engine's problem; Engine.initialize_device, set_state_device, state_device, chi_squared_device,
set_edge_levels_device, edge_levels_device).

Without a GPU: the exported symbols, the C entry points on no engine, and the Python wrappers' refusals before any library call.
On the GPU: every result bit for bit the host entry points' (fp64, fp32 and mixed engines, both linear solvers, every robust kernel,
fixed vertices, mono-only, stereo-only and repeated-pair problems, edge levels), structure reuse across the host and the device
calls, the host<->device bytes and launches each call moves, capture into a CUDA graph, stream order, refused problems and
landmark-sharded ranks under CUBA_DRY_SHARD."""
import ctypes
import subprocess

import numpy as np
import pytest

from conftest import KERNELS
from test_gpu_parity import REF_VARIANTS, _variant

NEW_SYMBOLS = ("cuba_engine_set_problem_device", "cuba_engine_set_state_device", "cuba_engine_get_state_device",
               "cuba_engine_get_chi2_device", "cuba_engine_set_edge_levels_device", "cuba_engine_get_edge_levels_device")
FIELDS = ("q", "t", "cam", "Xw", "idx2", "meas2", "omega2", "idx3", "meas3", "omega3")
STAT_KEYS = ("iteration", "trials", "chi2", "lambda_", "pcg_iters", "pcg_failed")
CHI2_MONO, CHI2_STEREO = 5.991, 7.815


def to_dev(prob, device="cuda:0"):
    import torch
    d = {k: torch.from_numpy(np.ascontiguousarray(getattr(prob, k))).to(device) for k in FIELDS}
    d.update(Pall=prob.Pall, numP=prob.numP, Lall=prob.Lall, numL=prob.numL)
    return d


def stats_bytes(stats):
    return np.array([[s[k] for k in STAT_KEYS] for s in stats], np.float64).tobytes()


def same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def mask_of(prob, seed=5, frac=0.1):
    rng = np.random.Generator(np.random.PCG64(seed))
    return (rng.random(prob.nedges) < frac).astype(np.uint8)


# ---- no GPU ---------------------------------------------------------------------------------------------------------------------------
def test_symbols_exported(pkg):
    out = subprocess.run(["nm", "-D", "--defined-only", pkg.library_path()], capture_output=True, text=True).stdout
    for s in NEW_SYMBOLS:
        assert s in pkg.binding.exported_symbols(), s
        assert " T " + s + "\n" in out, s


def test_null_engine(pkg):
    """a NULL engine fails as the host entry points do, before any device is touched"""
    L = pkg.load_library()
    P = pkg.binding._Problem()
    buf = (ctypes.c_double * 4)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    calls = {
        "set_problem": (L.cuba_engine_set_problem(None, ctypes.byref(P)), L.cuba_engine_set_problem_device(None, ctypes.byref(P), None)),
        "set_state": (L.cuba_engine_set_state(None, p, p, p), L.cuba_engine_set_state_device(None, p, p, p, None)),
        "get_state": (L.cuba_engine_get_state(None, p, p, p), L.cuba_engine_get_state_device(None, p, p, p, None)),
        "get_chi2": (L.cuba_engine_get_chi2(None, p), L.cuba_engine_get_chi2_device(None, p, None)),
        "set_edge_levels": (L.cuba_engine_set_edge_levels(None, p), L.cuba_engine_set_edge_levels_device(None, p, None)),
        "get_edge_levels": (L.cuba_engine_get_edge_levels(None, p), L.cuba_engine_get_edge_levels_device(None, p, None)),
    }
    for name, (host, dev) in calls.items():
        assert host == dev == -1, name
        assert L.cuba_last_error().decode() == "null engine"


class _NoLibrary:
    def __getattr__(self, name):
        raise AssertionError("the library was called: " + name)


def _bare_engine(pkg, prob=None):
    eng = object.__new__(pkg.Engine)
    eng.L, eng.h, eng._device, eng._stats = _NoLibrary(), None, 0, []
    eng.sizes = None if prob is None else dict(Pall=prob.Pall, numP=prob.numP, Lall=prob.Lall, numL=prob.numL, E2=prob.E2, E3=prob.E3)
    return eng


def test_wrappers_refuse_before_the_library(pkg):
    """numpy arrays, CPU tensors, wrong dtypes, non-contiguous tensors and wrong shapes raise before any library call"""
    torch = pytest.importorskip("torch")
    prob = pkg.graphio.flatten(pkg.synth.make_config("tiny"))
    eng = _bare_engine(pkg)
    cpu = {k: torch.from_numpy(np.ascontiguousarray(getattr(prob, k))) for k in FIELDS}
    cpu.update(Pall=prob.Pall, numP=prob.numP, Lall=prob.Lall, numL=prob.numL)
    meta = dict(cpu, **{k: cpu[k].to("meta") for k in FIELDS})
    with pytest.raises(ValueError, match="q is on cpu"):
        eng.initialize_device(cpu)
    with pytest.raises(ValueError, match="is on meta"):
        eng.initialize_device(meta)
    with pytest.raises(TypeError, match="meas2 must be a torch tensor"):
        eng.initialize_device(dict(meta, meas2=prob.meas2))
    with pytest.raises(TypeError, match="omega2 must be a torch tensor"):
        eng.initialize_device(dict(meta, omega2=prob.omega2))
    with pytest.raises(TypeError, match="idx2 is torch.int64"):
        eng.initialize_device(dict(meta, idx2=meta["idx2"].long()))
    with pytest.raises(TypeError, match="Xw is torch.float32"):
        eng.initialize_device(dict(meta, Xw=meta["Xw"].float()))
    with pytest.raises(ValueError, match="t is not contiguous"):
        eng.initialize_device(dict(meta, t=meta["t"].t().contiguous().t()))
    E2 = prob.E2
    with pytest.raises(ValueError, match="idx2 has shape \\(%d, 2\\), must be \\(%d, 2\\)" % (E2 - 1, E2)):
        eng.initialize_device(dict(meta, idx2=meta["idx2"][1:]))
    with pytest.raises(ValueError, match="idx2 has shape \\(%d, 2\\), must be \\(%d, 2\\)" % (E2, E2 + 1)):
        eng.initialize_device(dict(meta, E2=E2 + 1))
    with pytest.raises(ValueError, match="cam has shape"):
        eng.initialize_device(dict(meta, cam=meta["cam"][:, :4].contiguous()))
    with pytest.raises(ValueError, match="Xw has shape"):
        eng.initialize_device(dict(meta, Lall=prob.Lall + 1))
    with pytest.raises(TypeError, match="prob lacks meas3"):
        eng.initialize_device({k: v for k, v in meta.items() if k != "meas3"})

    # before a problem: no sizes to check against
    for call in (lambda: eng.state_device(), lambda: eng.chi_squared_device(), lambda: eng.edge_levels_device(),
                 lambda: eng.set_edge_levels_device(None), lambda: eng.set_state_device(meta["q"], meta["t"], meta["Xw"])):
        with pytest.raises(pkg.CubaError, match="before initialize"):
            call()
    eng = _bare_engine(pkg, prob)
    P, Lm, E = prob.Pall, prob.Lall, prob.nedges
    q, t, X = (torch.zeros(sh, dtype=torch.float64, device="meta") for sh in ((P, 4), (P, 3), (Lm, 3)))
    with pytest.raises(ValueError, match="Xw has shape"):
        eng.set_state_device(q, t, X[1:])
    with pytest.raises(TypeError, match="q is torch.float32"):
        eng.set_state_device(q.float(), t, X)
    with pytest.raises(TypeError, match="t must be a torch tensor"):
        eng.set_state_device(q, np.zeros((P, 3)), X)
    with pytest.raises(ValueError, match="q is on cpu"):
        eng.set_state_device(torch.zeros(P, 4, dtype=torch.float64), t, X)
    with pytest.raises(ValueError, match="q is not contiguous"):
        eng.set_state_device(torch.zeros(4, P, dtype=torch.float64, device="meta").t(), t, X)
    with pytest.raises(ValueError, match="is on meta"):
        eng.state_device(out=(q, t, X))
    with pytest.raises(ValueError, match="t has shape"):
        eng.state_device(out=(q, q, X))
    with pytest.raises(TypeError, match="out must be a tuple"):
        eng.state_device(out=[q, t, X])
    with pytest.raises(ValueError, match="out is on cpu"):
        eng.chi_squared_device(out=torch.zeros(E, dtype=torch.float64))
    with pytest.raises(ValueError, match="out has shape"):
        eng.chi_squared_device(out=torch.zeros(E + 1, dtype=torch.float64, device="meta"))
    with pytest.raises(TypeError, match="levels is torch.bool"):
        eng.set_edge_levels_device(torch.zeros(E, dtype=torch.bool, device="meta"))
    with pytest.raises(TypeError, match="levels must be a torch tensor"):
        eng.set_edge_levels_device(np.zeros(E, np.uint8))
    with pytest.raises(ValueError, match="levels has shape"):
        eng.set_edge_levels_device(torch.zeros(E - 1, dtype=torch.uint8, device="meta"))
    with pytest.raises(ValueError, match="levels is on cpu"):
        eng.set_edge_levels_device(torch.zeros(E, dtype=torch.uint8))
    with pytest.raises(TypeError, match="out is torch.int32"):
        eng.edge_levels_device(out=torch.zeros(E, dtype=torch.int32, device="meta"))
    with pytest.raises(ValueError, match="out is not contiguous"):
        eng.edge_levels_device(out=torch.zeros(E, 2, dtype=torch.uint8, device="meta")[:, 0])


# ---- on the GPU -------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    torch = pytest.importorskip("torch")
    torch.cuda.init()
    return torch


def _repeated_pair(pkg, prob):
    """tiny with its first monocular edge twice (its own measurement): two terms on the same (pose, landmark) pair"""
    p = prob.copy()
    p.idx2 = np.concatenate([prob.idx2, prob.idx2[:1]]); p.meas2 = np.concatenate([prob.meas2, prob.meas2[:1] + 0.5])
    p.omega2 = np.concatenate([prob.omega2, prob.omega2[:1]])
    return p


def gpu_problems(pkg, problems):
    tiny = problems("tiny")
    out = {"tiny": tiny, "repeated_pair": _repeated_pair(pkg, tiny),
           "mono_only": pkg.graphio.flatten(pkg.synth.make_graph(12, 300, 900, 0, 7)),
           "stereo_only": pkg.graphio.flatten(pkg.synth.make_graph(12, 300, 0, 900, 7))}
    for how in ("mixed", "pose_only", "landmark_only"):
        out["tiny-" + how] = _variant(pkg, tiny, **REF_VARIANTS[how](tiny))
    return out


def new_engine(pkg, rk, precision, solver, **kw):
    eng = pkg.Engine(device=0, use_fp32={"fp64": False, "fp32": True, "mixed": "mixed"}[precision], **kw)
    for et in (0, 1):
        eng.set_robust_kernels(rk[0][et], rk[1][et], et)
    eng.set_linear_solver(solver)
    return eng


def check_same_results(torch, host, dev, what):
    """state, per-edge chi2 and levels of two engines that must hold the same problem and estimate"""
    hq, ht, hX = host.state()
    dq, dt, dX = (a.cpu().numpy() for a in dev.state_device())
    assert same(hq, dq) and same(ht, dt) and same(hX, dX), (what, "state")
    assert same(host.chi_squared(), dev.chi_squared_device().cpu().numpy()), (what, "chi2")
    assert same(host.edge_levels(), dev.edge_levels_device().cpu().numpy()), (what, "levels")


def run_pair(torch, pkg, prob, rk, precision, solver, what):
    host = new_engine(pkg, rk, precision, solver)
    dev = new_engine(pkg, rk, precision, solver)
    assert host.initialize(prob) == dev.initialize_device(to_dev(prob)), what
    check_same_results(torch, host, dev, what + " initial")
    assert stats_bytes(host.optimize(5)) == stats_bytes(dev.optimize(5)), what
    check_same_results(torch, host, dev, what + " optimize(5)")
    assert host.classify_edges(CHI2_MONO, CHI2_STEREO) == dev.classify_edges(CHI2_MONO, CHI2_STEREO), what
    check_same_results(torch, host, dev, what + " classify_edges")
    assert stats_bytes(host.optimize(3)) == stats_bytes(dev.optimize(3)), what
    mask = mask_of(prob)
    host.set_edge_levels(mask)
    dev.set_edge_levels_device(torch.from_numpy(mask * 7).cuda())       # any non-zero value is level 1
    check_same_results(torch, host, dev, what + " set_edge_levels")
    host.set_state(prob.q, prob.t, prob.Xw)
    d = to_dev(prob)
    dev.set_state_device(d["q"], d["t"], d["Xw"])
    assert stats_bytes(host.optimize(4)) == stats_bytes(dev.optimize(4)), what
    check_same_results(torch, host, dev, what + " set_state + optimize(4)")
    host.set_edge_levels(None)
    dev.set_edge_levels_device(None)
    assert stats_bytes(host.optimize(2)) == stats_bytes(dev.optimize(2)), what
    check_same_results(torch, host, dev, what + " levels cleared")
    host.close(); dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp64", "fp32", "mixed"])
@pytest.mark.parametrize("solver", ["pcg", "dense"])
def test_bit_identical_to_host(pkg, problems, torch_cuda, precision, solver):
    for name, prob in gpu_problems(pkg, problems).items():
        for kernel in ("none", "huber", "tukey"):
            run_pair(torch_cuda, pkg, prob, KERNELS[kernel], precision, solver, "/".join((name, kernel, precision, solver)))


def _swap_landmarks(prob, kind="idx2"):
    """the same sizes, one (iP, iL) list changed: two edges of the list `kind` (idx2 monocular, idx3 stereo) of different poses and
    landmarks swap their landmarks"""
    p = prob.copy()
    idx = getattr(prob, kind).copy()
    k = next(k for k in range(1, len(idx)) if idx[k, 0] != idx[0, 0] and idx[k, 1] != idx[0, 1])
    idx[[0, k], 1] = idx[[k, 0], 1]
    setattr(p, kind, idx)
    return p


@pytest.mark.gpu
def test_structure_reuse_across_entry_points(pkg, problems, torch_cuda):
    """host -> device, device -> host and device -> device with the same lists reuse the structure; one changed index rebuilds; the
    results equal a fresh engine's either way"""
    prob = problems("small")
    moved = prob.copy(); moved.Xw = prob.Xw + 0.01; moved.meas2 = prob.meas2 + 0.25
    swapped = _swap_landmarks(prob)
    swapped3 = _swap_landmarks(prob, "idx3")                                 # the stereo half of the device comparison
    rk = KERNELS["huber"]

    def fresh(p):
        e = new_engine(pkg, rk, "fp64", "pcg")
        e.initialize(p)
        r = stats_bytes(e.optimize(3)), e.state(), e.chi_squared()
        e.close()
        return r

    eng = new_engine(pkg, rk, "fp64", "pcg")
    steps = [("host", prob, 0), ("device", moved, 1), ("device", prob, 1), ("host", moved, 1), ("host", prob, 1), ("device", swapped, 0),
             ("device", prob, 0), ("host", swapped, 0), ("device", swapped, 1), ("host", prob, 0), ("device", swapped3, 0),
             ("device", prob, 0), ("host", swapped3, 0), ("device", swapped3, 1), ("device", prob, 0)]
    for k, (how, p, reused) in enumerate(steps):
        before = eng.structure_reuses()
        if how == "host":
            eng.initialize(p)
        else:
            eng.initialize_device(to_dev(p))
        assert eng.structure_reuses() - before == reused, (k, how)
        want = fresh(p)
        got = stats_bytes(eng.optimize(3)), eng.state(), eng.chi_squared()
        assert got[0] == want[0] and all(same(a, b) for a, b in zip(got[1], want[1])) and same(got[2], want[2]), (k, how)
    eng.close()


@pytest.mark.gpu
def test_transfers_and_launches(pkg, problems, torch_cuda):
    """what each call moves between host and device (transfer_bytes) and launches, on the fp64 engine; the host-only formulas are
    those of the parent commit's build"""
    prob = problems("tiny")
    P, Lm, E2, E3 = prob.Pall, prob.Lall, prob.E2, prob.E3
    E = E2 + E3
    raw = 8 * E + 16 * E2 + 24 * E3 + 8 * E          # idx2 / idx3, meas2, meas3, omega2 / omega3
    state = 8 * (4 + 3 + 5) * P + 8 * 3 * Lm        # q, t, cam, Xw
    rk = KERNELS["huber"]
    tb = pkg.transfer_bytes
    host, dev = new_engine(pkg, rk, "fp64", "pcg"), new_engine(pkg, rk, "fp64", "pcg")

    def delta(eng, f):
        b0, l0 = np.array(tb()), eng.launch_count()
        f()
        return tuple(int(x) for x in np.array(tb()) - b0), eng.launch_count() - l0

    d = to_dev(prob)
    (h_fresh, hl_fresh) = delta(host, lambda: host.initialize(prob))
    (d_fresh, dl_fresh) = delta(dev, lambda: dev.initialize_device(d))
    # a fresh set_problem_device moves what set_problem moves without the raw arrays and the state: the builder's block pattern
    # (down), the PCG partition (up); the same launches
    assert h_fresh[0] - d_fresh[0] == raw + state and h_fresh[1] == d_fresh[1], (h_fresh, d_fresh)
    assert hl_fresh == dl_fresh
    # structure reuse: the host call uploads the values and the state (k_pack_state, k_edge_stream, k_pose_stream, jh4::k_emit);
    # the device call moves only the 4-byte flag of the comparison, and adds the comparison kernel
    (h_re, hl_re) = delta(host, lambda: host.initialize(prob))
    (d_re, dl_re) = delta(dev, lambda: dev.initialize_device(d))
    assert h_re == (16 * E2 + 24 * E3 + 8 * E + state, 0) and hl_re == 4
    assert d_re == (0, 4) and dl_re == hl_re + 1
    # the host getters and setters, unchanged: set_state uploads q, t, Xw (one k_pack_state); get_state reads the padded records
    # (8 + 4 doubles per pose / landmark); get_chi2 reads E doubles (k_chi_sqs); set_edge_levels uploads E bytes (k_mask_omega,
    # k_pose_omega, jh4::k_emit); get_edge_levels reads E bytes
    mask = mask_of(prob)
    assert delta(host, lambda: host.set_state(prob.q, prob.t, prob.Xw)) == ((8 * 7 * P + 8 * 3 * Lm, 0), 1)
    assert delta(host, lambda: host.state()) == ((0, 8 * (8 * P + 4 * Lm)), 0)
    assert delta(host, lambda: host.chi_squared()) == ((0, 8 * E), 1)
    assert delta(host, lambda: host.set_edge_levels(mask)) == ((E, 0), 3)
    assert delta(host, lambda: host.edge_levels()) == ((0, E), 0)
    # the device calls: nothing but the 8-byte count of set_edge_levels_device
    torch = torch_cuda
    out_state, out_chi, out_lv = dev.state_device(), dev.chi_squared_device(), dev.edge_levels_device()
    assert delta(dev, lambda: dev.set_state_device(d["q"], d["t"], d["Xw"])) == ((0, 0), 1)
    assert delta(dev, lambda: dev.state_device(out=out_state)) == ((0, 0), 1)
    assert delta(dev, lambda: dev.chi_squared_device(out=out_chi)) == ((0, 0), 1)
    assert delta(dev, lambda: dev.set_edge_levels_device(torch.from_numpy(mask).cuda()))[0] == (0, 8)
    assert delta(dev, lambda: dev.edge_levels_device(out=out_lv)) == ((0, 0), 0)
    torch.cuda.synchronize()
    check_same_results(torch, host, dev, "after the counted calls")
    host.close(); dev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_graph_capture(pkg, problems, torch_cuda, precision):
    """set_state_device + get_state_device + get_chi2_device captured into a CUDA graph after optimize(), replayed: the bytes of the
    direct calls"""
    torch = torch_cuda
    prob = problems("small")
    eng = new_engine(pkg, KERNELS["huber"], precision, "pcg")
    d = to_dev(prob)
    eng.initialize_device(d)
    eng.optimize(3)
    start = tuple((d[k] + 1e-3).contiguous() for k in ("q", "t", "Xw"))
    outs = eng.state_device(), eng.chi_squared_device()
    eng.set_state_device(*start)
    direct = [a.cpu().numpy() for a in eng.state_device()] + [eng.chi_squared_device().cpu().numpy()]
    eng.optimize(3)                                                        # the estimate moves on
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            eng.set_state_device(*start)
            eng.state_device(out=outs[0])
            eng.chi_squared_device(out=outs[1])
    torch.cuda.current_stream().wait_stream(side)
    for a in outs[0]:
        a.zero_()
    outs[1].fill_(-1.0)
    g.replay()
    torch.cuda.synchronize()
    got = [a.cpu().numpy() for a in outs[0]] + [outs[1].cpu().numpy()]
    assert all(same(a, b) for a, b in zip(got, direct))
    # and the engine's state is the captured one: optimize from it as from the direct set_state
    ref = new_engine(pkg, KERNELS["huber"], precision, "pcg")
    ref.initialize(prob)
    ref.set_state(*(a.cpu().numpy() for a in start))
    assert stats_bytes(eng.optimize(2)) == stats_bytes(ref.optimize(2))
    eng.close(); ref.close()


def _capture(torch, calls):
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(g, stream=side):
        calls()
    torch.cuda.current_stream().wait_stream(side)
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_captured_getters_hold_the_buffer_of_capture(pkg, problems, torch_cuda, precision):
    """a graph of get_state_device + get_chi2_device reads the working buffer that was current at capture (include/cuba_b200.h):
    replayed before the next LM step it gives the direct calls' bytes; after one accepted step (the buffers swapped) it gives the
    estimate of before the step, and a graph captured again gives the new one"""
    torch = torch_cuda
    prob = problems("small")
    eng = new_engine(pkg, KERNELS["huber"], precision, "pcg")
    eng.initialize_device(to_dev(prob))
    eng.optimize(2)
    outs = eng.state_device(), eng.chi_squared_device()

    def read():
        torch.cuda.synchronize()
        return [a.cpu().numpy().copy() for a in outs[0]] + [outs[1].cpu().numpy().copy()]

    def direct():
        return [a.cpu().numpy() for a in eng.state_device()] + [eng.chi_squared_device().cpu().numpy()]

    getters = lambda: (eng.state_device(out=outs[0]), eng.chi_squared_device(out=outs[1]))
    g = _capture(torch, getters)
    before = direct()
    g.replay()
    assert all(same(a, b) for a, b in zip(read(), before))
    eng.linearize()                                                        # one accepted LM step: the working buffers swap
    lam = 1e-4 * eng.max_diagonal()
    eng.solve(lam)
    eng.update(lam)
    eng.commit(True)
    after = direct()
    assert not same(after[2], before[2])
    g.replay()
    assert all(same(a, b) for a, b in zip(read(), before))                 # the stale graph: the estimate of before the step
    g2 = _capture(torch, getters)
    g2.replay()
    assert all(same(a, b) for a, b in zip(read(), after))
    eng.close()


@pytest.mark.gpu
def test_stream_order(pkg, problems, torch_cuda):
    """the state is written by a torch kernel on a side stream, after a long kernel there, and handed to set_state_device on that
    stream: optimize() then gives the host path's result"""
    torch = torch_cuda
    prob = problems("small")
    rk = KERNELS["huber"]
    host, dev = new_engine(pkg, rk, "fp64", "pcg"), new_engine(pkg, rk, "fp64", "pcg")
    host.initialize(prob)
    d = to_dev(prob)
    dev.initialize_device(d)
    host.set_state(-prob.q, prob.t, prob.Xw)                              # the same rotations, the other sign

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        q = -d["q"]
        dev.set_state_device(q, d["t"], d["Xw"])
    assert stats_bytes(host.optimize(4)) == stats_bytes(dev.optimize(4))
    check_same_results(torch, host, dev, "stream order")
    host.close(); dev.close()


@pytest.mark.gpu
def test_state_errors_before_a_problem(pkg, torch_cuda):
    """a fresh engine: every device call fails with the host call's code and message"""
    eng = pkg.Engine(device=0)
    L = pkg.load_library()
    buf = torch_cuda.zeros(16, dtype=torch_cuda.float64, device="cuda:0")
    p = ctypes.c_void_p(buf.data_ptr())
    pairs = [(L.cuba_engine_set_state(eng.h, p, p, p), L.cuba_engine_set_state_device(eng.h, p, p, p, None)),
             (L.cuba_engine_get_state(eng.h, None, None, None), L.cuba_engine_get_state_device(eng.h, None, None, None, None)),
             (L.cuba_engine_set_edge_levels(eng.h, None), L.cuba_engine_set_edge_levels_device(eng.h, None, None))]
    for host, dev in pairs:
        assert host == dev == -3
    msgs = []
    for f in (lambda: L.cuba_engine_get_chi2(eng.h, p), lambda: L.cuba_engine_get_chi2_device(eng.h, p, None),
              lambda: L.cuba_engine_get_edge_levels(eng.h, p), lambda: L.cuba_engine_get_edge_levels_device(eng.h, p, None)):
        assert f() == -3
        msgs.append(L.cuba_last_error().decode())
    assert msgs[0] == msgs[1] and msgs[2] == msgs[3]
    eng.close()


def _refused(pkg, eng, d, msg):
    with pytest.raises(pkg.CubaError, match=msg):
        eng.initialize_device(d)


@pytest.mark.gpu
def test_refused_problems(pkg, problems, torch_cuda):
    """an index out of range and an edge with both ends fixed fail with set_problem's messages; the host structure builder is
    refused; after each refusal the engine optimises a valid problem as a fresh engine does"""
    prob = problems("tiny")
    rk = KERNELS["huber"]
    ref = new_engine(pkg, rk, "fp64", "pcg")
    ref.initialize(prob)
    want = stats_bytes(ref.optimize(4)), ref.state()
    ref.close()
    # an edge whose landmark keeps other edges, so that no free landmark is left without one
    seen = np.bincount(np.concatenate([prob.idx2[:, 1], prob.idx3[:, 1]]), minlength=prob.Lall)
    k = next(k for k in range(prob.E2) if seen[prob.idx2[k, 1]] > 1 and prob.idx2[k, 1] != prob.Lall - 1)
    bad_index = prob.copy(); bad_index.idx2 = prob.idx2.copy(); bad_index.idx2[k, 1] = prob.Lall
    both_fixed = prob.copy(); both_fixed.idx2 = prob.idx2.copy(); both_fixed.idx2[k] = (prob.Pall - 1, prob.Lall - 1)
    both_fixed.numP, both_fixed.numL = prob.Pall - 1, prob.Lall - 1
    for bad, msg in ((bad_index, "edge index out of range"), (both_fixed, "edge with both ends fixed")):
        host = new_engine(pkg, rk, "fp64", "pcg")
        with pytest.raises(pkg.CubaError, match=msg) as ei:
            host.initialize(bad)
        for held in (False, True):
            eng = new_engine(pkg, rk, "fp64", "pcg")
            if held:
                eng.initialize(prob)
            with pytest.raises(pkg.CubaError) as ed:
                eng.initialize_device(to_dev(bad))
            assert str(ed.value) == str(ei.value)
            eng.initialize_device(to_dev(prob))
            got = stats_bytes(eng.optimize(4)), eng.state()
            assert got[0] == want[0] and all(same(a, b) for a, b in zip(got[1], want[1])), (msg, held)
            eng.close()
        host.close()
    ref = new_engine(pkg, rk, "fp64", "pcg", structure_on_host=True)
    ref.initialize(prob)
    want = stats_bytes(ref.optimize(4)), ref.state()
    ref.close()
    eng = new_engine(pkg, rk, "fp64", "pcg", structure_on_host=True)
    eng.initialize(prob)
    before = eng.state()
    with pytest.raises(pkg.CubaError, match="cuba error -1: set_problem_device: the host structure builder"):
        eng.initialize_device(to_dev(prob.copy()))
    assert all(same(a, b) for a, b in zip(eng.state(), before))
    eng.initialize(prob)
    got = stats_bytes(eng.optimize(4)), eng.state()
    assert got[0] == want[0] and all(same(a, b) for a, b in zip(got[1], want[1]))
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,world", [("small", 3), ("shard_edges", 3)])
def test_dry_shards(pkg, problems, torch_cuda, name, world, monkeypatch):
    """landmark sharding on one GPU (CUBA_DRY_SHARD): rank r's device calls give its host calls' state, chi2 and levels, and judge
    "no edge included" on its own edges alike"""
    torch = torch_cuda
    monkeypatch.setenv("CUBA_DRY_SHARD", "1")
    prob = problems(name)
    rk = KERNELS["huber"]
    mask = mask_of(prob, seed=9)
    for r in range(world):
        host, dev = new_engine(pkg, rk, "fp64", "pcg"), new_engine(pkg, rk, "fp64", "pcg")
        host.set_comm(r, world)
        dev.set_comm(r, world)
        host.initialize(prob)
        dev.initialize_device(to_dev(prob))
        check_same_results(torch, host, dev, (name, r, "initial"))
        assert host.linearize() == dev.linearize()
        host.set_edge_levels(mask)
        dev.set_edge_levels_device(torch.from_numpy(mask).cuda())
        check_same_results(torch, host, dev, (name, r, "levels"))
        assert host.linearize() == dev.linearize()
        if r == 0:
            assert stats_bytes(host.optimize(3)) == stats_bytes(dev.optimize(3))
            check_same_results(torch, host, dev, (name, r, "optimize"))
        own = (host.chi_squared() != 0).astype(np.uint8)                  # a rank reports its own edges' chi2 only
        host.set_edge_levels(own)
        dev.set_edge_levels_device(torch.from_numpy(own).cuda())
        assert host.optimize(3) == [] and dev.optimize(3) == []
        dev.set_edge_levels_device(None)
        host.set_edge_levels(None)
        check_same_results(torch, host, dev, (name, r, "cleared"))
        host.close(); dev.close()
