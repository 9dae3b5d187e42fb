"""The drop-in class's linear solver (include/cuba_b200_solver.h: cuba::setLinearSolver), through tests/cpp/solver_driver.cpp.

  CPU   the driver compiles against the drop-in headers; the stored choice (cuba::linearSolver) follows setLinearSolver without a GPU
  GPU   ORB-SLAM2's local-BA protocol (Huber optimize(5), classifyEdges, NONE optimize(10), classifyEdges) on local_ba with
        DENSE_CHOLESKY is bit for bit Engine with the dense solver on the same flat problem; switching back to PCG after an
        optimize() gives bit for bit a default engine started from that estimate
"""
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import KERNELS, ROOT

CHI2 = (5.991, 7.815)
MAX_POSES = 2730


def _build_driver(tmp_path_factory, pkg):
    out = str(tmp_path_factory.mktemp("cppsolver") / "solver_driver")
    libdir = os.path.dirname(pkg.library_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-DCUBA_FORCE_EIGEN_COMPAT", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "solver_driver.cpp"), "-L", libdir, "-lcuba_b200",
                           "-Wl,-rpath," + libdir, "-o", out])
    return out


def _drive(tmp_path_factory, pkg, g, ops):
    exe = _build_driver(tmp_path_factory, pkg)
    d = tmp_path_factory.mktemp("solver")
    path = str(d / "g.cubagraph"); dump = str(d / "state.bin")
    pkg.graphio.write_graph(path, g)
    out = subprocess.run([exe, path, ";".join(ops), dump], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr
    steps = json.loads(out.stdout)["steps"]
    if not os.path.exists(dump):
        return steps, None
    nP, nL = len(g["pose_id"]), len(g["lm_id"])
    raw = np.fromfile(dump, dtype=np.float64)
    return steps, (raw[:4 * nP].reshape(nP, 4), raw[4 * nP:7 * nP].reshape(nP, 3), raw[7 * nP:].reshape(nL, 3))


def _engine(pkg, prob, rk, solver):
    eng = pkg.Engine(device=0)
    for et in (0, 1):
        eng.set_robust_kernels(rk[0][et], rk[1][et], et)
    eng.set_linear_solver(solver)
    eng.initialize(prob)
    return eng


def _set_kernels(eng, rk):
    for et in (0, 1):
        eng.set_robust_kernels(rk[0][et], rk[1][et], et)


def _in_graph_order(pkg, g, prob, state):
    cur = {k: np.array(v, copy=True) for k, v in g.items()}
    pkg.graphio.write_back(cur, prob, *state)
    return cur


def _assert_state(cur, dump):
    for k, v in zip(("q", "t", "Xw"), dump):
        assert np.array_equal(cur[k], v), k


def test_driver_stores_the_choice_without_a_gpu(pkg, tmp_path_factory):
    g = pkg.synth.make_config("tiny")
    steps, state = _drive(tmp_path_factory, pkg, g, ["query", "solver:dense", "query", "solver:dense", "query", "solver:pcg", "query"])
    assert [s["solver"] for s in steps if s["op"] == "query"] == [0, 1, 1, 0]
    assert state is None
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", pkg.library_path()], capture_output=True, text=True).stdout
    for s in ("cuba::setLinearSolver(", "cuba::linearSolver("):
        assert s in out, s


@pytest.mark.gpu
def test_orbslam_local_ba_with_dense_cholesky(pkg, tmp_path_factory):
    g = pkg.synth.make_config("local_ba")
    ops = ["solver:dense", "kernel:huber", "init", "opt:5", "classify:%g:%g" % CHI2, "kernel:none", "opt:10", "classify:%g:%g" % CHI2]
    steps, dump = _drive(tmp_path_factory, pkg, g, ops)
    prob = pkg.graphio.flatten(g)
    eng = _engine(pkg, prob, KERNELS["huber"], "dense")
    chi_a = [s["chi2"] for s in eng.optimize(5)]
    c1 = eng.classify_edges(*CHI2)
    _set_kernels(eng, KERNELS["none"])
    chi_b = [s["chi2"] for s in eng.optimize(10)]
    c2 = eng.classify_edges(*CHI2)
    assert steps[3]["chi2"] == chi_a and steps[6]["chi2"] == chi_b
    assert steps[4]["counts"] == list(c1.values()) and steps[7]["counts"] == list(c2.values())
    assert eng.pcg_info()["kernel"] == "k_dense_chol"
    _assert_state(_in_graph_order(pkg, g, prob, eng.state()), dump)
    eng.close()


@pytest.mark.gpu
def test_switching_back_to_pcg(pkg, tmp_path_factory):
    """dense optimize(5), then setLinearSolver(PCG) and optimize(5): the second run is a default engine's from that estimate"""
    g = pkg.synth.make_config("local_ba")
    ops = ["solver:dense", "kernel:huber", "init", "opt:5", "solver:pcg", "opt:5"]
    steps, dump = _drive(tmp_path_factory, pkg, g, ops)
    prob = pkg.graphio.flatten(g)
    eng = _engine(pkg, prob, KERNELS["huber"], "dense")
    chi_a = [s["chi2"] for s in eng.optimize(5)]
    mid = _in_graph_order(pkg, g, prob, eng.state())
    eng.close()
    prob2 = pkg.graphio.flatten(mid)
    pcg = _engine(pkg, prob2, KERNELS["huber"], "pcg")
    chi_b = [s["chi2"] for s in pcg.optimize(5)]
    assert steps[3]["chi2"] == chi_a and steps[5]["chi2"] == chi_b
    assert pcg.pcg_info()["kernel"] != "k_dense_chol"
    _assert_state(_in_graph_order(pkg, mid, prob2, pcg.state()), dump)
    pcg.close()


@pytest.mark.gpu
def test_refused_upload_stays_pending(pkg, tmp_path_factory):
    """2 731 free poses optimised with the PCG, then DENSE_CHOLESKY: optimize() throws, and keeps throwing on the next call
    (the choice stays pending, the engine's PCG problem is not used under the dense name); back to PCG, optimize() runs"""
    g = pkg.synth.make_graph(MAX_POSES + 2, 20000, 20000, 40000, 31)        # the first pose is fixed
    ops = ["kernel:huber", "init", "opt:1", "solver:dense", "tryopt:1", "tryopt:1", "query", "solver:pcg", "tryopt:1", "query"]
    steps, dump = _drive(tmp_path_factory, pkg, g, ops)
    assert [s["threw"] for s in steps if s["op"] == "tryopt:1"] == [True, True, False]
    assert [s["solver"] for s in steps if s["op"] == "query"] == [1, 0]
    assert dump is not None
