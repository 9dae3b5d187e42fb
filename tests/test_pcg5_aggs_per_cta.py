"""Several coarse aggregates per CTA in the one-GPU tuned PCG (csrc/cuba_pcg5t.cuh): the plan that cuts every CTA's rows into
K contiguous groups (csrc/cuba_structure.cpp, checked by the library's own invariants), and the premise behind it -- smaller
rigid-motion aggregates cut the iteration count of the two-level PCG on the KITTI-00-shaped system."""
import numpy as np
import pytest

from conftest import have_fixture
from test_two_level_prototype import _adjoints, _pcg, _system


def _names():
    return ["kitti07_shaped", "kitti00_shaped"] + (["ba_kitti_00"] if have_fixture("ba_kitti_00") else [])


@pytest.mark.parametrize("name", _names())
@pytest.mark.parametrize("apc", [2, 3])
def test_plan_with_several_aggregates_per_cta(pkg, problems, name, apc):
    prob = problems(name)
    one = pkg.pcg5_plan_apc_host(prob, 1)
    info = pkg.pcg5_plan_apc_host(prob, apc)
    assert one["ok"] and info["ok"]
    # same rows over the same CTAs, K times the aggregates, none spanning CTAs
    assert info["G"] == one["G"] and info["maxRows"] == one["maxRows"] and info["needMax"] == one["needMax"]
    assert info["gs"] == 1 and info["A"] == apc * info["G"]
    assert one["maxNeedAgg"] <= info["maxNeedAgg"] <= apc * one["maxNeedAgg"]
    assert info["hash"] != one["hash"]


@pytest.mark.parametrize("name", _names())
def test_one_aggregate_per_cta_is_the_plan_of_k_pcg5(pkg, problems, name):
    prob = problems(name)
    one = pkg.pcg5_plan_apc_host(prob, 1)
    ref = pkg.pcg5_plan_host(prob, 1, 132, 148)
    assert {k: v for k, v in one.items() if k != "hash"} == ref
    assert one["hash"] == pkg.pcg5_plan_apc_host(prob, 1)["hash"] != 0


def test_several_aggregates_per_cta_only_on_one_gpu(pkg, problems):
    prob = problems("kitti00_shaped")
    assert pkg.pcg5_plan_apc_host(prob, 2, world=2)["ok"] == 0
    assert pkg.pcg5_plan_apc_host(prob, 1, world=2)["ok"] == 1
    with pytest.raises(pkg.CubaError):
        pkg.pcg5_plan_apc_host(prob, 4)


def test_smaller_aggregates_cut_the_iteration_count(pkg, oracle, problems):
    """K = 2 halves the aggregate size (about ten poses per CTA on 132 CTAs): exact coarse inverse, consecutive poses"""
    sp = pytest.importorskip("scipy.sparse")
    prob = problems("kitti00_shaped")
    P = prob.numP
    o = oracle.Oracle(prob, (0, 0), (0.0, 0.0))
    o.compute_errors(); o.build_system()
    lam = 1e-8 * o.max_diagonal()
    A, b = _system(o, P, lam)
    D = sp.block_diag([sp.csr_matrix(np.linalg.inv(A[6 * i:6 * i + 6, 6 * i:6 * i + 6].toarray())) for i in range(P)], format="csr")
    adj = _adjoints(prob, P)
    rr, cc = np.meshgrid(np.arange(6), np.arange(6), indexing="ij")
    I = np.concatenate([(6 * i + rr).ravel() for i in range(P)])
    V = np.concatenate([a.ravel() for a in adj])
    its, xs = {}, {}
    for m in (10, 5):
        na = -(-P // m)
        J = np.concatenate([(6 * (i // m) + cc).ravel() for i in range(P)])
        Z = sp.csr_matrix((V, (I, J)), shape=(6 * P, 6 * na))
        Aci = np.linalg.inv((Z.T @ A @ Z).toarray())
        xs[m], its[m] = _pcg(A, b, lambda r: D @ r + Z @ (Aci @ (Z.T @ r)))
    assert its[5] < 0.8 * its[10], its
    assert np.abs(xs[5] - xs[10]).max() <= 1e-6 * np.abs(xs[10]).max()
