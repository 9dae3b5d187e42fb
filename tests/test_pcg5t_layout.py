"""Shared-memory plan of the one-GPU tuned PCG (csrc/cuba_pcg5t.cuh): two coarse aggregates per CTA fit next to every Z^ and (all
but a few of) the cached blocks on an H100, the plan falls back to one aggregate per CTA when they do not, and on the GPU the
two-aggregate plan reaches the same solution in fewer iterations."""
import numpy as np
import pytest

from conftest import NONE, have_fixture, make_engine, relerr

H100_SMS = 132


def _names():
    return ["kitti00_shaped"] + (["ba_kitti_00"] if have_fixture("ba_kitti_00") else [])


@pytest.mark.parametrize("scalar_bytes", [8, 4])
@pytest.mark.parametrize("name", _names())
def test_two_aggregates_per_cta_fit_on_an_h100(pkg, problems, name, scalar_bytes):
    prob = problems(name)
    budget = pkg.binding.H100_SMEM_BUDGET
    one = pkg.binding.pcg5t_layout_host(prob, 1, H100_SMS, scalar_bytes, budget)
    two = pkg.binding.pcg5t_layout_host(prob, 2, H100_SMS, scalar_bytes, budget)
    plan = pkg.pcg5_plan_apc_host(prob, 2)
    print(name, scalar_bytes, one, two)
    assert one["ok"] and one["aggs_per_cta"] == 1 and one["streamed_blocks"] == 0 and one["zhInSmem"] == 1
    assert two["ok"] and two["aggs_per_cta"] == 2 and two["zhInSmem"] == 1
    assert two["total_bytes"] <= budget
    # Z^ never leaves the chip for the larger slice; at most one warp's share of a product round of blocks does
    assert 0 <= two["streamed_blocks"] <= 32
    assert two["capBlocks"] + two["streamed_blocks"] == max(plan["blkMax"] - 512, 0) == one["capBlocks"]
    # fp32 Z^ (36 words per needed column), the slice of the fp32 inverse (rows of this CTA x nc), 512 staging slots
    assert two["zh_bytes"] == one["zh_bytes"] == 36 * 4 * plan["needMax"]
    nc = 6 * plan["A"]
    assert two["slice_bytes"] == -(-nc // plan["G"]) * nc * 4 == 4 * one["slice_bytes"]
    assert one["staging_bytes"] == min(512, -(-plan["blkMax"] // 32) * 32) * 6 * 8
    assert two["rc_bytes"] == nc * scalar_bytes


@pytest.mark.parametrize("name", _names())
def test_plan_falls_back_to_one_aggregate_per_cta(pkg, problems, name):
    prob = problems(name)
    layout = pkg.binding.pcg5t_layout_host
    one = layout(prob, 1, H100_SMS, 8)
    two = layout(prob, 2, H100_SMS, 8)
    # shared memory that holds the one-aggregate plan but not the larger slice of the inverse, even with 32 blocks streamed
    tight = two["total_bytes"] - 33 * (36 * 8 + 4) - 2048
    assert tight >= one["total_bytes"] + 64
    back = layout(prob, 2, H100_SMS, 8, tight)
    assert back["ok"] and back["aggs_per_cta"] == 1 and back == layout(prob, 1, H100_SMS, 8, tight)
    assert back["streamed_blocks"] == 0 and back["capBlocks"] == one["capBlocks"]
    # nothing fits: no tuned plan at all (the engine then takes the 256-thread kernel)
    assert layout(prob, 2, H100_SMS, 8, 8192)["ok"] == 0
    with pytest.raises(pkg.CubaError):
        layout(prob, 4, H100_SMS, 8)


@pytest.mark.gpu
@pytest.mark.parametrize("name", _names())
def test_two_aggregates_per_cta_same_solution_fewer_iterations(pkg, problems, name, monkeypatch):
    """optimize(10) with every solve two-level: CUBA_PCG5_AGGS_PER_CTA=2 against the default plan (one aggregate per CTA)"""
    prob = problems(name)
    out = {}
    for apc in (1, 2):
        if apc == 2:
            monkeypatch.setenv("CUBA_PCG5_AGGS_PER_CTA", "2")
        eng = make_engine(pkg, prob, NONE, pcg_variant=5)
        stats = eng.optimize(10)
        info = eng.pcg_info()
        assert info["kernel"] == "k_pcg5t" and info["two_level"] and info["aggs_per_cta"] == apc and info["bj_retries"] == 0, info
        assert info["zhInSmem"] == 1, info
        out[apc] = (sum(s["pcg_iters"] for s in stats), np.array([s["chi2"] for s in stats]), [x.copy() for x in eng.state()])
        eng.close()
    print(name, "PCG iterations of optimize(10): K = 1 %d, K = 2 %d" % (out[1][0], out[2][0]))
    assert out[2][0] < out[1][0], (out[1][0], out[2][0])
    assert relerr(out[2][1], out[1][1]) < 1e-9
    for nme, a, b in zip(("q", "t", "Xw"), out[2][2], out[1][2]):
        assert relerr(a, b) < 1e-9, (nme, relerr(a, b))
