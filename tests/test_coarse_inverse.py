"""k_coarse_dense (csrc/cuba_coarse.cuh), the dense coarse inverse of the two-level PCG, on matrices of our own through
cuba_debug_coarse_inverse: the fp32 inverse against fp64, bit-reproducibility and the not-positive-definite path, which a solve
never takes (block-Jacobi alone carries on, silently).

The matrices are scaled like the real coarse matrix Ac = Z^T S Z, whose condition number of about 1e11 comes from its scaling
(translations of kilometres in the rigid-motion basis): D B D with B an SPD matrix of condition 1e4 and D spanning 2e4."""
import numpy as np
import pytest

from test_pcg_coarse import INV_RESIDUAL_FACTOR, packed_to_dense

SIZES = (38, 64, 133, 264)     # aggregates: smallest dense shape, 384 = 12 tiles exactly, one past 792, the K = 2 shape (1584)


def dense_to_packed(M, A):
    """symmetric [6A][6A] -> packed lower block triangle [A(A+1)/2][36], each block column-major (inverse of packed_to_dense)"""
    out = np.empty((A * (A + 1) // 2, 36))
    b = 0
    for ib in range(A):
        for jb in range(ib + 1):
            out[b] = M[6 * ib:6 * ib + 6, 6 * jb:6 * jb + 6].T.reshape(-1)
            b += 1
    return out


def scaled_spd(A, seed, cond_b=1e4, span=2e4):
    n = 6 * A
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    B = (Q * np.logspace(0, np.log10(cond_b), n)) @ Q.T
    d = np.logspace(0, np.log10(span), n)[rng.permutation(n)]
    M = d[:, None] * B * d[None, :]
    return 0.5 * (M + M.T)


def test_packing_round_trip():
    M = scaled_spd(5, 0)
    assert np.array_equal(packed_to_dense(dense_to_packed(M, 5), 5), M)


@pytest.fixture(scope="module")
def engine(pkg):
    eng = pkg.Engine(device=0)
    yield eng
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("A", SIZES)
def test_inverse_against_fp64(engine, A):
    """d_inv and |AcInv Ac - I| against the fp64 inverse rounded once to fp32, the criteria of test_pcg_coarse.py; exactly
    symmetric; the same bits on a second call"""
    M = scaled_spd(A, A)
    AcP = dense_to_packed(M, A)
    Ac = packed_to_dense(AcP, A)
    inv, info = engine.coarse_inverse(AcP)
    assert info == 0
    inv64 = np.linalg.inv(Ac)
    d_inv = np.abs(inv - inv64).max() / np.abs(inv64).max()
    eye = np.eye(6 * A)
    resid = np.abs(inv.astype(np.float64) @ Ac - eye).max()
    floor = np.abs(inv64.astype(np.float32).astype(np.float64) @ Ac - eye).max()
    print("A %3d nc %4d cond %.1e: d_inv %.1e, |AcInv Ac - I| %.1e = %.2f x the fp32 floor" % (A, 6 * A, np.linalg.cond(Ac), d_inv, resid, resid / floor))
    assert d_inv < 2e-6, d_inv
    assert resid <= INV_RESIDUAL_FACTOR * floor, (resid, floor)
    assert np.array_equal(inv, inv.T)
    again, info2 = engine.coarse_inverse(AcP)
    assert info2 == 0 and np.array_equal(again.view(np.uint32), inv.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("A", (38, 133))
def test_indefinite_matrix_is_refused(engine, A):
    """a negative eigenvalue: info 1 and an all-zero inverse (the PCG then runs block-Jacobi alone)"""
    n = 6 * A
    M = scaled_spd(A, 7)
    v = np.random.default_rng(8).standard_normal(n)
    v /= np.linalg.norm(v)
    lo = np.linalg.eigvalsh(M)[-1]
    M = M - 2 * lo * np.outer(v, v)                  # now v^T M v < 0
    M = 0.5 * (M + M.T)
    inv, info = engine.coarse_inverse(dense_to_packed(M, A))
    assert info == 1
    assert not inv.any()
