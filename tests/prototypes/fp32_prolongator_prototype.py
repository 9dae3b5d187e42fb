"""CPU prototype behind the fp32 prolongator of k_pcg5t (csrc/cuba_pcg5t.cuh): PCG iterations of the two-level preconditioner in
hat space, M^-1 = I + Z^ Ac^-1 Z^^T with A^ = L^-1 S L^-T, on the reduced pose system the CPU oracle assembles, with
  * K aggregates per CTA cut like the engine's (CTAs balanced by block count, a CTA's rows in K groups balanced by row count),
  * the engine's stopping rule r'r <= tol^2 r0'r0 in hat space (the block-Jacobi norm), tol 1e-11,
  * Ac^-1 rounded to fp32 as the engine stores it, and
  * Z^ in fp64, or rounded to fp32 in both places it is applied (what the kernel keeps in shared memory).
Test infrastructure (it uses the oracle); not collected by pytest.  Needs scipy.

    python tests/prototypes/fp32_prolongator_prototype.py [kitti00_shaped | ba_kitti_00 | ...]
"""
import os, sys
import numpy as np, scipy.sparse as sp
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge
pkg = ge.load_package(); oracle = ge.load_oracle()
name = sys.argv[1] if len(sys.argv) > 1 else 'kitti00_shaped'
if name.startswith('ba_'): g = pkg.graphio.read_graph(os.path.join(ROOT, 'oracle', '_ref', 'fixtures', '%s.cubagraph' % name))
else: g = pkg.synth.make_config(name)
prob = pkg.graphio.flatten(g)
o = oracle.Oracle(prob, (0, 0), (0.0, 0.0))
o.compute_errors(); o.build_system()
md = o.max_diagonal()
rp, ci = o.hsc_structure()
P = prob.numP
G = min(132, (P + 7) // 8)


def system(lam):
    """S (symmetric, full) and b of the reduced system at lambda"""
    assert o.solve(lam)
    Hsc, bsc, inv = o.schur()
    B = Hsc.reshape(-1, 6, 6).transpose(0, 2, 1)
    rows = np.repeat(np.arange(P), np.diff(rp))
    rr, cc = (x.ravel() for x in np.meshgrid(np.arange(6), np.arange(6), indexing='ij'))
    I = (6 * rows[:, None] + rr[None, :]).ravel(); J = (6 * np.asarray(ci)[:, None] + cc[None, :]).ravel()
    U = sp.csr_matrix((B.reshape(len(ci), 36).ravel(), (I, J)), shape=(6 * P, 6 * P))
    Dblk = sp.block_diag([U[6 * i:6 * i + 6, 6 * i:6 * i + 6].toarray() for i in range(P)], format='csr')
    Off = U - Dblk
    return (Dblk + Off + Off.T).tocsr(), bsc.reshape(-1).copy()


def adjoints():
    q = prob.q[:P]; t = prob.t[:P]; out = []
    for i in range(P):
        x, y, z, w = q[i]
        R = np.array([[1-2*(y*y+z*z), 2*(x*y-z*w), 2*(x*z+y*w)], [2*(x*y+z*w), 1-2*(x*x+z*z), 2*(y*z-x*w)], [2*(x*z-y*w), 2*(y*z+x*w), 1-2*(x*x+y*y)]])
        tx = np.array([[0, -t[i][2], t[i][1]], [t[i][2], 0, -t[i][0]], [-t[i][1], t[i][0], 0]])
        Ad = np.zeros((6, 6)); Ad[:3, :3] = R; Ad[3:, 3:] = R; Ad[3:, :3] = tx @ R
        out.append(Ad)
    return out


def aggregates(K):
    """first row of every aggregate: G CTAs with about the same number of blocks (upper and lower triangle), K groups of rows each"""
    full = np.zeros(P, np.int64)
    rows = np.repeat(np.arange(P), np.diff(rp))
    np.add.at(full, rows, 1); np.add.at(full, np.asarray(ci)[np.asarray(ci) != rows], 1)
    cum = np.concatenate([[0], np.cumsum(full)])
    cta = [0]
    for c in range(1, G):
        r = int(np.searchsorted(cum, cum[-1] * c / G))
        cta.append(min(max(r, cta[-1] + K), P - K * (G - c)))
    cta.append(P)
    return np.array([cta[c] + (cta[c + 1] - cta[c]) * j // K for c in range(G) for j in range(K)] + [P])


def pcg(A, b, Minv, tol=1e-11, maxit=5000):
    x = np.zeros_like(b); r = b.copy(); z = Minv(r); p = z.copy(); rz = r @ z; n0 = r @ r; it = 0
    while it < maxit:
        Ap = A @ p; al = rz / (p @ Ap); x += al * p; r -= al * Ap; it += 1
        if r @ r <= tol * tol * n0: break
        z = Minv(r); rzn = r @ z
        p = z + (rzn / rz) * p; rz = rzn
    return x, it


adj = adjoints()
rr, cc = np.meshgrid(np.arange(6), np.arange(6), indexing='ij')
print('%s: %d poses, %d CTAs' % (name, P, G), flush=True)
for scale in (1.0, 1e-2, 1e-4):
    S, b = system(1e-5 * md * scale)
    Ls = [np.linalg.cholesky(S[6 * i:6 * i + 6, 6 * i:6 * i + 6].toarray()) for i in range(P)]
    Linv = sp.block_diag([np.linalg.inv(L) for L in Ls], format='csr')
    Ah = (Linv @ S @ Linv.T).tocsr(); bh = Linv @ b
    line = 'lambda = 1e-5 maxdiag * %g:' % scale
    for K in (1, 2):
        first = aggregates(K)
        rowAgg = np.repeat(np.arange(G * K), np.diff(first))
        I = np.concatenate([(6 * i + rr).ravel() for i in range(P)])
        J = np.concatenate([(6 * rowAgg[i] + cc).ravel() for i in range(P)])
        Zh = sp.csr_matrix((np.concatenate([(Ls[i].T @ adj[i]).ravel() for i in range(P)]), (I, J)), shape=(6 * P, 6 * G * K))
        Aci = np.linalg.inv((Zh.T @ Ah @ Zh).toarray())
        Aci32 = Aci.astype(np.float32).astype(np.float64)
        Zh32 = Zh.copy(); Zh32.data = Zh32.data.astype(np.float32).astype(np.float64)
        x0, it0 = pcg(Ah, bh, lambda r: r + Zh @ (Aci @ (Zh.T @ r)))
        x1, it1 = pcg(Ah, bh, lambda r: r + Zh @ (Aci32 @ (Zh.T @ r)))
        x2, it2 = pcg(Ah, bh, lambda r: r + Zh32 @ (Aci32 @ (Zh32.T @ r)))
        line += '  K = %d (%d aggregates): fp64 %d, fp32 Ac^-1 %d, fp32 Ac^-1 and Z^ %d (|dx| rel %.1e)' % (
            K, G * K, it0, it1, it2, np.abs(x2 - x0).max() / np.abs(x0).max())
    print(line, flush=True)
