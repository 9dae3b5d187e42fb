"""The per-edge primitives of csrc/cuba_math.cuh -- se3_update, robust, edge_residual / edge_jacobians, sym3_inverse and
spd6_inverse -- compiled with g++ from the very header the kernels include (tests/cpp/math_driver.cpp), in their float and double
instantiations, against numpy longdouble restatements.  No GPU needed.

Every bound is K u |M|: u the unit roundoff of the type, M the magnitude the formula works with (written next to each bound) and K a
small constant.  The inputs are chosen where these primitives go wrong and the synthetic graphs never go: rotation angles on both
sides of the small-angle branch and through the range where 1 - cos(theta) cancels, rotations past 120 degrees (the trace <= 0
branch of the rotation -> quaternion conversion, each pivot), quaternions with w <= 0, poses at the origin, points 0.1 and 1e4 in
front of the camera or at the image border, robust-kernel thresholds to the ulp, and 3x3 / 6x6 inverses up to condition 1e7 (float)
and 1e14 (double)."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "cuda-bundle-adjustment_b200", "csrc")
U = {"float": 2.0 ** -24, "double": 2.0 ** -53}
NPT = {"float": np.float32, "double": np.float64}
LD = np.longdouble
TYPES = ["float", "double"]
K00 = (718.8560180664062, 718.8560180664062, 607.1928100585938, 185.2156982421875, 386.1448059082031)


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("cppmath") / "math_driver")
    # no FMA contraction on the host: every product and sum is rounded once, as the bounds below assume
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-I", CSRC,
                           os.path.join(ROOT, "tests", "cpp", "math_driver.cpp"), "-o", out])
    return out


def rnd(a, typ):
    """a rounded to the type (as float64): the driver's inputs are exactly representable, so the reference sees the same numbers"""
    return np.asarray(a, dtype=np.float64).astype(NPT[typ]).astype(np.float64)


def run(driver, typ, fn, rows):
    rows = np.atleast_2d(np.asarray(rows, dtype=np.float64))
    assert np.array_equal(rnd(rows, typ), rows)
    txt = "\n".join(" ".join(repr(float(v)) for v in r) for r in rows) + "\n"
    out = subprocess.run([driver, typ, fn], input=txt, capture_output=True, text=True, check=True).stdout
    res = np.array([[float(v) for v in line.split()] for line in out.splitlines()])
    assert res.shape[0] == rows.shape[0]
    return res


def report(label, err, bound):
    ratio = float(np.max(err / bound))
    print("%-40s max measured/bound %.3g" % (label, ratio))
    return ratio


# ---- SE(3) update --------------------------------------------------------------------------------------------------------------

def skew(w):
    O = np.zeros(w.shape[:-1] + (3, 3), dtype=w.dtype)
    O[..., 0, 1], O[..., 0, 2], O[..., 1, 2] = -w[..., 2], w[..., 1], -w[..., 0]
    O[..., 1, 0], O[..., 2, 0], O[..., 2, 1] = w[..., 2], -w[..., 1], w[..., 0]
    return O


def quat_mul(a, b):
    c = np.empty_like(a)
    c[:, 3] = a[:, 3] * b[:, 3] - (a[:, :3] * b[:, :3]).sum(1)
    c[:, :3] = a[:, 3:4] * b[:, :3] + b[:, 3:4] * a[:, :3] + np.cross(a[:, :3], b[:, :3])
    return c


def quat_rot(q):
    """rotation matrix of the unit quaternion q (x, y, z, w)"""
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.empty((len(q), 3, 3), dtype=q.dtype)
    R[:, 0, 0], R[:, 0, 1], R[:, 0, 2] = 1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)
    R[:, 1, 0], R[:, 1, 1], R[:, 1, 2] = 2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)
    R[:, 2, 0], R[:, 2, 1], R[:, 2, 2] = 2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)
    return R


def se3_exact(upd, q, t):
    """pose <- Exp([omega; upsilon]) * pose in longdouble, without cancellation: a2 = (1 - cos th) / th^2 = 1/2 (sin(th/2) / (th/2))^2,
    a3 = (th - sin th) / th^3 by its series below th = 1, the exponential's rotation as the quaternion (sin(th/2) n, cos(th/2)).
    Returns (q, t, R of the update, theta)."""
    upd, q, t = (np.asarray(a, dtype=LD) for a in (upd, q, t))
    w, v = upd[:, :3], upd[:, 3:]
    th = np.sqrt((w * w).sum(1))
    h = th / 2
    sh = np.where(h > 0, np.sin(h) / np.where(h > 0, h, 1), LD(1))          # sin(h) / h
    a2 = sh * sh / 2
    th2 = th * th
    ser, term = np.zeros_like(th), np.ones_like(th) / 6                       # sum_k (-th^2)^k / (2k + 3)!
    for k in range(14):
        ser = ser + term
        term = -term * th2 / ((2 * k + 4) * (2 * k + 5))
    a3 = np.where(th < 1, ser, (th - np.sin(th)) / np.where(th < 1, 1, th * th2))
    O1 = skew(w)
    O2 = O1 @ O1
    V = np.eye(3, dtype=LD) + a2[:, None, None] * O1 + a3[:, None, None] * O2
    eq = np.concatenate([w * (sh / 2)[:, None], np.cos(h)[:, None]], axis=1)
    Re = quat_rot(eq)
    tn = np.einsum("nij,nj->ni", V, v) + np.einsum("nij,nj->ni", Re, t)
    r = quat_mul(eq, q)
    r = r / np.sqrt((r * r).sum(1))[:, None]
    r = np.where(r[:, 3:4] < 0, -r, r)
    return r.astype(np.float64), tn.astype(np.float64), Re.astype(np.float64), th.astype(np.float64)


def unit(rng, n):
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1)[:, None]


def random_quat(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1)[:, None]
    return q * np.sign(q[:, 3:4] + 1e-300)


def se3_records(rng, typ, theta, dirs=None, q=None, tscale=10.0, vscale=0.3):
    n = len(theta)
    dirs = unit(rng, n) if dirs is None else dirs
    w = rnd(dirs * np.asarray(theta)[:, None], typ)
    v = rnd(rng.normal(0, vscale, (n, 3)), typ)
    q = rnd(random_quat(rng, n) if q is None else q, typ)
    t = rnd(rng.normal(0, tscale, (n, 3)), typ)
    return np.concatenate([w, v, q, t], axis=1)


def check_se3(driver, typ, rec, label, K_q=32, K_t=32):
    out = run(driver, typ, "se3", rec)
    q_ref, t_ref, _, th = se3_exact(rec[:, :6], rec[:, 6:10], rec[:, 10:13])
    u = U[typ]
    assert np.all(out[:, 3] >= 0), "quaternion not normalised to w >= 0"
    # q: rotation -> quaternion, product and normalisation, each a few roundings of numbers of magnitude 1
    eq = np.minimum(np.abs(out[:, :4] - q_ref).max(1), np.abs(out[:, :4] + q_ref).max(1))
    rq = report("se3<%s> %s q" % (typ, label), eq, K_q * u)
    # t = V upsilon + R t: M = |t| + |upsilon|.  The double instantiation keeps the reference's a2 = (1 - cos th) / th^2 above the
    # small-angle branch, whose cancellation leaves u / th^2 in a2 and so u / th |upsilon| in V upsilon (at most 1.1e-11 |upsilon|,
    # at th = 1e-5); the float instantiation has no such term.
    nt, nv = np.linalg.norm(rec[:, 10:13], axis=1), np.linalg.norm(rec[:, 3:6], axis=1)
    cancel = nv / np.maximum(th, 1e-5) if typ == "double" else 0.0
    bt = K_t * u * (nt + nv + cancel)
    et = np.abs(out[:, 4:7] - t_ref).max(1)
    rt = report("se3<%s> %s t" % (typ, label), et, bt)
    bad = np.argsort(-et / bt)[:3]
    assert rq <= 1 and rt <= 1, ("worst rows: theta", th[bad], "t err", et[bad], "bound", bt[bad], "q err", eq[bad])


def theta_ladder():
    return np.concatenate([np.logspace(-8, np.log10(3), 160),        # the whole range
                           np.linspace(0.5e-5, 2e-5, 61),             # both sides of the small-angle branch at 1e-5
                           np.logspace(-4, -2, 120)])                 # where 1 - cos(theta) and theta - sin(theta) cancel in fp32


@pytest.mark.parametrize("typ", TYPES)
def test_se3_update_theta_ladder(driver, typ):
    rng = np.random.default_rng(11)
    th = theta_ladder()
    check_se3(driver, typ, se3_records(rng, typ, th), "theta ladder")


@pytest.mark.parametrize("typ", TYPES)
def test_se3_update_near_the_origin(driver, typ):
    """poses whose translation is tiny next to the step: there V upsilon is the whole answer and its error is not hidden behind |t|"""
    rng = np.random.default_rng(12)
    th = theta_ladder()
    check_se3(driver, typ, se3_records(rng, typ, th, tscale=1e-4, vscale=1.0), "|t| ~ 1e-4")
    check_se3(driver, typ, se3_records(rng, typ, th, tscale=0.0, vscale=0.05), "t = 0")


@pytest.mark.parametrize("typ", TYPES)
def test_se3_update_large_rotations_take_every_pivot(driver, typ):
    """rotations of 120 .. 178 degrees: trace(R) <= 0, the conversion to a quaternion pivots on the largest diagonal entry"""
    rng = np.random.default_rng(13)
    recs, piv = [], []
    for i in range(3):
        n = 40
        d = rng.normal(0, 0.25, (n, 3)); d[:, i] = np.sign(rng.normal(size=n)) * (1 + rng.random(n))
        d /= np.linalg.norm(d, axis=1)[:, None]
        th = rng.uniform(2.1, 3.1, n)
        recs.append(se3_records(rng, typ, th, dirs=d))
    rec = np.concatenate(recs)
    _, _, Re, th = se3_exact(rec[:, :6], rec[:, 6:10], rec[:, 10:13])
    diag = np.einsum("nii->ni", Re)
    assert np.all(diag.sum(1) <= 0)
    piv = np.argmax(diag, axis=1)
    assert set(np.unique(piv)) == {0, 1, 2}
    check_se3(driver, typ, rec, "trace <= 0")


@pytest.mark.parametrize("typ", TYPES)
def test_se3_update_quaternion_sign(driver, typ):
    """input quaternions with w = 0, w tiny either side of 0 and w < 0: the result is the same rotation with w >= 0"""
    rng = np.random.default_rng(14)
    n = 60
    q = random_quat(rng, n)
    q[:20, 3] = 0.0
    q[20:40, 3] = rng.choice([-1, 1], 20) * 10.0 ** rng.uniform(-9, -4, 20)
    q[40:, 3] = -np.abs(q[40:, 3])
    q[:, :3] *= np.sqrt(1 - q[:, 3:4] ** 2) / np.linalg.norm(q[:, :3], axis=1)[:, None]
    th = np.concatenate([np.zeros(10), 10.0 ** rng.uniform(-7, 0, n - 10)])
    check_se3(driver, typ, se3_records(rng, typ, th, q=q), "w <= 0")


# ---- robust kernels ------------------------------------------------------------------------------------------------------------

def robust_ref(kind, delta, d2, e):
    """rho, rho' in longdouble with the branch threshold the kernel uses (its own rounded delta^2)"""
    e, delta, d2 = LD(e), LD(delta), LD(d2)
    if kind == 1:
        return (e, LD(1)) if e <= d2 else (2 * np.sqrt(e) * delta - delta * delta, delta / np.sqrt(e))
    if kind == 2:
        m = delta * delta / 3
        if e <= d2:
            u = 1 - e / (delta * delta)
            return m * (1 - u ** 3), u * u
        return m, LD(0)
    return e, LD(1)


@pytest.mark.parametrize("typ", TYPES)
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_robust_kernels_at_the_threshold(driver, typ, kind):
    T = NPT[typ]
    u = U[typ]
    rows = []
    for delta in (5.991 ** 0.5, 7.815 ** 0.5, 4.0, 5.0):
        dl = T(delta)
        d2 = T(dl * dl)
        es = [T(0), d2, np.nextafter(d2, T(0)), np.nextafter(d2, T(np.inf)), T(d2 * T(0.5)), T(d2 * T(1.5)), T(d2 * T(100))]
        es += list(np.asarray(np.logspace(-6, 3, 20), dtype=T))
        rows += [(kind, float(dl), float(e)) for e in es]
    rows = np.array(rows)
    out = run(driver, typ, "robust", rows)
    ref = np.array([[float(x) for x in robust_ref(kind, r[1], float(T(T(r[1]) * T(r[1]))), r[2])] for r in rows])
    d2s = np.array([float(T(T(r[1]) * T(r[1]))) for r in rows])
    # rho: a handful of roundings of numbers no larger than max(e, 2 sqrt(e) delta, delta^2)
    M = np.maximum(rows[:, 2], d2s) + 2 * np.sqrt(rows[:, 2] * d2s)
    report("robust<%s> kind %d rho" % (typ, kind), np.abs(out[:, 0] - ref[:, 0]), 16 * u * M)
    assert np.all(np.abs(out[:, 0] - ref[:, 0]) <= 16 * u * M)
    assert np.all(np.abs(out[:, 1] - ref[:, 1]) <= 16 * u * np.maximum(np.abs(ref[:, 1]), 1))
    # e = 0: rho = 0, rho' = 1 exactly
    z = rows[:, 2] == 0
    assert np.all(out[z, 0] == 0) and np.all(out[z, 1] == 1)
    # continuity across delta^2 (one ulp either side)
    for k in range(0, len(rows), 27):
        lo, at, hi = out[k + 2], out[k + 1], out[k + 3]
        d2 = d2s[k + 1]
        assert abs(hi[0] - lo[0]) <= 16 * u * d2 and abs(hi[0] - at[0]) <= 16 * u * d2, (lo, at, hi)
        assert abs(hi[1] - lo[1]) <= 16 * u, (lo, at, hi)
    if kind == 2:
        assert np.all(out[rows[:, 2] > d2s, 1] == 0)          # Tukey: rho' vanishes above delta^2
        assert np.all(out[rows[:, 2] <= d2s, 1] >= 0)


# ---- residual and Jacobians of one edge ------------------------------------------------------------------------------------------

def residual_ld(q, t, cam, Xw, m, stereo):
    """edge_residual in longdouble for a batch; q need not be unit (the kernel's rotate() uses it as given)"""
    q, t, cam, Xw, m = (np.asarray(a, dtype=LD) for a in (q, t, cam, Xw, m))
    qv = q[:, :3]
    a = 2 * np.cross(qv, Xw)
    Xc = Xw + q[:, 3:4] * a + np.cross(qv, a) + t
    iz = 1 / Xc[:, 2]
    uu = cam[:, 0] * Xc[:, 0] * iz + cam[:, 2]
    vv = cam[:, 1] * Xc[:, 1] * iz + cam[:, 3]
    r = np.stack([uu - m[:, 0], vv - m[:, 1], np.where(stereo, uu - cam[:, 4] * iz - m[:, 2], 0)], axis=1)
    return Xc, r


def project_ld(Xc, cam, m, stereo):
    iz = 1 / Xc[:, 2]
    uu = cam[:, 0] * Xc[:, 0] * iz + cam[:, 2]
    vv = cam[:, 1] * Xc[:, 1] * iz + cam[:, 3]
    return np.stack([uu - m[:, 0], vv - m[:, 1], np.where(stereo, uu - cam[:, 4] * iz - m[:, 2], 0)], axis=1)


def jacobians_fd(q, t, cam, Xw, m, stereo):
    """-d r / d(delta) under pose <- Exp(delta) pose (the LM's left update, which moves the camera-frame point to
    R(omega) Xc + V(omega) upsilon) and -d r / d Xw (which moves it by R(q) dXw), by a sixth-order central difference in longdouble"""
    n = len(q)
    cam, m = np.asarray(cam, LD), np.asarray(m, LD)
    Xc0, _ = residual_ld(q, t, cam, Xw, m, stereo)
    Z = np.abs(Xc0[:, 2])
    qn = np.asarray(q, LD) / np.sqrt((np.asarray(q, LD) ** 2).sum(1))[:, None]
    Rq = quat_rot(qn)
    JP = np.zeros((n, 3, 6)); JL = np.zeros((n, 3, 3))

    def r_pose(k, h):
        d = np.zeros((n, 6), dtype=LD); d[:, k] = h
        w, v = d[:, :3], d[:, 3:]
        th = np.sqrt((w * w).sum(1))
        sh = np.where(th > 0, np.sin(th / 2) / np.where(th > 0, th / 2, 1), LD(1))
        eq = np.concatenate([w * (sh / 2)[:, None], np.cos(th / 2)[:, None]], axis=1)
        # V(omega) upsilon with only one of omega, upsilon non-zero is upsilon itself
        return project_ld(np.einsum("nij,nj->ni", quat_rot(eq), Xc0) + v, cam, m, stereo)

    def r_lm(k, h):
        return project_ld(Xc0 + Rq[:, :, k] * h[:, None], cam, m, stereo)

    def d6(f, k, h):
        df = 45 * (f(k, h) - f(k, -h)) - 9 * (f(k, 2 * h) - f(k, -2 * h)) + (f(k, 3 * h) - f(k, -3 * h))
        return -(df / (60 * h)[:, None]).astype(np.float64)

    # steps: 1e-3 rad for the rotation, 1e-3 of the depth for translations and the point: truncation ~1e-18, rounding ~1e-16
    for k in range(6):
        JP[:, :, k] = d6(r_pose, k, np.full(n, LD(1e-3)) if k < 3 else LD(1e-3) * Z)
    for k in range(3):
        JL[:, :, k] = d6(r_lm, k, LD(1e-3) * Z)
    return JP, JL


def jacobian_magnitude(q, cam, Xc, stereo):
    """elementwise sum of |terms| of edge_jacobians' formulas (JP [n,3,6], JL [n,3,3]), the M of the bound K u M"""
    R = np.abs(quat_rot(np.asarray(q, dtype=np.float64)))
    iz = 1 / np.abs(Xc[:, 2]); xn, yn = np.abs(Xc[:, 0]) * iz, np.abs(Xc[:, 1]) * iz
    fu, fv, bf = cam[:, 0], cam[:, 1], cam[:, 4]
    fuZ, fvZ, bZZ = fu * iz, fv * iz, bf * iz * iz
    n = len(q)
    MP = np.zeros((n, 3, 6)); ML = np.zeros((n, 3, 3))
    ML[:, 0] = fuZ[:, None] * (R[:, 0] + xn[:, None] * R[:, 2])
    ML[:, 1] = fvZ[:, None] * (R[:, 1] + yn[:, None] * R[:, 2])
    MP[:, 0] = np.stack([fu * xn * yn, fu * (1 + xn * xn), fu * yn, fuZ, 0 * fu, fuZ * xn], axis=1)
    MP[:, 1] = np.stack([fv * (1 + yn * yn), fv * xn * yn, fv * xn, 0 * fv, fvZ, fvZ * yn], axis=1)
    s = np.asarray(stereo, dtype=bool)
    ML[s, 2] = ML[s, 0] + bZZ[s, None] * R[s, 2]
    P2 = MP[:, 0].copy(); P2[:, 0] += bZZ * np.abs(Xc[:, 1]); P2[:, 1] += bZZ * np.abs(Xc[:, 0]); P2[:, 4] = 0; P2[:, 5] += bZZ
    MP[s, 2] = P2[s]
    return MP, ML


def edge_records(rng, typ, n, Z, xn_max, stereo, tscale=1.0):
    q = rnd(random_quat(rng, n), typ)
    t = rnd(rng.normal(0, tscale, (n, 3)), typ)
    cam = np.tile(rnd(K00, typ), (n, 1))
    xn = rng.uniform(-xn_max, xn_max, n); yn = rng.uniform(-0.4, 0.4, n) * min(1, xn_max)
    z = Z * rng.uniform(0.9, 1.1, n)
    Xc = np.stack([xn * z, yn * z, z], axis=1)
    # Xw = R^T (Xc - t), rounded: the kernel's Xc is then close to (not exactly) the chosen point
    Xw = rnd(np.einsum("nji,nj->ni", quat_rot(q / np.linalg.norm(q, axis=1)[:, None]), Xc - t), typ)
    uu, vv = cam[:, 0] * xn + cam[:, 2], cam[:, 1] * yn + cam[:, 3]
    m = rnd(np.stack([uu, vv, uu - cam[:, 4] / z], axis=1) + rng.normal(0, 2, (n, 3)), typ)
    st = np.full((n, 1), 1.0 if stereo else 0.0)
    return np.concatenate([q, t, cam, Xw, m, st], axis=1)


@pytest.mark.parametrize("typ", TYPES)
@pytest.mark.parametrize("stereo", [False, True], ids=["mono", "stereo"])
@pytest.mark.parametrize("Z,xn_max", [(0.1, 0.5), (10.0, 0.5), (1e4, 0.5), (8.0, 1.0)], ids=["Z0.1", "Z10", "Z1e4", "xn1"])
def test_edge_residual_and_jacobians(driver, typ, stereo, Z, xn_max):
    rng = np.random.default_rng(int(Z * 10) + int(stereo) + 100 * int(xn_max))
    n = 64
    rec = edge_records(rng, typ, n, Z, xn_max, stereo, tscale=min(1.0, Z))
    q, t, cam, Xw, m = rec[:, 0:4], rec[:, 4:7], rec[:, 7:12], rec[:, 12:15], rec[:, 15:18]
    st = rec[:, 18] != 0
    out = run(driver, typ, "edge", rec)
    Xc_g, r_g = out[:, 0:3], out[:, 3:6]
    JP_g, JL_g = out[:, 6:24].reshape(n, 3, 6), out[:, 24:33].reshape(n, 3, 3)
    Xc_r, r_r = (a.astype(np.float64) for a in residual_ld(q, t, cam, Xw, m, st))
    u = U[typ]
    # the camera-frame point: rotate() and + t, magnitudes |R||Xw| + |t|
    MX = np.abs(quat_rot(q)) @ np.abs(Xw)[..., None]
    MX = MX[..., 0] + np.abs(t)
    ratio = report("Xc<%s> Z %g" % (typ, Z), np.abs(Xc_g - Xc_r), 16 * u * MX)
    assert ratio <= 1
    # its relative error carried into x/Z, y/Z: c = |MX| / |Z| (1 + |xn| + |yn|)
    c = MX.max(1) / np.abs(Xc_r[:, 2]) * (1 + np.abs(Xc_r[:, 0] / Xc_r[:, 2]) + np.abs(Xc_r[:, 1] / Xc_r[:, 2]))
    # residual: u - m cancels, so M holds |u| + |m| plus fu |x/Z| c
    Mr = np.abs(r_r) + np.abs(m) + cam[:, :3].max(1)[:, None] * (1 + c)[:, None]
    Mr[~st, 2] = 1
    ratio = report("r<%s> Z %g" % (typ, Z), np.abs(r_g - r_r), 16 * u * Mr)
    assert ratio <= 1
    if not stereo:
        assert np.all(r_g[:, 2] == 0) and np.all(JP_g[:, 2] == 0) and np.all(JL_g[:, 2] == 0)
    JP_r, JL_r = jacobians_fd(q, t, cam, Xw, m, st)
    MP, ML = jacobian_magnitude(q, cam, Xc_r, st)
    # K u (M (1 + c) + G c): M (1 + c) the formula's roundings and the relative error of 1/Z; G c the absolute error c u that x/Z and
    # y/Z carry into every entry, G bounding the entries' derivatives in x/Z, y/Z.  Plus the difference quotient's own error (below
    # 1e-13 of the largest entry).
    KJ = 32
    axn, ayn = np.abs(Xc_r[:, 0] / Xc_r[:, 2]), np.abs(Xc_r[:, 1] / Xc_r[:, 2])
    G = (cam[:, :2].max(1) * (1 + 2 * axn + 2 * ayn) + 3 * cam[:, 4] / np.abs(Xc_r[:, 2])) * c
    fd = 1e-13 * MP.max((1, 2))
    bp_ = KJ * u * (MP * (1 + c)[:, None, None] + G[:, None, None]) + fd[:, None, None]
    GL = cam[:, :2].max(1) / np.abs(Xc_r[:, 2]) * c                      # d JL / d(x/Z) = -f/Z R[2][k]
    bl_ = KJ * u * (ML * (1 + c)[:, None, None] + GL[:, None, None]) + 1e-13 * ML.max((1, 2))[:, None, None]
    rows = 3 if stereo else 2
    rp = report("JP<%s> Z %g %s" % (typ, Z, "stereo" if stereo else "mono"), np.abs(JP_g - JP_r)[:, :rows], bp_[:, :rows] + 1e-300)
    rl = report("JL<%s> Z %g" % (typ, Z), np.abs(JL_g - JL_r)[:, :rows], bl_[:, :rows] + 1e-300)
    assert rp <= 1 and rl <= 1


# ---- 3x3 and 6x6 inverses ------------------------------------------------------------------------------------------------------

def spd(rng, n, dim, kappa, profile):
    """random SPD matrices of 2-norm 1 and condition ~kappa: eigenvalues 1 .. 1/kappa spread log-uniformly ("spread"), one small
    ("one"), or all but the largest small ("many")"""
    Q, _ = np.linalg.qr(rng.normal(size=(n, dim, dim)))
    if profile == "spread":
        lam = np.logspace(0, -np.log10(kappa), dim)
    elif profile == "one":
        lam = np.ones(dim); lam[-1] = 1 / kappa
    else:
        lam = np.full(dim, 1 / kappa); lam[0] = 1
    A = np.einsum("nij,j,nkj->nik", Q, lam, Q)
    return (A + A.transpose(0, 2, 1)) / 2


def inv_ld(A):
    """batched Gauss-Jordan inverse with partial pivoting in longdouble"""
    A = np.asarray(A, dtype=LD).copy()
    n, d, _ = A.shape
    B = np.tile(np.eye(d, dtype=LD), (n, 1, 1))
    idx = np.arange(n)
    for k in range(d):
        p = k + np.argmax(np.abs(A[:, k:, k]), axis=1)
        A[idx, k], A[idx, p] = A[idx, p].copy(), A[idx, k].copy()
        B[idx, k], B[idx, p] = B[idx, p].copy(), B[idx, k].copy()
        piv = A[:, k, k].copy()
        A[:, k] /= piv[:, None]; B[:, k] /= piv[:, None]
        for i in range(d):
            if i != k:
                f = A[:, i, k].copy()
                A[:, i] -= f[:, None] * A[:, k]; B[:, i] -= f[:, None] * B[:, k]
    return B


KAPPAS = {"float": (1e1, 1e4, 1e7), "double": (1e1, 1e7, 1e14)}


@pytest.mark.parametrize("typ", TYPES)
@pytest.mark.parametrize("profile", ["spread", "one", "many"])
def test_sym3_inverse(driver, typ, profile):
    rng = np.random.default_rng(3)
    u = U[typ]
    checked = 0
    for kappa in KAPPAS[typ]:
        A = rnd(spd(rng, 64, 3, kappa, profile), typ)
        A = A[np.linalg.eigvalsh(A)[:, 0] > 0]            # at kappa 1e7 rounding to fp32 can take a matrix out of the cone
        assert len(A) >= 32
        a00, a01, a02, a11, a12, a22 = (A[:, i, j] for i, j in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)))
        out = run(driver, typ, "sym3", np.stack([a00, a01, a02, a11, a12, a22], axis=1))
        ref = inv_ld(A).astype(np.float64)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
        ev = np.linalg.eigvalsh(A)
        # the adjugate formula: cofactors C and det, each a sum of products rounded a few times, so with Cm and Dm the sums of their
        # terms' magnitudes, |B - A^-1| <= K u (Cm / det + |C| Dm / det^2).  Against K u kappa ||A^-1|| this carries an extra
        # lambda_max / lambda_mid: a 3x3 with two small eigenvalues loses accuracy in closed form (measured: 4e4 x the kappa bound in
        # double at kappa 1e7), which a Cholesky inverse would not -- the reference's formula, kept for parity.
        ab = np.abs
        Cm = np.stack([ab(a11 * a22) + a12 * a12, ab(a02 * a12) + ab(a01 * a22), ab(a01 * a12) + ab(a02 * a11),
                       ab(a00 * a22) + a02 * a02, ab(a02 * a01) + ab(a00 * a12), ab(a00 * a11) + a01 * a01], axis=1)
        Dm = ab(a00 * a11 * a22) + 2 * ab(a01 * a12 * a02) + ab(a00) * a12 * a12 + ab(a11) * a02 * a02 + ab(a22) * a01 * a01
        det = np.prod(ev, axis=1)
        # first order only while the rounded det keeps its sign (16 u Dm < det / 2); beyond that the closed form returns noise, which
        # in fp32 happens from kappa ~1e6 with spread eigenvalues -- those matrices are counted, not checked
        ok = 16 * u * Dm < det / 2
        checked += ok.sum()
        bound = 16 * u * (Cm / det[:, None] + ab(ref) * (Dm / det)[:, None])
        if ok.any():
            ratio = report("sym3<%s> %s kappa %g (%d of %d in range)" % (typ, profile, kappa, ok.sum(), len(A)), np.abs(out - ref)[ok], bound[ok])
            assert ratio <= 1
    assert checked >= 64


@pytest.mark.parametrize("typ", TYPES)
@pytest.mark.parametrize("profile", ["spread", "one", "many"])
def test_spd6_inverse(driver, typ, profile):
    rng = np.random.default_rng(6)
    u = U[typ]
    for kappa in KAPPAS[typ]:
        A = rnd(spd(rng, 64, 6, kappa, profile), typ)
        out = run(driver, typ, "spd6", A.transpose(0, 2, 1).reshape(-1, 36))
        assert np.all(out[:, 0] == 1)
        got = out[:, 1:].reshape(-1, 6, 6).transpose(0, 2, 1)
        assert np.array_equal(got, got.transpose(0, 2, 1))
        ref = inv_ld(A).astype(np.float64)
        ev = np.linalg.eigvalsh(A)
        bound = 64 * u * (ev[:, -1] / ev[:, 0]) / ev[:, 0]
        ratio = report("spd6<%s> %s kappa %g" % (typ, profile, kappa), np.abs(got - ref).max((1, 2)), bound)
        assert ratio <= 1


@pytest.mark.parametrize("typ", TYPES)
def test_spd6_inverse_rejects_indefinite_and_singular(driver, typ):
    rng = np.random.default_rng(7)
    A = spd(rng, 30, 6, 10.0, "spread")
    Q, _ = np.linalg.qr(rng.normal(size=(30, 6, 6)))
    lam = np.ones(6); lam[2] = -0.5
    B = np.einsum("nij,j,nkj->nik", Q, lam, Q)                          # indefinite
    C = A.copy(); C[:, 3, :] = 0; C[:, :, 3] = 0                          # a zero pivot
    D = A.copy(); D[:, 0, 0] = -1.0                                       # negative first pivot
    E = np.zeros((1, 6, 6))
    bad = rnd(np.concatenate([(B + B.transpose(0, 2, 1)) / 2, C, D, E]), typ)
    out = run(driver, typ, "spd6", bad.transpose(0, 2, 1).reshape(-1, 36))
    assert np.all(out[:, 0] == 0)
