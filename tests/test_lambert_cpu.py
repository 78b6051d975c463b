"""K9 Lambert solver without a GPU: the scalar C statement (tests/lambert_oracle) against textbook cases and an
independent universal-variable Kepler propagator, the edge cases of the status rules, the host build of the device core
(tests/host_emul/emul_lambert.cu) bit for bit against the statement, and the C ABI's argument checks, which run before
any device is touched.  The device runs are in tests/test_gpu_lambert.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import lambert_oracle as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "host_emul")
MU = 398600.5
OK, NO_SOLUTION, DEGENERATE, NOT_CONVERGED = 0, 1, 2, 3


@pytest.fixture(scope="module")
def emul():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = os.path.join(EMUL_DIR, "libemul_lambert.so")
    src = os.path.join(EMUL_DIR, "emul_lambert.cu")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("az_lambert.cuh", "az_math.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-I" + csrc, "-o", so, src], check=True,
                       capture_output=True)
    return C.CDLL(so)


def run_emul(lib, r1, r2, tof, mu, *, max_revs=0, normal=None):
    r1 = np.ascontiguousarray(np.asarray(r1, dtype=np.float64).reshape(-1, 3))
    n = len(r1)
    r2 = np.ascontiguousarray(np.asarray(r2, dtype=np.float64).reshape(n, 3))
    tof = np.ascontiguousarray(np.broadcast_to(np.asarray(tof, dtype=np.float64), (n,)))
    nrm = None if normal is None else np.ascontiguousarray(np.broadcast_to(np.asarray(normal, dtype=np.float64), (n, 3)))
    S = 2 * max_revs + 1
    v1, v2 = np.zeros((n, S, 3)), np.zeros((n, S, 3))
    st, it = np.zeros((n, S), dtype=np.uint8), np.zeros((n, S), dtype=np.uint8)
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    lib.emul_lambert(p(r1), p(r2), p(tof), p(nrm), C.c_uint32(n), C.c_double(mu), C.c_uint32(max_revs), p(v1), p(v2),
                     p(st), p(it))
    return v1, v2, st, it


def same_bits(a, b):
    return all(np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)) for x, y in zip(a, b))


# ---- an independent two-body propagator: universal variables, Laguerre-Conway iteration ------------------------------
def _stumpff(z):
    c, s = np.empty_like(z), np.empty_like(z)
    small, pos, neg = np.abs(z) < 1e-3, z >= 1e-3, z <= -1e-3
    zs = z[small]
    c[small] = 1 / 2 - zs / 24 + zs ** 2 / 720 - zs ** 3 / 40320
    s[small] = 1 / 6 - zs / 120 + zs ** 2 / 5040 - zs ** 3 / 362880
    q = np.sqrt(z[pos])
    c[pos], s[pos] = (1 - np.cos(q)) / z[pos], (q - np.sin(q)) / q ** 3
    q = np.sqrt(-z[neg])
    c[neg], s[neg] = (np.cosh(q) - 1) / -z[neg], (np.sinh(q) - q) / q ** 3
    return c, s


def kepler(r0, v0, dt, mu):
    """(r, v) after dt for every row of r0, v0 (n, 3); an elliptic dt is reduced modulo the period first."""
    r0n = np.linalg.norm(r0, axis=1)
    vr0 = np.einsum("ij,ij->i", r0, v0) / r0n
    alpha = 2 / r0n - np.einsum("ij,ij->i", v0, v0) / mu
    ell = alpha > 0
    dt = np.array(dt, dtype=np.float64)
    dt[ell] = np.fmod(dt[ell], 2 * np.pi / np.sqrt(mu * alpha[ell] ** 3))
    sm = np.sqrt(mu)
    chi = sm * np.abs(alpha) * dt
    chi[~ell] = np.sign(dt[~ell]) * np.sqrt(-1 / alpha[~ell]) * np.log(
        (-2 * mu * alpha[~ell] * np.abs(dt[~ell])) / (r0n[~ell] * vr0[~ell] * np.sign(dt[~ell]) +
                                                      np.sqrt(-mu / alpha[~ell]) * (1 - r0n[~ell] * alpha[~ell])) + 1e-300)
    a1, a2 = r0n * vr0 / sm, 1 - alpha * r0n
    for _ in range(200):
        z = alpha * chi ** 2
        c, s = _stumpff(z)
        F = a1 * chi ** 2 * c + a2 * chi ** 3 * s + r0n * chi - sm * dt
        dF = a1 * chi * (1 - z * s) + a2 * chi ** 2 * c + r0n
        d2F = a1 * (1 - z * c) + a2 * chi * (1 - z * s)
        step = 5 * F / (dF + np.sign(dF) * np.sqrt(np.abs(16 * dF ** 2 - 20 * F * d2F)))
        chi = chi - step
        if np.all(np.abs(step) <= 1e-15 * np.maximum(1, np.abs(chi))):
            break
    z = alpha * chi ** 2
    c, s = _stumpff(z)
    f, g = 1 - chi ** 2 / r0n * c, dt - chi ** 3 * s / sm
    r = f[:, None] * r0 + g[:, None] * v0
    rn = np.linalg.norm(r, axis=1)
    fd, gd = sm / (rn * r0n) * (alpha * chi ** 3 * s - chi), 1 - chi ** 2 / rn * c
    return r, fd[:, None] * r0 + gd[:, None] * v0


def conic(r1, v1, mu):
    """(perigee radius, eccentricity, period or inf) of the conics through (r1, v1)"""
    h = np.cross(r1, v1)
    hn2 = np.einsum("ij,ij->i", h, h)
    e = np.linalg.norm(np.cross(v1, h) / mu - r1 / np.linalg.norm(r1, axis=1)[:, None], axis=1)
    alpha = 2 / np.linalg.norm(r1, axis=1) - np.einsum("ij,ij->i", v1, v1) / mu
    period = np.where(alpha > 0, 2 * np.pi / np.sqrt(mu * np.abs(alpha) ** 3), np.inf)
    return hn2 / mu / (1 + e), e, period


def closure(r1, r2, tof, v1, v2, status, mu):
    """Check every OK slot of (n, S) outputs: closure where the perigee is >= 1000 km, finiteness elsewhere, and the
    revolution count of every elliptic slot.  Returns the number of slots checked for closure."""
    n, S = status.shape
    idx = np.argwhere(status == OK)
    assert len(idx)
    i, s = idx[:, 0], idx[:, 1]
    R1, R2, V1, V2, T = r1[i], r2[i], v1[i, s], v2[i, s], tof[i]
    assert np.all(np.isfinite(V1)) and np.all(np.isfinite(V2))
    rp, e, period = conic(R1, V1, mu)
    M = (s + 1) // 2
    ell = np.isfinite(period)
    assert np.all(M[ell] * period[ell] < T[ell]) and np.all(T[ell] < (M[ell] + 1) * period[ell])
    assert np.all(M[~ell] == 0)
    good = rp >= 1000.0
    r, v = kepler(R1[good], V1[good], T[good], mu)
    scale = np.maximum(np.linalg.norm(R1[good], axis=1), np.linalg.norm(R2[good], axis=1))
    dr = np.linalg.norm(r - R2[good], axis=1) / scale
    dv = np.linalg.norm(v - V2[good], axis=1) / np.linalg.norm(V2[good], axis=1)
    assert dr.max() < 1e-9, (dr.max(), np.argmax(dr))
    assert dv.max() < 1e-9, (dv.max(), np.argmax(dv))
    return int(good.sum())


def random_problems(rng, n, max_revs):
    """LEO to GEO and HEO radii, |sin dnu| >= 1e-3, tof from 5 min to 2 days (hyperbolic at the short end), both
    directions (a random sign of the normal)."""
    def unit(k):
        u = rng.normal(size=(k, 3))
        return u / np.linalg.norm(u, axis=1)[:, None]
    rad = lambda k: np.exp(rng.uniform(np.log(6600.0), np.log(45000.0), k))  # noqa: E731
    u1 = unit(n)
    w = unit(n)
    w -= np.einsum("ij,ij->i", w, u1)[:, None] * u1
    w /= np.linalg.norm(w, axis=1)[:, None]
    ang = rng.uniform(0, 2 * np.pi, n)
    ang = np.where(np.abs(np.sin(ang)) < 1e-3, ang + 0.01, ang)
    u2 = np.cos(ang)[:, None] * u1 + np.sin(ang)[:, None] * w
    r1, r2 = u1 * rad(n)[:, None], u2 * rad(n)[:, None]
    heo = rng.random(n) < 0.1   # a HEO apogee at one end
    r2[heo] *= (80000.0 / np.linalg.norm(r2[heo], axis=1))[:, None]
    tof = np.exp(rng.uniform(np.log(300.0), np.log(2 * 86400.0), n))
    normal = np.cross(r1, r2) * rng.choice([-1.0, 1.0], n)[:, None]
    normal /= np.linalg.norm(normal, axis=1)[:, None]
    return r1, r2, tof, normal


# ---- textbook cases -------------------------------------------------------------------------------------------------
def test_vallado_7_5_and_curtis_5_2(emul):
    # Vallado, Fundamentals of Astrodynamics, Example 7-5 (printed to 1e-6 km/s from rounded inputs)
    r1, r2 = [15945.34, 0.0, 0.0], [12214.83899, 10249.46731, 0.0]
    v1, v2, st, _ = L.solve(r1, r2, 76 * 60.0, 398600.4418)
    assert st[0, 0] == OK
    assert np.abs(v1[0, 0] - [2.058913, 2.915965, 0.0]).max() < 1e-6
    assert np.abs(v2[0, 0] - [-3.451565, 0.910315, 0.0]).max() < 1e-6
    assert same_bits((v1, v2), run_emul(emul, r1, r2, 76 * 60.0, 398600.4418)[:2])
    # Curtis, Orbital Mechanics for Engineering Students, Example 5.2 (printed to 1e-5 km/s: within half a unit of the
    # last printed digit)
    r1, r2 = [5000.0, 10000.0, 2100.0], [-14600.0, 2500.0, 7000.0]
    v1, v2, st, _ = L.solve(r1, r2, 3600.0, 398600.0)
    assert st[0, 0] == OK
    assert np.abs(v1[0, 0] - [-5.99249, 1.92536, 3.24564]).max() < 5e-6
    assert np.abs(v2[0, 0] - [-3.31246, -4.19662, -0.38529]).max() < 5e-6
    assert same_bits((v1, v2), run_emul(emul, r1, r2, 3600.0, 398600.0)[:2])


def test_random_geometries_close_under_two_body_motion(emul):
    rng = np.random.default_rng(9)
    r1, r2, tof, normal = random_problems(rng, 3000, 10)
    out = L.solve(r1, r2, tof, MU, max_revs=10, normal=normal)
    v1, v2, st, it = out
    assert np.all(np.isin(st, [OK, NO_SOLUTION]))
    assert np.all(it[st == OK] <= 10)
    # every slot zero-filled unless OK
    assert not np.any(v1[st != OK]) and not np.any(v2[st != OK])
    checked = closure(r1, r2, tof, v1, v2, st, MU)
    assert checked > 5000
    # multi-revolution slots of both branches, hyperbolic transfers and long-way transfers all occur
    assert np.any(st[:, 10 * 2 - 1] == OK) and np.any(st[:, 10 * 2] == OK)
    assert np.any(np.einsum("ij,ij->i", np.cross(r1, r2), normal) < 0)
    assert np.any(np.isinf(conic(r1[st[:, 0] == OK], v1[st[:, 0] == OK, 0], MU)[2]))
    assert same_bits(out, run_emul(emul, r1, r2, tof, MU, max_revs=10, normal=normal))


def test_default_normal_is_plus_z_and_a_negated_normal_flies_the_other_way(emul):
    r1, r2 = [7000.0, 0, 0], [0, 7100.0, 100.0]
    a = L.solve(r1, r2, 2700.0, MU)
    b = L.solve(r1, r2, 2700.0, MU, normal=[0, 0, 1.0])
    c = L.solve(r1, r2, 2700.0, MU, normal=[0, 0, -1.0])
    assert same_bits(a, b)
    assert a[2][0, 0] == OK and c[2][0, 0] == OK
    assert np.cross(r1, a[0][0, 0])[2] > 0 and np.cross(r1, c[0][0, 0])[2] < 0
    for res in (a, c):
        closure(np.array([r1]), np.array([r2]), np.array([2700.0]), *res[:3], MU)
    assert same_bits(c, run_emul(emul, r1, r2, 2700.0, MU, normal=[0, 0, -1.0]))


# ---- edge cases -----------------------------------------------------------------------------------------------------
def _tof_for(T, r1, r2, mu, normal=(0, 0, 1.0)):
    lam, T0 = L.geometry(r1, r2, 1.0, mu, normal)
    return T / T0


@pytest.mark.parametrize("M", [1, 2, 5])
def test_status_on_each_side_of_the_minimum_time_of_flight(emul, M):
    r1, r2 = np.array([7000.0, 0, 0]), np.array([-3000.0, 8000.0, 500.0])
    lam, _ = L.geometry(r1, r2, 1.0, MU)
    tmin = _tof_for(L.t_min(lam, M), r1, r2, MU)
    below = L.solve(r1, r2, tmin * (1 - 1e-9), MU, max_revs=M)
    above = L.solve(r1, r2, tmin * (1 + 1e-9), MU, max_revs=M)
    assert below[2][0, 2 * M - 1] == NO_SOLUTION and below[2][0, 2 * M] == NO_SOLUTION
    assert np.all(below[2][0, : 2 * M - 1] == OK)
    # just above T_min the two roots nearly coincide (a double root at T_min): each branch is solved or, when the
    # Householder steps do not settle within 15, NOT_CONVERGED -- never NO_SOLUTION
    assert set(above[2][0, 2 * M - 1:].tolist()) <= {OK, NOT_CONVERGED}
    clear = L.solve(r1, r2, tmin * (1 + 1e-6), MU, max_revs=M)
    assert clear[2][0, 2 * M - 1] == OK and clear[2][0, 2 * M] == OK
    # the two branches meet at T_min: just above it their velocities nearly agree
    assert np.linalg.norm(clear[0][0, 2 * M - 1] - clear[0][0, 2 * M]) < 0.05
    closure(r1[None], r2[None], np.array([tmin * (1 + 1e-6)]), *clear[:3], MU)
    for tof, res in ((tmin * (1 - 1e-9), below), (tmin * (1 + 1e-9), above), (tmin * (1 + 1e-6), clear)):
        assert same_bits(res, run_emul(emul, r1, r2, tof, MU, max_revs=M))


def test_tof_not_positive_zero_vectors_collinear_and_perpendicular_normal(emul):
    R = 7000.0
    cases = [  # (r1, r2, tof, normal, expected status of every slot or None for "not degenerate")
        ([R, 0, 0], [0, R, 0], 0.0, [0, 0, 1], NO_SOLUTION),
        ([R, 0, 0], [0, R, 0], -60.0, [0, 0, 1], NO_SOLUTION),
        ([0, 0, 0], [0, R, 0], 3000.0, [0, 0, 1], DEGENERATE),
        ([R, 0, 0], [0, 0, 0], 3000.0, [0, 0, 1], DEGENERATE),
        ([R, 0, 0], [2 * R, 0, 0], 3000.0, [0, 0, 1], DEGENERATE),
        ([R, 0, 0], [-R, 0, 0], 3000.0, [0, 0, 1], DEGENERATE),
        ([R, 0, 0], [R * math.cos(5e-13), R * math.sin(5e-13), 0], 3000.0, [0, 0, 1], DEGENERATE),
        ([R, 0, 0], [R * math.cos(2e-12), R * math.sin(2e-12), 0], 3000.0, [0, 0, 1], None),
        ([R, 0, 0], [-R * math.cos(5e-13), R * math.sin(5e-13), 0], 3000.0, [0, 0, 1], DEGENERATE),
        ([R, 0, 0], [-R * math.cos(2e-12), R * math.sin(2e-12), 0], 3000.0, [0, 0, 1], None),
        ([R, 0, 0], [0, R, 0], 3000.0, [1, 0, 0], DEGENERATE),
        ([R, 0, 0], [0, R, 0], 3000.0, [0, 0, 0], DEGENERATE),
    ]
    for r1, r2, tof, n, want in cases:
        res = L.solve(r1, r2, tof, MU, max_revs=2, normal=n)
        v1, v2, st, it = res
        if want is None:
            assert not np.any(st == DEGENERATE), (r1, r2)
        else:
            assert np.all(st == want), (r1, r2, tof, n, st)
            assert not np.any(v1) and not np.any(v2) and not np.any(it)
        assert same_bits(res, run_emul(emul, r1, r2, tof, MU, max_revs=2, normal=n))


@pytest.mark.parametrize("lam_sign", [1.0, -1.0])
def test_near_parabolic_switch_points_of_the_time_of_flight(emul, lam_sign):
    """x on each side of the Battin (|x - 1| = 0.01) and Lagrange (|x - 1| = 0.2) switch points: the solver returns a
    solution that closes, with the same bits as the statement."""
    r1, r2 = np.array([7000.0, 0, 0]), np.array([-5000.0, 9000.0, 0.0])
    normal = [0, 0, lam_sign]
    lam, _ = L.geometry(r1, r2, 1.0, MU, normal)
    xs = [1 + s * (b + d) for s in (-1, 1) for b in (0.01, 0.2) for d in (-1e-6, 1e-6)]
    tofs = np.array([_tof_for(L.tof_of_x(x, lam, 0), r1, r2, MU, normal) for x in xs])
    R1, R2 = np.tile(r1, (len(xs), 1)), np.tile(r2, (len(xs), 1))
    res = L.solve(R1, R2, tofs, MU, normal=normal)
    assert np.all(res[2] == OK)
    closure(R1, R2, tofs, *res[:3], MU)
    assert same_bits(res, run_emul(emul, R1, R2, tofs, MU, normal=normal))
    # the time-of-flight forms agree across each switch point to rounding
    for b in (0.01, 0.2):
        for s in (-1, 1):
            lo, hi = L.tof_of_x(1 + s * (b - 1e-12), lam, 0), L.tof_of_x(1 + s * (b + 1e-12), lam, 0)
            assert abs(hi - lo) < 1e-9 * abs(lo)


def test_porkchop_cell_keeps_the_cheapest_slot(emul):
    """The host build of the porkchop cell: n = rc x vc, the slot of least |dv1| + |dv2| over the statement's slots,
    slot 0's status when no slot is OK."""
    rng = np.random.default_rng(4)
    n = 300
    r1, r2, tof, _ = random_problems(rng, n, 3)
    vc = np.cross([0, 0, 1.0], r1)
    vc *= (np.sqrt(MU / np.linalg.norm(r1, axis=1)) / np.linalg.norm(vc, axis=1))[:, None]
    vt = rng.normal(size=(n, 3))
    tof[:5] = [0.0, -10.0, 0.0, 1.0, 2.0]
    dv, slot, st = np.zeros((n, 2)), np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.uint8)
    p = lambda a: C.c_void_p(np.ascontiguousarray(a).ctypes.data)  # noqa: E731
    arrs = [np.ascontiguousarray(a) for a in (r1, vc, r2, vt, tof)]
    emul.emul_porkchop(*map(p, arrs), C.c_uint32(n), C.c_double(MU), C.c_uint32(3), p(dv), p(slot), p(st))
    v1, v2, s_all, _ = L.solve(r1, r2, tof, MU, max_revs=3, normal=np.cross(r1, vc))
    for i in range(n):
        ok = np.flatnonzero(s_all[i] == OK)
        if not len(ok):
            assert st[i] == s_all[i, 0] and slot[i] == 0 and not np.any(dv[i])
            continue
        cost = np.linalg.norm(v1[i, ok] - vc[i], axis=1) + np.linalg.norm(vt[i] - v2[i, ok], axis=1)
        assert st[i] == OK and slot[i] == ok[np.argmin(cost)]
        assert abs(dv[i].sum() - cost.min()) < 1e-12 * max(1.0, cost.min())
    assert np.all(st[:2] == NO_SOLUTION)


# ---- C ABI and frontend argument checks (no device needed) ----------------------------------------------------------
def test_cabi_refuses_bad_arguments_and_writes_nothing():
    from astroz_b200._abi import DEFINES
    from astroz_b200._lib import lib

    VALUE_ERROR = DEFINES["ASTROZ_VALUE_ERROR"]
    lb = lib()
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    r1, r2, tof = np.array([[7000.0, 0, 0]]), np.array([[0, 7000.0, 0]]), np.array([3000.0])
    bad_r1 = np.array([[np.nan, 0, 0]])
    for args in [  # (r1, tof, mu, max_revs, device)
        (r1, tof, 0.0, 0, 0), (r1, tof, -1.0, 0, 0), (r1, tof, np.nan, 0, 0), (r1, tof, np.inf, 0, 0),
        (r1, tof, MU, 128, 0), (r1, tof, MU, 0, -1), (bad_r1, tof, MU, 0, 0), (r1, np.array([np.inf]), MU, 0, 0),
    ]:
        a_r1, a_tof, mu, mr, dev = args
        S = 2 * mr + 1
        v1, v2 = np.full((1, S, 3), 7.0), np.full((1, S, 3), 7.0)
        st, it = np.full((1, S), 9, dtype=np.uint8), np.full((1, S), 9, dtype=np.uint8)
        assert lb.astroz_cuda_lambert(p(a_r1), p(r2), p(a_tof), None, 1, mu, mr, dev, p(v1), p(v2), p(st),
                                      p(it)) == VALUE_ERROR, args
        assert np.all(v1 == 7.0) and np.all(v2 == 7.0) and np.all(st == 9) and np.all(it == 9)
        if a_r1 is r1 and a_tof is tof:   # the device call checks the scalars only
            assert lb.astroz_cuda_lambert_device(p(a_r1), p(r2), p(a_tof), None, 1, mu, mr, dev, p(v1), p(v2), p(st),
                                                 p(it), None) == VALUE_ERROR, args
    dv = np.full(2, 7.0)
    b = np.full(1, 9, dtype=np.uint8)
    st6 = np.zeros(6)
    t = np.zeros(1)
    for mu, mr, dev in ((0.0, 0, 0), (np.nan, 0, 0), (MU, 128, 0), (MU, 0, -1)):
        assert lb.astroz_cuda_lambert_porkchop_device(p(st6), None, p(st6), None, 1, p(t), p(t), 1, p(t), p(t), 1, mu,
                                                      mr, dev, p(dv), p(b), p(b), None) == VALUE_ERROR
    # a grid whose cell count would not fit one launch
    assert lb.astroz_cuda_lambert_porkchop_device(p(st6), None, p(st6), None, 0xFFFFFFFF, p(t), p(t), 0xFFFFFFFF,
                                                  p(t), p(t), 0xFFFFFFFF, MU, 0, 0, p(dv), p(b), p(b),
                                                  None) == VALUE_ERROR
    assert np.all(dv == 7.0) and np.all(b == 9)
    # a null handle
    assert lb.astroz_cuda_constellation_porkchop(None, None, None, 1, None, None, 1, None, None, 1, MU, 0, None, None,
                                                 None) == DEFINES["ASTROZ_NULL_POINTER"]


def test_frontend_lambert_raises_the_references_errors():
    from astroz_b200.frontend import lambert

    msg = "Lambert solver failed"
    for r1, r2, tof in (([7000, 0, 0], [0, 7000, 0], 0.0), ([7000, 0, 0], [0, 7000, 0], -5.0),
                        ([0, 0, 0], [0, 7000, 0], 100.0), ([7000, 0, 0], [0, 0, 0], 100.0),
                        ([7000, 0, 0], [8000, 0, 0], 100.0), ([7000, 0, 0], [-8000, 0, 0], 100.0)):
        with pytest.raises(ValueError, match=msg):
            lambert(MU, r1, r2, tof)
    with pytest.raises(ValueError):
        lambert(MU, [7000, 0], [0, 7000, 0], 100.0)
