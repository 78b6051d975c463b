"""Model lists for numerical propagation (astroz_b200.numerical.propagate_models_batch) on the CPU:
- the scalar restatement (tests/numerical_oracle/numerical_oracle_models.c) against the reference's own ForceModel tests and against
  an independent numpy statement of every model, at every edge;
- the K7 model-list cores (az_numerical.cuh) under host emulation, bit-identical to the restatement;
- the SPICE example's loop, scipy's DOP853, and the C ABI's argument errors.
The device run is in tests/test_gpu_numerical_models.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from astroz_b200 import numerical as P
from tests.numerical_oracle import models as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "host_emul")
MU, R_EQ, J2 = 398600.5, 6378.137, 0.00108262998905
J3, J4 = -0.00000253215306, -0.00000161098761        # ForceModel.zig:401-402
SUN_MU, MOON_MU, AU = 1.32712e11, 4902.80, 1.495978707e8
OMEGA = 7.2921150e-5


# ---- an independent numpy statement of each model (ForceModel.zig), vectorised over states s (m, 6) ----------------
def np_two_body(s, mu):
    r = np.sqrt(s[:, 0] ** 2 + s[:, 1] ** 2 + s[:, 2] ** 2)
    f = -mu / (r * r * r)
    return np.stack([f * s[:, 0], f * s[:, 1], f * s[:, 2]], axis=1)


def np_zonal(s, mu, coef, r_eq, n):
    x, y, z = s[:, 0], s[:, 1], s[:, 2]
    r2 = x * x + y * y + z * z
    r = np.sqrt(r2)
    if n == 2:
        f = -1.5 * coef * mu * r_eq * r_eq / (r2 * r2 * r)
        q = (z * z) / r2
        return np.stack([f * x * (5.0 * q - 1.0), f * y * (5.0 * q - 1.0), f * z * (5.0 * q - 3.0)], axis=1)
    if n == 3:   # the x / y coefficient has the extra 1/r (reference quirk)
        f = 2.5 * coef * mu * (r_eq * r_eq * r_eq) / (r2 * r2 * r2 * r)
        q = (z * z) / r2
        xy = 3.0 * z / r - 7.0 * z * q / r
        zc = 6.0 * z * z - 7.0 * z * z * q - 0.6 * r2
        return np.stack([f * x * xy, f * y * xy, f * zc], axis=1)
    r4 = r2 * r2     # J4 over r^9 (reference quirk)
    z2 = z * z
    q2, q4 = z2 / r2, (z2 * z2) / r4
    f = 1.875 * coef * mu * (r_eq * r_eq * r_eq * r_eq) / (r4 * r4 * r)
    xy = 3.0 - 42.0 * q2 + 63.0 * q4
    zt = 15.0 - 70.0 * q2 + 63.0 * q4
    return np.stack([f * x * xy, f * y * xy, f * z * zt], axis=1)


def np_drag(s, r_eq, rho0, H, cd, area, mass, max_alt):
    v = np.sqrt(s[:, 3] ** 2 + s[:, 4] ** 2 + s[:, 5] ** 2)
    alt = np.sqrt(s[:, 0] ** 2 + s[:, 1] ** 2 + s[:, 2] ** 2) - r_eq
    on = ~(alt > max_alt) & ~(v < 1e-10)
    rho = rho0 * np.array([math.exp(-a / H) for a in alt])
    f = -0.5 * cd * area * rho * v * 1e3 / mass
    with np.errstate(all="ignore"):
        a = np.stack([f * s[:, 3] / v, f * s[:, 4] / v, f * s[:, 5] / v], axis=1)
    return np.where(on[:, None], a, 0.0)


LAYERS = [(100.0, 5.297e-7, 5.877), (200.0, 2.789e-10, 37.105), (400.0, 3.725e-12, 62.822), (600.0, 2.418e-13, 79.864),
          (1000.0, 3.561e-15, 200.0)]


def np_improved_drag(s, r_eq, cd, area, mass, max_alt, f107):
    x, y = s[:, 0], s[:, 1]
    alt = np.sqrt(x * x + y * y + s[:, 2] ** 2) - r_eq
    vr = np.stack([s[:, 3] + OMEGA * y, s[:, 4] - OMEGA * x, s[:, 5]], axis=1)
    v = np.sqrt(vr[:, 0] ** 2 + vr[:, 1] ** 2 + vr[:, 2] ** 2)
    on = ~(alt > max_alt) & ~(alt < 100.0) & ~(v < 1e-10)
    rho = np.zeros(len(s))
    for j, h in enumerate(alt):
        base, r0, H = LAYERS[max([i for i, L in enumerate(LAYERS) if h >= L[0]], default=0)]
        rho[j] = r0 * math.exp(-(h - base) / H) * (f107 / 150.0)
    f = -0.5 * cd * area * rho * v * 1e3 / mass
    with np.errstate(all="ignore"):
        a = f[:, None] * vr / v[:, None]
    return np.where(on[:, None], a, 0.0)


def np_srp(s, cr, area, mass, r_eq, sun):
    sun = np.asarray(sun, dtype=np.float64)
    d = sun[None, :] - s[:, :3]
    dist = np.sqrt(d[:, 0] ** 2 + d[:, 1] ** 2 + d[:, 2] ** 2)
    sd = math.sqrt(sun[0] ** 2 + sun[1] ** 2 + sun[2] ** 2)
    if sd < 1e-10:
        return np.zeros((len(s), 3))
    hat = sun / sd
    proj = s[:, 0] * hat[0] + s[:, 1] * hat[1] + s[:, 2] * hat[2]
    perp = s[:, :3] - proj[:, None] * hat[None, :]
    rho = np.sqrt(perp[:, 0] ** 2 + perp[:, 1] ** 2 + perp[:, 2] ** 2)
    on = ~(dist < 1e-10) & ~((proj < 0) & (rho < r_eq))
    with np.errstate(all="ignore"):
        f = -cr * 4.56e-6 * ((AU / dist) * (AU / dist)) * area / mass * 1e-3
        a = f[:, None] * (d / dist[:, None])
    return np.where(on[:, None], a, 0.0)


def np_third_body(s, mu, q):
    q = np.asarray(q, dtype=np.float64)
    qm = math.sqrt(q[0] ** 2 + q[1] ** 2 + q[2] ** 2)
    if qm < 1e-10:
        return np.zeros((len(s), 3))
    d = q[None, :] - s[:, :3]
    dm = np.sqrt(d[:, 0] ** 2 + d[:, 1] ** 2 + d[:, 2] ** 2)
    with np.errstate(all="ignore"):
        a = mu * (d / (dm * dm * dm)[:, None] - q[None, :] / (qm * qm * qm))
    return np.where((dm < 1e-10)[:, None], 0.0, a)


def random_states(rng, m):
    r = rng.uniform(R_EQ + 50, 50000, m)
    u = rng.standard_normal((m, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    v = rng.standard_normal((m, 3)) * np.sqrt(MU / r)[:, None] / np.sqrt(3)
    return np.concatenate([u * r[:, None], v], axis=1)


def same(a, b):
    return np.array_equal(a.view(np.uint64) if a.dtype == np.float64 else a, b.view(np.uint64))


def test_numpy_statement_of_each_model_at_random_states():
    """No exp: bit-identical (the same IEEE operations in the same order).  Drag kinds: math.exp is the C library's,
    as in the restatement, so these are bit-identical too."""
    rng = np.random.default_rng(7)
    s = random_states(rng, 400)
    sun, moon = (AU * 0.3, -AU * 0.9, AU * 0.2), (384400.0 * 0.5, 384400.0 * 0.8, -1000.0)
    cases = [
        ([P.TwoBody(MU)], np_two_body(s, MU)),
        ([P.J2(MU, J2, R_EQ)], np_zonal(s, MU, J2, R_EQ, 2)),
        ([P.J3(MU, J3, R_EQ)], np_zonal(s, MU, J3, R_EQ, 3)),
        ([P.J4(MU, J4, R_EQ)], np_zonal(s, MU, J4, R_EQ, 4)),
        ([P.Drag(R_EQ, 1.225, 7.249, 2.2, 4.0, 300.0, 1500.0)], np_drag(s, R_EQ, 1.225, 7.249, 2.2, 4.0, 300.0, 1500.0)),
        ([P.ImprovedDrag(R_EQ, 2.2, 4.0, 300.0, 1500.0, 180.0)], np_improved_drag(s, R_EQ, 2.2, 4.0, 300.0, 1500.0, 180)),
        ([P.SolarRadiationPressure(1.5, 20.0, 1000.0, R_EQ, sun)], np_srp(s, 1.5, 20.0, 1000.0, R_EQ, sun)),
        ([P.SolarRadiationPressure(1.5, 20.0, 1000.0, R_EQ)], np_srp(s, 1.5, 20.0, 1000.0, R_EQ, (AU, 0, 0))),
        ([P.ThirdBody(SUN_MU, sun)], np_third_body(s, SUN_MU, sun)),
        ([P.ThirdBody(MOON_MU, moon)], np_third_body(s, MOON_MU, moon)),
    ]
    for models, ref in cases:
        assert same(M.accel(models, s), ref), models
    # Composite: a total from zero, in list order
    models = [c[0][0] for c in cases]
    total = np.zeros((len(s), 3))
    for _, ref in cases:
        total = total + ref
    assert same(M.accel(models, s), total)


def test_numpy_statement_at_every_edge():
    """The shadow cylinder's boundary, each ImprovedDrag layer boundary and 100 km, max_altitude, and each zero guard."""
    e = lambda x: [x, np.nextafter(x, -np.inf), np.nextafter(x, np.inf)]  # noqa: E731
    # shadow cylinder, Sun on +X: behind the Earth at a perpendicular distance of r_eq and one ulp either side
    rows = [[-7000.0, y, 0.0, 0.0, 7.5, 0.0] for y in e(R_EQ)] + [[-7000.0, 0, z, 0.0, 7.5, 0.0] for z in e(R_EQ)]
    rows += [[0.0, R_EQ * 0.5, 0, 0, 7.5, 0], [1e-300, 7000.0, 0, 0, 7.5, 0], [-1e-300, 7000.0, 0, 0, 7.5, 0]]
    s = np.array(rows)
    srp = [P.SolarRadiationPressure(1.5, 20.0, 1000.0, R_EQ)]
    a = M.accel(srp, s)
    assert same(a, np_srp(s, 1.5, 20.0, 1000.0, R_EQ, (AU, 0, 0)))
    assert (a[[1, 4]] == 0).all() and (a[[0, 2, 3, 5], 0] != 0).all() and (a[6:, 0] != 0).all()
    # altitude edges: each layer base, 100 km, max_altitude (both drag kinds)
    alts = [b for L in LAYERS for b in e(L[0])] + e(1500.0) + e(1200.0) + [50.0, 99.0, 2000.0]
    s = np.array([[R_EQ + h, 0.0, 0.0, 0.0, 7.6, 0.1] for h in alts] +
                 [[0.0, 0.0, R_EQ + h, 7.6, 0.0, 0.0] for h in alts])
    for models, ref in (([P.ImprovedDrag(R_EQ, 2.2, 4.0, 300.0, 1200.0, 150.0)],
                         np_improved_drag(s, R_EQ, 2.2, 4.0, 300.0, 1200.0, 150.0)),
                        ([P.Drag(R_EQ, 1.225, 7.249, 2.2, 4.0, 300.0, 1500.0)],
                         np_drag(s, R_EQ, 1.225, 7.249, 2.2, 4.0, 300.0, 1500.0))):
        assert same(M.accel(models, s), ref)
    # zero guards: v < 1e-10, vrel < 1e-10 (co-rotating), dist < 1e-10, sunDist < 1e-10, qMag < 1e-10, dMag < 1e-10
    x, y = 6778.0, 100.0
    still = np.array([[x, y, 0, 0, 0, 0], [x, y, 0, -OMEGA * y, OMEGA * x, 0.0], [x, y, 0, 0, 0, 5e-11]])
    assert (M.accel([P.Drag(R_EQ, 1.225, 7.249, 2.2, 4, 300, 1500)], still[[0, 2]]) == 0).all()
    assert (M.accel([P.ImprovedDrag(R_EQ, 2.2, 4, 300, 1500, 150)], still[[1]]) == 0).all()
    at = np.array([[AU, 0, 0, 0, 0, 0], [AU, 1e-11, 0, 0, 0, 0]])
    assert (M.accel(srp, at) == 0).all()
    assert (M.accel([P.SolarRadiationPressure(1.5, 20, 1000, R_EQ, (0, 0, 0))], still) == 0).all()
    assert (M.accel([P.ThirdBody(SUN_MU, (0, 0, 5e-11))], still) == 0).all()
    assert (M.accel([P.ThirdBody(SUN_MU, (AU, 0, 0))], at) == 0).all()
    for models, ref in (([P.ThirdBody(SUN_MU, (AU, 0, 0))], np_third_body(at, SUN_MU, (AU, 0, 0))),
                        (srp, np_srp(at, 1.5, 20, 1000, R_EQ, (AU, 0, 0)))):
        assert same(M.accel(models, at), ref)


def test_reference_force_model_tests():
    """ForceModel.zig:377-504, restated on the restatement."""
    s = np.array([7000.0, 0, 0, 0, 7.5, 0])
    assert M.accel([P.TwoBody(398600.4418)], s)[0, 0] < 0
    assert M.accel([P.TwoBody(398600.4418), P.J2(398600.4418, 0.00108263, 6378.137)], s)[0, 0] < 0
    s3 = np.array([6000.0, 1000, 2000, 0, 7.5, 0])
    mags = [np.linalg.norm(M.accel([m], s3)) for m in (P.J2(398600.5, 0.00108262998905, R_EQ), P.J3(398600.5, J3, R_EQ),
                                                      P.J4(398600.5, J4, R_EQ))]
    assert 0 < mags[1] < mags[0] and 0 < mags[2] < mags[0]
    srp = lambda sun=None: [P.SolarRadiationPressure(1.5, 10.0, 500.0, 6378.137, sun)]  # noqa: E731
    assert M.accel(srp(), s)[0, 0] < 0 and M.accel(srp(), [-7000.0, 0, 0, 0, 7.5, 0])[0, 0] == 0
    a = M.accel(srp((0, AU, 0)), s)[0]
    assert abs(a[1] / -1.368e-10 - 1) < 1e-3 and abs(a[0]) < abs(a[1])
    assert M.accel(srp((0, AU, 0)), [0, -7000.0, 0, 0, 7.5, 0])[0, 1] == 0
    a1, a2 = M.accel(srp((AU, 0, 0)), s)[0, 0], M.accel(srp((AU / 2, 0, 0)), s)[0, 0]
    d1, d2 = AU - 7000.0, AU / 2 - 7000.0
    assert abs((d1 / d2) ** 2 / (abs(a2) / abs(a1)) - 1) < 1e-10
    tb = [P.ThirdBody(SUN_MU, (AU, 0, 0))]
    assert M.accel(tb, [0, 0, 0, 0, 7.5, 0])[0, 0] == 0
    assert abs(np.linalg.norm(M.accel(tb, [0, 7000.0, 0, 0, 0, 7.5])) / 2.775e-10 - 1) < 1e-2
    assert np.linalg.norm(M.accel([P.ThirdBody(SUN_MU, (1e12, 0, 0))], s)) < 1e-10
    a = M.accel([P.ImprovedDrag(6378.137, 2.2, 10.0, 500.0, 1500.0, 150.0)], [6778.137, 0, 0, 0, 7.67, 0])[0]
    assert a[1] < 0 and np.linalg.norm(a) > 0
    low = [P.ImprovedDrag(6378.137, 2.2, 10.0, 500.0, 1000.0, 150.0)]
    assert (M.accel(low, [8378.137, 0, 0, 0, 6.9, 0]) == 0).all() and (M.accel(low, [6428.137, 0, 0, 0, 7.8, 0]) == 0).all()


# ---- host emulation of the K7 model-list cores --------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = os.path.join(EMUL_DIR, "libemul_numerical_models.so")
    src = os.path.join(EMUL_DIR, "emul_numerical_models.cu")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("az_numerical.cuh", "az_math.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-I" + csrc, "-o", so, src], check=True,
                       capture_output=True)
    return C.CDLL(so)


def _steps(t0, duration, dt):
    t, out = t0, []
    while t < t0 + duration:
        out.append(min(dt, t0 + duration - t))
        t += out[-1]
    return np.array(out)


def run_emul(L, states, t0, duration, dt, models, integrator="dp87", rtol=1e-9, atol=1e-12):
    states = np.ascontiguousarray(np.atleast_2d(states), dtype=np.float64)
    n = len(states)
    steps = _steps(t0, duration, dt)
    K = len(steps)
    descs, keep = M.descriptors(models, n, K)
    out = np.zeros((n, K + 1, 6))
    st = np.zeros(n, dtype=np.uint8)
    cnt = np.zeros((n, 2), dtype=np.uint64)
    p = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    assert L.emul_numerical_models(p(states), n, p(steps), K, C.c_double(dt), C.cast(descs, C.c_void_p), len(descs),
                                   C.c_double(rtol), C.c_double(atol), 0 if integrator == "rk4" else 1, p(out), p(st),
                                   p(cnt)) == 0
    del keep
    return out, st, cnt


def fixtures():
    """LEO, SSO, an eccentric 250 km perigee, GEO, Molniya, and a circular orbit at 180 km (ImprovedDrag's steep
    bottom layer)."""
    def kep(a, e, inc, M_):
        E = M_
        for _ in range(60):
            E -= (E - e * math.sin(E) - M_) / (1 - e * math.cos(E))
        p = a * (1 - e * e)
        c, s = (math.cos(E) - e) / (1 - e * math.cos(E)), math.sqrt(1 - e * e) * math.sin(E) / (1 - e * math.cos(E))
        r, h = p / (1 + e * c), math.sqrt(MU * p)
        x, y, vx, vy = r * c, r * s, -MU / h * s, MU / h * (e + c)
        return [x, y * math.cos(inc), y * math.sin(inc), vx, vy * math.cos(inc), vy * math.sin(inc)]
    return np.array([kep(6778, 0.001, 0.9, 0.1), kep(7078, 0.0012, 1.71, 2.0),
                     kep(R_EQ + 900, 1 - (R_EQ + 250) / (R_EQ + 900), 0.6, -0.4), kep(42164, 0.0002, 0.001, 1.0),
                     kep(26600, 0.72, 1.1, 0.2), kep(R_EQ + 180, 0.0, 0.5, 0.0)])


def sun_moon_tables(K, every, t0=0.0, dt=60.0):
    """Seeded circular test orbits for the Sun and the Moon (test data, not an ephemeris), one row per interval,
    changing every `every` intervals"""
    k = (np.arange(K) // every) * every
    t = t0 + k * dt
    w_s, w_m = 2 * math.pi / (365.25 * 86400), 2 * math.pi / (27.32 * 86400)
    sun = AU * np.stack([np.cos(w_s * t + 0.3), 0.917 * np.sin(w_s * t + 0.3), 0.398 * np.sin(w_s * t + 0.3)], axis=1)
    moon = 384400.0 * np.stack([np.cos(w_m * t + 1.1), 0.9 * np.sin(w_m * t + 1.1), 0.45 * np.sin(w_m * t + 1.1)], axis=1)
    return np.ascontiguousarray(sun), np.ascontiguousarray(moon)


def spice_list(sun, moon, order=(0, 1, 2, 3, 4), cr=1.5, area=20.0, mass=1000.0):
    """spice_propagation.zig:35-47: TwoBody + J2 + SRP + Sun + Moon"""
    ms = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.SolarRadiationPressure(cr, area, mass, R_EQ, sun),
          P.ThirdBody(SUN_MU, sun), P.ThirdBody(MOON_MU, moon)]
    return [ms[i] for i in order]


def single_lists(n, K):
    rng = np.random.default_rng(3)
    sun, moon = sun_moon_tables(K, 7)
    return {
        "two_body": [P.TwoBody(MU)], "j2": [P.J2(MU, J2, R_EQ)], "j3": [P.TwoBody(MU), P.J3(MU, J3, R_EQ)],
        "j4": [P.TwoBody(MU), P.J4(MU, J4, R_EQ)],
        "drag": [P.TwoBody(MU), P.Drag(R_EQ, 1.225, 7.249, rng.uniform(1.8, 2.6, n), rng.uniform(1, 30, n), 300.0,
                                       1500.0)],
        "improved_drag": [P.TwoBody(MU), P.ImprovedDrag(R_EQ, 2.2, rng.uniform(1, 30, n), rng.uniform(100, 900, n),
                                                        1500.0, 170.0)],
        "srp": [P.TwoBody(MU), P.SolarRadiationPressure(rng.uniform(1, 2, n), 20.0, rng.uniform(100, 2000, n), R_EQ)],
        "srp_table": [P.TwoBody(MU), P.SolarRadiationPressure(1.3, 20.0, 500.0, R_EQ, sun)],
        "third_body": [P.TwoBody(MU), P.ThirdBody(MOON_MU, (384400.0, 1000.0, -3000.0))],
        "third_body_table": [P.TwoBody(MU), P.ThirdBody(MOON_MU, moon), P.ThirdBody(SUN_MU, sun)],
        "spice": spice_list(sun, moon),
        "spice_reordered": spice_list(sun, moon, (4, 2, 0, 3, 1)),
    }


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_cores_equal_the_restatement(emul, integrator):
    """With K7's step factor the host build of the model-list cores is bit-identical to the restatement: states, steps
    and status, for each model, per-state arrays, tables and the SPICE list in two orders (which differ)."""
    y = fixtures()
    K = len(_steps(0.0, 10800.0, 60.0))
    outs = {}
    for name, models in single_lists(len(y), K).items():
        out, st, cnt = run_emul(emul, y, 0.0, 10800.0, 60.0, models, integrator)
        _, ref, rst, rcnt = M.propagate(y, 0.0, 10800.0, 60.0, models, integrator=integrator, k7_step_factor=True)
        assert same(out, ref) and np.array_equal(st, rst) and np.array_equal(cnt, rcnt), name
        outs[name] = out
    assert not np.array_equal(outs["spice"], outs["spice_reordered"])      # the order is part of the result
    assert not np.array_equal(outs["srp_table"], outs["two_body"])


def test_equal_rows_give_the_fixed_vector_bits(emul):
    y = fixtures()
    K = len(_steps(0.0, 7200.0, 60.0))
    sun, moon = (AU * 0.4, AU * 0.8, AU * 0.3), (300000.0, -200000.0, 40000.0)
    fixed = spice_list(sun, moon)
    tab = spice_list(np.tile(sun, (K, 1)), np.tile(moon, (K, 1)))
    for integ in ("rk4", "dp87"):
        a = run_emul(emul, y, 0.0, 7200.0, 60.0, fixed, integ)
        b = run_emul(emul, y, 0.0, 7200.0, 60.0, tab, integ)
        assert all(same(u, v) if u.dtype == np.float64 else np.array_equal(u, v) for u, v in zip(a, b))


def test_list_with_k7_forces_equals_the_fixed_path(emul):
    """[TwoBody, J2, Drag(1.225, 7.249, 1500)] through the list cores is the fixed kForceJ2 | kForceDrag path, bit for
    bit, both integrators (host emulation of both cores)."""
    from tests.test_numerical_host_emulation import run_emul as run_fixed

    y = fixtures()
    area = np.linspace(1, 20, len(y))
    models = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.Drag(R_EQ, 1.225, 7.249, 2.2, area, 300.0, 1500.0)]
    for integ in ("rk4", "dp87"):
        a = run_emul(emul, y, 0.0, 21600.0, 60.0, models, integ)
        b = run_fixed(emul_fixed(), y, 0.0, 21600.0, 60.0, j2=J2, r_eq=R_EQ, drag=(2.2, area, 300.0), integrator=integ)
        assert same(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def emul_fixed():
    so = os.path.join(EMUL_DIR, "libemul_numerical.so")
    src = os.path.join(EMUL_DIR, "emul_numerical.cu")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    deps = [src] + [os.path.join(csrc, f) for f in ("az_numerical.cuh", "az_math.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-I" + csrc, "-o", so, src], check=True,
                       capture_output=True)
    return C.CDLL(so)


def test_spice_example_loop():
    """spice_propagation.zig:61-86 restated in Python floats: RK4 at dt 10 s, the Sun (for SRP and the Sun's third body)
    and the Moon moved between steps every 600 s (60 intervals), over 3 hours.  The batch call with per-interval tables
    reproduces it bit for bit."""
    r0 = R_EQ + 420.0
    v0 = math.sqrt(MU / r0)
    inc = 51.6 * math.pi / 180.0
    initial = [r0, 0.0, 0.0, 0.0, v0 * math.cos(inc), v0 * math.sin(inc)]
    duration, dt = 10800.0, 10.0
    K = len(_steps(0.0, duration, dt))
    sun, moon = sun_moon_tables(K, 60, dt=dt)

    def acc(s, sp, mp):
        x, y, z = s[0], s[1], s[2]
        out = [0.0, 0.0, 0.0]
        terms = [np_two_body(np.array([s]), MU)[0], np_zonal(np.array([s]), MU, J2, R_EQ, 2)[0],
                 np_srp(np.array([s]), 1.5, 20.0, 1000.0, R_EQ, sp)[0], np_third_body(np.array([s]), SUN_MU, sp)[0],
                 np_third_body(np.array([s]), MOON_MU, mp)[0]]
        del x, y, z
        for a in terms:
            out = [out[0] + float(a[0]), out[1] + float(a[1]), out[2] + float(a[2])]
        return out

    def deriv(s, sp, mp):
        a = acc(s, sp, mp)
        return [s[3], s[4], s[5], a[0], a[1], a[2]]

    state, t, k = list(initial), 0.0, 0
    traj = [list(state)]
    sp, mp = sun[0], moon[0]
    while t < duration:
        if k % 60 == 0:   # updateSunPos / updatePos every 600 s
            sp, mp = sun[k], moon[k]
        h = min(dt, duration - t)
        k1 = deriv(state, sp, mp)
        k2 = deriv([state[c] + k1[c] * (0.5 * h) for c in range(6)], sp, mp)
        k3 = deriv([state[c] + k2[c] * (0.5 * h) for c in range(6)], sp, mp)
        k4 = deriv([state[c] + k3[c] * h for c in range(6)], sp, mp)
        f = h / 6.0
        state = [state[c] + f * (k1[c] + 2.0 * k2[c] + 2.0 * k3[c] + k4[c]) for c in range(6)]
        t += h
        k += 1
        traj.append(list(state))
    ref = np.array(traj)
    _, out, st, _ = M.propagate([initial], 0.0, duration, dt, spice_list(sun, moon), integrator="rk4")
    assert st[0] == 0 and same(out[0], ref)


def test_dp87_agrees_with_scipy_dop853():
    """TwoBody + SRP + Sun + Moon at GEO over two days, fixed Sun and Moon: the restatement's DP87 against scipy's
    DOP853 on the numpy right-hand side, both at tight tolerances."""
    from scipy.integrate import solve_ivp

    sun, moon = (AU * 0.6, AU * 0.75, AU * 0.3), (300000.0, 240000.0, 80000.0)
    models = [P.TwoBody(MU), P.SolarRadiationPressure(1.5, 20.0, 1000.0, R_EQ, sun), P.ThirdBody(SUN_MU, sun),
              P.ThirdBody(MOON_MU, moon)]
    y0 = fixtures()[3]

    def rhs(_, s):
        a = sum(f for f in (np_two_body(s[None], MU), np_srp(s[None], 1.5, 20.0, 1000.0, R_EQ, sun),
                            np_third_body(s[None], SUN_MU, sun), np_third_body(s[None], MOON_MU, moon)))[0]
        return np.concatenate([s[3:], a])

    t, out, st, _ = M.propagate(y0, 0.0, 172800.0, 3600.0, models, rtol=1e-12, atol=1e-12)
    sol = solve_ivp(rhs, (0.0, 172800.0), y0, method="DOP853", t_eval=t, rtol=1e-13, atol=1e-13)
    assert st[0] == 0 and sol.success
    assert np.max(np.abs(out[0][:, :3] - sol.y.T[:, :3])) < 1e-5
    assert np.max(np.abs(out[0][:, 3:] - sol.y.T[:, 3:])) < 1e-9
    # the perturbations are really there: two-body alone drifts far from it
    _, kep, _, _ = M.propagate(y0, 0.0, 172800.0, 3600.0, models[:1], rtol=1e-12, atol=1e-12)
    assert np.max(np.abs(kep[0][:, :3] - out[0][:, :3])) > 1.0


# ---- C ABI argument errors ---------------------------------------------------------------------------------------
def test_cabi_refuses_bad_model_lists_and_writes_nothing():
    from astroz_b200._lib import lib

    L = lib()
    y = np.zeros((1, 6))
    y[0, 0] = 7000.0
    out = np.full((1, 11, 6), 7.0)
    st = np.full(1, 9, dtype=np.uint8)
    p = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731

    def desc(kind, flags=0, **kw):
        d = P._ForceModelC()
        d.kind, d.flags = kind, flags
        for f in ("mu", "coef", "r_eq", "rho0", "scale_height", "max_altitude", "f107", "c", "area", "mass"):
            setattr(d, f, 1.0)
        d.pos[:] = [AU, 0.0, 0.0]
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    ok = desc(0, mu=MU)
    bad_lists = [
        [],                                                   # empty
        [ok] * 17,                                            # more than 16
        [desc(8)], [desc(-1)],                                # unknown kinds
        [desc(0, mu=math.nan)], [desc(1, coef=math.inf)], [desc(2, r_eq=math.nan)],
        [desc(4, rho0=math.nan)], [desc(4, scale_height=math.inf)], [desc(4, c=math.nan)], [desc(5, f107=math.nan)],
        [desc(5, max_altitude=math.nan)], [desc(6, mass=math.inf)], [desc(6, pos=(C.c_double * 3)(math.nan, 0, 0))],
        [desc(7, mu=math.nan)],
        [desc(4, 1)], [desc(5, 2)], [desc(6, 4)], [desc(6, 8)], [desc(7, 8)],   # flag set, pointer NULL
        [desc(0, 1)], [desc(7, 1)], [desc(1, 8)], [desc(6, 16)],                 # flags the kind does not take
    ]
    cases = [(lst, 0.0, 100.0, 10.0, 1, 1e-9, 1e-12, 0) for lst in bad_lists]
    cases += [([ok], 0.0, 100.0, 0.0, 1, 1e-9, 1e-12, 0), ([ok], 0.0, math.inf, 10.0, 1, 1e-9, 1e-12, 0),
              ([ok], 0.0, 100.0, 10.0, 2, 1e-9, 1e-12, 0), ([ok], 0.0, 100.0, 10.0, 1, math.nan, 1e-12, 0),
              ([ok], 1e17, 1000.0, 1.0, 1, 1e-9, 1e-12, 0), ([ok], 0.0, 100.0, 10.0, 1, 1e-9, 1e-12, -1)]
    for lst, t0, dur, dt, integ, rtol, atol, dev in cases:
        arr = (P._ForceModelC * max(1, len(lst)))(*lst)
        for fn in (L.astroz_cuda_propagate_numerical_models, L.astroz_cuda_propagate_numerical_models_device):
            extra = [None] if fn is L.astroz_cuda_propagate_numerical_models_device else []
            rc = fn(p(y), 1, t0, dur, dt, C.cast(arr, C.c_void_p), len(lst), integ, rtol, atol, dev, p(out), p(st),
                    None, *extra)
            assert rc == -20, (lst[:1] and (lst[0].kind, lst[0].flags), t0, dur, dt, integ, dev)
    assert (out == 7.0).all() and st[0] == 9
    # n = 0 on device -1 is still refused; a NULL list pointer too
    arr = (P._ForceModelC * 1)(ok)
    assert L.astroz_cuda_propagate_numerical_models(p(y), 0, 0.0, 100.0, 10.0, C.cast(arr, C.c_void_p), 1, 1, 1e-9,
                                                    1e-12, -1, p(out), p(st), None) == -20
    assert L.astroz_cuda_propagate_numerical_models(p(y), 1, 0.0, 100.0, 10.0, None, 1, 1, 1e-9, 1e-12, 0, p(out),
                                                    p(st), None) == -20
    assert (out == 7.0).all() and st[0] == 9


def test_python_wrapper_validates_shapes():
    y = np.zeros((2, 6))
    with pytest.raises(ValueError, match="non-empty"):
        P.propagate_models_batch(y, 0.0, 100.0, 10.0, [])
    with pytest.raises(ValueError, match="at most 16"):
        P.propagate_models_batch(y, 0.0, 100.0, 10.0, [P.TwoBody(MU)] * 17)
    with pytest.raises(ValueError, match="shape"):
        P.propagate_models_batch(y, 0.0, 100.0, 10.0, [P.Drag(R_EQ, 1.225, 7.249, [2.2] * 3, 1.0, 1.0, 1500.0)])
    with pytest.raises(ValueError, match="shape"):
        P.propagate_models_batch(y, 0.0, 100.0, 10.0, [P.ThirdBody(MOON_MU, np.zeros((11, 3)))])   # K is 10
    with pytest.raises(ValueError, match="3-vector"):
        P.propagate_models_batch(y, 0.0, 100.0, 10.0, [P.ThirdBody(MOON_MU, (1.0, 2.0))])


def test_frontend_exports_sun_and_moon_mu():
    from astroz_b200 import frontend

    assert frontend.SUN_MU == 1.32712e11 and frontend.MOON_MU == 4902.80
    assert {"SUN_MU", "MOON_MU"} <= set(frontend.__all__)
