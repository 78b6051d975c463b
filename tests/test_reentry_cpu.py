"""K19 reentry prediction (az_reentry.cuh, az_reentry.cu) on the CPU.

The host build of the device source (tests/host_emul/emul_reentry.cu) against the independent numpy / scipy statement
(tests/fit_oracle/reentry.py): the atmosphere table and its continuity, the force and the sign of its J2 term, the
analytic decay of a circular orbit, crossings against scipy's DOP853 with a height event, the Hermite locator against
exact two-body motion, the draws against K14's host build, the split / order / batch invariants, the rules, every
refusal of the C ABI and the wrapper's window().  The device runs are in tests/test_gpu_reentry.py."""
import ctypes as C

import numpy as np
import pytest

from tests.fit_oracle import conjunction_mc as mc
from tests.fit_oracle import reentry as ro

G = ro.WGS72
EPOCH = 2460400.5


@pytest.fixture(scope="module")
def L():
    lib = ro.emul_library()
    if lib is None:
        pytest.skip("nvcc unavailable")
    return lib


def leo(hp, ha, incl=51.6, node=30.0, argp=40.0, ma=0.0, bstar=2e-4, epoch=EPOCH):
    """element columns (8,) of an orbit with perigee / apogee heights hp, ha [km] above the WGS-72 radius"""
    a = G["req"] + 0.5 * (hp + ha)
    e = (ha - hp) / (2 * G["req"] + hp + ha)
    n = np.sqrt(G["mu"] / a ** 3) * 86400.0 / (2 * np.pi)
    return np.array([epoch, n, e, incl, node, argp, ma, bstar])


def kepler_state(a, e, M, mu=G["mu"], incl=0.3):
    """TEME-like state of a two-body orbit at mean anomaly M (periapsis on +x, then inclined about x)"""
    E = M
    for _ in range(50):
        E = E - (E - e * np.sin(E) - M) / (1 - e * np.cos(E))
    r = a * (1 - e * np.cos(E))
    x, y = a * (np.cos(E) - e), a * np.sqrt(1 - e * e) * np.sin(E)
    n = np.sqrt(mu / a ** 3)
    vx, vy = -a * n * np.sin(E) / (1 - e * np.cos(E)), a * n * np.sqrt(1 - e * e) * np.cos(E) / (1 - e * np.cos(E))
    ci, si = np.cos(incl), np.sin(incl)
    assert abs(np.hypot(x, y) - r) < 1e-6
    return np.array([x, y * ci, y * si, vx, vy * ci, vy * si])


# ---- 1. density -----------------------------------------------------------------------------------------------------
def test_density_table(L):
    edges = ro.H0
    mids = 0.5 * (ro.H0[:-1] + ro.H0[1:])
    h = np.r_[edges, mids, 1500.0, 3000.0, -1.0]
    got, ref = ro.emul_density(L, h), ro.density(h)
    assert np.allclose(got, ref, rtol=1e-15, atol=0)
    assert ro.emul_density(L, 0.0)[0] == 1.225
    # the last band holds above 1000 km
    assert ro.emul_density(L, 2000.0)[0] == pytest.approx(3.019e-15 * np.exp(-1000.0 / 268.0), rel=1e-15)
    # each band, extended to the next band's base, meets the next rho0 within 0.2 %: a mistyped row cannot pass
    ext = ro.RHO0[:-1] * np.exp(-(ro.H0[1:] - ro.H0[:-1]) / ro.HS[:-1])
    gap = np.abs(ext / ro.RHO0[1:] - 1)
    print(f"largest band-edge gap {gap.max():.2%} at {ro.H0[gap.argmax()]:.0f} km")
    assert gap.max() < 2e-3
    below = ro.emul_density(L, ro.H0[1:] - 1e-9)
    assert np.allclose(below / ro.RHO0[1:], 1.0, atol=2e-3)


# ---- 2. force -------------------------------------------------------------------------------------------------------
def _states(rng, n):
    out = []
    for _ in range(n):
        hp, ha = rng.uniform(100, 600), rng.uniform(600, 36000)
        a = G["req"] + 0.5 * (hp + ha) + 6378.0 * 0
        e = (ha - hp) / (2 * G["req"] + hp + ha)
        s = kepler_state(a, e, rng.uniform(0, 2 * np.pi), incl=rng.uniform(0, np.pi))
        out.append(s)
    return np.array(out)


def test_force_matches_the_statement(L):
    rng = np.random.default_rng(3)
    s = _states(rng, 400)
    B = 0.02
    got = ro.emul_accel(L, s, G["mu"], G["req"], G["j2"], ro.OMEGA, B)
    ref = ro.accel(s, G["mu"], G["req"], G["j2"], ro.OMEGA, B)
    rel = np.linalg.norm(got - ref, axis=1) / np.linalg.norm(ref, axis=1)
    print(f"total acceleration: worst relative difference {rel.max():.2e}")
    assert rel.max() < 1e-14
    # the drag term alone (gravity of both subtracted)
    dg = got - ro.emul_accel(L, s, G["mu"], G["req"], G["j2"], ro.OMEGA, 0.0)
    dr = ref - ro.accel(s, G["mu"], G["req"], G["j2"], ro.OMEGA, 0.0)
    big = np.linalg.norm(dr, axis=1) > 1e-12
    assert np.allclose(dg[big], dr[big], rtol=1e-8, atol=0)


def test_j2_is_the_gradient_of_the_potential(L):
    """the J2 term equals the finite-difference gradient of the geopotential's J2 part U = -mu J2 R^2 / (2 r^3)
    (3 z^2 / r^2 - 1), a = grad U: pins its sign (the bulge pulls harder at the equator)"""
    mu, R, J2 = G["mu"], G["req"], G["j2"]
    U = lambda r: -mu * J2 * R ** 2 / (2 * np.linalg.norm(r) ** 3) * (3 * r[2] ** 2 / np.linalg.norm(r) ** 2 - 1)  # noqa
    rng = np.random.default_rng(5)
    for s in _states(rng, 20):
        a = ro.emul_accel(L, s, mu, R, J2, 0.0, 0.0)[0] - ro.emul_accel(L, s, mu, R, 0.0, 0.0, 0.0)[0]
        h = 1e-3
        grad = np.array([(U(s[:3] + h * e) - U(s[:3] - h * e)) / (2 * h) for e in np.eye(3)])
        assert np.linalg.norm(a - grad) < 1e-6 * np.linalg.norm(a)   # a - two-body loses ~1e-8 of the J2 term


def test_drag_is_quadratic_and_zero_at_zero_relative_speed(L):
    r = np.array([6378.137 + 150.0, 0.0, 0.0])
    corot = np.r_[r, np.cross([0, 0, ro.OMEGA], r)]
    a0 = ro.emul_accel(L, corot, G["mu"], G["req"], 0.0, ro.OMEGA, 0.0)
    assert np.array_equal(ro.emul_accel(L, corot, G["mu"], G["req"], 0.0, ro.OMEGA, 0.05), a0)
    drag = []
    for k in (1.0, 2.0):
        s = np.r_[r, k * np.array([0.0, 7.8, 0.0])]
        drag.append(ro.emul_accel(L, s, G["mu"], G["req"], 0.0, 0.0, 0.05)[0]
                    - ro.emul_accel(L, s, G["mu"], G["req"], 0.0, 0.0, 0.0)[0])
    assert drag[1][1] / drag[0][1] == pytest.approx(4.0, rel=1e-12)
    assert drag[0][1] < 0


# ---- 3. analytic decay ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h0,days", [(300.0, 38.75), (200.0, 2.01)])
def test_circular_decay_matches_the_quadrature(L, h0, days):
    """equatorial circular orbit, J2 = 0, no rotation, B = 0.01: geodetic height = |r| - R, and the time from h0 to
    120 km is the quadrature of da/dt = -B rho 1e3 sqrt(mu a)"""
    from scipy.integrate import quad

    mu, R, B = 398600.4418, 6378.137, 0.01
    a0 = R + h0
    y0 = np.array([a0, 0, 0, 0, np.sqrt(mu / a0), 0])
    got = ro.emul_integrate(L, y0, B, 120.0, 80 * 86400.0, mu, R, 0.0, omega=0.0)
    assert got["status"] == 0
    ts = []
    for lo, hi in zip(np.r_[120.0, ro.H0[(ro.H0 > 120) & (ro.H0 < h0)]], np.r_[ro.H0[(ro.H0 > 120) & (ro.H0 < h0)], h0]):
        ts.append(quad(lambda a: 1.0 / (B * ro.density(a - R) * 1e3 * np.sqrt(mu * a)), R + lo, R + hi,
                       epsabs=0, epsrel=1e-12)[0])
    t = sum(ts) / 86400.0
    print(f"from {h0:.0f} km: integrated {got['dt'] / 1440:.4f} d, quadrature {t:.4f} d")
    assert t == pytest.approx(days, abs=0.01)
    assert got["dt"] / 1440.0 == pytest.approx(t, rel=5e-3)


# ---- 4. independent integrator --------------------------------------------------------------------------------------
def _cases():
    out = []
    rng = np.random.default_rng(11)
    for q in range(10):   # low LEO: perigees 110-140 km, apogees up to 400 km
        hp, ha = rng.uniform(110, 140), rng.uniform(140, 400)
        a = G["req"] + 0.5 * (hp + ha)
        e = (ha - hp) / (2 * G["req"] + hp + ha)
        out.append(kepler_state(a, e, rng.uniform(0.3, 6.0), incl=rng.uniform(0.1, 2.0)))
    hp, ha = 75.0, 35786.0   # a GTO whose perigee is below the interface: it crosses on its first descent
    a = G["req"] + 0.5 * (hp + ha)
    out.append(kepler_state(a, (ha - hp) / (2 * G["req"] + hp + ha), 5.9, incl=0.48))
    return out


def test_crossings_match_dop853(L):
    worst = [0.0, 0.0]
    for y0 in _cases():
        got = ro.emul_integrate(L, y0, 0.02, 80.0, 3 * 86400.0, G["mu"], G["req"], G["j2"], epoch=EPOCH)
        t, s = ro.integrate(y0, 0.02, 80.0, 3 * 86400.0, G["mu"], G["req"], G["j2"])
        assert got["status"] == 0 and np.isfinite(t)
        lat, lon = ro.footprint(s[:3], EPOCH + t / 86400.0)
        dlon = (got["lon"] - lon + 180.0) % 360.0 - 180.0
        worst = [max(worst[0], abs(got["dt"] * 60 - t)), max(worst[1], abs(got["lat"] - lat), abs(dlon))]
        # DP87 at K7's rtol 1e-9 against DOP853 at 1e-12: the crossing moves by up to 0.45 s after a day of decay, a few
        # km along a track that descends at about 1 deg, and the footprint moves with it
        assert abs(got["dt"] * 60.0 - t) < 1.0
        assert np.linalg.norm(got["y"][:3] - s[:3]) < 8.0 * abs(got["dt"] * 60.0 - t) + 0.2
        p1, p2 = (np.radians([got["lat"], got["lon"]]), np.radians([lat, lon]))
        c = np.sin(p1[0]) * np.sin(p2[0]) + np.cos(p1[0]) * np.cos(p2[0]) * np.cos(p1[1] - p2[1])
        assert 6378.0 * np.arccos(min(c, 1.0)) < 11.0 * abs(got["dt"] * 60.0 - t) + 0.5
    print(f"against DOP853: worst |dt| {worst[0]:.3e} s, worst footprint {worst[1]:.2e} deg")


# ---- 5. locator ----------------------------------------------------------------------------------------------------
def test_hermite_crossing_against_exact_two_body(L):
    """end states 60 s apart on an exact two-body arc: the Hermite crossing within 1e-3 s of the exact one"""
    from scipy.optimize import brentq

    mu = G["mu"]
    a, e = G["req"] + 0.5 * (60.0 + 2000.0), (2000.0 - 60.0) / (2 * G["req"] + 2060.0)
    n = np.sqrt(mu / a ** 3)
    M0 = -0.25
    h = lambda t: ro.geodetic(kepler_state(a, e, M0 + n * t)[:3])[2]  # noqa: E731
    t_cross = brentq(lambda t: h(t) - 80.0, 0.0, -M0 / n, xtol=1e-12)   # before perigee
    t0 = np.floor(t_cross / 60.0) * 60.0
    s = ro.emul_locate(L, kepler_state(a, e, M0 + n * t0), kepler_state(a, e, M0 + n * (t0 + 60.0)), 60.0, 80.0)
    print(f"Hermite crossing {t0 + 60 * s:.6f} s, exact {t_cross:.6f} s")
    assert abs(t0 + 60.0 * s - t_cross) < 2e-3   # 1.5e-3 s on this grazing arc (flight-path angle -0.6 deg)


def test_perigee_dip_and_start_below(L):
    mu = G["mu"]
    # a perigee 1 km below the interface in the middle of a 300 s interval; both ends are above it
    hp = 79.0 + 0.0
    a, e = G["req"] + 0.5 * (hp + 1000.0), (1000.0 - hp) / (2 * G["req"] + hp + 1000.0)
    n = np.sqrt(mu / a ** 3)
    y0, y1 = kepler_state(a, e, -150 * n, incl=0.0), kepler_state(a, e, 150 * n, incl=0.0)
    hs = ro.emul_height(L, np.array([y0[:3], y1[:3]]))
    assert (hs > 80.0).all()
    s = ro.emul_locate(L, y0, y1, 300.0, 80.0)
    assert 0.0 < s < 0.5
    assert ro.emul_locate(L, y0, y1, 300.0, 78.0) == -1.0   # the dip stays above 78 km
    # a start at or below the interface crosses at dt = 0
    got = ro.emul_integrate(L, kepler_state(a, e, 0.0, incl=0.0), 0.02, 80.0, 86400.0, mu, G["req"], G["j2"])
    assert got["status"] == 0 and got["dt"] == 0.0 and got["acc"] == 0


# ---- 6. draws ------------------------------------------------------------------------------------------------------
def _cat():
    el = np.stack([leo(150, 250, bstar=3e-3), leo(180, 300, incl=97.0, bstar=2e-3), leo(160, 220, incl=28.5, bstar=3e-3)], 1)
    P = np.zeros((3, 28))
    # a small diagonal covariance on row 1 (n, e cos w, e sin w, i, node, lambda, B*)
    idx = [0, 7, 13, 18, 22, 25, 27]
    P[1, idx] = np.array([1e-9, 1e-9, 1e-9, 1e-8, 1e-8, 1e-8, 1e-10])
    return el, P


def test_zero_covariance_samples_equal_the_nominal(L):
    el, P = _cat()
    rec, _, nst, counts, out, st = ro.emul(L, el, P, None, [0, 2], samples=5, record=5, horizon_days=3.0)
    assert (st == 0).all() and (nst == 0).all() and (counts[:, 0] == 5).all()
    for i in range(2):
        assert (out[i, :, 0] == rec[i, 0]).all() and (out[i, :, 1] == rec[i, 1]).all()
        assert (out[i, :, 2] == rec[i, 2]).all() and (out[i, :, 3] == rec[i, 6] + rec[i, 7]).all()


def test_drawn_set_is_k14s_primary_draw(L):
    Lmc = mc.emul_library()
    el, P = _cat()
    k = np.arange(100, 164, dtype=np.uint64)
    st, x, B, f, y, built = ro.emul_draw(L, el[:, 1], 0, P[1], 99, k, sigma=0.0)
    x14, st14 = mc.emul_draw(Lmc, el[:, 1], 0, P[1], 99, 0, k)
    assert st == 0 and st14 == 0 and np.array_equal(x, x14)
    assert np.array_equal(B, 12.741621 * el[7, 1] + 12.741621 * (x[:, 6] - el[7, 1]))
    assert (f == 1.0).all() and built.all()


def test_density_draws_order_the_crossings(L):
    el, P = _cat()
    sigma, seed = 0.5, 7
    _, x, B, f, _, _ = ro.emul_draw(L, el[:, 0], 0, P[0], seed, np.arange(16, dtype=np.uint64), sigma=sigma)
    z7 = mc.normals(seed, np.arange(16, dtype=np.uint64))[:, 7]
    assert np.allclose(f, np.exp(sigma * z7), rtol=1e-15)
    _, _, _, _, out, _ = ro.emul(L, el, P, None, [0], samples=16, seed=seed, sigma=sigma, record=16,
                                 horizon_days=3.0)
    dt = out[0, :, 0]
    order = np.argsort(z7)
    assert (np.diff(dt[order]) < 0).all()   # denser atmosphere, earlier crossing


def test_split_order_and_batch_invariance(L):
    el, P = _cat()
    kw = dict(horizon_days=3.0, sigma=0.3, seed=5)
    rec, _, nst, counts, out, st = ro.emul(L, el, P, None, [1, 0, 1], samples=8, record=8, **kw)
    a = ro.emul(L, el, P, None, [1], samples=4, record=4, **kw)
    b = ro.emul(L, el, P, None, [1], samples=4, first=4, record=4, **kw)
    assert np.array_equal(a[3] + b[3], counts[:1])
    same = lambda x, y: np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))  # noqa: E731
    assert same(np.concatenate([a[4], b[4]], 1), out[:1])
    assert same(rec[0], rec[2]) and same(out[0], out[2])   # a duplicated row
    perm = ro.emul(L, el, P, None, [0, 1], samples=8, record=8, **kw)
    assert same(perm[0][0], rec[1]) and same(perm[4][1], out[0])


# ---- 7. rules ------------------------------------------------------------------------------------------------------
def test_ballistic_rules_and_statuses(L):
    el, P = _cat()
    el = np.concatenate([el, leo(150, 200, bstar=-1e-4)[:, None], leo(600, 700, bstar=1e-5)[:, None],
                         leo(120, 200)[:, None]], 1)
    el[1, 5] = 100.0   # 100 rev/day: no set can be built
    P = np.concatenate([P, np.zeros((3, 28))])
    P6 = P.copy()
    P6[0, 0] = -1e-9   # a negative variance: NOT_PSD
    rec, _, nst, counts, _, st = ro.emul(L, el, P6, None, [0, 1, 2, 3, 4, 5], samples=3, horizon_days=1.0)
    assert list(st) == [2, 0, 0, 0, 0, 1]   # NOT_PSD; row 5 (100 rev/day) INIT_FAILED
    assert rec[2, 5] == 12.741621 * el[7, 2]   # the default B
    assert nst[3] == ro_nonphysical() and (counts[3] == [0, 0, 3]).all()   # B* <= 0
    assert nst[4] == 1 and (counts[4] == [0, 3, 0]).all()                  # ABOVE at a 1-day horizon
    assert nst[2] == 0
    bad = ro.emul(L, el, P, None, [5, 1], samples=1, horizon_days=1.0)
    assert list(bad[5]) == [1, 0]
    el2 = el.copy()
    el2[1, 1] = 100.0
    r2 = ro.emul(L, el2, P, None, [1, 7], samples=1)
    assert list(r2[5]) == [1, 3] and (r2[2] == 2).all()   # INIT_FAILED, BAD_ROW; the nominals are not run
    # given ballistic coefficients override B*; a draw with B <= 0 counts as failed
    r3 = ro.emul(L, el, P, None, [0, 0], ballistic=[0.03, -0.01], samples=2, horizon_days=1.0)
    assert r3[0][0, 5] == 0.03 and r3[2][1] == ro_nonphysical() and (r3[3][1] == [0, 0, 2]).all()


def ro_nonphysical():
    return 3


def test_stopped_trajectory(L):
    """K7's stop rule: a drag so strong (B = 1e9 m^2/kg at 100 km) that no step down to hMin meets the tolerance;
    and a non-finite state"""
    r = G["req"] + 100.0
    y0 = np.array([r, 0.0, 0.0, 0.0, np.sqrt(G["mu"] / r), 0.0])
    got = ro.emul_integrate(L, y0, 1e9, 60.0, 86400.0, G["mu"], G["req"], G["j2"])
    assert got["status"] == 4 and np.isnan(got["dt"]) and got["rej"] > 0
    bad = ro.emul_integrate(L, np.array([7000.0, 0, 0, np.nan, 0, 0]), 0.02, 80.0, 86400.0, G["mu"], G["req"], G["j2"])
    assert bad["status"] == 4 and np.isnan(bad["dt"])


# ---- the C ABI's refusals and the wrapper ---------------------------------------------------------------------------
def _abi(**over):
    el, P = _cat()
    m = 3
    a = dict(el=np.ascontiguousarray(el), P=np.ascontiguousarray(P), model=np.zeros(3, np.uint8),
             rows=np.array([0, 1, 2], np.uint32), bc=None, ns=np.full(m, 4, np.uint64), first=np.zeros(m, np.uint64),
             seed=np.zeros(m, np.uint64), hi=80.0, hor=30.0, step=60.0, scale=1.0, sigma=0.0, grav=1, device=0,
             record=2, out=True)
    a.update(over)
    return a


def _call(a):
    from astroz_b200 import _lib

    m = len(a["rows"])
    rec, nst, st = np.full((m, 8), 7.0), np.full(m, 9, np.uint8), np.full(m, 9, np.uint8)
    counts = np.full((m, 3), 7, np.uint64)
    so = np.full((m, a["record"], 4), 7.0) if a["out"] else None
    p = lambda x: None if x is None else C.c_void_p(x.ctypes.data)  # noqa: E731
    rc = _lib.lib().astroz_cuda_reentry(p(a["el"]), a["el"].shape[1], a["grav"], p(a["P"]), p(a["model"]),
                                        p(a["rows"]), p(a["bc"]), p(a["ns"]), p(a["first"]), p(a["seed"]), m, a["hi"],
                                        a["hor"], a["step"], a["scale"], a["sigma"], a["record"], a["device"], p(rec),
                                        None, p(nst), p(counts), p(so), p(st))
    untouched = (rec == 7.0).all() and (nst == 9).all() and (st == 9).all() and (counts == 7).all() and \
        (so is None or (so == 7.0).all())
    return rc, untouched


def _nan_el():
    el, _ = _cat()
    el[2, 1] = np.nan
    return np.ascontiguousarray(el)


REFUSALS = {
    "device": (dict(device=-1), "runs on one device"), "grav": (dict(grav=7), "grav must be"),
    "hi_low": (dict(hi=59.9), "h_i"), "hi_high": (dict(hi=200.1), "h_i"), "horizon0": (dict(hor=0.0), "horizon_days"),
    "horizon_big": (dict(hor=3660.5), "horizon_days"), "step_low": (dict(step=0.5), "step_s"),
    "step_high": (dict(step=3601.0), "step_s"), "sigma_neg": (dict(sigma=-0.1), "density_sigma"),
    "sigma_big": (dict(sigma=2.5), "density_sigma"), "scale0": (dict(scale=0.0), "density_scale"),
    "scale_inf": (dict(scale=np.inf), "density_scale"), "row": (dict(rows=np.array([0, 3, 1], np.uint32)), "outside"),
    "ballistic": (dict(bc=np.array([0.01, np.nan, 0.02])), "ballistic"),
    "overflow": (dict(first=np.array([0, 2 ** 64 - 2, 0], np.uint64)), "2^64"),
    "no_sample_out": (dict(out=False), "needs sample_out"), "nan_el": (dict(el=_nan_el()), "elements must be"),
    "model": (dict(model=np.array([0, 2, 0], np.uint8)), "model byte"),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_c_abi_refusals(case):
    from astroz_b200 import _lib
    from astroz_b200._abi import DEFINES as D

    over, text = REFUSALS[case]
    rc, untouched = _call(_abi(**over))
    assert rc == D["ASTROZ_VALUE_ERROR"]
    assert text in _lib.lib().astroz_cuda_last_error().decode()
    assert untouched


def test_valid_input_without_a_device_writes_nothing():
    from astroz_b200 import _lib
    from astroz_b200._abi import DEFINES as D

    if _lib.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    rc, untouched = _call(_abi())
    assert rc == D["ASTROZ_NO_DEVICE"] and untouched
    b = C.c_uint64(5)
    assert _lib.lib().astroz_cuda_reentry_scratch_bytes(4, C.byref(b)) == D["ASTROZ_NO_DEVICE"] and b.value == 5


def test_window_counts_above_as_inf():
    from astroz_b200.reentry import ReentryResult

    words = np.full((2, 10, 4), np.nan)
    words[0, :, 0] = np.r_[np.arange(1.0, 8.0), np.inf, np.inf, np.nan]   # 7 crossings, 2 ABOVE, 1 failed
    words[1, :3, 0] = np.inf
    res = ReentryResult(np.zeros((2, 8)), np.full(2, 2460000.5), np.zeros(2), None, np.zeros(2, np.uint8),
                        np.array([[7, 2, 1], [0, 3, 0]], np.uint64), np.array([10, 3], np.uint64), words,
                        np.zeros(2, np.uint8))
    lo, hi = res.window(0.05, 0.95)   # epochs: the row's epoch plus dt
    assert lo[0] == 2460000.5 + 1.0 / 1440.0 and hi[0] == np.inf and lo[1] == np.inf
    assert lo[0] < res.window(0.5, 0.5)[0][0] < np.inf
    assert np.allclose(res.fraction_reentered(), [7 / 9, 0.0])
