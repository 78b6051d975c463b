"""K18 sensor tasking (az_tasking.cuh, az_tasking.cu) on the CPU.

The host build of the device source (tests/host_emul/emul_tasking.cu): its visibility against a numpy statement of
the rules on the oracle's SGP4 / SDP4 states; its gain, spread and posterior against numpy's m x m and Joseph forms
and a linear Monte Carlo; its schedule against a brute-force statement of the greedy rule; sun_direction against
published equinox and solstice instants; the C ABI's refusals.  The device runs are in tests/test_gpu_tasking.py."""
import ctypes as C

import numpy as np
import pytest

from tests.fit_oracle import covariance as K
from tests.fit_oracle import obs as O
from tests.fit_oracle import tasking as TK


@pytest.fixture(scope="module")
def L():
    lib = TK.emul_library()
    if lib is None:
        pytest.skip("nvcc unavailable")
    return lib


@pytest.fixture(scope="module")
def sc():
    return TK.scene(n_per=10, T=60)


def _oracle_states(el, jd, fr):
    return O.states_of(el, jd, fr)


# ---- 1. visibility --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("optical", [False, True])
def test_visibility_against_the_numpy_statement(L, optical):
    """every rule (elevation, range, shadow, station darkness, exclusion) on LEO, SSO, GEO and Molniya rows, radar and
    optical sites over a day: the host build's visible cells equal the numpy statement on the oracle's states, except
    cells within 1e-9 rad / 1e-6 km of a threshold (counted)"""
    kw = dict(radar=np.zeros((0, 3)), optical=TK.OPTICAL_SITES) if optical else dict(range_max=4000.0)
    sc = TK.scene(n_per=2, T=96, step_min=15.0, **kw)
    seen, excluded, compared = 0, 0, 0
    states = [_oracle_states(sc.el[:, s], sc.jd, sc.fr) for s in range(sc.n)]
    for t in range(sc.T):
        _, _, vis, fail, _, rs = TK.emul_slot(L, sc, t, sc.P)
        assert np.all(rs == 0) and np.all(fail == 0)
        jdf = sc.jd[t] + sc.fr[t]
        for k in range(sc.S):
            st = np.array([states[s][t] for s in range(sc.n)])
            v, margin = TK.visibility(st, np.full(sc.n, jdf), sc.stations[sc.station[k]], sc.kind[k],
                                      sc.limits[k], sc.sun[t])
            mine = (vis >> k) & 1 == 1
            keep = margin > 1e-6
            excluded += int((~keep).sum())
            compared += int(keep.sum())
            assert np.array_equal(mine[keep], v[keep]), (t, k)
            seen += int(mine.sum())
    print(f"visible cells {seen}, compared {compared}, excluded near a threshold {excluded}")
    assert seen > 0 and excluded < 0.01 * compared


def test_geo_over_its_station_is_seen_in_every_dark_slot(L):
    """a GEO row at the optical site's longitude is visible whenever the site is dark and the row is lit"""
    sc = TK.scene(n_per=1, T=48, step_min=30.0, radar=np.zeros((0, 3)), optical=[[0.0, 80.0, 0.0]],
                  exclusion=0.0)
    geo = 2
    # put the GEO row over longitude 80 at t0
    _, _, _, _, f0, _ = TK.emul_slot(L, sc, 0, sc.P)
    lon = np.rad2deg(np.arctan2(*(O.ecef_state(f0[geo], sc.jd[0] + sc.fr[0])[0][0, [1, 0]])))
    sc.el[6, geo] = (sc.el[6, geo] + 80.0 - lon) % 360.0
    dark = 0
    for t in range(sc.T):
        _, _, vis, _, f0, _ = TK.emul_slot(L, sc, t, sc.P)
        jdf = sc.jd[t] + sc.fr[t]
        up = O.enu_basis(sc.stations[0])[2]
        u = sc.sun[t] / np.linalg.norm(sc.sun[t])
        if (O.rot(O.gmst(jdf)) @ u) @ up > np.sin(np.deg2rad(-12.0)):
            continue
        r = f0[geo, :3]
        rs = r @ u
        if rs < 0 and np.linalg.norm(r - rs * u) <= TK.R_EARTH:
            continue
        dark += 1
        assert vis[geo] & 1, t
    assert dark >= 8


def test_no_optical_task_at_local_noon_or_in_shadow(L):
    """an optical sensor sees nothing while its Sun is up, and never tasks a row inside the shadow cylinder"""
    sc = TK.scene(n_per=4, T=72, step_min=20.0, radar=np.zeros((0, 3)), optical=TK.OPTICAL_SITES[:1])
    out = TK.emul(L, sc)
    lit_up = 0
    for t in range(sc.T):
        jdf = sc.jd[t] + sc.fr[t]
        u = sc.sun[t] / np.linalg.norm(sc.sun[t])
        _, _, vis, _, f0, _ = TK.emul_slot(L, sc, t, sc.P)
        if (O.rot(O.gmst(jdf)) @ u) @ O.enu_basis(sc.stations[0])[2] > 0.0:
            lit_up += 1
            assert not np.any(vis & 1) and out["task_row"][0, t] == TK.IDLE
        s = out["task_row"][0, t]
        if s != TK.IDLE:
            r = f0[s, :3]
            assert r @ u >= 0 or np.linalg.norm(r - (r @ u) * u) > TK.R_EARTH
    assert lit_up > 0 and np.any(out["task_row"][0] != TK.IDLE)


# ---- 2. gain, spread, posterior -------------------------------------------------------------------------------------
def _cells(L, sc, count=60):
    """(G (4, 7), P (28,), sigma (4,), gain, spread) of visible cells of the scene"""
    out = []
    for t in range(0, sc.T, 3):
        gain, cell, vis, _, _, _ = TK.emul_slot(L, sc, t, sc.P)
        for k in range(sc.S):
            for s in np.nonzero((vis >> k) & 1)[0]:
                out.append((cell[k, s, 8:].reshape(4, 7), sc.P[s], sc.sigma[k], gain[k, s], cell[k, s, 4:8]))
    assert len(out) >= count
    return out


def test_gain_spread_and_posterior_against_numpy(L, sc):
    """g within 1e-10 of 1/2 log det(I + G P G^T) in the m x m form, = 1/2 log(det P / det P+) for definite P; the
    spread is sqrt(diag(G P G^T)) sigma; P+ within 1e-10 of its trace of the Joseph form, symmetric and PSD"""
    worst = {"g": 0.0, "ratio": 0.0, "spread": 0.0, "P+": 0.0}
    for G, Pw, sigma, g, spread in _cells(L, sc):
        P = K.unpack7(Pw)
        used = np.any(G != 0.0, axis=1)
        Gm = G[used]
        S = Gm @ P @ Gm.T
        g_ref = 0.5 * np.linalg.slogdet(np.eye(len(Gm)) + S)[1]
        worst["g"] = max(worst["g"], abs(g - g_ref) / abs(g_ref))
        rc, g2, sp2, Pp = TK.emul_update(L, G, Pw, sigma)
        assert rc == 0 and g2 == g and np.array_equal(sp2, spread)
        sref = np.where(np.isfinite(sigma), np.sqrt(np.diag(G @ P @ G.T)) * np.where(np.isfinite(sigma), sigma, 0), 0)
        worst["spread"] = max(worst["spread"], np.max(np.abs(spread - sref) / np.maximum(sref, 1e-300)))
        Kg = P @ Gm.T @ np.linalg.inv(np.eye(len(Gm)) + S)
        A = np.eye(7) - Kg @ Gm
        Pj = A @ P @ A.T + Kg @ Kg.T
        Pm = K.unpack7(Pp)
        worst["P+"] = max(worst["P+"], np.max(np.abs(Pm - Pj)) / np.trace(Pj))
        assert np.array_equal(Pm, Pm.T) and np.linalg.eigvalsh(Pm).min() >= -1e-12 * np.trace(Pm)
        if np.linalg.eigvalsh(P).min() > 0:
            ratio = 0.5 * (np.linalg.slogdet(P)[1] - np.linalg.slogdet(Pm)[1])
            worst["ratio"] = max(worst["ratio"], abs(g - ratio) / abs(g))
    print(worst)
    assert worst["g"] < 1e-10 and worst["P+"] < 1e-10 and worst["spread"] < 1e-10 and worst["ratio"] < 1e-8


def test_zero_and_singular_covariance(L, sc):
    """P = 0: g = 0 exactly, P+ = 0, and such rows are never tasked; a held B* row (zero row) stays zero"""
    G, Pw, sigma, _, _ = _cells(L, sc)[0]
    rc, g, spread, Pp = TK.emul_update(L, G, np.zeros(28), sigma)
    assert rc == 0 and g == 0.0 and np.all(spread == 0.0) and np.all(Pp == 0.0)
    P = K.unpack7(Pw)
    P[6, :] = P[:, 6] = 0.0
    rc, g, _, Pp = TK.emul_update(L, G, K.pack7(P), sigma)
    Pm = K.unpack7(Pp)
    assert rc == 0 and g > 0 and np.all(Pm[6] == 0.0) and np.all(Pm[:, 6] == 0.0)
    cov = sc.P.copy()
    cov[::2] = 0.0
    out = TK.emul(L, sc, cov=cov)
    tasked = out["task_row"][out["task_row"] != TK.IDLE]
    assert len(tasked) and np.all(tasked % 2 == 1)
    assert np.all(out["posterior"][::2] == 0.0) and np.all(out["n_tasks"][::2] == 0)


def test_posterior_is_the_linear_mmse_error_covariance(L, sc):
    """10^5 draws x ~ N(0, P), y = G x + e, e ~ N(0, I) (weighted units): the error covariance of the linear MMSE
    estimate equals P+ within sampling error"""
    G, Pw, sigma, _, _ = next(c for c in _cells(L, sc) if np.linalg.eigvalsh(K.unpack7(c[1])).min() > 0)
    _, _, _, Pp = TK.emul_update(L, G, Pw, sigma)
    P = K.unpack7(Pw)
    rng = np.random.default_rng(11)
    N = 100_000
    x = rng.multivariate_normal(np.zeros(7), P, size=N, method="eigh")
    y = x @ G.T + rng.standard_normal((N, 4))
    Kg = P @ G.T @ np.linalg.inv(G @ P @ G.T + np.eye(4))
    err = x - y @ Kg.T
    emp = err.T @ err / N
    Pm = K.unpack7(Pp)
    d = np.sqrt(np.diag(Pm))
    assert np.max(np.abs(emp - Pm) / np.outer(d, d)) < 5 * np.sqrt(2.0 / N)


# ---- 3. schedule ----------------------------------------------------------------------------------------------------
def test_schedule_against_the_brute_force_statement(L, sc):
    """40 mixed rows x 3 sensors x 60 slots: task_row, task_gain, n_candidates and posterior equal the brute-force
    statement's exactly"""
    out = TK.emul(L, sc)
    rows, gains, cands, P = TK.greedy(L, sc)
    assert np.array_equal(out["task_row"], rows)
    assert np.array_equal(out["task_gain"], gains)
    assert np.array_equal(out["n_candidates"], cands)
    assert np.array_equal(out["posterior"], P)
    assert np.sum(rows != TK.IDLE) > 20
    assert np.array_equal(out["n_tasks"], np.bincount(rows[rows != TK.IDLE].astype(np.int64), minlength=sc.n))


def test_ties_go_to_the_lower_row(L, sc):
    """a catalogue of each row twice: every task goes to the lower copy first, and a row's copy is taken only by a
    later sensor of the same slot"""
    n = sc.n
    dup = TK.Scene(np.ascontiguousarray(np.concatenate([sc.el, sc.el], axis=1)), np.concatenate([sc.model] * 2),
                   np.concatenate([sc.P, sc.P]), sc.kind, sc.station, sc.sigma, sc.limits, sc.stations, sc.jd[:20],
                   sc.fr[:20], sc.sun[:20])
    out = TK.emul(L, dup)
    rows, _, _, _ = TK.greedy(L, dup)
    assert np.array_equal(out["task_row"], rows)
    tasks = np.zeros(2 * n, np.int64)   # tasks before the slot: equal counts mean equal covariances
    upper = 0
    for t in range(dup.T):
        picked = [int(r) for r in out["task_row"][:, t] if r != TK.IDLE]
        for q, r in enumerate(picked):
            if r >= n:
                upper += 1
                assert r - n in picked[:q] or tasks[r - n] != tasks[r], (t, r)
        tasks[picked] += 1
    print(f"tasks {int(tasks.sum())}, upper copies taken {upper}")
    assert tasks[:n].sum() > 0


def test_statuses_and_counters(L, sc):
    """INIT_FAILED rows (a set below the surface, a deep-space set of e 0.96 with B* 0) take part in nothing: no
    visible cell, no task, the posterior their input covariance; the other counters are consistent"""
    el = sc.el.copy()
    el[1, 0] = 40.0                       # a near-earth row below the surface: init fails
    el[2, 25], el[7, 25] = 0.96, 0.0      # a deep-space row of e 0.96: cells fail near perigee or not at all
    bad = TK.Scene(el, sc.model, sc.P, sc.kind, sc.station, sc.sigma, sc.limits, sc.stations, sc.jd, sc.fr, sc.sun)
    out = TK.emul(L, bad)
    for s in (0, 25):
        assert out["row_status"][s] == 1 and out["n_visible"][s] == 0 and out["n_tasks"][s] == 0
        assert out["n_failed"][s] == 0 and np.array_equal(out["posterior"][s], sc.P[s])
    assert np.sum(out["row_status"] != 0) == 2
    ok = out["task_row"] != TK.IDLE
    assert np.all(out["n_candidates"][ok] >= 1) and np.all(out["n_candidates"][~ok] == 0)
    assert np.all(out["task_gain"][ok] > 0) and np.all(out["task_gain"][~ok] == 0)
    assert out["n_visible"].sum() > 0 and np.all(out["n_tasks"] <= out["n_visible"])


# ---- 4. the Sun -----------------------------------------------------------------------------------------------------
def test_sun_direction():
    """against an independent statement (ecliptic longitude from the equation of centre, rotated by the obliquity),
    the 2024 equinoxes and solstices within 0.02 deg of 0 / +-23.44 deg declination, the distance in 0.983 .. 1.017"""
    from astroz_b200.tasking import sun_direction

    # 2024-03-20 03:06, 2024-06-20 20:51, 2024-09-22 12:44, 2024-12-21 09:21 UT
    inst = np.array([2460389.5 + (3 + 6 / 60) / 24, 2460481.5 + (20 + 51 / 60) / 24,
                     2460575.5 + (12 + 44 / 60) / 24, 2460665.5 + (9 + 21 / 60) / 24])
    v = sun_direction(inst)
    dec = np.rad2deg(np.arcsin(v[:, 2] / np.linalg.norm(v, axis=1)))
    assert np.max(np.abs(dec - [0.0, 23.44, 0.0, -23.44])) < 0.02
    jd = 2451545.0 + np.linspace(-9000, 18000, 500)
    v = sun_direction(jd)
    r = np.linalg.norm(v, axis=1)
    assert r.min() > 0.983 and r.max() < 1.017
    T = (jd - 2451545.0) / 36525.0
    M = np.deg2rad(357.52911 + 35999.05029 * T)
    L0 = 280.46646 + 36000.76983 * T
    lam = np.deg2rad(L0 + (1.914602 - 0.004817 * T) * np.sin(M) + 0.019993 * np.sin(2 * M))
    eps = np.deg2rad(23.439291 - 0.0130042 * T)
    ref = np.stack([np.cos(lam), np.cos(eps) * np.sin(lam), np.sin(eps) * np.sin(lam)], axis=1)
    ang = np.rad2deg(np.arccos(np.clip(np.einsum("ni,ni->n", v / r[:, None], ref), -1, 1)))
    assert ang.max() < 0.02


# ---- 5. the C ABI's refusals ----------------------------------------------------------------------------------------
def _call(sc, **over):
    from astroz_b200._lib import lib

    a = dict(el=sc.el, n=sc.n, grav=1, cov=sc.P, model=sc.model, kind=sc.kind, station=sc.station, sigma=sc.sigma,
             limits=sc.limits, s=sc.S, stations=sc.stations, k=len(sc.stations), jd=sc.jd, fr=sc.fr, t=sc.T,
             sun=sc.sun, gain_min=0.0, device=0)
    a.update(over)
    S, T, n = a["s"], a["t"], a["n"]
    outs = [np.full((max(S, 1), max(T, 1)), 7, np.uint32), np.full((max(S, 1), max(T, 1)), 7.0),
            np.full((max(S, 1), max(T, 1), 4), 7.0), np.full((max(S, 1), max(T, 1), 4), 7.0),
            np.full((max(S, 1), max(T, 1)), 7, np.uint32), np.full((n, 28), 7.0), np.full(n, 7, np.uint32),
            np.full(n, 7, np.uint32), np.full(n, 7, np.uint32), np.full(n, 7, np.uint8)]
    vp = lambda x: None if x is None else C.c_void_p(np.ascontiguousarray(x).ctypes.data)  # noqa: E731
    keep = [np.ascontiguousarray(a[q]) if a[q] is not None else None
            for q in ("el", "cov", "model", "kind", "station", "sigma", "limits", "stations", "jd", "fr", "sun")]
    el, cov, md, kind, st, sig, lim, sts, jd, fr, sun = keep
    rc = lib().astroz_cuda_tasking(vp(el), n, a["grav"], vp(cov), vp(md), vp(kind), vp(st), vp(sig), vp(lim), S,
                                   vp(sts), a["k"], vp(jd), vp(fr), T, vp(sun), a["gain_min"], a["device"],
                                   *[C.c_void_p(o.ctypes.data) for o in outs])
    return rc, outs


def _refusals(sc):
    kind = sc.kind.copy(); kind[0] = 1                          # noqa: E702
    st = sc.station.copy(); st[0] = len(sc.stations)            # noqa: E702
    sg0 = sc.sigma.copy(); sg0[0, 1] = 0.0                      # noqa: E702
    sgn = sc.sigma.copy(); sgn[0] = np.inf                      # noqa: E702
    lel = sc.limits.copy(); lel[0, 0] = 2.0                     # noqa: E702
    lsun = sc.limits.copy(); lsun[-1, 2] = -1.6                 # noqa: E702
    lrng = sc.limits.copy(); lrng[0, 1] = 0.0                   # noqa: E702
    lexc = sc.limits.copy(); lexc[-1, 3] = 3.5                  # noqa: E702
    jdn = sc.jd.copy(); jdn[3] = np.nan                         # noqa: E702
    frd = sc.fr.copy(); frd[5] = frd[4] - 1e-6                  # noqa: E702
    sun0 = sc.sun.copy(); sun0[2] = 0.0                         # noqa: E702
    sunn = sc.sun.copy(); sunn[2, 1] = np.inf                   # noqa: E702
    eln = sc.el.copy(); eln[3, 2] = np.nan                      # noqa: E702
    covn = sc.P.copy(); covn[1, 1] = np.inf                     # noqa: E702
    md = sc.model.copy(); md[0] = 2                             # noqa: E702
    return [
        (dict(device=-1), "sensor tasking runs on one device: pass its ordinal"),
        (dict(grav=7), "grav must be ASTROZ_WGS72 or ASTROZ_WGS84"),
        (dict(s=0), "s must be in [1, ASTROZ_TASK_MAX_SENSORS]"),
        (dict(s=33), "s must be in [1, ASTROZ_TASK_MAX_SENSORS]"),
        (dict(t=0), "t must be at least 1"),
        (dict(gain_min=-1e-3), "gain_min must be finite and >= 0"),
        (dict(gain_min=np.nan), "gain_min must be finite and >= 0"),
        (dict(kind=kind), "a sensor kind is not ASTROZ_OBS_RADAR or ASTROZ_OBS_OPTICAL"),
        (dict(station=st), "a sensor's station index is not below the station count k"),
        (dict(sigma=sg0), "sensor sigma must be > 0 (+inf: component not measured)"),
        (dict(sigma=sgn), "a sensor measures no component"),
        (dict(limits=lel), "an elevation limit is outside [-pi/2, pi/2]"),
        (dict(limits=lsun), "an elevation limit is outside [-pi/2, pi/2]"),
        (dict(limits=lrng), "range_max must be > 0 (+inf allowed)"),
        (dict(limits=lexc), "an exclusion angle is outside [0, pi]"),
        (dict(jd=jdn), "slot times must be finite"),
        (dict(fr=frd), "slot times must be non-decreasing"),
        (dict(sun=None), "an optical sensor needs the Sun's direction at every slot"),
        (dict(sun=sun0), "a Sun direction is zero or not finite"),
        (dict(sun=sunn), "a Sun direction is zero or not finite"),
        (dict(el=eln), "elements must be finite"),
        (dict(cov=covn), "covariance words must be finite"),
        (dict(model=md), "a model byte is not 0 (near-earth) or 1 (deep space)"),
    ]


def test_refusals_write_nothing(sc):
    """every refusal of the host call: ASTROZ_VALUE_ERROR with its text, every output untouched"""
    from astroz_b200._lib import lib

    last_error = lambda: lib().astroz_cuda_last_error().decode()  # noqa: E731
    small = TK.Scene(sc.el[:, :4].copy(), sc.model[:4].copy(), sc.P[:4].copy(), sc.kind, sc.station, sc.sigma,
                     sc.limits, sc.stations, sc.jd[:8].copy(), sc.fr[:8].copy(), sc.sun[:8].copy())
    for over, text in _refusals(small):
        rc, outs = _call(small, **over)
        assert rc == -20, (over.keys(), rc)
        assert last_error() == text, (over.keys(), last_error())
        for o in outs:
            assert np.all(o == 7), over.keys()


def test_scratch_bytes_and_zig_bindings():
    import subprocess
    import sys

    from astroz_b200.tasking import plan_scratch_bytes

    L = TK.emul_library()
    if L is not None:
        assert plan_scratch_bytes(1000, 9) == L.emul_task_scratch_bytes(1000, 9)
    with pytest.raises(Exception):
        plan_scratch_bytes(10, 0)
    r = subprocess.run([sys.executable, "tools/gen_zig_bindings.py", "--check"], capture_output=True, text=True,
                       cwd=TK._ROOT)
    assert r.returncode == 0, r.stdout + r.stderr
