"""Element fits from sensor observations (az_obs.cuh, az_fit_obs.cu) on the CPU.

The measurement models of the host build of the device source (tests/host_emul/emul_fit_obs.cu) against an independent
numpy statement (tests/fit_oracle/obs.py) and against geometry with known answers; the sigma = inf rule; noise-free
round trips that recover known element sets from perturbed guesses out of radar, GPS (ECEF) and optical tracks made
on the oracle's SGP4 / SDP4; the formal covariance against 300 noisy replicas; the element-covariance mapping; the C
ABI's refusals.  The device runs are in tests/test_gpu_fit_obs.py."""
import ctypes as C

import numpy as np
import pytest

from tests import fit_oracle as R
from tests.fit_oracle import obs as O

TWO_PI = 2 * np.pi


@pytest.fixture(scope="module")
def L():
    lib = O.emul_library()
    if lib is None:
        pytest.skip("nvcc unavailable")
    return lib


def _leo(k):
    from astroz_b200 import synth

    return synth.elements_from_tles(synth.near_earth_catalog(600))[:, :k]


def _grid(days, step_min=1.0):
    from astroz_b200 import synth

    jd, fr = synth.time_grid(int(days * 1440 / step_min))
    return jd, np.arange(len(jd)) * step_min / 1440.0 + fr[0]


# ---- measurement models ------------------------------------------------------------------------------------------
def test_station_round_trips_through_ecef_to_geodetic(L):
    """Stations on the ground come back from ecef_to_geodetic within 2e-9 km.  That converter takes one Bowring step,
    sized for satellite altitudes; at the surface its latitude is good to ~1.6e-13 rad (1e-9 km), which sets the bound."""
    rng = np.random.default_rng(4)
    llh = np.column_stack([rng.uniform(-89.9, 89.9, 200), rng.uniform(-180, 180, 200), rng.uniform(-0.4, 5.0, 200)])
    llh = np.concatenate([llh, [[90.0 - 1e-9, 10.0, 1.0], [-45.0, 0.0, 0.0], [0.0, 179.999, 0.0]]])
    for row in llh:
        ecef, back = np.zeros(3), np.zeros(3)
        L.emul_station(O._p(np.ascontiguousarray(row)), O._p(ecef), O._p(back))
        assert np.abs(ecef - O.station_ecef(row)).max() < 1e-9
        lat, lon, h = back
        assert abs(h - row[2]) < 1e-9, row
        assert abs(lat - np.radians(row[0])) * 6378.137 < 2e-9, row
        dl = np.mod(lon - np.radians(row[1]) + np.pi, TWO_PI) - np.pi
        assert abs(dl) * 6378.137 * np.cos(np.radians(row[0])) < 1e-9, row


def _teme_of_ecef(r_ecef, jd_full):
    return np.einsum("ji,j->i", O.rot(O.gmst(jd_full)), r_ecef)


def test_zenith_and_due_north_on_the_horizon(L):
    jdf = 2460437.3
    for llh in ([42.6, -71.5, 0.12], [-31.0, 136.0, 0.15], [0.0, 0.0, 0.0], [80.0, 200.0, 1.0]):
        llh = np.array(llh)
        e, n, u = O.enu_basis(llh)
        rs = O.station_ecef(llh)
        for target, az, el in ((rs + 800.0 * u, None, np.pi / 2), (rs + 1500.0 * n, 0.0, 0.0)):
            state = np.concatenate([_teme_of_ecef(target, jdf), np.zeros(3)])
            h = O.emul_observe(L, state, jdf, 0.0, O.RADAR, 0, llh)[0]
            assert abs(h[2] - el) < 1e-9, (llh, h)
            if az is not None:
                assert abs(np.mod(h[1] - az + np.pi, TWO_PI) - np.pi) < 1e-12, (llh, h)
            assert abs(h[0] - np.linalg.norm(target - rs)) < 1e-9


@pytest.mark.parametrize("kind", [O.TEME, O.ECEF, O.RADAR, O.OPTICAL])
def test_models_match_the_numpy_statement(L, kind):
    el = _leo(4)
    jd, fr = _grid(1.0, 2.0)
    site = O.RADAR_SITES[0]
    for s in range(4):
        st = O.states_of(el[:, s], jd, fr)
        got = O.emul_observe(L, st, jd, fr, kind, 0, site)
        ref = O.observe(kind, st, jd + fr, site)
        c = O.COUNTS[kind]
        assert (got[:, c:] == 0).all()
        for q in range(c):
            d = got[:, q] - ref[:, q]
            if (kind, q) in ((O.RADAR, 1), (O.OPTICAL, 0)):
                d = np.mod(d + np.pi, TWO_PI) - np.pi
            scale = np.abs(ref[:, q]).max() if (kind, q) not in ((O.RADAR, 1), (O.RADAR, 2), (O.OPTICAL, 0),
                                                                 (O.OPTICAL, 1)) else 1.0
            # the numpy GMST (one fp64 polynomial on jd + fr) and the library's uncontracted one differ by rounding
            assert np.abs(d).max() <= 1e-11 * scale, (kind, q, np.abs(d).max())


def test_range_rate_and_earth_fixed_velocity_are_derivatives(L):
    """range-rate = d(range)/dt and the Earth-fixed velocity = d(r_ecef)/dt, by central differences over SGP4 positions.
    SGP4's own velocity is not the derivative of its position (they differ by up to ~2e-4 km/s), so the states carry
    the central difference of the positions as their velocity: the kinds are then checked, not SGP4."""
    el = _leo(3)
    jd, fr = _grid(1.0, 7.0)
    h = 0.05 / 86400.0
    site = O.RADAR_SITES[1]
    # the step as the propagation sees it: jd + fr rounds to 4.7e-10 day (40 us), so 2 h is taken from the sums
    dt = ((jd + (fr + h)) - (jd + (fr - h)))[:, None] * 86400.0
    for s in range(3):
        pos = lambda f: O.states_of(el[:, s], jd, f)[:, :3]   # noqa: E731
        p2, p1, p0, m1, m2 = pos(fr + 2 * h), pos(fr + h), pos(fr), pos(fr - h), pos(fr - 2 * h)
        state = lambda c, p, m: np.concatenate([c, (p - m) / dt], axis=1)   # noqa: E731
        rad = O.emul_observe(L, state(p0, p1, m1), jd, fr, O.RADAR, 0, site)
        rp = O.emul_observe(L, state(p1, p2, p0), jd, fr + h, O.RADAR, 0, site)
        rm = O.emul_observe(L, state(m1, p0, m2), jd, fr - h, O.RADAR, 0, site)
        ecef = O.emul_observe(L, state(p0, p1, m1), jd, fr, O.ECEF, 0, site)
        ep = O.emul_observe(L, state(p1, p2, p0), jd, fr + h, O.ECEF, 0, site)
        em = O.emul_observe(L, state(m1, p0, m2), jd, fr - h, O.ECEF, 0, site)
        # O(h^2) truncation (~2e-7 km/s at 0.1 s) and 1e-9 km of position rounding over the 0.1 s step
        dr = (rp[:, 0] - rm[:, 0]) / dt[:, 0]
        assert np.abs(dr - rad[:, 3]).max() < 1e-6, np.abs(dr - rad[:, 3]).max()
        dp = (ep[:, :3] - em[:, :3]) / dt
        assert np.abs(dp - ecef[:, 3:]).max() < 1e-6, np.abs(dp - ecef[:, 3:]).max()
        # leaving omega x r out (the ECEF output mode's velocity) would miss by |omega x r| ~ 0.5 km/s
        v_rot = np.einsum("nij,nj->ni", O.rot(O.gmst(jd + fr)), p1 - m1)
        assert np.abs(v_rot - dp).max() > 0.1


def _sums(L, el, jd, fr, kind, value, sigma, station, stations):
    words, nres = np.zeros(4 + 28 + 7), np.zeros(1, dtype=np.uint32)
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (el, jd, fr, value, sigma)]
    kd = np.ascontiguousarray(kind, dtype=np.uint8)
    sta = np.ascontiguousarray(station, dtype=np.uint32)
    st = np.ascontiguousarray(stations, dtype=np.float64).reshape(-1, 3)
    rc = L.emul_obs_sums(O._p(a[0]), 1, C.c_uint32(len(a[1])), O._p(a[1]), O._p(a[2]), O._p(a[3]), O._p(a[4]),
                         O._p(sta), O._p(kd), O._p(st), O._p(words), O._p(nres))
    assert rc == 0
    return words, int(nres[0])


def _radar_batch(el, days=1.0):
    jd, fr = _grid(days, 1.0)
    return O.tracks(el, O.RADAR, O.RADAR_SITES[:3], jd, fr)


def test_unused_components_leave_the_sums_unchanged(L):
    el = _leo(1)[:, 0]
    guess = R.perturbed(el[:, None], seed=2)[:, 0]
    jd, fr, kd, val, sig, sta = _radar_batch(el)
    sig[:, 3] = np.inf                                        # a radar without range-rate
    words, nres = _sums(L, guess, jd, fr, kd, val, sig, sta, O.RADAR_SITES[:3])
    assert nres == 3 * len(jd) and words[0] > 0
    # garbage in the unused range-rate and past the kind's count, and an extra observation with every sigma = inf
    val2 = val.copy()
    val2[:, 3] = np.nan
    val2[:, 4:] = 1e300
    sig2 = sig.copy()
    sig2[:, 4:] = -1.0                                        # past the kind's count: never read
    extra = lambda a, v: np.concatenate([a, v])               # noqa: E731
    w2, n2 = _sums(L, guess, extra(jd, jd[:1]), extra(fr, fr[:1]), extra(kd, kd[:1]),
                   extra(val2, np.full((1, 6), 7.0)), extra(sig2, np.full((1, 6), np.inf)), extra(sta, sta[:1]),
                   O.RADAR_SITES[:3])
    assert n2 == nres and w2.tobytes() == words.tobytes()
    # a position-only GPS fix: sigma = inf on the velocity counts 3 residuals
    _, n3 = _sums(L, guess, jd[:5], fr[:5], np.full(5, O.ECEF, np.uint8), np.ones((5, 6)),
                  np.array([[1e-3] * 3 + [np.inf] * 3] * 5), np.zeros(5), np.zeros((0, 3)))
    assert n3 == 15


def test_angle_wraps_at_zero_and_two_pi(L):
    """Observed azimuth / right ascension given on the far side of 0 / 2 pi gives the same cost"""
    el = _leo(1)[:, 0]
    guess = R.perturbed(el[:, None], seed=2)[:, 0]
    jd, fr, kd, val, sig, sta = _radar_batch(el)
    words, _ = _sums(L, guess, jd, fr, kd, val, sig, sta, O.RADAR_SITES[:3])
    for shift in (TWO_PI, -TWO_PI):
        v = val.copy()
        v[:, 1] += shift
        w, _ = _sums(L, guess, jd, fr, kd, v, sig, sta, O.RADAR_SITES[:3])
        assert abs(w[0] - words[0]) <= 1e-9 * words[0]
    # azimuths straddling north: an observation at 2 pi - 1e-7 against a model at +1e-7 is a 2e-7 rad residual
    el_st = O.states_of(el, jd[:1], fr[:1])
    site = O.RADAR_SITES[0]
    h = O.emul_observe(L, el_st, jd[:1], fr[:1], O.RADAR, 0, site)[0]
    for obs_az in (h[1] + 1e-7, h[1] + 1e-7 - TWO_PI, h[1] + 1e-7 + TWO_PI):
        v = h.copy()
        v[1] = obs_az
        s = np.array([[np.inf, 1e-7, np.inf, np.inf, np.inf, np.inf]])
        w, n = _sums(L, el, jd[:1], fr[:1], [O.RADAR], v[None], s, [0], site)
        assert n == 1 and abs(np.sqrt(w[0]) - abs(np.cos(h[2]))) < 1e-4


def _accumulate(L, kind, states, inv, jdf, value, sigma, llh):
    words = np.zeros(4 + 28 + 7)
    f = np.ascontiguousarray(states, dtype=np.float64)
    iv = np.ascontiguousarray(inv, dtype=np.float64)
    v, s, st = (np.ascontiguousarray(x, dtype=np.float64) for x in (value, sigma, llh))
    L.emul_obs_accumulate(kind, O._p(f), len(f) - 1, O._p(iv), C.c_double(jdf), O._p(v), O._p(s), O._p(st),
                          O._p(words))
    return words


def test_wraps_where_the_model_crosses_north_and_zero_ra(L):
    """An observation whose nominal model lies just east of north (azimuth +d) while the stepped set lies just west of
    it (2 pi - d), and the same for right ascension at 0 / 2 pi: the Jacobian column is the wrapped difference -2 d,
    not 2 pi - 2 d, and an observed angle on the far side of the cut gives the wrapped residual."""
    jdf = 2460437.3
    llh = np.array([42.6, -71.5, 0.12])
    e, n, u = O.enu_basis(llh)
    rs = O.station_ecef(llh)
    R_ = O.rot(O.gmst(jdf))
    d, step = 1e-9, 1e-8
    inv = np.array([0.0, 1.0 / step])
    el_ang = 0.4
    cases = []
    # radar: azimuth +d and -d at the same range and elevation
    for az in (d, -d):
        rho = 1500.0 * (np.cos(el_ang) * (np.sin(az) * e + np.cos(az) * n) + np.sin(el_ang) * u)
        cases.append(np.concatenate([R_.T @ (rs + rho), np.zeros(3)]))
    radar = np.array(cases)
    # optical: right ascension +d and -d in TEME from the station
    st_teme = R_.T @ rs
    optical = np.array([np.concatenate([st_teme + 36000.0 * np.array([np.cos(el_ang) * np.cos(a),
                                                                    np.cos(el_ang) * np.sin(a), np.sin(el_ang)]),
                                        np.zeros(3)]) for a in (d, -d)])
    for kind, states, q in ((O.RADAR, radar, 1), (O.OPTICAL, optical, 0)):
        h = O.emul_observe(L, states, jdf, 0.0, kind, 0, llh)
        assert h[0, q] < 1e-8 and h[1, q] > TWO_PI - 1e-8          # the two sets straddle the cut
        sig_q = 1e-6
        sigma = np.full(6, np.inf)
        sigma[q] = sig_q
        obs = h[0].copy()
        obs[q] = TWO_PI - 1e-7                                       # observed just west of the cut
        words = _accumulate(L, kind, states, inv, jdf, obs, sigma, llh)
        w = np.cos(obs[q + 1]) / sig_q
        r = (-1e-7 - h[0, q]) * w                                   # wrapped residual
        jcol = -2 * d * w / step                                     # wrapped Jacobian entry
        assert abs(words[0] - r * r) <= 1e-6 * r * r, (kind, words[0], r * r)
        assert abs(words[4] - jcol * jcol) <= 1e-6 * jcol * jcol, (kind, words[4], jcol * jcol)
        assert abs(words[4 + 28] - jcol * r) <= 1e-6 * abs(jcol * r), (kind, words[4 + 28], jcol * r)


# ---- round trips -------------------------------------------------------------------------------------------------
def _arc_error(truth, fitted, jd, fr):
    return max(np.abs(O.states_of(truth[:, s], jd, fr)[:, :3] - O.states_of(fitted[:, s], jd, fr)[:, :3]).max()
               for s in range(truth.shape[1]))


def _at_floor(wrms, sigma_km):
    """noise-free tracks: the weighted residual left is the two SGP4s' rounding (~1e-8 km), not model error"""
    return (wrms * sigma_km < 5e-8).all()


def _fit(L, el, per, stations, **kw):
    jd, fr, kd, val, sig, sta, off = O.concat(per)
    return O.emul_fit(L, el, jd, fr, kd, val, sig, sta, off, stations, **kw)


def _config2_leo():
    from astroz_b200 import synth

    el = synth.elements_from_tles(synth.near_earth_catalog(600))
    a = (398600.8 / (el[1] * 2 * np.pi / 86400.0) ** 2) ** (1.0 / 3.0)
    # the 2 % eccentric shells and a few ordinary ones.  (The low-perigee high-drag sets need more than 25 steps back
    # from a doubled B*, as in the TEME fit.)
    pick = np.unique(np.concatenate([np.flatnonzero((el[2] > 0.02) & (a * (1 - el[2]) - 6378.135 > 300.0))[:3],
                                     [0, 1, 2]]))
    return el[:, pick]


def test_leo_from_radar_at_three_stations_over_two_days(L):
    el = _config2_leo()
    jd, fr = _grid(2.0, 1.0)
    per = [O.tracks(el[:, s], O.RADAR, O.RADAR_SITES[:3], jd, fr) for s in range(el.shape[1])]
    f, wrms, nres, cov, it, st = _fit(L, R.perturbed(el, seed=1), per, O.RADAR_SITES[:3])
    assert (st == R.CONVERGED).all(), (st, it)
    err = _arc_error(el, f, jd, fr)
    assert err < 1e-6, err
    assert _at_floor(wrms, 1e-5)                 # the range-rate's sigma, the tightest
    assert (nres == [4 * len(p[0]) for p in per]).all()
    assert (cov[:, 0] > 0).all()


def test_leo_from_ecef_gps_states(L):
    el = _config2_leo()
    jd, fr = _grid(1.0, 10.0)
    per = [O.tracks(el[:, s], O.ECEF, None, jd, fr) for s in range(el.shape[1])]
    f, wrms, nres, cov, it, st = _fit(L, R.perturbed(el, seed=1), per, np.zeros((0, 3)))
    assert (st == R.CONVERGED).all(), (st, it)
    err = _arc_error(el, f, jd, fr)
    assert err < 1e-6, err
    assert _at_floor(wrms, 1e-6)


def _optical_nights(el, nights, step_min=5.0):
    """two stations 25 deg either side of the set's sub-satellite longitude at epoch; 10-hour nights a day apart"""
    t = np.concatenate([np.arange(0.0, 600.0, step_min) + 1440.0 * k for k in range(nights)]) / 1440.0
    jd, fr = np.full(len(t), np.floor(el[0]) + 0.5), t + 0.3
    r, _ = O.ecef_state(O.states_of(el, jd[:1], fr[:1]), jd[0] + fr[0])
    lon = np.degrees(np.arctan2(r[0, 1], r[0, 0]))
    return jd, fr, np.array([[30.0, lon - 25.0, 2.0], [-25.0, lon + 25.0, 2.4]])


def test_geo_and_gps_from_optical_angles_over_two_nights(L):
    from tests.test_fit_deep_cpu import deep_cases, guesses

    cases, held = deep_cases()
    pick = [0, 1, 2, 9, 10, 11]                     # GEO, GPS-like
    el = cases[:, pick]
    guess = guesses(el, held[pick])
    per, stations = [], []
    for s in range(el.shape[1]):
        jd, fr, sites = _optical_nights(el[:, s], 2)
        t = O.tracks(el[:, s], O.OPTICAL, sites, jd, fr)
        per.append(t[:5] + (t[5] + 2 * s,))
        stations.append(sites)
    f, wrms, nres, cov, it, st = _fit(L, guess, per, np.concatenate(stations), fit_bstar=False)
    assert (st == R.CONVERGED).all(), (st, it)
    errs = [_arc_error(el[:, [s]], f[:, [s]], p[0], p[1]) for s, p in enumerate(per)]
    assert max(errs) < 1e-4, errs
    assert _at_floor(wrms * 4.8e-6 * 36000.0, 1.0)  # 1" at GEO range: ~0.17 km of sky per unit of wrms
    assert (f[7] == guess[7]).all() and (cov[:, 6] == 0).all() and (cov[:, 27] == 0).all()


def test_molniya_from_radar(L):
    from tests.test_fit_deep_cpu import deep_cases, guesses

    cases, held = deep_cases()
    el = cases[:, [13, 14]]
    jd, fr = _grid(2.0, 1.0)
    per = [O.tracks(el[:, s], O.RADAR, O.RADAR_SITES[:3], jd, fr) for s in range(2)]
    f, wrms, nres, cov, it, st = _fit(L, guesses(el, held[[13, 14]]), per, O.RADAR_SITES[:3])
    assert (st == R.CONVERGED).all(), (st, it)
    err = _arc_error(el, f, jd, fr)
    assert err < 1e-6, err
    assert _at_floor(wrms, 1e-5)


def test_too_few_counts_used_residuals(L):
    el = _leo(1)
    jd, fr, kd, val, sig, sta = _radar_batch(el[:, 0])
    sig[:, 1:] = np.inf                                   # range only
    k = 6                                                 # 6 ranges < 7 variables
    f, wrms, nres, cov, it, st = O.emul_fit(L, el, jd[:k], fr[:k], kd[:k], val[:k], sig[:k], sta[:k],
                                            np.array([0, k]), O.RADAR_SITES[:3])
    assert st[0] == R.TOO_FEW and nres[0] == 6 and (cov == 0).all() and wrms[0] == 0 and it[0] == 0
    f, wrms, nres, cov, it, st = O.emul_fit(L, el, jd[:k], fr[:k], kd[:k], val[:k], sig[:k], sta[:k],
                                            np.array([0, k]), O.RADAR_SITES[:3], fit_bstar=False)
    assert st[0] != R.TOO_FEW and nres[0] == 6


# ---- covariance --------------------------------------------------------------------------------------------------
def _replicas(L, el, per, stations, deep, fit_bstar, nrep=300, seed=11):
    jd, fr, kd, val, sig, sta, off = O.concat(per)
    rng = np.random.default_rng(seed)
    m = len(jd)
    used = np.isfinite(sig)
    noise = np.where(used[None], rng.standard_normal((nrep, m, 6)) * np.where(used, sig, 0.0)[None], 0.0)
    vals = val[None] + noise
    wr = 1 if kd[0] == O.RADAR else 0 if kd[0] == O.OPTICAL else -1
    if wr >= 0:   # the azimuth / RA noise is an arc on the sky: divide by cos of the elevation / declination
        vals[:, :, wr] = val[None, :, wr] + noise[:, :, wr] / np.cos(val[None, :, wr + 1])
    rep = lambda a: np.tile(a, (nrep,) + (1,) * (a.ndim - 1))   # noqa: E731
    offs = np.arange(nrep + 1, dtype=np.uint32) * m
    f, wrms, nres, cov, it, st = O.emul_fit(L, np.repeat(el[:, None], nrep, axis=1), rep(jd), rep(fr), rep(kd),
                                            vals.reshape(-1, 6), rep(sig), rep(sta), offs, stations,
                                            fit_bstar=fit_bstar, max_iter=60)
    # with noise the stopping rule (a step changes the cost by <= 1e-10 of it) takes ~20 steps: allow 60
    assert (st == R.CONVERGED).all(), np.bincount(st)
    x = np.array([O.fit_vars(f[:, r], deep) for r in range(nrep)])
    x0 = O.fit_vars(el, deep)
    for c in ((4, 5) if not deep else (5,)):
        x[:, c] = x0[c] + np.mod(x[:, c] - x0[c] + np.pi, TWO_PI) - np.pi
    return x - x0, cov, wrms


def _check_covariance(dx, cov, nvar):
    from scipy import stats

    nrep = len(dx)
    P = np.zeros((nrep, 7, 7))
    P[:, np.triu_indices(7)[0], np.triu_indices(7)[1]] = cov
    P = P + np.triu(P, 1).transpose(0, 2, 1)
    Pm = P.mean(axis=0)[:nvar, :nvar]
    emp = np.cov(dx[:, :nvar].T)
    lo, hi = stats.chi2.ppf([0.0005, 0.9995], nrep - 1) / (nrep - 1)
    ratio = np.diag(emp) / np.diag(Pm)
    assert ((ratio > lo) & (ratio < hi)).all(), (ratio, lo, hi)
    d2 = np.array([dx[r, :nvar] @ np.linalg.solve(P[r, :nvar, :nvar], dx[r, :nvar]) for r in range(nrep)])
    se = np.sqrt(2.0 * nvar / nrep)
    assert abs(d2.mean() - nvar) < 3 * se, (d2.mean(), nvar, se)
    return ratio, d2.mean()


def test_formal_covariance_matches_replicas_leo_radar(L):
    el = _leo(1)[:, 0]
    jd, fr = _grid(2.0, 2.0)
    per = [O.tracks(el, O.RADAR, O.RADAR_SITES[:3], jd, fr)]
    dx, cov, wrms = _replicas(L, el, per, O.RADAR_SITES[:3], deep=False, fit_bstar=True)
    _check_covariance(dx, cov, 7)
    assert abs(np.mean(wrms) - 1.0) < 0.05                 # the sigmas are right: wrms ~ 1


def test_formal_covariance_matches_replicas_geo_optical(L):
    from tests.test_fit_deep_cpu import deep_cases

    cases, _ = deep_cases()
    el = cases[:, 0]
    jd, fr, sites = _optical_nights(el, 2, step_min=10.0)
    per = [O.tracks(el, O.OPTICAL, sites, jd, fr)]
    dx, cov, wrms = _replicas(L, el, per, sites, deep=True, fit_bstar=False)
    _check_covariance(dx, cov, 6)
    assert abs(np.mean(wrms) - 1.0) < 0.05


def test_element_covariance_is_the_jacobian_mapping():
    from astroz_b200.fit import FitResult, element_jacobian

    from tests.test_fit_deep_cpu import deep_cases

    cases, _ = deep_cases()
    for el, deep in ((_leo(3)[:, 2], False), (cases[:, 0], True), (cases[:, 13], True)):
        x0 = O.fit_vars(el, deep)

        def elements(x):
            d = 180.0 / np.pi
            e = np.hypot(x[1], x[2])
            peri = np.arctan2(x[2], x[1])
            if not deep:
                return np.array([x[0], e, x[3], x[4], peri, x[5] - peri, x[6]])
            node = np.arctan2(x[4], x[3])
            return np.array([x[0], e, 2 * np.arctan(np.hypot(x[3], x[4])), node, peri - node, x[5] - peri, x[6]])

        Jfd = np.zeros((7, 7))
        for j in range(7):
            h = 1e-7 * max(abs(x0[j]), 1e-3)
            xp, xm = x0.copy(), x0.copy()
            xp[j] += h
            xm[j] -= h
            Jfd[:, j] = (elements(xp) - elements(xm)) / (2 * h)
        Ja = element_jacobian(el, deep)
        assert np.abs(Ja - Jfd).max() <= 1e-6 * max(1.0, np.abs(Jfd).max()), (Ja - Jfd)
        rng = np.random.default_rng(1)
        A = rng.standard_normal((7, 7))
        P = A @ A.T * 1e-10
        res = FitResult(el[:, None], np.zeros(1), np.zeros(1), np.zeros(1, np.uint32), np.zeros(1, np.uint8),
                        covariance=P[np.triu_indices(7)][None], deep_space=np.array([deep]))
        assert np.allclose(res.covariance_matrix(0), P, rtol=0, atol=1e-25)
        E = res.element_covariance(0)
        assert np.abs(E - Jfd @ P @ Jfd.T).max() <= 1e-6 * np.abs(E).max()


# ---- C ABI refusals ----------------------------------------------------------------------------------------------
def _abi(n=2, m=4):
    el = np.tile(np.array([[2460437.0], [15.5], [1e-3], [53.0], [10.0], [20.0], [30.0], [1e-4]]), (1, n))
    a = dict(el=el, off=np.array([0, 2, m], dtype=np.uint32)[: n + 1], jd=np.full(m, 2460437.0), fr=np.zeros(m),
             value=np.tile([1000.0, 1.0, 0.5, 0.1, 0.0, 0.0], (m, 1)), sigma=np.tile([0.01, 1e-4, 1e-4, 1e-5,
                                                                                      np.inf, np.inf], (m, 1)),
             station=np.zeros(m, dtype=np.uint32), kind=np.full(m, O.RADAR, dtype=np.uint8),
             stations=np.array([[42.6, -71.5, 0.1]]))
    out = [np.full((8, n), -7.0), np.full(n, -7.0), np.full(n, 7, dtype=np.uint32), np.full((n, 28), -7.0),
           np.full(n, 7, dtype=np.uint32), np.full(n, 9, dtype=np.uint8), np.full(n, 9, dtype=np.uint8)]
    return a, out


def _abi_call(a, out, *, n=2, m=4, k=1, grav=1, max_iter=25, device=0, mixed=False):
    from astroz_b200 import _lib

    p = lambda x: None if x is None else C.c_void_p(x.ctypes.data)  # noqa: E731
    f = _lib.lib().astroz_cuda_fit_observations_mixed if mixed else _lib.lib().astroz_cuda_fit_observations
    return f(p(a["el"]), n, grav, p(a["off"]), p(a["jd"]), p(a["fr"]), p(a["value"]), p(a["sigma"]),
             p(a["station"]), p(a["kind"]), m, p(a["stations"]), k, 1, max_iter, device, *[p(o) for o in out])


def _untouched(out):
    return all((o == v).all() for o, v in zip(out, (-7, -7, 7, -7, 7, 9, 9)))


def test_cabi_value_errors_write_nothing():
    pytest.importorskip("astroz_b200")
    edits = {
        "device": (lambda a: None, dict(device=-1)),
        "max_iter": (lambda a: None, dict(max_iter=0)),
        "grav": (lambda a: None, dict(grav=7)),
        "unknown kind": (lambda a: a["kind"].__setitem__(1, 4), {}),
        "station index": (lambda a: a["station"].__setitem__(2, 1), {}),
        "station count": (lambda a: None, dict(k=0)),
        "sigma zero": (lambda a: a["sigma"].__setitem__((0, 0), 0.0), {}),
        "sigma negative": (lambda a: a["sigma"].__setitem__((3, 2), -1e-4), {}),
        "sigma nan": (lambda a: a["sigma"].__setitem__((1, 3), np.nan), {}),
        "value nan": (lambda a: a["value"].__setitem__((2, 0), np.nan), {}),
        "value inf": (lambda a: a["value"].__setitem__((2, 3), np.inf), {}),
        "elevation of a used azimuth": (lambda a: (a["sigma"].__setitem__((0, 2), np.inf),
                                                   a["value"].__setitem__((0, 2), np.nan)), {}),
        "latitude": (lambda a: a["stations"].__setitem__((0, 0), 90.5), {}),
        "station nan": (lambda a: a["stations"].__setitem__((0, 2), np.nan), {}),
        "offsets total": (lambda a: None, dict(m=3)),
        "offsets decrease": (lambda a: (a["off"].__setitem__(1, 3), a["off"].__setitem__(2, 2)), dict(m=2)),
        "element nan": (lambda a: a["el"].__setitem__((3, 1), np.nan), {}),
        "time nan": (lambda a: a["jd"].__setitem__(3, np.nan), {}),
    }
    for name, (edit, kw) in edits.items():
        for mixed in (False, True):
            a, out = _abi()
            edit(a)
            assert _abi_call(a, out, mixed=mixed, **kw) == -20, name
            assert _untouched(out), name


def test_cabi_accepts_unused_garbage_and_empty_batches():
    from astroz_b200 import _lib

    a, out = _abi()
    a["value"][:, 3] = np.nan
    a["sigma"][:, 3] = np.inf            # range-rate not used: its value is not read
    a["sigma"][:, 4:] = -1.0             # past the radar's four components: ignored
    rc = _abi_call(a, out)
    assert rc == (0 if _lib.device_count() > 0 else -201)
    a, out = _abi()
    assert _abi_call(a, out, n=0) == 0 and _untouched(out)


def test_python_refuses_kinds_and_stations_that_do_not_fit_their_integer_type():
    from astroz_b200.fit import fit_observations, observe

    el = _abi()[0]["el"]
    for kind, station in (([256, 2], [0, 0]), ([-1, 2], [0, 0]), ([2, 2], [0, 2 ** 32]), ([2, 2], [-1, 0])):
        with pytest.raises(ValueError):
            fit_observations(el[:, :1], [0, 0], [2460437.0] * 2, [0.0] * 2, kind, np.ones((2, 4)),
                             np.ones((2, 4)), station, [[0.0, 0.0, 0.0]])
    with pytest.raises(ValueError):
        observe(np.ones((1, 6)), 2460437.0, 0.0, 258, 0, [[0.0, 0.0, 0.0]])


def test_element_covariance_of_a_teme_fit_result_is_refused():
    from astroz_b200.fit import FitResult

    res = FitResult(_leo(1), np.zeros(1), np.zeros(1), np.zeros(1, np.uint32), np.zeros(1, np.uint8))
    with pytest.raises(ValueError):
        res.element_covariance(0)


def test_cabi_observe_refusals():
    from astroz_b200 import _lib

    p = lambda x: None if x is None else C.c_void_p(x.ctypes.data)  # noqa: E731
    m = 3
    st, jd, fr = np.ones((m, 6)) * 7000.0, np.full(m, 2460437.0), np.zeros(m)
    for kind, sta, stations, dev in (([0, 4, 1], [0, 0, 0], [[0.0, 0.0, 0.0]], 0),
                                     ([2, 2, 3], [0, 1, 0], [[0.0, 0.0, 0.0]], 0),
                                     ([2, 2, 3], [0, 0, 0], [[-91.0, 0.0, 0.0]], 0),
                                     ([0, 0, 0], [0, 0, 0], [[0.0, 0.0, 0.0]], -1)):
        out = np.full((m, 6), -3.0)
        kd, sa, ss = np.array(kind, np.uint8), np.array(sta, np.uint32), np.array(stations, dtype=np.float64)
        rc = _lib.lib().astroz_cuda_observe(p(st), p(jd), p(fr), p(kd), p(sa), m, p(ss), len(ss), dev, p(out))
        assert rc == -20 and (out == -3.0).all(), (kind, sta, stations, dev)


# ---- the host build against the independent C restatement (tests/fit_oracle/fit_oracle_obs.c) -------------------------
def _noisy(per, seed):
    rng = np.random.default_rng(seed)
    out = []
    for jd, fr, kd, val, sig, sta in per:
        used = np.isfinite(sig)
        noise = np.where(used, rng.standard_normal(val.shape) * np.where(used, sig, 0.0), 0.0)
        v = val + noise
        wr = {O.RADAR: 1, O.OPTICAL: 0}.get(int(kd[0]), -1) if len(kd) else -1
        if wr >= 0:
            v[:, wr] = val[:, wr] + noise[:, wr] / np.cos(val[:, wr + 1])
        out.append((jd, fr, kd, v, sig, sta))
    return out


def _restatement_cases():
    from tests.test_fit_deep_cpu import deep_cases, guesses

    el = _config2_leo()
    jd, fr = _grid(2.0, 1.0)
    jd2, fr2 = _grid(1.0, 10.0)
    out = [("LEO radar", el, R.perturbed(el, seed=1), False, True, O.RADAR_SITES[:3],
            [O.tracks(el[:, s], O.RADAR, O.RADAR_SITES[:3], jd, fr) for s in range(el.shape[1])]),
           ("LEO ECEF", el, R.perturbed(el, seed=1), False, True, np.zeros((0, 3)),
            [O.tracks(el[:, s], O.ECEF, None, jd2, fr2) for s in range(el.shape[1])])]
    dc, held = deep_cases()
    pick = [0, 1, 9, 10]
    e3 = dc[:, pick]
    per, sites = [], []
    for s in range(len(pick)):
        j, f, st = _optical_nights(e3[:, s], 2)
        t = O.tracks(e3[:, s], O.OPTICAL, st, j, f)
        per.append(t[:5] + (t[5] + 2 * s,))
        sites.append(st)
    out.append(("GEO / GPS optical", e3, guesses(e3, held[pick]), True, False, np.concatenate(sites), per))
    e4 = dc[:, [13, 14]]
    out.append(("Molniya radar", e4, guesses(e4, held[[13, 14]]), True, True, O.RADAR_SITES[:3],
                [O.tracks(e4[:, s], O.RADAR, O.RADAR_SITES[:3], jd, fr) for s in range(2)]))
    return out


def _compare(E, Rr, deep):
    n = E[0].shape[1]
    dx = np.array([O.fit_vars(E[0][:, s], deep) - O.fit_vars(Rr[0][:, s], deep) for s in range(n)])
    dx[:, 4:6] = np.mod(dx[:, 4:6] + np.pi, TWO_PI) - np.pi
    iu = np.triu_indices(7)
    diag = Rr[3][:, np.cumsum([0, 7, 6, 5, 4, 3, 2])]
    scale = np.sqrt(np.abs(diag[:, iu[0]] * diag[:, iu[1]]))
    dcov = np.abs(E[3] - Rr[3]) / np.where(scale > 0, scale, 1.0)
    return np.abs(dx[:, 0] / Rr[0][1]).max(), np.abs(dx[:, 1:6]).max(), dcov.max()


def test_host_build_matches_the_restatement_noise_free(L):
    """Noise-free tracks: the same steps and statuses; n within 1e-9 relative and the other variables within 1e-9
    (measured: 4e-14 and 7e-12).  wRMS is then what separates the library's SGP4 from the oracle's, a few 1e-9 km over
    the sigmas, so it is compared in absolute (measured 1.2e-6 for the 1e-6 km/s velocity sigmas of ECEF states).  The
    covariance words agree to 1e-2 of their scale (measured 4e-3): J is a forward difference over 1e-8 steps, and the
    two SGP4s' rounding of the states reaches it at ~1e-4."""
    for name, el, guess, deep, fb, sites, per in _restatement_cases():
        a = O.concat(per)
        E = O.emul_fit(L, guess, *a[:6], a[6], sites, fit_bstar=fb)
        Rr = O.restated_fit(guess, *a[:6], a[6], sites, fit_bstar=fb)
        assert (E[5] == 0).all() and (E[5] == Rr[5]).all() and (E[4] == Rr[4]).all(), (name, E[4], Rr[4])
        assert (E[2] == Rr[2]).all(), name
        dn, dx, dcov = _compare(E, Rr, deep)
        print(f"{name}: n {dn:.1e} relative, variables {dx:.1e}, wRMS {np.abs(E[1] - Rr[1]).max():.1e} absolute, "
              f"covariance {dcov:.1e}")
        assert dn <= 1e-9 and dx <= 1e-9, (name, dn, dx)
        assert np.abs(E[1] - Rr[1]).max() <= 5e-6, name
        assert dcov <= 1e-2, (name, dcov)


def test_host_build_matches_the_restatement_with_noise(L):
    """Noisy tracks at the stated sigmas (wRMS ~ 1): the same statuses.  The fits take 5-30 steps to the stopping rule,
    whose 1e-10 relative cost test the two SGP4s' differences cross at different steps, so the step counts differ and
    the stopping points lie within the flat bottom of the cost.  Radar and optical: variables within 1e-9, wRMS within
    5e-9 relative (measured 8e-10, 3e-9).  ECEF states, whose 1e-6 km/s velocity sigmas magnify the SGP4 differences:
    variables within 2e-8 and wRMS within 1e-7 relative (measured 7e-9, 3e-8)."""
    for name, el, guess, deep, fb, sites, per in _restatement_cases():
        a = O.concat(_noisy(per, 3))
        E = O.emul_fit(L, guess, *a[:6], a[6], sites, fit_bstar=fb, max_iter=60)
        Rr = O.restated_fit(guess, *a[:6], a[6], sites, fit_bstar=fb, max_iter=60)
        assert (E[5] == 0).all() and (E[5] == Rr[5]).all(), name
        dn, dx, dcov = _compare(E, Rr, deep)
        dw = np.abs(E[1] / Rr[1] - 1.0).max()
        print(f"{name}: n {dn:.1e} relative, variables {dx:.1e}, wRMS {dw:.1e} relative, covariance {dcov:.1e}")
        ecef = name == "LEO ECEF"
        assert dn <= (2e-8 if ecef else 1e-9) and dx <= (2e-8 if ecef else 1e-9), (name, dn, dx)
        assert dw <= (1e-7 if ecef else 5e-9), (name, dw)
        assert dcov <= 1e-2, (name, dcov)
