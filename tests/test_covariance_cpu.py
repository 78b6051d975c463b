"""K10 state covariance (az_covariance.cuh, az_covariance.cu) on the CPU.

The host build of the device source (tests/host_emul/emul_covariance.cu) against the independent C restatement on the
oracle's SGP4 / SDP4 (tests/fit_oracle/covariance.c); the hat-matrix invariant that ties it to the covariance the
element fit inverted; a Monte Carlo of the fit's variables through the oracle; frames and algebra; the B*, zero-P,
model and status rules; chunk independence; the C ABI's refusals and the Python wrapper's order.  The device runs are
in tests/test_gpu_covariance.py."""
import ctypes as C

import numpy as np
import pytest

from tests import fit_oracle as R
from tests.fit_oracle import covariance as K
from tests.fit_oracle import obs as O

@pytest.fixture(scope="module")
def L():
    lib = K.emul_library()
    if lib is None:
        pytest.skip("nvcc unavailable")
    return lib


def _catalogue():
    """LEO sets and deep-space ones (GEO, Molniya, GPS-like) of the synthetic catalogues, with their model bytes"""
    from astroz_b200 import synth

    leo = synth.elements_from_tles(synth.near_earth_catalog(600))[:, :4]
    mix = synth.elements_from_tles(synth.mixed_catalog(64, n_geo=4, n_molniya=4, n_gps=4))
    deep = mix[:, 1440.0 / mix[1] > 225.0]
    geo = deep[:, np.abs(deep[1] - 1.0027) < 0.01][:, :2]
    mol = deep[:, (deep[2] > 0.6)][:, :2]
    gps = deep[:, (np.abs(deep[1] - 2.0056) < 0.01) & (deep[2] < 0.05)][:, :2]
    el = np.concatenate([leo, geo, mol, gps], axis=1)
    model = np.array([0] * leo.shape[1] + [1] * (el.shape[1] - leo.shape[1]), np.uint8)
    return el, model


def _P(n, seed=3, bstar=True):
    """PSD covariances in the fit's variables at the scale of a radar fit: n 1e-7 rev/day, e-terms 1e-6, angles 1e-5
    rad (deep: tan(i/2) terms 1e-6), B* 1e-5 / ER; random correlations"""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 28))
    d = np.array([1e-7, 1e-6, 1e-6, 1e-5, 1e-5, 1e-5, 1e-5 if bstar else 0.0])
    for s in range(n):
        A = rng.standard_normal((7, 7))
        Cm = A @ A.T / 7.0 + 0.3 * np.eye(7)
        Cm /= np.sqrt(np.outer(np.diag(Cm), np.diag(Cm)))
        out[s] = K.pack7(Cm * np.outer(d, d))
    return out


def _queries(n, days=3.0, count=61):
    """count times per satellite spread over epoch +- days"""
    sat = np.repeat(np.arange(n), count)
    offsets = np.arange(n + 1, dtype=np.uint32) * count
    return sat, offsets


def _times(el, sat, days=3.0, count=61):
    t = np.tile(np.linspace(-days, days, count), el.shape[1])
    ep = el[0][sat]
    jd = np.floor(ep + t - 0.5) + 0.5
    return jd, (ep + t) - jd


def _column_errors(jac, rjac, P, sat):
    """per query and block (position rows, velocity rows): max |dJ D| / max |J D|, D = diag(sqrt(P_jj)) -- the columns
    as the state moves of a one-sigma step in each variable.  The deep-space B* column is rounding noise in both
    builds (SDP4's drag moves a GPS orbit by ~1e-11 km over a 1e-8 step), and this scale says how little it weighs."""
    D = np.sqrt(np.stack([np.diag(K.unpack7(p)) for p in P]))[sat][:, None, :]
    out = []
    for rows in (slice(0, 3), slice(3, 6)):
        d = (np.abs(jac[:, rows] - rjac[:, rows]) * D).max(axis=(1, 2))
        out.append(d / (np.abs(rjac[:, rows]) * D).max(axis=(1, 2)))
    return max(o.max() for o in out)


# ---- 1. the host build against the restatement ----------------------------------------------------------------------
@pytest.mark.parametrize("frame", [0, 1])
def test_host_build_matches_the_restatement(L, frame):
    """LEO, GEO, Molniya and GPS-like sets over +-3 days: statuses equal; states, J columns and Sigma within the two
    SGP4 / SDP4 builds' agreement.  Measured: state 7.9e-9 km and 5.6e-12 km/s, J 4.0e-6 and Sigma 5.8e-6 of their
    scale -- far inside the ~1e-4 that the forward differences over 1e-8 steps could move between two builds."""
    el, model = _catalogue()
    n = el.shape[1]
    sat, off = _queries(n)
    jd, fr = _times(el, sat)
    P = _P(n)
    st, sig, jac, status = K.emul(L, el, P, model, off, jd, fr, frame)
    rst, rsig, rjac, rstatus = K.restated(el, P, model, off, jd, fr, frame)
    assert (status == rstatus).all() and (status == 0).all()
    dpos = np.abs(st[:, :3] - rst[:, :3]).max()
    dvel = np.abs(st[:, 3:] - rst[:, 3:]).max()
    ej = _column_errors(jac, rjac, P, sat)
    S, RS = K.unpack6(sig), K.unpack6(rsig)
    es = (np.abs(S - RS).max(axis=(1, 2)) / np.abs(RS).max(axis=(1, 2))).max()
    print(f"frame {frame}: state {dpos:.2e} km {dvel:.2e} km/s, J {ej:.2e}, Sigma {es:.2e} of scale")
    assert dpos < 1e-7 and dvel < 1e-10
    assert ej < 1e-4 and es < 1e-4


# ---- 2. the hat-matrix invariant ------------------------------------------------------------------------------------
def _teme_fit(el_true, deep, fit_bstar, seed):
    """a fit of the host build to noisy oracle TEME states over one day at 10 min: (fitted (8, 1), cov (1, 28), model,
    jd, fr, sigma)"""
    jd, fr = np.full(145, np.floor(el_true[0] - 0.5) + 0.5), np.zeros(145)
    fr = (el_true[0] - jd) + np.arange(145) / 144.0
    st = O.states_of(el_true, jd, fr)
    sig = np.array([1e-3] * 3 + [1e-6] * 3)
    rng = np.random.default_rng(seed)
    val = st + rng.standard_normal(st.shape) * sig
    m = len(jd)
    guess = R.perturbed(el_true[:, None], seed=seed)
    if not fit_bstar:
        guess[7] = el_true[7]
    Lf = O.emul_library()
    fitted, wrms, nres, cov, iters, status = O.emul_fit(
        Lf, guess, jd, fr, np.zeros(m, np.uint8), val, np.tile(sig, (m, 1)), np.zeros(m, np.uint32),
        np.array([0, m], np.uint32), np.zeros((0, 3)), fit_bstar=fit_bstar, mixed=deep)
    assert status[0] == 0 and abs(wrms[0] - 1.0) < 0.2
    return fitted, cov, np.array([int(deep)], np.uint8), jd, fr, sig


@pytest.mark.parametrize("case,fit_bstar", [("LEO", True), ("LEO", False), ("GEO", False)])
def test_hat_matrix_invariant(L, case, fit_bstar):
    """sum_i tr(W_i Sigma_i) over the fit's own observations = tr(N N^-1) = the number of fitted variables, when Sigma
    is propagated from the covariance the fit returned at the fit's observation times.  (A GEO fit with B* free has no
    covariance: at GEO the B* column is zero and the normal matrix is singular.)  Measured: within 2e-7 of nvar; a
    wrong step or variable map moves the sum by more than 0.05."""
    el, model = _catalogue()
    deep = case == "GEO"
    true = el[:, int(np.flatnonzero(model == 1)[0])] if deep else el[:, 0]
    fitted, cov, md, jd, fr, sig = _teme_fit(true, deep, fit_bstar, seed=5)
    _, S, _, status = K.emul(L, fitted, cov, md, np.array([0, len(jd)], np.uint32), jd, fr, 0)
    assert (status == 0).all()
    diag = K.unpack6(S)[:, range(6), range(6)]
    total = float((diag / sig ** 2).sum())
    nvar = 7 if fit_bstar else 6
    print(f"{case} fit_bstar={fit_bstar}: sum tr(W Sigma) = {total:.9f} (nvar {nvar})")
    assert abs(total - nvar) < 1e-5


# ---- 3. linear against Monte Carlo ----------------------------------------------------------------------------------
def _obs_fit(case):
    """a LEO radar fit (two days, three stations) or a GEO optical fit (three nights), noisy, by the host build"""
    el, model = _catalogue()
    rng = np.random.default_rng(11)
    if case == "LEO":
        true = el[:, 0]
        jd0 = np.floor(true[0] - 0.5) + 0.5
        fr = (true[0] - jd0) + np.arange(2 * 1440) / 1440.0
        trk = O.tracks(true, O.RADAR, O.RADAR_SITES[:3], np.full(len(fr), jd0), fr)
    else:
        true = el[:, int(np.flatnonzero(model == 1)[0])]
        jd0 = np.floor(true[0] - 0.5) + 0.5
        fr = (true[0] - jd0) + np.arange(3 * 144) / 144.0
        trk = O.tracks(true, O.OPTICAL, O.RADAR_SITES[:3], np.full(len(fr), jd0), fr)
    jd, fr, kd, val, sigma, sta = trk
    used = np.isfinite(sigma)
    noise = np.where(used, rng.standard_normal(val.shape) * np.where(used, sigma, 0.0), 0.0)
    v = val + noise
    wr = 1 if case == "LEO" else 0
    v[:, wr] = val[:, wr] + noise[:, wr] / np.cos(val[:, wr + 1])
    deep = case == "GEO"
    fitted, wrms, nres, cov, iters, status = O.emul_fit(
        O.emul_library(), R.perturbed(true[:, None], seed=2), jd, fr, kd, v, sigma, sta,
        np.array([0, len(jd)], np.uint32), O.RADAR_SITES[:3], fit_bstar=not deep, mixed=deep)
    assert status[0] == 0
    return fitted[:, 0], cov[0], deep


def _monte_carlo(L, fitted, cov, deep, t_days, draws, seed):
    """(K10's RTN Sigma (6, 6), the sample RTN covariance of `draws` oracle propagations of N(x, P))"""
    jd = np.array([np.floor(fitted[0] + t_days - 0.5) + 0.5])
    fr = (fitted[0] + t_days) - jd
    md = np.array([int(deep)], np.uint8)
    st, S, _, status = K.emul(L, fitted[:, None], cov[None], md, np.array([0, 1], np.uint32), jd, fr, 1)
    assert status[0] == 0
    P = K.unpack7(cov)
    x = O.fit_vars(fitted, deep)
    w, V = np.linalg.eigh(P)
    rng = np.random.default_rng(seed)
    xs = x + (rng.standard_normal((draws, 7)) * np.sqrt(np.clip(w, 0, None))) @ V.T
    els = K.elements_of(xs, fitted[0], deep)
    off = np.arange(draws + 1, dtype=np.uint32)
    states, _, _, stat = K.restated(els, np.zeros((draws, 28)), np.full(draws, int(deep), np.uint8), off,
                                    np.full(draws, jd[0]), np.full(draws, fr[0]), 0)
    assert (stat == 0).all()
    Rm = K.rtn(st)[0]
    d = states - states.mean(axis=0)
    d = np.concatenate([d[:, :3] @ Rm.T, d[:, 3:] @ Rm.T], axis=1)
    return K.unpack6(S[0]), d.T @ d / (draws - 1)


@pytest.mark.parametrize("case", ["LEO", "GEO"])
def test_linear_covariance_matches_monte_carlo_at_one_day(L, case):
    """20,000 draws of the fit's variables from N(x, P), mapped to element sets by a numpy statement of elements_of and
    propagated by the oracle: at +1 day the RTN variances lie within 5 sigma of their chi-square sampling spread."""
    fitted, cov, deep = _obs_fit(case)
    draws = 20000
    S, Smc = _monte_carlo(L, fitted, cov, deep, 1.0, draws, seed=7)
    ratio = np.diag(Smc) / np.diag(S)
    bound = 5.0 * np.sqrt(2.0 / (draws - 1))
    print(f"{case} +1 day: sample / linear RTN variances {np.array2string(ratio, precision=4)}, bound 1 +- {bound:.3f}")
    assert np.abs(ratio - 1.0).max() < bound


def test_linear_model_limit_at_seven_days_leo(L):
    """Printed, not asserted: how far the along-track variance of the linear model departs from the sample one a week
    out, where the along-track error is curved in the variables (recorded in DESIGN §3, K10)."""
    fitted, cov, deep = _obs_fit("LEO")
    S, Smc = _monte_carlo(L, fitted, cov, deep, 7.0, 20000, seed=8)
    ratio = np.diag(Smc) / np.diag(S)
    print(f"LEO +7 days: sample / linear RTN variances {np.array2string(ratio, precision=4)}")


# ---- 4. frames and algebra ------------------------------------------------------------------------------------------
def test_frames_and_algebra(L):
    el, model = _catalogue()
    n = el.shape[1]
    sat, off = _queries(n)
    jd, fr = _times(el, sat)
    P = _P(n)
    st, sT, jT, _ = K.emul(L, el, P, model, off, jd, fr, 0)
    st2, sR, jR, _ = K.emul(L, el, P, model, off, jd, fr, 1)
    assert st.tobytes() == st2.tobytes()
    ST, SR = K.unpack6(sT), K.unpack6(sR)
    Rm = K.rtn(st)
    R6 = np.zeros((len(st), 6, 6))
    R6[:, :3, :3] = R6[:, 3:, 3:] = Rm
    scale = np.abs(ST).max(axis=(1, 2))
    rot = np.einsum("nij,njk,nlk->nil", R6, ST, R6)
    assert (np.abs(rot - SR).max(axis=(1, 2)) / scale).max() < 1e-12
    tr = np.trace(ST, axis1=1, axis2=2)
    assert (np.abs(np.trace(SR, axis1=1, axis2=2) - tr) / tr).max() < 1e-12
    for S in (ST, SR):
        ev = np.linalg.eigvalsh(S)
        assert (ev.min(axis=1) >= -1e-12 * np.abs(ev).max(axis=1)).all()
    for J, S in ((jT, ST), (jR, SR)):
        JPJ = np.einsum("nij,njk,nlk->nil", J, np.stack([K.unpack7(p) for p in P])[sat], J)
        assert (np.abs(JPJ - S).max(axis=(1, 2)) / scale).max() < 1e-12
    assert (np.abs(np.einsum("nij,njk->nik", R6, jT) - jR).max(axis=(1, 2)) /
            np.abs(jT).max(axis=(1, 2))).max() < 1e-12


# ---- 5. rules -------------------------------------------------------------------------------------------------------
def test_a_zero_bstar_row_is_the_six_variable_case(L):
    el, model = _catalogue()
    n = el.shape[1]
    sat, off = _queries(n, count=21)
    jd, fr = _times(el, sat, count=21)
    P = _P(n)
    P6 = P.copy()
    for s in range(n):
        M = K.unpack7(P6[s])
        M[6, :] = M[:, 6] = 0.0
        P6[s] = K.pack7(M)
    for frame in (0, 1):
        _, _, j7, _ = K.emul(L, el, P, model, off, jd, fr, frame)
        _, s6, j6, status = K.emul(L, el, P6, model, off, jd, fr, frame)
        assert (status == 0).all()
        assert (j6[:, :, 6] == 0).all() and j6[:, :, :6].tobytes() == j7[:, :, :6].tobytes()
        Pm = np.stack([K.unpack7(p)[:6, :6] for p in P])[sat]
        ref = np.einsum("nij,njk,nlk->nil", j7[:, :, :6], Pm, j7[:, :, :6])
        S6 = K.unpack6(s6)
        assert (np.abs(S6 - ref).max(axis=(1, 2)) / np.abs(ref).max(axis=(1, 2))).max() < 1e-12


def test_a_zero_covariance_gives_zero_sigma_and_the_state(L):
    el, model = _catalogue()
    n = el.shape[1]
    sat, off = _queries(n, count=5)
    jd, fr = _times(el, sat, count=5)
    st, sig, jac, status = K.emul(L, el, np.zeros((n, 28)), model, off, jd, fr, 1)
    st_ref, _, _, _ = K.emul(L, el, _P(n), model, off, jd, fr, 1)
    assert (status == 0).all() and (sig == 0).all()
    assert st.tobytes() == st_ref.tobytes() and (np.abs(st[:, :3]).max(axis=1) > 1000.0).all()
    assert (jac[:, :, :6] != 0).any(axis=(1, 2)).all() and (jac[:, :, 6] == 0).all()


def _assert_zero_filled(st, sig, jac, mask):
    assert (st[mask] == 0).all() and (sig[mask] == 0).all() and (jac[mask] == 0).all()


def test_a_model_byte_that_contradicts_the_set_is_init_failed(L):
    el, model = _catalogue()
    n = el.shape[1]
    sat, off = _queries(n, count=5)
    jd, fr = _times(el, sat, count=5)
    wrong = (1 - model).astype(np.uint8)
    for frame in (0, 1):
        st, sig, jac, status = K.emul(L, el, _P(n), wrong, off, jd, fr, frame)
        assert (status == 1).all()
        _assert_zero_filled(st, sig, jac, status != 0)
        assert (K.restated(el, _P(n), wrong, off, jd, fr, frame)[3] == 1).all()


def test_a_decaying_deep_space_set_is_cell_failed(L):
    """A GTO with a large drag term: SDP4 stops it (decay, eccentricity) after some 60 days.  Queries before that are
    OK, later ones CELL_FAILED and zero-filled, as in the restatement."""
    from astroz_b200 import synth

    gto = synth.elements_from_tles([synth.tle_lines(7, 24, 127.5, 27.0, 40.0, 0.73, 180.0, 10.0, 2.25, 0.5)])
    t = np.linspace(0.0, 120.0, 241)
    jd = np.full(len(t), np.floor(gto[0, 0] - 0.5) + 0.5)
    fr = (gto[0, 0] - jd) + t
    off = np.array([0, len(t)], np.uint32)
    md = np.ones(1, np.uint8)
    st, sig, jac, status = K.emul(L, gto, _P(1), md, off, jd, fr, 0)
    rstatus = K.restated(gto, _P(1), md, off, jd, fr, 0)[3]
    print("first CELL_FAILED at", t[np.argmax(status == 2)], "days")
    assert status[0] == 0 and (status == 2).any() and set(np.unique(status)) <= {0, 2}
    assert (status == rstatus).all()
    _assert_zero_filled(st, sig, jac, status != 0)


# ---- 6. chunking ----------------------------------------------------------------------------------------------------
def test_results_do_not_depend_on_the_chunking(L):
    """One satellite's queries cut by chunk boundaries, and chunks over many small satellites (some with no queries)
    give the same bytes"""
    el, model = _catalogue()
    n = el.shape[1]
    rng = np.random.default_rng(2)
    counts = rng.integers(0, 40, n)
    counts[0], counts[-1] = 700, 0
    sat = np.repeat(np.arange(n), counts)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    t = rng.uniform(-3.0, 3.0, len(sat))
    jd = np.floor(el[0][sat] + t - 0.5) + 0.5
    fr = (el[0][sat] + t) - jd
    ref = K.emul(L, el, _P(n), model, off, jd, fr, 1)
    for chunk in (1, 7, 32, 100, 10 ** 6):
        got = K.emul(L, el, _P(n), model, off, jd, fr, 1, chunk=chunk)
        for a, b in zip(got, ref):
            assert a.tobytes() == b.tobytes(), chunk
    # and a query's bytes do not depend on the other queries of the batch
    one = K.emul(L, el[:, :1], _P(n)[:1], model[:1], np.array([0, 1], np.uint32), jd[5:6], fr[5:6], 1)
    for a, b in zip(one, ref):
        assert a[0].tobytes() == b[5].tobytes()


# ---- 7. the C ABI and the Python wrapper ----------------------------------------------------------------------------
def test_cabi_refusals_write_nothing():
    from astroz_b200 import _lib

    p = lambda x: None if x is None else C.c_void_p(x.ctypes.data)  # noqa: E731
    el, model = _catalogue()
    el, model = el[:, :3], model[:3].copy()
    n, m = 3, 6
    good = dict(el=el, cov=_P(n), model=model, off=np.array([0, 2, 4, 6], np.uint32), jd=np.full(m, 2460437.5),
                fr=np.zeros(m), frame=0, grav=1, dev=0)
    bad = []
    for key, val in (("dev", -1), ("grav", 7), ("frame", 2), ("off", np.array([0, 3, 2, 6], np.uint32)),
                     ("off", np.array([0, 2, 4, 5], np.uint32)), ("off", np.array([1, 2, 4, 6], np.uint32)),
                     ("model", np.array([0, 2, 0], np.uint8))):
        bad.append({**good, key: val})
    for key in ("el", "cov", "jd", "fr"):
        a = good[key].copy()
        a.reshape(-1)[1] = np.nan if key != "jd" else np.inf
        bad.append({**good, key: a})
    for a in bad:
        st, sig, jac, status = np.full((m, 6), -3.0), np.full((m, 21), -3.0), np.full((m, 42), -3.0), \
            np.full(m, 9, np.uint8)
        rc = _lib.lib().astroz_cuda_propagate_covariance(
            p(a["el"]), n, a["grav"], p(a["cov"]), p(a["model"]), p(a["off"]), p(a["jd"]), p(a["fr"]), m,
            a["frame"], a["dev"], p(st), p(sig), p(jac), p(status))
        assert rc == -20, a
        assert (st == -3.0).all() and (sig == -3.0).all() and (jac == -3.0).all() and (status == 9).all()
    for key, val in (("dev", -1), ("grav", 7), ("frame", 2)):
        a = {**good, key: val}
        rc = _lib.lib().astroz_cuda_propagate_covariance_device(
            None, n, a["grav"], None, None, None, None, None, m, a["frame"], a["dev"], None, None, None, None, None)
        assert rc == -20, key


class _EmulLib:
    """astroz_cuda_propagate_covariance served by the host build, for the wrapper's checks without a device"""

    def __init__(self, L):
        self.L = L

    def astroz_cuda_propagate_covariance(self, el, n, grav, cov, model, off, jd, fr, m, frame, device, st, sig, jac,
                                         status):
        return self.L.emul_propagate_covariance(el, C.c_uint32(n), grav, cov, model, off, jd, fr, C.c_uint32(m),
                                                frame, C.c_uint32(self.L.emul_cov_chunk(m)), st, sig, jac, status)


def test_python_wrapper_returns_caller_order(L, monkeypatch):
    from astroz_b200 import covariance as cv
    from astroz_b200.fit import FitResult

    el, model = _catalogue()
    n = el.shape[1]
    P = _P(n)
    monkeypatch.setattr(cv, "lib", lambda: _EmulLib(L))
    rng = np.random.default_rng(4)
    sat = rng.integers(0, n, 300)
    t = rng.uniform(-2.0, 2.0, 300)
    jd = np.floor(el[0][sat] + t - 0.5) + 0.5
    fr = (el[0][sat] + t) - jd
    fit = FitResult(el, np.zeros(n), np.zeros(n), np.zeros(n, np.uint32), np.zeros(n, np.uint8), covariance=P,
                    deep_space=model == 1)
    res = cv.propagate_covariance(fit, sat, jd, fr, frame=cv.RTN, jacobian=True)
    mats = np.stack([K.unpack7(p) for p in P])
    res2 = cv.propagate_covariance(el, sat, jd, fr, covariance=mats, model=model, frame=cv.RTN)
    assert res2.jacobian is None and res.covariance.tobytes() == res2.covariance.tobytes()
    for i in (0, 17, 299):
        one = K.emul(L, el[:, sat[i]:sat[i] + 1], P[sat[i]:sat[i] + 1], model[sat[i]:sat[i] + 1],
                     np.array([0, 1], np.uint32), jd[i:i + 1], fr[i:i + 1], 1)
        assert res.state[i].tobytes() == one[0][0].tobytes() and res.jacobian[i].tobytes() == one[2][0].tobytes()
        assert res.status[i] == one[3][0]
        assert (res.matrix(i) == K.unpack6(one[1][0])).all()
    with pytest.raises(ValueError):
        cv.propagate_covariance(el, sat, jd, fr)                       # no covariance
    with pytest.raises(ValueError):
        cv.propagate_covariance(el, sat, jd, fr, covariance=P, model=np.full(n, 2))
    with pytest.raises(ValueError):
        cv.propagate_covariance(el, [n], jd[:1], fr[:1], covariance=P)
