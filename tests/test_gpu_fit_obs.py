"""Element fits from sensor observations on the device (fit_obs_kernel, fit_obs_deep_kernel, observe_kernel): the device
against the host build of the same source on 2,000+ mixed sets of every kind, bit-identity with astroz_cuda_fit_elements
for TEME observations, the residual invariant through create_from_elements + propagate_pairs + observe, host vs device
calls and batch independence, and observe against the host emulation."""
import numpy as np
import pytest

from tests import fit_oracle as R
from tests.fit_oracle import obs as O

pytestmark = pytest.mark.gpu
TWO_PI = 2 * np.pi


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def emul():
    _lib()
    L = O.emul_library()
    if L is None:
        pytest.skip("nvcc unavailable")
    return L


def _library_tracks(el, kinds, jd, fr, sites, min_el_deg=10.0):
    """Tracks of every column of el made by the library itself: propagate_pairs TEME states, then observe; satellite s
    gets kind kinds[s] at every site (radar and optical above min_el_deg), or every epoch (state kinds)."""
    from astroz_b200.constellation import Constellation
    from astroz_b200.fit import observe

    n, t = el.shape[1], len(jd)
    c = Constellation.from_elements(*el)
    p, v, st = c.propagate_pairs(np.repeat(np.arange(n), t), np.tile(jd, n), np.tile(fr, n))
    c.deinit()
    states = np.concatenate([np.asarray(p), np.asarray(v)], axis=1).reshape(n, t, 6)
    ok = (np.asarray(st).reshape(n, t) == 0)
    per = []
    for s in range(n):
        k = kinds[s]
        if k in (O.TEME, O.ECEF):
            keep = np.flatnonzero(ok[s][::10])
            idx = keep * 10
            val = observe(states[s, idx], jd[idx], fr[idx], k)
            sig = np.array([1e-3] * 3 + [1e-6] * 3)
            rows = [(idx, np.zeros(len(idx), np.uint32), val)]
        else:
            rows = []
            for q in range(len(sites)):
                elev = observe(states[s], jd, fr, O.RADAR, q, sites)[:, 2]
                idx = np.flatnonzero(ok[s] & (elev > np.deg2rad(min_el_deg)))
                rows.append((idx, np.full(len(idx), q, np.uint32), observe(states[s, idx], jd[idx], fr[idx], k, q,
                                                                           sites)))
            sig = O.RADAR_SIGMA if k == O.RADAR else O.OPTICAL_SIGMA
        idx = np.concatenate([r[0] for r in rows])
        sig6 = np.full((len(idx), 6), np.inf)
        sig6[:, :len(sig)] = sig
        per.append((jd[idx], fr[idx], np.full(len(idx), k, np.uint8), np.concatenate([r[2] for r in rows]), sig6,
                    np.concatenate([r[1] for r in rows])))
    return per


@pytest.fixture(scope="module")
def mixed_case():
    """2,000 config-2 near-earth sets and 200 config-3 deep-space sets; kinds cycle TEME, ECEF, radar, optical over
    the satellites; one day, radar and optical at the six sites above 10 deg."""
    _lib()
    from astroz_b200 import synth

    ne = synth.elements_from_tles(synth.near_earth_catalog(2000))
    mc = synth.elements_from_tles(synth.mixed_catalog(13478))
    deep = mc[:, 1440.0 / mc[1] > 225.0][:, :200]
    el = np.concatenate([ne, deep], axis=1)
    n = el.shape[1]
    kinds = np.arange(n) % 4
    jd, fr = synth.time_grid(720)
    fr = np.arange(720) * 2.0 / 1440.0 + fr[0]
    per = _library_tracks(el, kinds, jd, fr, O.RADAR_SITES)
    guess = R.perturbed(el, seed=3)
    guess[3] = np.abs(guess[3])
    guess[7] = el[7]                 # B* held at its generating value: one day of tracks says little about drag
    return el, guess, per


def _device_fit(guess, per, stations, **kw):
    from astroz_b200.fit import fit_observations

    jd, fr, kd, val, sig, sta, off = O.concat(per)
    sat = np.repeat(np.arange(len(per)), np.diff(off))
    return fit_observations(guess, sat, jd, fr, kd, val, sig, sta, stations, **kw)


def test_device_matches_host_emulation(mixed_case, emul):
    """The device against the host build of the same source.  Status bytes and residual counts are equal; the step
    counts are equal on 99 % of the sets, not all; the fitted variables agree to 1e-9 on the sets that take the same
    steps.  A 1e-6 relative bound on the covariance is NOT met: the words agree to 1e-3 of their scale (3.2e-4
    measured), for the reason given at the assertion.  The independent check of the covariance is the CPU restatement
    (tests/fit_oracle/fit_oracle_obs.c) and the replica statistics in tests/test_fit_obs_cpu.py."""
    el, guess, per = mixed_case
    res = _device_fit(guess, per, O.RADAR_SITES, deep_space=True, fit_bstar=False)
    jd, fr, kd, val, sig, sta, off = O.concat(per)
    f, wrms, nres, cov, it, st = O.emul_fit(emul, guess, jd, fr, kd, val, sig, sta, off, O.RADAR_SITES,
                                            fit_bstar=False)
    deep = np.arange(el.shape[1]) >= 2000
    print("status", np.bincount(res.status, minlength=5), "iterations", np.bincount(res.iterations))
    assert (res.status == st).all() and (res.n_residuals == nres).all()
    # The host build does not contract a * b + c into FMAs, so a trial cost can land on the other side of the stopping
    # rule (a step changes the cost by <= 1e-10 of it) and the two stop some steps apart: 7 of these 2,200 sets on an
    # H100.  The rest take the same steps and agree as below.
    same = res.iterations == it
    print(f"iterations equal on {same.sum()} of {len(same)} sets")
    assert same.mean() >= 0.99
    assert (st[~deep] == 0).mean() > 0.99 and (st[deep] == 0).mean() > 0.9
    ok = (st == 0) & same
    # the fit's own variables (near-earth, or equinoctial for the deep rows): n to 1e-9 relative, the others to 1e-9
    xd = np.array([O.fit_vars(res.elements[:, s], deep[s]) for s in np.flatnonzero(ok)])
    xe = np.array([O.fit_vars(f[:, s], deep[s]) for s in np.flatnonzero(ok)])
    dx = xd - xe
    for c in (4, 5):
        dx[:, c] = np.mod(dx[:, c] + np.pi, TWO_PI) - np.pi
    print(f"n {np.abs(dx[:, 0] / xe[:, 0]).max():.1e} relative, others {np.abs(dx[:, 1:6]).max():.1e}, "
          f"wrms {np.abs(res.wrms[ok] - wrms[ok]).max():.1e} (of up to {wrms[ok].max():.1e})")
    assert np.abs(dx[:, 0] / xe[:, 0]).max() <= 1e-9 and np.abs(dx[:, 1:6]).max() <= 1e-9
    # noise-free tracks: wRMS is what is left of the rounding of two builds (~1e-7), so it is compared in absolute
    assert np.abs(res.wrms[ok] - wrms[ok]).max() <= 1e-5
    # Covariance words relative to the scale of their row and column.  J is a forward difference over steps of 1e-8, so
    # the two builds' rounding of the states (~1e-12 relative) reaches it at ~1e-4 relative, and the inverse of the
    # correlated normal matrix carries that: 3.2e-4 on an H100.
    iu = np.triu_indices(7)
    diag = cov[ok][:, np.cumsum([0, 7, 6, 5, 4, 3, 2])]
    scale = np.sqrt(np.abs(diag[:, iu[0]] * diag[:, iu[1]]))
    dcov = np.abs(res.covariance[ok] - cov[ok]) / np.where(scale > 0, scale, 1.0)
    print(f"covariance: max relative difference {dcov.max():.2e}")
    assert dcov.max() <= 1e-3


def _grid_states(n, t):
    from astroz_b200 import synth
    from astroz_b200.constellation import Constellation, Layout

    el = synth.elements_from_tles(synth.near_earth_catalog(n))
    c = Constellation.from_elements(*el)
    jd, fr = synth.time_grid(t)
    pos, vel = c.propagate(jd, fr, layout=Layout.satelliteMajor)
    c.deinit()
    return el, np.repeat(np.arange(n), t), np.tile(jd, n), np.tile(fr, n), np.array(pos).reshape(-1, 3), \
        np.array(vel).reshape(-1, 3)


def test_teme_observations_are_bit_identical_to_fit_elements():
    """Kind-0 observations whose sigmas equal fit_elements' pos_sigma / vel_sigma: the same fitted columns, iterations
    and status bytes, near-earth and mixed, with and without velocities."""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.fit import fit_elements, fit_observations

    el, sat, jd, fr, pos, vel = _grid_states(2000, 1440)
    guess = R.perturbed(el, seed=3)
    m = len(sat)
    for with_vel in (True, False):
        ref = fit_elements(guess, sat, jd, fr, pos, vel if with_vel else None)
        val = np.concatenate([pos, vel], axis=1)
        sig = np.tile([1.0] * 3 + ([1e-3] if with_vel else [np.inf]) * 3, (m, 1))
        got = fit_observations(guess, sat, jd, fr, np.zeros(m, np.uint8), val, sig)
        assert got.elements.tobytes() == ref.elements.tobytes(), with_vel
        assert got.iterations.tobytes() == ref.iterations.tobytes() and got.status.tobytes() == ref.status.tobytes()
    # mixed: config-3 deep-space sets with B* held, as the deep-space TEME fit's tests run them
    mc = synth.elements_from_tles(synth.mixed_catalog(13478))
    deep = mc[:, 1440.0 / mc[1] > 225.0][:, :300]
    cols = np.concatenate([el[:, :100], deep], axis=1)
    from astroz_b200.constellation import Constellation, Layout

    c = Constellation.from_elements(*cols)
    jd1, fr1 = synth.time_grid(1440)
    p, v = c.propagate(jd1, fr1, layout=Layout.satelliteMajor)
    c.deinit()
    n = cols.shape[1]
    s2 = np.repeat(np.arange(n), 1440)
    p, v = np.array(p).reshape(-1, 3), np.array(v).reshape(-1, 3)
    g = R.perturbed(cols, seed=5)
    g[3] = np.abs(g[3])
    g[7, 100:] = cols[7, 100:]
    ref = fit_elements(g, s2, np.tile(jd1, n), np.tile(fr1, n), p, v, deep_space=True, fit_bstar=False)
    got = fit_observations(g, s2, np.tile(jd1, n), np.tile(fr1, n), np.zeros(len(s2), np.uint8),
                           np.concatenate([p, v], axis=1), np.tile([1.0] * 3 + [1e-3] * 3, (len(s2), 1)),
                           deep_space=True, fit_bstar=False)
    print("mixed statuses", np.bincount(ref.status, minlength=5))
    assert got.elements.tobytes() == ref.elements.tobytes()
    assert got.iterations.tobytes() == ref.iterations.tobytes() and got.status.tobytes() == ref.status.tobytes()


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


def test_residual_invariant(mixed_case):
    """Fitted columns -> Constellation.from_elements -> propagate_pairs (TEME) -> observe give back the reported wRMS.
    Noisy tracks (wRMS ~ 1).  The handle's own element init (host libm) and time model move each state by rounding,
    within the 1e-8 km / 1e-11 km/s K8's invariant allows; through the 1e-6 km/s velocity sigmas of the state kinds
    that is up to 1e-5 of a sigma per residual.  Measured: 9e-9 relative in wRMS; bound 1e-7."""
    from astroz_b200.constellation import Constellation
    from astroz_b200.fit import observe

    el, guess, per = mixed_case
    rows = np.arange(0, 2000, 7)
    sub = _noisy([per[s] for s in rows], seed=9)
    res = _device_fit(guess[:, rows], sub, O.RADAR_SITES, fit_bstar=False, max_iter=60)
    assert (res.status == 0).mean() > 0.98, np.bincount(res.status)
    jd, fr, kd, val, sig, sta, off = O.concat(sub)
    sat = np.repeat(np.arange(len(rows)), np.diff(off))
    c = Constellation.from_elements(*res.elements)
    p, v, st = c.propagate_pairs(sat, jd, fr)
    c.deinit()
    h = observe(np.concatenate([np.asarray(p), np.asarray(v)], axis=1), jd, fr, kd, sta, O.RADAR_SITES)
    d = val - h
    for k, q in ((O.RADAR, 1), (O.OPTICAL, 0)):
        m = kd == k
        d[m, q] = (np.mod(d[m, q] + np.pi, TWO_PI) - np.pi) * np.cos(val[m, q + 1])
    w = np.where(np.isfinite(sig), d / sig, 0.0)
    F = np.bincount(sat, (w ** 2).sum(1), minlength=len(rows))
    nres = np.bincount(sat, np.isfinite(sig).sum(1), minlength=len(rows))
    ok = res.status == 0
    assert (nres == res.n_residuals).all()
    wrms = np.sqrt(F / nres)
    rel = np.abs(wrms[ok] / res.wrms[ok] - 1.0)
    print(f"residual invariant: wrms median {np.median(res.wrms[ok]):.3f}, max relative difference {rel.max():.2e}")
    assert rel.max() < 1e-7


def test_host_vs_device_calls_and_batch_independence(mixed_case):
    import torch

    from astroz_b200.fit import fit_observations, fit_observations_device

    el, guess, per = mixed_case
    rows = np.concatenate([np.arange(0, 2000, 40), np.arange(2000, 2200, 10)])
    sub = [per[s] for s in rows]
    g = guess[:, rows]
    res = _device_fit(g, sub, O.RADAR_SITES, deep_space=True)
    jd, fr, kd, val, sig, sta, off = O.concat(sub)
    n, m = len(rows), len(jd)
    sat = np.repeat(np.arange(n), np.diff(off))
    # The C call with pinned host buffers (direct DMA, no staging ring) and with pageable ones, the observations already
    # grouped by satellite so nothing is re-indexed on the way: the bytes of fit_observations
    import ctypes as C

    from astroz_b200 import _lib

    def direct(bufs):
        outs = [np.zeros((8, n)), np.zeros(n), np.zeros(n, np.uint32), np.zeros((n, 28)), np.zeros(n, np.uint32),
                np.zeros(n, np.uint8), np.zeros(n, np.uint8)]
        p = lambda a: C.c_void_p(a.ctypes.data)   # noqa: E731
        el_, off_, jd_, fr_, val_, sig_, sta_, kd_, st_ = bufs
        assert _lib.lib().astroz_cuda_fit_observations_mixed(
            p(el_), n, 1, p(off_), p(jd_), p(fr_), p(val_), p(sig_), p(sta_), p(kd_), m, p(st_), len(st_), 1, 25, 0,
            *[p(o) for o in outs]) == 0
        return outs

    def pinned(a, dtype):
        b = _lib.pinned_empty(np.shape(a), dtype)
        b[...] = a
        return b

    host = [(g, np.float64), (off, np.uint32), (jd, np.float64), (fr, np.float64), (val, np.float64),
            (sig, np.float64), (sta, np.uint32), (kd, np.uint8), (O.RADAR_SITES, np.float64)]
    pageable = direct([np.ascontiguousarray(a, dtype=dt) for a, dt in host])
    pin = direct([pinned(a, dt) for a, dt in host])
    for a, b in zip(pageable, pin):
        assert a.tobytes() == b.tobytes()
    assert pin[0].tobytes() == res.elements.tobytes() and pin[3].tobytes() == res.covariance.tobytes()
    assert pin[1].tobytes() == res.wrms.tobytes() and (pin[6] == res.deep_space).all()
    assert (res.deep_space == (rows >= 2000)).all()            # the deep-space pass ran on the deep-space rows
    # the device call
    dev = torch.device("cuda", 0)
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a)).to(dev, dt)   # noqa: E731
    out = dict(fitted=torch.empty((8, n), dtype=torch.float64, device=dev),
               wrms=torch.empty(n, dtype=torch.float64, device=dev),
               n_residuals=torch.empty(n, dtype=torch.int32, device=dev),
               covariance=torch.empty((n, 28), dtype=torch.float64, device=dev),
               iterations=torch.empty(n, dtype=torch.int32, device=dev),
               status=torch.empty(n, dtype=torch.uint8, device=dev),
               model=torch.empty(n, dtype=torch.uint8, device=dev))
    fit_observations_device(t(g), t(off, torch.int32), t(jd), t(fr), t(kd, torch.uint8), t(val), t(sig),
                            t(sta, torch.int32), t(O.RADAR_SITES), **out, deep_space=True)
    torch.cuda.synchronize()
    assert out["fitted"].cpu().numpy().tobytes() == res.elements.tobytes()
    assert out["covariance"].cpu().numpy().tobytes() == res.covariance.tobytes()
    assert out["wrms"].cpu().numpy().tobytes() == res.wrms.tobytes()
    assert out["iterations"].cpu().numpy().astype(np.uint32).tobytes() == res.iterations.tobytes()
    assert (out["model"].cpu().numpy() == res.deep_space).all()
    assert out["status"].cpu().numpy().tobytes() == res.status.tobytes()
    # alone, shuffled (observations interleaved across satellites), inside the larger batch
    for j in (0, 3, n - 1):
        one = _device_fit(g[:, [j]], [sub[j]], O.RADAR_SITES, deep_space=True)
        assert one.elements[:, 0].tobytes() == res.elements[:, j].tobytes()
        assert one.covariance[0].tobytes() == res.covariance[j].tobytes() and one.wrms[0] == res.wrms[j]
    perm = np.random.default_rng(5).permutation(n)
    inv = np.argsort(perm)
    order = np.lexsort((inv[sat], np.arange(m) - off[sat]))   # interleaved, each set's own order kept
    shuffled = fit_observations(g[:, perm], inv[sat][order], jd[order], fr[order], kd[order], val[order], sig[order],
                                sta[order], O.RADAR_SITES, deep_space=True)
    assert shuffled.elements.tobytes() == res.elements[:, perm].tobytes()
    assert shuffled.covariance.tobytes() == res.covariance[perm].tobytes()
    full = _device_fit(guess, per, O.RADAR_SITES, deep_space=True)
    assert full.elements[:, rows].tobytes() == res.elements.tobytes()
    assert full.covariance[rows].tobytes() == res.covariance.tobytes()


@pytest.mark.parametrize("kind", [O.TEME, O.ECEF, O.RADAR, O.OPTICAL])
def test_observe_on_the_device_matches_host_emulation(emul, kind):
    from astroz_b200.fit import observe

    rng = np.random.default_rng(kind)
    m = 20000
    u = rng.standard_normal((m, 3))
    r = rng.uniform(6600, 45000, m)[:, None] * u / np.linalg.norm(u, axis=1)[:, None]
    states = np.concatenate([r, rng.standard_normal((m, 3)) * 4.0], axis=1)
    jd = np.full(m, 2460437.0) + rng.integers(-400, 400, m)
    fr = rng.uniform(0, 1, m)
    sta = rng.integers(0, len(O.RADAR_SITES), m).astype(np.uint32)
    got = observe(states, jd, fr, kind, sta, O.RADAR_SITES)
    ref = O.emul_observe(emul, states, jd, fr, kind, sta, O.RADAR_SITES)
    d = got - ref
    if kind in (O.RADAR, O.OPTICAL):
        q = 1 if kind == O.RADAR else 0
        d[:, q] = np.mod(d[:, q] + np.pi, TWO_PI) - np.pi
    scale = np.maximum(np.abs(ref), 1.0)
    print(f"kind {kind}: max relative difference {np.abs(d / scale).max():.2e}")
    assert np.abs(d / scale).max() <= 1e-12
