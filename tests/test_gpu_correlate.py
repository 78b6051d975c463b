"""K12 track correlation on the device (correlate_kernel, correlate_deep_kernel): the device against the host build of
the same source on device-fitted mixed rows and radar, optical, ECEF, unknown-object and clustered tracks; host
pageable / pinned / device-call, order, split and single-track byte identity; a closed loop of fit, correlate,
assign and refit; a catalogue-scale run checked on sampled tracks."""
import numpy as np
import pytest

from tests import fit_oracle as R
from tests.fit_oracle import correlate as cr
from tests.fit_oracle import obs as O

pytestmark = pytest.mark.gpu
SIG = np.array([1e-3] * 3 + [1e-6] * 3)


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def emul():
    _lib()
    L = cr.emul_library()
    if L is None:
        pytest.skip("nvcc unavailable")
    return L


def _pairs_states(el, sat, jd, fr):
    from astroz_b200.constellation import Constellation

    c = Constellation.from_elements(*el)
    p, v, st = c.propagate_pairs(sat, jd, fr)
    c.deinit()
    return np.concatenate([np.asarray(p), np.asarray(v)], axis=1), np.asarray(st)


@pytest.fixture(scope="module")
def fitted():
    """~1,000 mixed rows fitted on the device from TEME states (as the K10 / K11 device tests fit them), deep-space rows
    with B* held; a co-located GEO cluster and a launch train appended as rows with the same covariance"""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.fit import OBS_TEME_STATE, fit_observations

    el = synth.elements_from_tles(synth.mixed_catalog(1000, n_geo=64, n_molniya=16, n_gps=16))
    n, t = el.shape[1], 49
    jd0 = np.floor(el[0] - 0.5) + 0.5
    sat = np.repeat(np.arange(n), t)
    jd = jd0[sat]
    fr = (el[0] - jd0)[sat] + np.tile(np.arange(t) / 48.0, n)
    st, status = _pairs_states(el, sat, jd, fr)
    val = st + np.random.default_rng(3).standard_normal(st.shape) * SIG
    keep = status == 0
    res = fit_observations(R.perturbed(el, seed=4), sat[keep], jd[keep], fr[keep],
                           np.full(keep.sum(), OBS_TEME_STATE), val[keep], np.tile(SIG, (keep.sum(), 1)),
                           deep_space=True)
    P = res.covariance.copy()
    bstar = np.array([q for q, (j, k) in enumerate(zip(*np.triu_indices(7))) if j == 6 or k == 6])
    P[np.ix_(np.flatnonzero(res.deep_space), bstar)] = 0.0
    ok = np.flatnonzero(np.isin(res.status, (0, 1)) & np.any(P != 0, axis=1))
    cat = res.elements.copy()
    model = res.deep_space.astype(np.uint8)
    extra_el, extra_P, extra_m = [], [], []
    geo = [s for s in ok if model[s] == 1 and cat[1, s] < 1.1][:1] or [s for s in ok if model[s] == 1][:1]
    leo = [s for s in ok if model[s] == 0][:1]
    for s, dm in [(geo[0], d) for d in (0.0005, 0.001, 0.002)] + [(leo[0], d) for d in (0.01, 0.02, 0.05)]:
        e = cat[:, s].copy()
        e[6] = (e[6] + dm) % 360.0
        extra_el.append(e)
        extra_P.append(P[s])
        extra_m.append(model[s])
    cat = np.concatenate([cat, np.stack(extra_el, 1)], axis=1)
    P = np.concatenate([P, np.stack(extra_P)])
    model = np.concatenate([model, np.array(extra_m, np.uint8)])
    return cat, P, model, ok


def _tracks(cat, model, ok, seed, count=600):
    """radar passes at six stations (near-earth rows), optical nights (GEO rows), ECEF fixes, tracks of objects that are
    not in the catalogue (a row perturbed by 0.5 deg in M) and tracks of the cluster rows; returns Tracks and the true
    row (-1: not in the catalogue)"""
    rng = np.random.default_rng(seed)
    per, truth = [], []
    n = cat.shape[1]
    cluster = list(range(n - 6, n))
    while len(per) < count:
        u = rng.uniform()
        s = int(rng.choice(cluster)) if u < 0.1 else int(rng.choice(ok))
        el = cat[:, s].copy()
        unknown = 0.1 <= u < 0.2
        if unknown:
            el[6] = (el[6] + 0.5) % 360.0
        t0 = el[0] + rng.uniform(0.0, 1.0)
        if model[s] == 1:
            kind, minutes, step = (O.OPTICAL, 60, 300.0) if rng.uniform() < 0.8 else (O.ECEF, 30, 300.0)
        else:
            kind, minutes, step = (O.RADAR, 8, 30.0) if rng.uniform() < 0.8 else (O.ECEF, 5, 60.0)
        tr = cr.track_of(el, kind, t0, minutes, step, rng=rng)
        if tr is None or not len(tr[0]):
            continue
        per.append(tr)
        truth.append(-1 if unknown else s)
    return cr.Tracks(per, O.RADAR_SITES), np.array(truth)


def _device(cat, P, model, tr, best=4, gate=0.999):
    from astroz_b200.correlate import correlate

    return correlate(cat, tr.track_ids(), tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station, tr.stations,
                     covariance=P, model=model, best=best, gate_probability=gate)


def _against_host(res, host, picks=None, row_status=True, tol=1e-4):
    """statuses, used, n_gate and n_failed equal; d2 within tol relative (the device contracts to FMA where the host
    build does not, and |z|^2 - b^T (...) magnifies that rounding); rows equal wherever the d2 gap to the neighbouring
    slots exceeds tol.  Returns the worst relative d2 difference."""
    rows, d2, used, ng, nf, status, rs = host
    sel = slice(None) if picks is None else picks
    assert np.array_equal(res.status[sel], status) and np.array_equal(res.used[sel], used)
    assert np.array_equal(res.n_gate[sel], ng) and np.array_equal(res.n_failed[sel], nf)
    if row_status:
        assert np.array_equal(res.row_status, rs)
    er = np.where(rows == cr.EMPTY, -1, rows.astype(np.int64))
    fin = np.isfinite(d2)
    assert np.array_equal(np.isfinite(res.d2[sel]), fin)
    rel = np.abs(res.d2[sel][fin] - d2[fin]) / np.maximum(1.0, d2[fin])
    assert rel.max() < tol
    gap = np.diff(np.concatenate([d2, np.full((len(d2), 1), np.inf)], axis=1), axis=1)   # gap to the next slot
    prev = np.concatenate([np.full((len(d2), 1), np.inf), gap[:, :-1]], axis=1)
    clear = (gap > tol * np.maximum(1.0, d2)) & (prev > tol * np.maximum(1.0, d2)) & fin
    assert np.array_equal(res.rows[sel][clear], er[clear])
    assert np.all(res.rows[sel][~fin] == -1)
    return rel.max()


def test_device_matches_the_host_build(emul, fitted):
    """2,000 tracks against ~1,000 device-fitted mixed rows plus the cluster rows"""
    cat, P, model, ok = fitted
    tr, truth = _tracks(cat, model, ok, seed=1, count=2000)
    res = _device(cat, P, model, tr)
    host = cr.emul_threaded(emul, cat, P, model, tr)
    worst = _against_host(res, host)
    ng, status = host[3], host[5]
    print(f"d2 device vs host build: worst relative {worst:.2e} over {np.isfinite(host[1]).sum()} slots")
    amb = np.sum(ng > 1)
    unc = np.sum(status == 1)
    print(f"{tr.t} tracks: {amb} ambiguous, {unc} uncorrelated, {np.sum(truth < 0)} of objects not in the catalogue")
    assert amb > 0 and unc > 0


def test_byte_identity_across_calls_orders_and_splits(fitted):
    import torch

    from astroz_b200.correlate import correlate_device, correlate_scratch_bytes

    cat, P, model, ok = fitted
    tr, _ = _tracks(cat, model, ok, seed=2, count=300)
    base = _device(cat, P, model, tr)
    # pinned host buffers
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()  # noqa: E731
    tp = cr.Tracks([(tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station)], tr.stations)
    tp.jd, tp.fr, tp.value, tp.sigma = pin(tr.jd), pin(tr.fr), pin(tr.value), pin(tr.sigma)
    tp.offsets, tp.t = tr.offsets, tr.t
    r2 = _device(pin(cat), pin(P), model, tp)
    assert np.array_equal(r2.rows, base.rows) and np.array_equal(r2.d2, base.d2)
    # the device call
    dev = torch.device("cuda", 0)
    g = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
    n, t, best = cat.shape[1], tr.t, 4
    out = dict(rows=torch.zeros((t, best), dtype=torch.int32, device=dev), d2=torch.zeros((t, best), dtype=torch.float64,
               device=dev), used=torch.zeros(t, dtype=torch.int32, device=dev),
               n_gate=torch.zeros(t, dtype=torch.int32, device=dev), n_failed=torch.zeros(t, dtype=torch.int32, device=dev),
               status=torch.zeros(t, dtype=torch.uint8, device=dev), row_status=torch.zeros(n, dtype=torch.uint8, device=dev))
    scratch = torch.zeros(correlate_scratch_bytes(n, t, best), dtype=torch.uint8, device=dev)
    correlate_device(g(cat, torch.float64), g(P, torch.float64), g(model, torch.uint8), g(tr.offsets.astype(np.int32),
                     torch.int32), g(tr.jd, torch.float64), g(tr.fr, torch.float64), g(tr.kind, torch.uint8),
                     g(tr.value, torch.float64), g(tr.sigma, torch.float64), g(tr.station.astype(np.int32), torch.int32),
                     g(tr.stations, torch.float64), scratch, **out)
    torch.cuda.synchronize()
    rows = out["rows"].cpu().numpy().astype(np.int64)
    assert np.array_equal(rows, base.rows) and np.array_equal(out["d2"].cpu().numpy(), base.d2)
    assert np.array_equal(out["status"].cpu().numpy(), base.status)
    assert np.array_equal(out["n_gate"].cpu().numpy(), base.n_gate.astype(np.int32))
    # shuffled track order with duplicates, a split batch, and one track against the whole catalogue
    rng = np.random.default_rng(9)
    perm = rng.permutation(tr.t)
    perm = np.concatenate([perm, perm[:20]])
    ids = tr.track_ids()
    sel = np.concatenate([np.flatnonzero(ids == j) for j in perm])
    new_id = np.concatenate([np.full(np.sum(ids == j), q) for q, j in enumerate(perm)])
    from astroz_b200.correlate import correlate

    r3 = correlate(cat, new_id, tr.jd[sel], tr.fr[sel], tr.kind[sel], tr.value[sel], tr.sigma[sel], tr.station[sel],
                   tr.stations, covariance=P, model=model)
    assert np.array_equal(r3.rows, base.rows[perm]) and np.array_equal(r3.d2, base.d2[perm])
    half = tr.offsets[tr.t // 2]
    a = correlate(cat, ids[:half], tr.jd[:half], tr.fr[:half], tr.kind[:half], tr.value[:half], tr.sigma[:half],
                  tr.station[:half], tr.stations, covariance=P, model=model)
    assert np.array_equal(a.d2, base.d2[:tr.t // 2]) and np.array_equal(a.rows, base.rows[:tr.t // 2])
    for j in (0, 7, tr.t - 1):
        b, e = tr.offsets[j], tr.offsets[j + 1]
        one = correlate(cat, np.zeros(e - b, int), tr.jd[b:e], tr.fr[b:e], tr.kind[b:e], tr.value[b:e],
                        tr.sigma[b:e], tr.station[b:e], tr.stations, covariance=P, model=model)
        assert np.array_equal(one.rows[0], base.rows[j]) and np.array_equal(one.d2[0], base.d2[j])
        assert one.n_gate[0] == base.n_gate[j] and one.status[0] == base.status[j]


SIG_LOOP = np.array([0.2] * 3 + [2e-4] * 3)   # a coarse day-1 source: 200 m, 20 cm/s


def test_closed_loop_fit_correlate_assign_refit():
    """The catalogue fitted on the device from day-1 states of the truth (200 m, 20 cm/s); day-2 radar, optical and ECEF
    tracks made from the truth, beyond the fit span, mixed with tracks of objects not in the catalogue.  The true row
    falls inside the 0.99 gate in a fraction within 4 sigma of 0.99.  The same tracks against the catalogue without its
    covariance fall far below it, so the gate's coverage comes from the fitted covariance.  The assignments feed
    fit_observations directly."""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.fit import OBS_TEME_STATE, fit_observations

    truth = synth.elements_from_tles(synth.mixed_catalog(600, n_geo=48, n_molniya=8, n_gps=8))
    n, t = truth.shape[1], 49
    jd0 = np.floor(truth[0] - 0.5) + 0.5
    sat = np.repeat(np.arange(n), t)
    jd = jd0[sat]
    fr = (truth[0] - jd0)[sat] + np.tile(np.arange(t) / 48.0, n)   # day 1: [epoch, epoch + 1]
    st, status = _pairs_states(truth, sat, jd, fr)
    val = st + np.random.default_rng(13).standard_normal(st.shape) * SIG_LOOP
    keep = status == 0
    fit = fit_observations(R.perturbed(truth, seed=14), sat[keep], jd[keep], fr[keep],
                           np.full(keep.sum(), OBS_TEME_STATE), val[keep], np.tile(SIG_LOOP, (keep.sum(), 1)),
                           deep_space=True)
    cat, model = fit.elements, fit.deep_space.astype(np.uint8)
    P = fit.covariance.copy()
    bstar = np.array([q for q, (j, k) in enumerate(zip(*np.triu_indices(7))) if j == 6 or k == 6])
    P[np.ix_(np.flatnonzero(fit.deep_space), bstar)] = 0.0
    conv = np.flatnonzero((fit.status == 0) & np.any(P != 0, axis=1))
    rng = np.random.default_rng(15)
    per, true_row = [], []
    while len(per) < 1000:
        s = int(rng.choice(conv))
        el = truth[:, s].copy()
        unknown = rng.uniform() < 0.1
        if unknown:
            el[6] = (el[6] + 0.5) % 360.0
        t0 = truth[0, s] + 1.0 + rng.uniform(0.0, 1.0)                 # day 2
        if model[s] == 1:
            kind, minutes, step = (O.OPTICAL, 60, 300.0) if rng.uniform() < 0.8 else (O.ECEF, 30, 300.0)
        else:
            kind, minutes, step = (O.RADAR, 8, 30.0) if rng.uniform() < 0.8 else (O.ECEF, 5, 60.0)
        trk = cr.track_of(el, kind, t0, minutes, step, rng=rng)
        if trk is None or not len(trk[0]):
            continue
        per.append(trk)
        true_row.append(-1 if unknown else s)
    tr, true_row = cr.Tracks(per, O.RADAR_SITES), np.array(true_row)
    p = 0.99
    known = true_row >= 0

    def inside(res):
        return np.array([true_row[j] in res.rows[j][res.d2[j] <= res.gate_d2[j]] for j in range(tr.t)])[known].mean()

    res = _device(cat, P, model, tr, best=8, gate=p)
    frac = inside(res)
    frac_zero = inside(_device(cat, np.zeros_like(P), model, tr, best=8, gate=p))
    sd = np.sqrt(p * (1 - p) / known.sum())
    sat = res.assigned()
    wrong = np.sum((sat >= 0) & known & (sat != true_row))
    false_pos = np.sum((sat >= 0) & ~known)
    print(f"closed loop: true row inside the {p} gate for {frac:.4f} of {known.sum()} day-2 tracks (4 sigma "
          f"{4 * sd:.4f}; {frac_zero:.4f} without the covariance); {wrong} wrong assignments, {false_pos} of "
          f"{np.sum(~known)} tracks of objects not in the catalogue assigned, {np.sum(res.status == 1)} uncorrelated")
    assert abs(frac - p) <= 4 * sd
    assert frac_zero < p - 20 * sd
    take = sat[tr.track_ids()] >= 0
    ids = tr.track_ids()[take]
    refit = fit_observations(cat, sat[ids], tr.jd[take], tr.fr[take], tr.kind[take], tr.value[take], tr.sigma[take],
                             tr.station[take], tr.stations, deep_space=True)
    assert np.all(np.isin(refit.status[np.unique(sat[ids])], (0, 1, 4)))


def test_catalogue_scale_sampled_against_the_host_build(emul):
    """The config-2 catalogue refitted on the device from radar tracks of six stations over two days (an OT1-like refit:
    six tracks of 10 observations per object; geometric, visibility is not modelled), its covariances as the rows' P,
    against 10,000 day-3 radar tracks of the truth; 200 sampled tracks checked against the host build over every row"""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.fit import fit_observations

    truth = synth.elements_from_tles(synth.near_earth_catalog(13478, 13478))
    n = truth.shape[1]
    rows = np.repeat(np.arange(n), 6)
    ids, jd, fr, kind, value, sigma, station = cr.device_tracks(truth, rows, O.RADAR, 10, 30.0, 21, span=2.0)
    fit = fit_observations(R.perturbed(truth, seed=22), rows[ids], jd, fr, kind, value, sigma, station,
                           O.RADAR_SITES)
    cat, P = fit.elements, fit.covariance
    rng = np.random.default_rng(4)
    ids, jd, fr, kind, value, sigma, station = cr.device_tracks(truth, rng.integers(0, n, 10000), O.RADAR, 10, 10.0,
                                                                5, start=2.0)
    tr = cr.Tracks([(jd, fr, kind, value, sigma, station)], O.RADAR_SITES)
    tr.offsets = np.searchsorted(ids, np.arange(10001)).astype(np.uint32)
    tr.t = 10000
    res = _device(cat, P, None, tr)
    pick = rng.choice(tr.t, 200, replace=False)
    host = cr.emul_threaded(emul, cat, P, None, cr.subset(tr, pick))
    worst = _against_host(res, host, picks=pick)
    print(f"catalogue scale: {np.sum(fit.status == 0)} of {n} rows converged in the refit; {np.sum(res.status == 0)} of "
          f"{tr.t} tracks correlated, {np.sum(res.n_gate == 1)} with one row in the gate; 200 sampled tracks equal "
          f"the host build, d2 within {worst:.2e}")
