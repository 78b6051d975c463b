"""K11 conjunction assessment on the device (conjunction_kernel, conjunction_deep_kernel): the device against the host
build of the same source on a few thousand engineered candidates among device-fitted mixed rows, the TCA states against
from_elements + propagate_pairs, a Monte Carlo assessed by the call itself, and batch / order / duplication and host /
pinned / device-call byte identity."""
import numpy as np
import pytest

from tests import fit_oracle as R
from tests.fit_oracle import conjunction as cj
from tests.fit_oracle import covariance as K

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
    L = cj.emul_library()
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
    """~1,000 mixed rows fitted on the device (as the K10 device tests fit them), deep-space rows with B* held"""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.fit import OBS_TEME_STATE, fit_observations

    el = synth.elements_from_tles(synth.mixed_catalog(1024, n_geo=64, n_molniya=16, n_gps=16))
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
    P[np.ix_(np.flatnonzero(res.deep_space), bstar)] = 0.0   # deep-space B* held (K10's header note)
    return res, P


def _candidates(res, P, m, seed):
    """m candidates over the fitted catalogue with engineered partners appended as extra rows:
      - 1/2 crossings of a converged row with a copy of itself, inclination changed by 0.5 .. 60 deg
        (conjunction_cases.crossings; near-earth +-2 min, deep-space +-30 min), the copy carrying the row's P;
      - 1/4 LEO-deep crossings: a converged near-earth row against a 12 h deep-space set whose perigee lies on the
        row's node at its radius (conjunction_cases.leo_deep_partner), +-2 min, a synthetic deep-space P with B* held;
      - 1/4 random near-earth / deep-space pairs at a common time, +-10 min (mostly window edges).
    Returns ((elements, P, model), (primary, secondary, jd, fr, window, hbr), engineered mask)."""
    from tests.fit_oracle import conjunction_cases as cc

    rng = np.random.default_rng(seed)
    el, deep = res.elements, res.deep_space
    n = el.shape[1]
    good = np.flatnonzero(res.status == 0)
    ne, ds = good[~deep[good]], good[deep[good]]
    k1, k2 = m // 2, m // 4
    k3 = m - k1 - k2
    rows1 = rng.choice(good, k1)
    cp, jd1, fr1 = cc.crossings(el, rows1, rng.uniform(0.5, 60.0, k1))
    rows2 = rng.choice(ne, k2)
    _, jd2, fr2 = cc.crossings(el, rows2, np.zeros(k2))
    dp = np.stack([cc.leo_deep_partner(el[:, r], j, f) for r, j, f in zip(rows2, jd2, fr2)], axis=1)
    Pd = cc.P_words(k2, scale=0.1, bstar=False, deep=np.ones(k2, bool), seed=seed)
    t0 = float(np.max(el[0]))
    jd0 = np.floor(t0 - 0.5) + 0.5
    cat = (np.concatenate([el, cp, dp], axis=1), np.concatenate([P, P[rows1], Pd]),
           np.concatenate([deep, deep[rows1], np.ones(k2, bool)]).astype(np.uint8))
    pr = np.concatenate([rows1, rows2, rng.choice(ne, k3)])
    se = np.concatenate([n + np.arange(k1), n + k1 + np.arange(k2), rng.choice(ds, k3)])
    jd = np.concatenate([jd1, jd2, np.full(k3, jd0)])
    fr = np.concatenate([fr1, fr2, (t0 - jd0) + rng.uniform(0.0, 1.0, k3)])
    w = np.concatenate([np.where(deep[rows1], 30.0, 2.0), np.full(k2, 2.0), np.full(k3, 10.0)])
    engineered = np.arange(m) < k1 + k2
    return cat, (pr, se, jd, fr, w, np.full(m, 0.02)), engineered


def _device_call(cat, cand, frame=0, states=True):
    from astroz_b200.collision import conjunctions

    el, P, model = cat
    pr, se, jd, fr, w, r = cand
    return conjunctions(el, pr, se, jd, fr, window_min=w, hbr_km=r, covariance=P, model=model, frame=frame,
                        states=states)


def _plane_d(states):
    dr, dv = states[:, 1, :3] - states[:, 0, :3], states[:, 1, 3:] - states[:, 0, 3:]
    z = dv / np.linalg.norm(dv, axis=1)[:, None]
    return np.linalg.norm(dr - np.sum(dr * z, axis=1)[:, None] * z, axis=1)


@pytest.mark.parametrize("frame", [0, 1])
def test_device_matches_the_host_build(emul, fitted, frame):
    """Equal status bytes on 3,000 candidates (near-earth and deep-space crossings, LEO-deep crossings, random
    near-earth / deep-space pairs).  Against the host build: |dTCA| |dv| and the miss within 1e-6 km on the
    engineered crossings (a random far pair's minimum can be flat, where the TCA moves along a near-constant range);
    each Sigma within 1e-3 of its scale on near-earth rows (K10's device tolerance; measured 3.4e-4) and 1e-4 on
    deep-space rows (1.5e-6); C2 within 1e-3; the device's Pc within 1e-9 relative (or 1e-300) of the host build's
    integrator on the device's own plane, since a tail Pc amplifies the C2 difference by (d / sigma)^2."""
    res, P = fitted
    cat, cand, engineered = _candidates(res, P, 3000, seed=1)
    got = _device_call(cat, cand, frame)
    rec, st, sig, status = cj.emul(emul, *cat, *cand, frame=frame)
    bad = np.flatnonzero(got.status != status)
    print(f"frame {frame}: statuses device {np.bincount(got.status, minlength=6).tolist()} host "
          f"{np.bincount(status, minlength=6).tolist()}; differing {bad[:10].tolist()}")
    assert len(bad) == 0
    ok = np.isin(status, (0, 3))
    close = ok & engineered
    mixed = close & (cat[2][cand[0]] != cat[2][cand[1]])
    assert ok.sum() > 0.9 * len(status) and close.sum() > 2000 and (status[mixed] == 0).sum() > 500
    dt = np.abs(got.record[close, 0] - rec[close, 0]) * 60.0 * rec[close, 2]
    dmiss = np.abs(got.record[close, 1] - rec[close, 1])
    deep_pair = (cat[2][cand[0]] | cat[2][cand[1]]).astype(bool)
    deep_obj = np.stack([cat[2][cand[0]], cat[2][cand[1]]], axis=1).astype(bool)[ok]
    es = (np.abs(got.state_covariance - sig).max(axis=2) / np.maximum(np.abs(sig).max(axis=2), 1e-300))[ok]
    ec = np.abs(got.record[:, 9:12] - rec[:, 9:12]).max(axis=1) / np.maximum(np.abs(rec[:, 9:12]).max(axis=1), 1e-300)
    d = _plane_d(got.states[ok])
    own = np.array([cj.emul_pc(emul, *c2, dd, 0.02) for c2, dd in zip(got.record[ok, 9:12], d)])
    epc = np.abs(got.record[ok, 12] - own) / np.maximum(own, 1e-300)
    print(f"frame {frame}: {close.sum()} engineered candidates ({mixed.sum()} LEO-deep) of {ok.sum()}; "
          f"|dTCA||dv| {dt.max():.2e} km, miss "
          f"{dmiss.max():.2e} km; Sigma near-earth rows {es[~deep_obj].max():.2e} deep rows {es[deep_obj].max():.2e}"
          f"; C2 near-earth {ec[ok & ~deep_pair].max():.2e} deep {ec[ok & deep_pair].max():.2e}; Pc vs own plane "
          f"{epc.max():.2e}; Pc host vs device {np.abs(got.pc - rec[:, 12]).max():.2e} abs, max Pc {rec[:, 12].max():.3e}")
    assert dt.max() < 1e-6 and dmiss.max() < 1e-6
    assert es[~deep_obj].max() < 1e-3 and es[deep_obj].max() < 1e-4
    assert ec[ok & ~deep_pair].max() < 1e-3 and epc.max() < 1e-9


def test_tca_states_match_propagate_pairs(fitted):
    """Both TEME states at the TCA against from_elements + propagate_pairs at (jd, fr + dt / 1440): within K8's 2.4e-9
    km plus |v| times one ulp of the jd (4.7e-10 day).  The TCA is the guess's jd + fr, rounded as K10 rounds it, plus
    dt; the pairs path rounds jd + (fr + dt / 1440) once more, so the two times differ by up to one ulp (measured 1.8
    half-ulps)."""
    res, P = fitted
    cat, cand, _ = _candidates(res, P, 400, seed=2)
    got = _device_call(cat, cand)
    ok = np.isin(got.status, (0, 3))
    for o, rows in ((0, cand[0][ok]), (1, cand[1][ok])):
        ref, st = _pairs_states(cat[0], rows, got.tca_jd[ok], got.tca_fr[ok])
        s = got.states[ok][:, o]
        good = st == 0
        v = np.linalg.norm(s[:, 3:], axis=1)
        allow = 2.4e-9 + v * 86400.0 * 4.7e-10
        dp = np.linalg.norm(s[good, :3] - ref[good, :3], axis=1)
        print(f"object {o}: TCA state vs propagate_pairs {dp.max():.2e} km over {good.sum()} (allowed "
              f"{allow[good].min():.1e} ..); worst/allowed {(dp / allow[good]).max():.2f}")
        assert (dp <= allow[good]).all()


def test_monte_carlo_assessed_by_the_call(fitted):
    """10^5 draws of both rows' variables; each drawn pair is assessed by the call itself with P = 0, which gives its
    exact miss at its own TCA, and the fraction of misses below R is compared with the linear Pc of the nominal pair,
    within 4 binomial sigma plus the linearisation allowance of 0.01 (measured through the oracle in
    tests/test_conjunction_cpu.py)"""
    from astroz_b200.collision import conjunctions

    from tests.fit_oracle import conjunction_cases as cc

    def assess(el, P, hbr):
        jd = np.floor(el[0, 0] - 0.5) + 0.5
        return conjunctions(el, [0], [1], jd, el[0, 0] - jd, window_min=1.0, hbr_km=hbr, covariance=P).record[0]

    el2, P2, hbr = cc.high_pc_leo(assess)
    jd = np.floor(el2[0, 0] - 0.5) + 0.5
    fr = el2[0, 0] - jd
    pc = assess(el2, P2, hbr)[12]
    draws = 100000
    rng = np.random.default_rng(21)
    cols = []
    for o in range(2):
        e = el2[:, o]
        wr = np.radians(e[5])
        x = np.array([e[1], e[2] * np.cos(wr), e[2] * np.sin(wr), np.radians(e[3]), np.radians(e[4]),
                      np.radians(e[6]) + wr, e[7]])
        cols.append(K.elements_of(rng.multivariate_normal(x, K.unpack7(P2[o]), size=draws, method="eigh"), e[0],
                                  False))
    el = np.empty((8, 2 * draws))
    el[:, 0::2], el[:, 1::2] = cols
    got = conjunctions(el, np.arange(0, 2 * draws, 2), np.arange(1, 2 * draws, 2), jd, fr, window_min=1.0,
                       hbr_km=hbr, covariance=np.zeros((2 * draws, 28)))
    ok = np.isin(got.status, (0, 3))
    frac = (got.miss_km[ok] < hbr).mean()
    sig = np.sqrt(pc * (1 - pc) / ok.sum())
    print(f"device Monte Carlo: Pc {pc:.4f}, hit fraction {frac:.4f} over {ok.sum()} draws, 4 sigma {4 * sig:.4f}")
    assert 0.1 < pc < 0.3 and abs(frac - pc) <= 4 * sig + 0.01


def test_batch_order_duplication_and_call_independence(fitted):
    """A candidate's bytes do not depend on the batch, its position or duplicates; the pageable, pinned and _device
    calls give identical bytes"""
    import torch

    from astroz_b200.collision import conjunctions, conjunctions_device

    res, P = fitted
    cat, cand, _ = _candidates(res, P, 600, seed=3)
    base = _device_call(cat, cand)
    perm = np.random.default_rng(4).permutation(600)
    dup = np.concatenate([perm, perm[:100]])
    sub = tuple(np.asarray(c)[dup] for c in cand)
    other = _device_call(cat, sub)
    assert (other.record.view(np.uint64) == base.record[dup].view(np.uint64)).all()
    assert (other.states.view(np.uint64) == base.states[dup].view(np.uint64)).all()
    assert (other.status == base.status[dup]).all()
    one = _device_call(cat, tuple(np.asarray(c)[[7]] for c in cand))
    assert (one.record.view(np.uint64) == base.record[[7]].view(np.uint64)).all()
    # pinned host buffers
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()  # noqa: E731
    pinned = conjunctions(pin(cat[0]), cand[0], cand[1], pin(cand[2]), pin(cand[3]), window_min=pin(cand[4]),
                          hbr_km=pin(cand[5]), covariance=pin(cat[1]), model=cat[2], states=True)
    assert (pinned.record.view(np.uint64) == base.record.view(np.uint64)).all()
    # device pointers
    dev = torch.device("cuda:0")
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
    m = 600
    rec, st = torch.zeros((m, 13), dtype=torch.float64, device=dev), torch.zeros((m, 2, 6), dtype=torch.float64, device=dev)
    sg, stat = torch.zeros((m, 2, 21), dtype=torch.float64, device=dev), torch.zeros(m, dtype=torch.uint8, device=dev)
    conjunctions_device(t(cat[0]), t(cat[1]), t(cat[2], torch.uint8),
                        t(cand[0], torch.int32), t(cand[1], torch.int32), t(cand[2]), t(cand[3]), t(cand[4]),
                        t(cand[5]), rec, st, sg, stat)
    torch.cuda.synchronize()
    assert (rec.cpu().numpy().view(np.uint64) == base.record.view(np.uint64)).all()
    assert (sg.cpu().numpy().view(np.uint64) == base.state_covariance.view(np.uint64)).all()
    assert (stat.cpu().numpy() == base.status).all()


def test_device_call_flags_bad_pairs(fitted):
    import torch

    from astroz_b200.collision import BAD_PAIR, conjunctions_device

    res, P = fitted
    n = res.elements.shape[1]
    dev = torch.device("cuda:0")
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
    pr, se = np.array([0, 5, n + 3]), np.array([0, 6, 1])
    rec = torch.full((3, 13), 7.0, dtype=torch.float64, device=dev)
    stat = torch.zeros(3, dtype=torch.uint8, device=dev)
    conjunctions_device(t(res.elements), t(P), t(res.deep_space.astype(np.uint8), torch.uint8), t(pr, torch.int32),
                        t(se, torch.int32), t(np.full(3, 2460000.5)), t(np.zeros(3)), t(np.ones(3)),
                        t(np.full(3, 0.01)), rec, None, None, stat)
    torch.cuda.synchronize()
    s = stat.cpu().numpy()
    assert s[0] == BAD_PAIR and s[2] == BAD_PAIR and s[1] != BAD_PAIR
    assert (rec.cpu().numpy()[[0, 2]] == 0.0).all()
