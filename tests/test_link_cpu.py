"""K17 track linking on the CPU: the host build of the device source (tests/host_emul/emul_link.cu) against exact
two-body truth and against an independent numpy restatement (tests/fit_oracle/link.py, K9's C statement for Lambert);
pair symmetry and batch invariance; statuses; the C ABI's refusals."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from tests.fit_oracle import correlate as cr
from tests.fit_oracle import iod as I
from tests.fit_oracle import link as K
from tests.fit_oracle import obs as O

MU, RE = I.MU[1], I.RE[1]
R_MIN, R_MAX = 6578.0, 50000.0
T0 = 2460000.5 + 0.3


@pytest.fixture(scope="module")
def L():
    lib = K.emul_library()
    if lib is None:
        pytest.skip("nvcc unavailable")
    return lib


def _site_under(s, jdf, lat, dlon):
    """a site at latitude lat, dlon degrees east of the sub-satellite longitude of s at jdFull jdf"""
    r = O.rot(O.gmst(np.array([jdf])))[0] @ s[:3]
    return np.array([lat, np.rad2deg(np.arctan2(r[1], r[0])) + dlon, 0.3])


def _pair(s0, gap, kinds=(O.OPTICAL, O.OPTICAL), n=12, span=55 * 60.0, sites=((20.0, 10.0), (-10.0, -5.0))):
    """two noise-free tracks of the exact two-body orbit s0 (state at T0): the first from T0, the second gap seconds
    later, n observations over span seconds each, each from a site near the sub-satellite point at its start.  Returns
    (tracks, true state at the second track's anchor, true (revs, retrograde))."""
    per, st, truth = [], [], []
    for k, (kind, (lat, dlon)) in enumerate(zip(kinds, sites)):
        t0 = T0 + k * gap / 86400.0
        site = _site_under(I.kepler(s0, k * gap, MU), t0, lat, dlon)
        tp, S = K.two_body_track(s0, t0, kind, site, np.linspace(0.0, span, n), t_state=T0)
        per.append(tp)
        st.append(site)
        truth.append(S)
    tr = K.tracks_with_sites(per, st)
    a = 1.0 / (2.0 / np.linalg.norm(s0[:3]) - s0[3:] @ s0[3:] / MU)
    period = 2 * np.pi * np.sqrt(a ** 3 / MU)
    anchor_gap = gap   # both anchors are the middle observation of equal tracks
    revs = int(anchor_gap // period)
    retro = int(np.cross(s0[:3], s0[3:])[2] < 0)
    return tr, truth[1][n // 2], (revs, retro)


# the noise-free cases: (name, elements a, e, i deg, gap seconds, kinds, n, span, r_max)
CASES = [("GEO same night", (42164.0, 0.0002, 0.05), 2 * 3600.0, (O.OPTICAL, O.OPTICAL), 12, 3300.0, R_MAX),
         ("GEO next night", (42164.0, 0.0002, 0.05), 86400.0, (O.OPTICAL, O.OPTICAL), 12, 3300.0, R_MAX),
         ("GEO next night, inclined", (42164.0, 0.0003, 5.0), 86400.0 - 1800.0, (O.OPTICAL, O.OPTICAL), 12, 3300.0,
          R_MAX),
         ("GPS", (26560.0, 0.01, 55.0), 6 * 3600.0, (O.OPTICAL, O.OPTICAL), 12, 3300.0, R_MAX),
         ("Molniya", (26600.0, 0.7, 63.4), 3 * 3600.0, (O.OPTICAL, O.OPTICAL), 12, 3300.0, 60000.0),
         ("LEO, two stations in one pass", (7000.0, 0.001, 51.6), 420.0, (O.OPTICAL, O.OPTICAL), 12, 180.0, R_MAX),
         ("radar then optical", (26560.0, 0.01, 55.0), 4 * 3600.0, (O.RADAR, O.OPTICAL), 12, 3300.0, R_MAX),
         ("optical then radar, LEO", (7200.0, 0.002, 98.0), 600.0, (O.OPTICAL, O.RADAR), 10, 240.0, R_MAX)]
# Measured worst |state - truth| component over the cases: position 1.6e-10 km (GEO), velocity 1.2e-12 km/s; asserted
# at K13's 1e-8 km for exact two-body tracks, and 1e-10 km/s.
POS_TOL, VEL_TOL = 1e-8, 1e-10


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_noise_free_pairs_recover_the_truth(L, case):
    name, (a, e, i), gap, kinds, n, span, r_max = case
    s0 = I.coe2rv(a, e, np.deg2rad(i), 0.7, 0.4, 0.2, MU)
    tr, truth, (revs, retro) = _pair(s0, gap, kinds, n, span)
    o = K.emul(L, tr, [[0, 1]], R_MIN, r_max, max_revs=1)
    dr = np.abs(o["state"][0, :3] - truth[:3]).max()
    dv = np.abs(o["state"][0, 3:] - truth[3:]).max()
    print(f"{name}: status {o['status'][0]} revs {o['revs'][0]} flags {o['flags'][0]} hypotheses "
          f"{o['hypotheses'][0]} wrms {o['wrms'][0]:.2e} |dr| {dr:.2e} km |dv| {dv:.2e} km/s")
    assert o["status"][0] == K.OK
    assert o["revs"][0] == revs and (o["flags"][0] & K.RETROGRADE) == retro * K.RETROGRADE
    assert dr <= POS_TOL and dv <= VEL_TOL
    assert o["elements"][0, 0] == tr.jd[tr.offsets[1] + n // 2] + tr.fr[tr.offsets[1] + n // 2]
    assert o["used"][0] == sum(len(O.RADAR_SIGMA) if k == O.RADAR else 2 for k in kinds for _ in range(n))


def test_range_bounds_and_grid(L):
    """The range interval's ends within 1e-12 relative of numpy's polynomial roots; the grid geometric with exact
    ends"""
    s0 = I.coe2rv(42164.0, 0.0002, 0.05, 0.7, 0.4, 0.2, MU)
    tr, _, _ = _pair(s0, 7200.0)
    for j in (0, 1):
        idx, t, R, Lv, lo, hi, n = K.emul_anchor(L, tr, j, R_MIN, R_MAX)
        assert idx == tr.offsets[j] + 6 and n == K.RANGES
        for r, got in ((R_MIN, lo), (R_MAX, hi)):
            ref = K.range_roots(R, Lv, r)
            assert abs(got - ref) <= 1e-12 * ref
            assert abs(np.linalg.norm(R + got * Lv) - r) <= 1e-12 * r
        g = np.array([L.emul_link_range(lo, hi, n, k) for k in range(n)])
        assert g[0] == lo and g[-1] == hi
        np.testing.assert_allclose(g[1:] / g[:-1], (hi / lo) ** (1.0 / (n - 1)), rtol=1e-13)


@pytest.mark.parametrize("case", [0, 1, 6], ids=["GEO same night", "GEO next night", "radar then optical"])
def test_probe_scores_and_seeds_match_the_restatement(L, case):
    """Every admissible hypothesis of the pair: the same keys as the restatement (K9's C statement for Lambert, K13's
    admissibility restated), F_probe within 1e-9 relative (plus 1e-9 absolute for the near-zero scores at the truth),
    and the host build's seeds are the restatement's kLinkSeeds least"""
    name, (a, e, i), gap, kinds, n, span, r_max = CASES[case]
    s0 = I.coe2rv(a, e, np.deg2rad(i), 0.7, 0.4, 0.2, MU)
    tr, _, _ = _pair(s0, gap, kinds, n, span)
    keys, F, states, probes = K.emul_hypotheses(L, tr, 0, 1, R_MIN, r_max)
    anchors = {}
    for j in (0, 1):
        idx, t, R, Lv, lo, hi, nh = K.emul_anchor(L, tr, j, R_MIN, r_max)
        anchors[j] = (idx, R, Lv, lo if nh == 1 else None)
    ref = K.restated_hypotheses(tr, 0, 1, R_MIN, r_max, anchors)
    assert sorted(keys.tolist()) == sorted(ref)
    worst = 0.0
    for k, f in zip(keys, F):
        worst = max(worst, abs(f - ref[int(k)]) / max(ref[int(k)], 1.0))
    assert worst <= 1e-9, worst
    seeds = K.emul(L, tr, [[0, 1]], R_MIN, r_max)["seed_key"][0]
    want = sorted(ref, key=lambda k: (ref[k], k))[:K.SEEDS]
    assert list(seeds) == want
    print(f"{name}: {len(keys)} hypotheses, worst F_probe difference {worst:.2e}; probes {list(probes)}")


def _scene():
    """four optical GEO tracks (two objects, two nights each) and a GPS radar + optical pair"""
    per, sites = [], []
    for q, (a, e, i) in enumerate([(42164.0, 0.0002, 0.05), (42164.0, 0.0004, 2.0), (26560.0, 0.01, 55.0)]):
        s0 = I.coe2rv(a, e, np.deg2rad(i), 0.7 + q, 0.4, 0.2 + q, MU)
        gap = 86400.0 if q < 2 else 4 * 3600.0
        kinds = (O.OPTICAL, O.OPTICAL) if q < 2 else (O.RADAR, O.OPTICAL)
        tr, _, _ = _pair(s0, gap + 600.0 * q, kinds)
        for j in (0, 1):
            per.append(tuple(x[tr.offsets[j]:tr.offsets[j + 1]] for x in (tr.jd, tr.fr, tr.kind, tr.value, tr.sigma,
                                                                          tr.station)))
            sites.append(tr.stations[j])
    return K.tracks_with_sites(per, sites)


def test_pair_order_and_batches_do_not_change_the_bytes(L):
    tr = _scene()
    pairs = np.array([(a, b) for a in range(tr.t) for b in range(a + 1, tr.t)])
    full = K.emul(L, tr, pairs, R_MIN, R_MAX)
    fields = ("elements", "state", "rho", "revs", "flags", "wrms", "used", "hypotheses", "conv", "deep", "status")

    def same(o, picks):
        for f in fields:
            x = full[f][:, picks] if f == "elements" else full[f][picks]
            assert x.tobytes() == o[f].tobytes(), f

    same(K.emul(L, tr, pairs[:, ::-1], R_MIN, R_MAX), np.arange(len(pairs)))
    perm = np.random.default_rng(4).permutation(len(pairs))
    same(K.emul(L, tr, pairs[perm], R_MIN, R_MAX), perm)
    half = len(pairs) // 2
    same(K.emul(L, tr, pairs[half:], R_MIN, R_MAX), np.arange(half, len(pairs)))
    dup = np.concatenate([np.arange(len(pairs)), [0, 3, 3]])
    same(K.emul(L, tr, pairs[dup], R_MIN, R_MAX), dup)
    ok = full["status"] == K.OK
    print(f"{len(pairs)} pairs, statuses {np.bincount(full['status'], minlength=6)}")
    assert ok[[0, 5, 14]].all()   # the three true pairs (0, 1), (2, 3), (4, 5)


def test_every_status(L):
    s0 = I.coe2rv(42164.0, 0.0002, 0.05, 0.7, 0.4, 0.2, MU)
    tr, _, _ = _pair(s0, 7200.0)
    base = [tuple(x[tr.offsets[j]:tr.offsets[j + 1]] for x in (tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station))
            for j in (0, 1)]
    one_angle = list(base[1])
    one_angle[4] = one_angle[4].copy()
    one_angle[4][:, 1] = np.inf                                    # declinations unused: no anchor
    rev = tuple(x[::-1] for x in base[1])                          # out of time order
    same_t = list(base[1])
    same_t[0], same_t[1] = base[0][0].copy(), base[0][1].copy()    # the first track's times
    sc = K.tracks_with_sites([base[0], base[1], tuple(one_angle), rev, tuple(same_t)], tr.stations)
    pairs = [[0, 1], [0, 2], [0, 3], [0, 4], [1, 1], [0, 9]]
    o = K.emul(L, sc, pairs, R_MIN, R_MAX)
    assert list(o["status"]) == [K.OK, K.TOO_FEW, K.BAD_TRACK, K.BAD_PAIR, K.BAD_PAIR, K.BAD_PAIR]
    for q in range(1, 6):
        assert o["hypotheses"][q] == 0 and o["used"][q] == 0
        assert not o["state"][q].any() and not o["elements"][:, q].any()
    # NO_CANDIDATE: two TEME positions 60 s apart and 5,000 km away from each other: every transfer is hyperbolic
    st = np.full((1, 6), np.inf)
    st[0, :3] = 1e-3
    p1 = (np.array([2460000.5]), np.array([0.3]), np.zeros(1, np.uint8), np.array([[7000.0, 0, 0, 0, 0, 0]]), st,
          np.zeros(1, np.uint32))
    p2 = (np.array([2460000.5]), np.array([0.3 + 60 / 86400]), np.zeros(1, np.uint8),
          np.array([[7000.0, 5000.0, 0, 0, 0, 0]]), st, np.zeros(1, np.uint32))
    o = K.emul(L, cr.Tracks([p1, p2], tr.stations), [[0, 1]], R_MIN, R_MAX)
    assert o["status"][0] == K.NO_CANDIDATE and o["hypotheses"][0] == 0 and o["used"][0] == 6
    # CONVERSION_FAILED: TEME positions of an exact two-body orbit of 224.95 min osculating period: the osculating set
    # is a deep-space one (its mean motion crosses 225 min), and the fit under SDP4 cannot reach the state
    a = (MU * (224.95 * 60.0 / (2 * np.pi)) ** 2) ** (1.0 / 3.0)
    s0 = I.coe2rv(a, 0.001, np.deg2rad(30.0), 0.1, 0.0, 0.0, MU)
    per = []
    for dt in (0.0, 600.0):
        s = I.kepler(s0, dt, MU)
        per.append((np.array([2460000.5]), np.array([0.3 + dt / 86400]), np.zeros(1, np.uint8),
                    np.concatenate([s[:3], np.zeros(3)])[None], st, np.zeros(1, np.uint32)))
    o = K.emul(L, cr.Tracks(per, tr.stations), [[0, 1]], R_MIN, R_MAX)
    assert o["status"][0] == K.CONVERSION_FAILED, o["status"]
    assert o["state"][0].any() and o["conv"][0].any()


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def _abi(tr, pairs, *, r_min=R_MIN, r_max=R_MAX, max_revs=1, grav=1, device=0, bstar=None, offsets=None,
         stations=None):
    from astroz_b200._lib import lib

    pairs = np.ascontiguousarray(np.asarray(pairs, np.uint32).reshape(-1, 2))
    p = len(pairs)
    off = tr.offsets if offsets is None else np.ascontiguousarray(offsets, np.uint32)
    sta = tr.stations if stations is None else np.ascontiguousarray(stations, np.float64)
    outs = [np.full((8, p), 7.0), np.full((p, 6), 7.0), np.full((p, 2), 7.0), np.full(p, 7, np.uint8),
            np.full(p, 7, np.uint8), np.full(p, 7.0), np.full(p, 7, np.uint32), np.full(p, 7, np.uint32),
            np.full((p, 2), 7.0), np.full(p, 7, np.uint8), np.full(p, 7, np.uint8)]
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    rc = lib().astroz_cuda_link_tracks(ptr(off), tr.t, ptr(tr.jd), ptr(tr.fr), ptr(tr.kind), ptr(tr.value),
                                       ptr(tr.sigma), ptr(tr.station), len(tr.jd), ptr(sta), len(sta), ptr(pairs), p,
                                       ptr(bstar), C.c_double(r_min), C.c_double(r_max), max_revs, grav, device,
                                       *[ptr(o) for o in outs])
    return rc, outs


def test_abi_refusals_write_nothing():
    from astroz_b200._abi import DEFINES as D

    VE = D["ASTROZ_VALUE_ERROR"]
    s0 = I.coe2rv(42164.0, 0.0002, 0.05, 0.7, 0.4, 0.2, MU)
    tr, _, _ = _pair(s0, 7200.0)
    base = [tuple(x[tr.offsets[j]:tr.offsets[j + 1]] for x in (tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station))
            for j in (0, 1)]
    same_t = list(base[1])
    same_t[0], same_t[1] = base[0][0].copy(), base[0][1].copy()
    three = K.tracks_with_sites([base[0], base[1], tuple(same_t)], np.concatenate([tr.stations, tr.stations[:1]]))

    def refused(t=tr, pairs=((0, 1),), **kw):
        rc, outs = _abi(t, pairs, **kw)
        assert rc == VE, kw
        assert all(np.all(o == 7) for o in outs)

    def with_obs(**change):
        t = cr.Tracks([(tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station)], tr.stations)
        t.offsets, t.t = tr.offsets.copy(), tr.t
        for k, v in change.items():
            setattr(t, k, v)
        return t

    refused(pairs=((0, 2),))
    refused(pairs=((1, 1),))
    refused(three, pairs=((0, 1), (0, 2)))                    # equal anchor times
    refused(max_revs=128)
    refused(r_min=6300.0)                                      # not above the stations' radius
    refused(r_min=np.nan)
    refused(r_max=R_MIN)
    refused(r_max=np.inf)
    refused(bstar=np.array([np.nan]))
    refused(grav=7)
    refused(device=-1)
    bad = tr.offsets.copy()
    bad[1] = bad[0]
    refused(offsets=bad)
    bad = tr.offsets.copy()
    bad[-1] -= 1
    refused(offsets=bad)
    sig = tr.sigma.copy()
    sig[tr.offsets[0]:tr.offsets[1]] = np.inf
    refused(with_obs(sigma=sig))
    kd = tr.kind.copy()
    kd[0] = 4
    refused(with_obs(kind=kd))
    sta = tr.station.copy()
    sta[0] = 99
    refused(with_obs(station=sta))
    val = tr.value.copy()
    val[0, 0] = np.nan
    refused(with_obs(value=val))
    sig = tr.sigma.copy()
    sig[0, 0] = -1.0
    refused(with_obs(sigma=sig))
    # valid input gets past every check: without a device that is NO_DEVICE, with one OK
    rc, outs = _abi(tr, ((0, 1), (1, 0)))
    assert rc in (D["ASTROZ_OK"], D["ASTROZ_NO_DEVICE"])


def test_python_pair_selection():
    """anchor_times restates the anchor rule in numpy; candidate_pairs takes every pair within the gap"""
    from astroz_b200.iod import anchor_times, candidate_pairs

    tr = _scene()
    at = anchor_times(tr.track_ids(), tr.jd, tr.fr, tr.kind, tr.sigma)
    L = K.emul_library()
    if L is not None:
        for j in range(tr.t):
            assert at[j] == K.emul_anchor(L, tr, j, R_MIN, R_MAX)[1]
    pr = candidate_pairs(at, 1.5)
    ref = [(a, b) for a in range(tr.t) for b in range(a + 1, tr.t) if abs(at[a] - at[b]) <= 1.5 and at[a] != at[b]]
    assert [tuple(x) for x in pr] == ref


def test_fit_links_chooses_each_tracks_best_links():
    """best_links ranks every OK link once within each of its tracks, over all of that track's OK links: with best = 1
    the chosen links are each track's least-wrms link, whichever column the track is in"""
    from astroz_b200.iod import LINK_NO_CANDIDATE, LINK_OK, best_links

    pairs = np.array([(0, 1), (0, 2), (1, 2), (1, 3), (2, 3)])
    wrms = np.array([5.0, 1.0, 2.0, 3.0, 4.0])
    ok = np.full(5, LINK_OK, np.uint8)
    # track 0: (0, 2); track 1: (1, 2); track 2: (0, 2); track 3: (1, 3)
    assert best_links(pairs, wrms, ok, 1).tolist() == [1, 2, 3]
    assert best_links(pairs, wrms, ok, 2).tolist() == [0, 1, 2, 3, 4]
    # a link that is not OK is neither chosen nor ranked: track 0's best is then (0, 1), track 2's (1, 2)
    st = ok.copy()
    st[1] = LINK_NO_CANDIDATE
    assert best_links(pairs, wrms, st, 1).tolist() == [0, 2, 3]
    # equal wrms: the lower link index first (tracks 0 and 1: (0, 1), track 2: (0, 2), track 3: (1, 3)); the pair's
    # column order does not matter
    assert best_links(pairs[:, ::-1], np.ones(5), ok, 1).tolist() == best_links(pairs, np.ones(5), ok, 1).tolist() \
        == [0, 1, 3]
    assert best_links(np.zeros((0, 2), int), np.zeros(0), np.zeros(0, np.uint8), 4).tolist() == []
    # against a direct statement of the rule on random links
    rng = np.random.default_rng(7)
    for _ in range(20):
        t, p = 12, 40
        pr = np.array([rng.choice(t, 2, replace=False) for _ in range(p)])
        w = rng.uniform(0.5, 5.0, p).round(1)
        st = np.where(rng.uniform(size=p) < 0.8, LINK_OK, LINK_NO_CANDIDATE).astype(np.uint8)
        for b in (1, 2, 4):
            want = set()
            for j in range(t):
                mine = [q for q in range(p) if st[q] == LINK_OK and j in pr[q]]
                want |= set(sorted(mine, key=lambda q: (w[q], q))[:b])
            assert best_links(pr, w, st, b).tolist() == sorted(want)
