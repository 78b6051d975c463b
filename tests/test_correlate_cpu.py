"""K12 track correlation (az_correlate.cuh, az_correlate.cu) on the CPU.

The host build of the device source (tests/host_emul/emul_correlate.cu): its rows and d2 against the independent C
restatement on the oracle's SGP4 / SDP4 (tests/fit_oracle/correlate.c, the stacked form) and against a 40-digit mpmath
evaluation; its sums against the element fit's own; its selection against numpy brute force over the full d2 matrix;
the chi-square gate against scipy; the gate's coverage on draws from P; the C ABI's refusals.  The device runs are in
tests/test_gpu_correlate.py."""
import ctypes as C

import mpmath as mp
import numpy as np
import pytest

from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import correlate as cr
from tests.fit_oracle import covariance as K
from tests.fit_oracle import obs as O


@pytest.fixture(scope="module")
def L():
    lib = cr.emul_library()
    if lib is None:
        pytest.skip("nvcc unavailable")
    return lib


T0 = 2460000.25 + 0.3


@pytest.fixture(scope="module")
def scene():
    """4 rows (LEO, SSO, GEO, Molniya) with covariances; tracks of every kind, 1 .. 64 observations"""
    el, model = cr.base_rows()
    P = cc.P_words(4, scale=1.0, seed=7, deep=model == 1)
    rng = np.random.default_rng(1)
    per, owner = [], []
    for s in range(4):
        for kind, minutes, step in ((O.RADAR, 10, 20.0), (O.OPTICAL, 30, 30.0), (O.ECEF, 4, 60.0), (O.TEME, 0, 60.0)):
            for t0 in (T0, T0 + 0.25, T0 + 0.5, T0 + 0.75):
                tr = cr.track_of(el[:, s], kind, t0, minutes if s < 2 or kind != O.RADAR else 60,
                                 step if s < 2 else 120.0, rng=rng)
                if tr is not None and len(tr[0]):
                    per.append(tuple(a[:64] for a in tr))
                    owner.append(s)
    return el, model, P, cr.Tracks(per, O.RADAR_SITES), np.array(owner)


# ---- 1. per pair ----------------------------------------------------------------------------------------------------
def test_rows_and_d2_against_the_restatement(L, scene):
    """every kind, near-earth and deep-space rows, tracks of 1 .. 64 observations: z within 1e-5 sigma and G within 1e-5 of its scale
    (the two SGP4s differ by ~1e-9 km, magnified by the sigmas and the 1e-8 steps), d2 within 1e-5 relative"""
    el, model, P, tr, owner = scene
    worst = {"z": 0.0, "G": 0.0, "d2": 0.0}
    kinds, lens = set(), set()
    for j in range(tr.t):
        s = owner[j]
        z, G, _, _, d2 = cr.emul_pair(L, el, P, model, tr, s, j)
        rc, zr, Gr, d2r = cr.restated_pair(el, P, model, tr, s, j)
        assert rc == 0 and np.isfinite(d2)
        kinds.add(int(tr.kind[tr.offsets[j]]))
        lens.add(int(tr.offsets[j + 1] - tr.offsets[j]))
        Gt = np.transpose(G, (0, 2, 1))
        worst["z"] = max(worst["z"], np.max(np.abs(z - zr)) / max(1.0, np.max(np.abs(zr))))
        worst["G"] = max(worst["G"], np.max(np.abs(Gt - Gr)) / np.max(np.abs(Gr)))
        worst["d2"] = max(worst["d2"], abs(d2 - d2r) / max(1.0, d2r))
    print("host build vs restatement, worst:", {k: f"{v:.2e}" for k, v in worst.items()})
    assert kinds == {0, 1, 2, 3} and min(lens) == 1 and max(lens) >= 30
    assert worst["z"] < 1e-5 and worst["G"] < 1e-5 and worst["d2"] < 1e-5


def _mp_d2(z, G, P7):
    with mp.workdps(40):
        Zm, Gm, Pm = mp.matrix(z.tolist()), mp.matrix(G.tolist()), mp.matrix(P7.tolist())
        A = Gm * Pm * Gm.T
        for i in range(A.rows):
            A[i, i] += 1
        return float((Zm.T * mp.lu_solve(A, Zm))[0])


def test_d2_against_a_40_digit_evaluation(L, scene):
    """zT (I + G P GT)^-1 z on the stacked rows in 40 digits, for the fitted P, a singular P, P = 0 and P scaled by 1e4
    and 1e8 until |z|^2 / d2 passes 1e6.  The normal-matrix form squares the conditioning of the stacked one: within
    1e-6 relative at the fitted scale (measured 4.7e-13), 1e-3 at the inflated ones (measured 4e-4, where I + P N has a
    condition number near 1e16)"""
    el, model, P, tr, owner = scene
    rng = np.random.default_rng(2)
    worst, worst_big, ratio_max = 0.0, 0.0, 0.0
    for j in range(0, tr.t, 3):
        s = owner[j]
        if tr.offsets[j + 1] - tr.offsets[j] > 12:
            continue
        P7 = K.unpack7(P[s])
        v = rng.standard_normal(7)
        singular = P7 - np.outer(P7 @ v, P7 @ v) / (v @ P7 @ v)      # rank 6
        for big, Pc in ((0, P7), (0, singular), (0, np.zeros((7, 7))), (1, P7 * 1e4), (1, P7 * 1e8)):
            Pw = np.tile(K.pack7(Pc), (el.shape[1], 1))
            z, G, sums, _, d2 = cr.emul_pair(L, el, Pw, model, tr, s, j)
            zs, gs = cr.stacked(z, G, Pc)
            ref = _mp_d2(zs, gs, Pc) if np.any(Pc) else float(zs @ zs)
            err = abs(max(d2, 0.0) - ref) / ref
            if big:
                worst_big = max(worst_big, err)
            else:
                worst = max(worst, err)
            ratio_max = max(ratio_max, sums[0] / ref)
    print(f"d2 vs 40-digit: worst relative {worst:.2e} (fitted P), {worst_big:.2e} (inflated P), largest |z|^2/d2 "
          f"{ratio_max:.1e}")
    assert worst < 1e-6 and worst_big < 1e-3
    assert ratio_max > 1e6


# ---- 2. identities with the fit -------------------------------------------------------------------------------------
def test_sums_are_the_fits_and_zero_p_skips_the_stepped_sets(L, scene):
    """N and b equal fit_accumulate_obs's over the same observations bit for bit; |z|^2 equals its cost (to rounding:
    K8's TEME path sums the components in another order); with P = 0 the d2 is |z|^2 exactly and equals d2 with the
    stepped sets built under a P whose only nonzero word is negligible"""
    el, model, P, tr, owner = scene
    for j in range(tr.t):
        s = owner[j]
        z, G, sums, _, d2 = cr.emul_pair(L, el, P, model, tr, s, j)
        rc, fs = cr.emul_fit_sums(L, el, P, model, tr, s, j)
        assert rc == 0
        assert np.array_equal(sums[4:], fs[4:]), j
        assert abs(sums[0] - fs[0]) <= 1e-14 * fs[0]
        Z = np.zeros_like(P)
        z0, _, s0, _, d0 = cr.emul_pair(L, el, Z, model, tr, s, j)
        assert np.array_equal(z0, z) and d0 == s0[0] == sums[0]


def test_nominal_state_is_propagate_covariances(L, scene):
    from tests.fit_oracle import covariance as KV

    el, model, P, tr, owner = scene
    Lc = KV.emul_library()
    for j in range(0, tr.t, 5):
        s = owner[j]
        b, e = tr.offsets[j], tr.offsets[j + 1]
        _, _, _, f0, _ = cr.emul_pair(L, el, P, model, tr, s, j)
        off = np.zeros(el.shape[1] + 1, np.uint32)
        off[s + 1:] = e - b
        st, _, _, status = KV.emul(Lc, el, P, model, off, tr.jd[b:e], tr.fr[b:e])
        assert np.array_equal(st, f0) and np.all(status == 0)


@pytest.mark.parametrize("s, kind", [(0, O.RADAR), (2, O.OPTICAL)])
def test_a_fits_own_observations_against_its_own_row(L, s, kind):
    """a converged host-build fit (LEO from radar, GEO from optical angles) correlated with its own observations as one
    track against its own row and covariance: d2 = cost - b^T (I + P N)^-1 P b (the numpy statement on the pair's own
    sums, within 1e-9 of the cost), and b ~ 0 at the optimum, so d2 ~ wrms^2 x n_residuals (within 1e-6)"""
    el, model = cr.base_rows()
    truth = el[:, s]
    jd = np.full(1440, np.floor(T0 - 0.5) + 0.5)
    fr = (T0 - jd) + np.arange(1440) / 1440.0
    obs = O.tracks(truth, kind, O.RADAR_SITES, jd, fr)
    keep = np.sort(np.random.default_rng(6).choice(len(obs[0]), min(200, len(obs[0])), replace=False))
    jd_, fr_, kd, val, sig, sta = (a[keep] for a in obs)
    rng = np.random.default_rng(7)
    fin = np.isfinite(sig)
    val = val.copy()
    val[fin] += rng.standard_normal(fin.sum()) * sig[fin]
    val[:, 0 if kind == O.OPTICAL else 1] %= 2 * np.pi
    guess = truth.copy()
    guess[1] += 1e-6
    guess[6] += 0.002
    Lf = O.emul_library()
    off = np.array([0, len(jd_)], np.uint32)
    fitted, wrms, nres, cov, iters, status = O.emul_fit(Lf, guess[:, None], jd_, fr_, kd, val, sig, sta, off,
                                                        O.RADAR_SITES, fit_bstar=not model[s], mixed=True)
    assert status[0] == 0
    tr = cr.Tracks([(jd_, fr_, kd, val, sig, sta)], O.RADAR_SITES)
    _, _, sums, _, d2 = cr.emul_pair(L, fitted, cov, model[s:s + 1], tr, 0, 0)
    F, b = sums[0], sums[4 + 28:4 + 35]
    N, P = K.unpack7(sums[4:4 + 28]), K.unpack7(cov[0])
    ref = F - b @ np.linalg.solve(np.eye(7) + P @ N, P @ b)
    cost = wrms[0] ** 2 * nres[0]
    print(f"row {s}: d2 {d2:.9g}, cost - b^T(I+PN)^-1 Pb {ref:.9g}, wrms^2 n {cost:.9g} ({nres[0]} residuals)")
    assert abs(d2 - ref) <= 1e-9 * F
    assert abs(d2 - cost) <= 1e-6 * cost


# ---- 3. selection ----------------------------------------------------------------------------------------------------
def test_selection_against_brute_force(L, scene):
    el, model, P, tr, owner = scene
    # duplicated rows make exact ties; a row that cannot be built (a near-earth set under model 1) takes no part
    dup = [0, 2, 0, 3, 1, 2]
    el2 = np.concatenate([el, el[:, dup]], axis=1)
    P2 = np.concatenate([P, P[dup]])
    md2 = np.concatenate([model, model[dup]])
    md2[-2] = 1                              # row 1 (near-earth) under the deep-space model: INIT_FAILED
    for best in (1, 4, 8):
        rows, d2, used, ng, nf, status, rs, full = cr.emul(L, el2, P2, md2, tr, best=best, full=True)
        assert rs[-2] == 1 and np.all(np.delete(rs, -2) == 0)
        for j in range(tr.t):
            gate = L.emul_chi2_quantile(int(used[j]), 0.999)
            ok = np.flatnonzero(np.isfinite(full[j]))
            order = ok[np.lexsort((ok, full[j][ok]))][:best]
            want_rows = np.full(best, cr.EMPTY, np.uint32)
            want_rows[:len(order)] = order
            assert np.array_equal(rows[j], want_rows)
            assert np.array_equal(d2[j][:len(order)], full[j][order])
            assert ng[j] == np.sum(full[j][ok] <= gate)
            assert nf[j] == np.sum(np.isnan(full[j])) - 1
            assert status[j] == (0 if ng[j] else 1)
        if best == 1:
            continue
        ties = [j for j in range(tr.t) if np.sum(full[j] == full[j][rows[j][0]]) > 1]
        assert ties   # the duplicates tie, and the lower row index comes first
        for j in ties:
            assert rows[j][0] < rows[j][1] and d2[j][0] == d2[j][1]


# ---- 4. the gate ------------------------------------------------------------------------------------------------------
def test_chi2_quantile_against_scipy(L):
    from scipy.stats import chi2

    worst = 0.0
    for p in (0.9, 0.99, 0.999, 0.9999):
        ks = np.arange(1, 1537)
        ref = chi2.ppf(p, ks)
        got = np.array([L.emul_chi2_quantile(int(k), p) for k in ks])
        worst = max(worst, np.max(np.abs(got - ref) / ref))
    print(f"chi2 quantile vs scipy: worst relative {worst:.2e}")
    assert worst < 1e-12


# ---- 5. statistics --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [O.RADAR, O.OPTICAL])
def test_true_row_falls_inside_the_gate_at_its_probability(L, kind):
    """rows drawn as truth + a sample of P: the truth's noisy track falls inside the p-gate of its row in a fraction
    within 4 sigma of p (k = 4L radar, 2L optical; 2,000 tracks each)"""
    el, model = cr.base_rows()
    s = 0 if kind == O.RADAR else 2
    truth = el[:, s]
    deep = bool(model[s])
    p, N = 0.99, 2000
    P = cc.P_words(1, scale=0.3, seed=11, deep=[deep])[0]
    P7 = K.unpack7(P)
    Lc = np.linalg.cholesky(P7 + 1e-30 * np.eye(7))
    x0 = O.fit_vars(truth, deep)
    rng = np.random.default_rng(5)
    inside = 0
    tracks = []
    for q in range(20 * N):
        tr = cr.track_of(truth, kind, T0 + rng.uniform(0.0, 1.0), 6 if kind == O.RADAR else 20, 60.0, rng=rng)
        if tr is not None and len(tr[0]):
            tracks.append(tr)
        if len(tracks) == N:
            break
    rows = []
    for q in range(len(tracks)):
        x = x0 + Lc @ rng.standard_normal(7)
        rows.append(K.elements_of(x, truth[0], deep))
    cat = np.stack(rows, axis=1)
    for q, t in enumerate(tracks):
        tr = cr.Tracks([t], O.RADAR_SITES)
        _, _, _, _, d2 = cr.emul_pair(L, cat[:, q:q + 1], P[None], np.array([model[s]]), tr, 0, 0)
        k = int(np.sum(np.isfinite(t[4])))
        inside += d2 <= L.emul_chi2_quantile(k, p)
    n = len(tracks)
    sd = np.sqrt(p * (1 - p) / n)
    print(f"kind {kind}: {inside} of {n} inside the {p} gate ({inside / n:.4f}, 4 sigma = {4 * sd:.4f})")
    assert n >= 2000
    assert abs(inside / n - p) <= 4 * sd


# ---- 6. the C ABI ----------------------------------------------------------------------------------------------------
def _abi_call(el, cov, model, tr, *, gate=0.999, best=4, grav=1, device=0, offsets=None):
    from astroz_b200._lib import lib

    n, t = el.shape[1], tr.t
    off = tr.offsets if offsets is None else np.ascontiguousarray(offsets, np.uint32)
    outs = [np.full((t, best), 7, np.uint32), np.full((t, best), 7.0), np.full(t, 7, np.uint32),
            np.full(t, 7, np.uint32), np.full(t, 7, np.uint32), np.full(t, 7, np.uint8), np.full(n, 7, np.uint8)]
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    rc = lib().astroz_cuda_correlate(p(el), n, grav, p(cov), p(model), p(off), t, p(tr.jd), p(tr.fr), p(tr.kind),
                                     p(tr.value), p(tr.sigma), p(tr.station), len(tr.jd), p(tr.stations),
                                     len(tr.stations), gate, best, device, *[p(o) for o in outs])
    return rc, outs


def test_abi_refusals_write_nothing(scene):
    from astroz_b200._abi import DEFINES as D

    el, model, P, tr, owner = scene
    el, P = np.ascontiguousarray(el), np.ascontiguousarray(P)
    VE = D["ASTROZ_VALUE_ERROR"]

    def refused(**kw):
        e, c, m_, t = kw.pop("el", el), kw.pop("cov", P), kw.pop("model", model), kw.pop("tr", tr)
        rc, outs = _abi_call(e, c, m_, t, **kw)
        assert rc == VE, kw
        assert all(np.all(o == 7) for o in outs)

    def with_obs(**change):
        t = cr.Tracks([(tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station)], tr.stations)
        t.offsets = tr.offsets.copy()
        t.t = tr.t
        for k, v in change.items():
            setattr(t, k, v)
        return t

    refused(grav=7)
    refused(device=-1)
    refused(best=0)
    refused(best=9)
    refused(gate=0.0)
    refused(gate=1.0)
    bad = tr.offsets.copy()
    bad[2], bad[3] = bad[3], bad[2]
    refused(offsets=bad)                                   # decreasing
    bad = tr.offsets.copy()
    bad[-1] -= 1
    refused(offsets=bad)                                   # not ending at m
    bad = tr.offsets.copy()
    bad[1] = bad[0]
    refused(offsets=bad)                                   # an empty track
    long = cr.Tracks([tuple(np.concatenate([a] * 300)[:257] for a in
                            (tr.jd[:1], tr.fr[:1], tr.kind[:1], tr.value[:1], tr.sigma[:1], tr.station[:1]))],
                     tr.stations)
    refused(tr=long)                                       # longer than 256 observations
    sig = tr.sigma.copy()
    sig[tr.offsets[0]:tr.offsets[1]] = np.inf
    refused(tr=with_obs(sigma=sig))                        # k = 0
    kd = tr.kind.copy()
    kd[0] = 4
    refused(tr=with_obs(kind=kd))                          # unknown kind
    sta = tr.station.copy()
    sta[np.flatnonzero(tr.kind == O.RADAR)[0]] = 99
    refused(tr=with_obs(station=sta))                      # station index
    sig = tr.sigma.copy()
    sig[0, 0] = -1.0
    refused(tr=with_obs(sigma=sig))                        # sigma <= 0
    val = tr.value.copy()
    val[0, 0] = np.nan
    refused(tr=with_obs(value=val))                        # a used value not finite
    jd = tr.jd.copy()
    jd[0] = np.inf
    refused(tr=with_obs(jd=jd))                            # time
    e2 = el.copy()
    e2[1, 0] = np.nan
    refused(el=e2)                                         # element
    c2 = P.copy()
    c2[0, 0] = np.inf
    refused(cov=c2)                                        # covariance word
    m2 = model.copy()
    m2[0] = 2
    refused(model=m2)                                      # model byte
