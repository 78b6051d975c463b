"""K14 Monte Carlo collision probability (az_conjunction_mc.cuh, az_conjunction_mc.cu) on the CPU.

The host build of the device source (tests/host_emul/emul_conjunction_mc.cu) against the independent numpy statement of
the draws (tests/fit_oracle/conjunction_mc.py): Philox known answers and a million counters, the normals, the factor's
rules and the draws' covariance; per sample against each drawn pair assessed by the C restatement of K11 with P = 0;
the zero-P, split-range and batch invariants; the C ABI's refusals and the Python wrapper.  The device runs are in
tests/test_gpu_conjunction_mc.py."""
import ctypes as C

import numpy as np
import pytest

from tests.fit_oracle import conjunction as cj
from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import conjunction_mc as mc
from tests.fit_oracle.covariance import pack7

KAT = [  # Random123's known answers for Philox4x32-10: counter, key, output
    ([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
    ([0xFFFFFFFF] * 4, [0xFFFFFFFF] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
     [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]),
]


@pytest.fixture(scope="module")
def L():
    lib = mc.emul_library()
    if lib is None:
        pytest.skip("nvcc unavailable")
    return lib


# ---- 1. the generator -----------------------------------------------------------------------------------------------
def test_philox_known_answers(L):
    ctr = np.array([k[0] for k in KAT], np.uint32)
    key = np.array([k[1] for k in KAT], np.uint32)
    want = np.array([k[2] for k in KAT], np.uint32)
    assert (mc.philox(ctr, key) == want).all()
    assert (mc.emul_philox(L, ctr, key) == want).all()


def test_philox_and_normals_match_the_statement(L):
    """10^6 random counters and keys bit for bit; the 14 normals of 10^5 samples within 4 ulp"""
    rng = np.random.default_rng(7)
    ctr = rng.integers(0, 2 ** 32, (10 ** 6, 4), dtype=np.uint64).astype(np.uint32)
    key = rng.integers(0, 2 ** 32, (10 ** 6, 2), dtype=np.uint64).astype(np.uint32)
    assert np.array_equal(mc.emul_philox(L, ctr, key), mc.philox(ctr, key))
    for seed in (0, 0x123456789ABCDEF0):
        k = np.concatenate([np.arange(50000, dtype=np.uint64),
                            rng.integers(0, 2 ** 63, 50000, dtype=np.uint64) * np.uint64(2)])
        got, ref = mc.emul_normals(L, seed, k), mc.normals(seed, k)
        ulp = np.abs(got - ref) / np.spacing(np.abs(ref))
        print(f"normals, seed {seed:#x}: worst {ulp.max():.1f} ulp, mean {got.mean():+.4f}, var {got.var():.4f}")
        assert ulp.max() <= 4
        assert abs(ref.mean()) < 5 / np.sqrt(ref.size) and abs(ref.var() - 1) < 5 * np.sqrt(2 / ref.size)


# ---- 2. the factor and the draws ------------------------------------------------------------------------------------
D7 = np.array([1e-7, 1e-6, 1e-6, 1e-5, 1e-5, 1e-5, 1e-5])


def _P(S, d=D7):
    return pack7(S * np.outer(d, d))


def _unit(rng, rank=7):
    A = rng.standard_normal((7, rank))
    S = A @ A.T
    return S / np.sqrt(np.outer(np.diag(S), np.diag(S)))


def _pair(rho2):
    """unit-diagonal S whose (1, 2) pivot is 1 - rho2"""
    S = np.eye(7)
    S[1, 2] = S[2, 1] = np.sqrt(rho2)
    return S


CASES = {
    "full rank": lambda rng: (_P(_unit(rng)), True, 7),
    "B* held": lambda rng: (_P(_unit(rng), D7 * (np.arange(7) < 6)), True, 6),
    "rank 3": lambda rng: (_P(_unit(rng, 3)), True, 3),
    "zero P": lambda rng: (np.zeros(28), True, 0),
    "zero-variance variable": lambda rng: (_P(_unit(rng), D7 * (np.arange(7) != 3)), True, 6),
    "pivot -0.5e-12": lambda rng: (_P(_pair(1 + 0.5e-12)), True, 6),
    "pivot -2e-12": lambda rng: (_P(_pair(1 + 2e-12)), False, None),
}


@pytest.mark.parametrize("case", list(CASES))
def test_factor_rules(L, case):
    """The host build's factor equals the statement's, with the same PSD verdict and rank; L L^T reproduces S"""
    P, psd, rank = CASES[case](np.random.default_rng(3))
    sd, Lm, ok = mc.emul_factor(L, P)
    rsd, rL, rok = mc.factor(P)
    assert ok == rok == psd
    if not psd:
        return
    assert np.array_equal(sd, rsd)
    assert np.abs(Lm - rL).max() <= 1e-12
    assert np.linalg.matrix_rank(Lm, tol=1e-9) == rank
    nv = mc.nvar_of(P)
    live = np.flatnonzero(sd[:nv] > 0)
    S = np.zeros((7, 7))
    Pm = mc.unpack7(P)
    S[np.ix_(live, live)] = Pm[np.ix_(live, live)] / np.outer(sd[live], sd[live])
    assert np.abs(Lm @ Lm.T - S).max() <= 1e-12


@pytest.mark.parametrize("case", ["full rank", "B* held", "rank 3", "zero P"])
def test_draws_have_covariance_P(L, case):
    """20,000 draws of a LEO row: the host build's draws equal the statement's within 1e-15 of scale, and their sample
    covariance is P by a chi-square bound at 1e-6 on the whitened draws (over the factor's rank)"""
    from scipy.stats import chi2

    P, _, rank = CASES[case](np.random.default_rng(3))
    e = cc.leo()
    k = np.arange(20000, dtype=np.uint64)
    x, st = mc.emul_draw(L, e, 0, P, 99, 0, k)
    ref = mc.draws(e, False, P, 99, 0, k)
    assert st == 0
    assert (np.abs(x - ref) <= 1e-15 * np.maximum(np.abs(ref), 1e-3)).all()
    dx = ref - mc.vars_of(e, False)
    if rank == 0:
        assert (dx == 0).all()
        return
    sd, Lm, _ = mc.factor(P)
    cols = np.flatnonzero(np.abs(np.diag(Lm)) > 0)
    Lr = Lm[:, cols] * sd[:, None]
    w = np.linalg.lstsq(Lr, dx.T, rcond=None)[0].T     # whitened draws: N(0, I_rank)
    # the draws lie in the factor's span, to the rounding of x^ + dx and the solve's
    tol = 8 * np.spacing(np.maximum(np.abs(ref), np.abs(mc.vars_of(e, False)))) + 1e-9 * np.abs(dx).max(axis=0)
    assert (np.abs(dx - w @ Lr.T) <= tol).all()
    n = len(w)
    Wc = w.T @ w / n
    T = n / 2.0 * ((Wc - np.eye(rank)) ** 2).sum()
    bound = chi2.ppf(1 - 1e-6, rank * (rank + 1) // 2)
    print(f"{case}: rank {rank}, T {T:.1f} (bound {bound:.1f})")
    assert T < bound


# ---- 3. per sample against the restatement ---------------------------------------------------------------------------
def _high_pc_leo(L):
    el, P, hbr = cc.high_pc_leo(lambda el, P, hbr: cj.emul(cj.emul_library(), el, P, np.zeros(2, np.uint8), [0], [1],
                                                           *_guess(el, 0), [1.0], hbr)[0][0])
    return el, np.zeros(2, np.uint8), P, (0, 1, 1.0), hbr


def _guess(el, p):
    jd = np.floor(el[0, p] - 0.5) + 0.5
    return jd, el[0, p] - jd


def _scenes(L):
    """(label, elements, model, P, (p, s, window), hbr)"""
    out = [("high-Pc LEO",) + _high_pc_leo(L)]
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], scale=300.0, deep=model.astype(bool))
    for p, s, w, label in cands:
        if label in ("LEO-Molniya", "LEO-GTO"):
            out.append((label, el, model, P, (p, s, w), 1.0))
    geo = cc.pair(cc.geo(), 0.05, dnode=0.0, dm=0.0)
    out.append(("GEO slow pair", geo, np.ones(2, np.uint8), cc.P_words(2, scale=0.2, bstar=False, deep=np.ones(2, bool)),
                (0, 1, 30.0), 0.05))
    lp = cc.pair(cc.leo(), 60.0, dnode=0.003, dm=0.0)
    out.append(("window edge", lp, np.zeros(2, np.uint8), cc.P_words(2, scale=30.0), (0, 1, 0.05), 0.5))
    # a near-earth row at a 223-minute period with a large n variance: draws whose period passes 225 minutes are not
    # near-earth sets and cannot be built under the row's model
    edge225 = cc.pair(np.array([2460000.25, 6.45, 0.001, 51.6, 120.0, 80.0, 0.0, 0.0]), 30.0, dnode=0.003)
    Pn = cc.P_words(2, scale=30.0, bstar=False)
    Pn[0, 0] = 0.05 ** 2
    out.append(("n variance across 225 min", edge225, np.zeros(2, np.uint8), Pn, (0, 1, 1.0), 0.5))
    return out


SAMPLES = 256


@pytest.fixture(scope="module")
def scenes(L):
    res = []
    for label, el, model, P, (p, s, w), hbr in _scenes(L):
        jd, fr = _guess(el, p)
        counts, out, status = mc.emul(L, el, P, model, [p], [s], jd, fr, w, hbr, SAMPLES, 0, 5, record=SAMPLES)
        dt, miss, rstatus, speed = _restated(el, P, model, p, s, jd, fr, w)
        res.append((label, hbr, counts[0], out[0], status[0], dt, miss, rstatus, speed))
    return res


def _restated(el, P, model, p, s, jd, fr, w):
    dt, miss, rstatus = mc.restated(el, P, model, p, s, jd, fr, w, SAMPLES, 0, 5)
    k = np.arange(SAMPLES, dtype=np.uint64)
    cols = [mc.elements_of(mc.draws(el[:, r], bool(model[r]), P[r], 5, o, k), el[0, r], bool(model[r]))
            for o, r in enumerate((p, s))]
    sel = np.empty((8, 2 * SAMPLES))
    sel[:, 0::2], sel[:, 1::2] = cols
    md = np.repeat(model[[p, s]][None], SAMPLES, axis=0).reshape(-1)
    _, st, _, _ = cj.restated(sel, np.zeros((2 * SAMPLES, 28)), md, np.arange(0, 2 * SAMPLES, 2),
                              np.arange(1, 2 * SAMPLES, 2), jd, fr, np.full(SAMPLES, w))
    return dt, miss, rstatus, np.linalg.norm(st[:, 1, 3:] - st[:, 0, 3:], axis=1)


def test_samples_match_the_restatement(scenes):
    """Failed and edge samples equal the restatement's; |d dt| |dv| and the miss within K11's host-vs-restatement
    allowance of 1e-7 km; hits equal where no miss lies within 1e-6 km of the radius"""
    for label, hbr, counts, out, status, dt, miss, rstatus, speed in scenes:
        assert status == 0, label
        failed = np.isnan(out[:, 0])
        assert np.array_equal(failed, ~np.isin(rstatus, (0, 3))), label
        ok = ~failed
        assert int(counts[2]) == failed.sum(), label
        assert int(counts[1]) == (rstatus == 3).sum(), label
        e_dt = (np.abs(out[ok, 0] - dt[ok]) * 60.0 * speed[ok]).max(initial=0.0)
        e_miss = np.abs(out[ok, 1] - miss[ok]).max(initial=0.0)
        print(f"{label}: hits {counts[0]}, edge {counts[1]}, failed {counts[2]}; |d dt| |dv| {e_dt:.1e} km, "
              f"miss {e_miss:.1e} km")
        assert e_dt <= 1e-7 and e_miss <= 1e-7, label
        assert np.abs(miss[ok] - hbr).min(initial=1.0) > 1e-6, label
        assert int(counts[0]) == (miss[ok] < hbr).sum(), label
    by = {s[0]: s for s in scenes}
    assert by["n variance across 225 min"][2][2] > 0            # some draws cannot be built
    assert by["window edge"][2][1] > 0                               # some searches end at a window end
    assert 0 < by["high-Pc LEO"][2][0] < SAMPLES


# ---- 4. invariants --------------------------------------------------------------------------------------------------
def _catalogue_inputs():
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], scale=30.0, deep=model.astype(bool))
    pr = np.array([c[0] for c in cands])
    se = np.array([c[1] for c in cands])
    w = np.array([c[2] for c in cands])
    jd = np.floor(el[0][pr] - 0.5) + 0.5
    return el, model, P, pr, se, jd, el[0][pr] - jd, w


def test_zero_P_gives_k11s_tca_and_miss(L):
    """P = 0: every sample is the nominal pair, with K11's host-build dt and miss bit for bit"""
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    P = np.zeros_like(P)
    rec, _, _, st11 = cj.emul(cj.emul_library(), el, P, model, pr, se, jd, fr, w, 1.0)
    counts, out, status = mc.emul(L, el, P, model, pr, se, jd, fr, w, 1.0, 20, 0, 3, record=20)
    assert (status == 0).all() and (st11 == 0).all()
    assert (out[:, :, 0] == rec[:, 0:1]).all() and (out[:, :, 1] == rec[:, 1:2]).all()
    assert (counts[:, 0] == 20 * (rec[:, 1] < 1.0)).all() and (counts[:, 2] == 0).all()


def test_split_ranges_add_up(L):
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    c0, o0, _ = mc.emul(L, el, P, model, pr, se, jd, fr, w, 0.5, 40, 0, 9, record=40)
    c1, o1, _ = mc.emul(L, el, P, model, pr, se, jd, fr, w, 0.5, 17, 0, 9, record=17)
    c2, o2, _ = mc.emul(L, el, P, model, pr, se, jd, fr, w, 0.5, 23, 17, 9, record=30)
    assert np.array_equal(c0, c1 + c2)
    assert np.array_equal(o0[:, :17], o1, equal_nan=True) and np.array_equal(o0[:, 17:], o2[:, :23], equal_nan=True)
    assert np.isnan(o2[:, 23:]).all()   # past samples[i]


def test_batch_order_and_duplicates_change_no_byte(L):
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    seeds = np.arange(len(pr), dtype=np.uint64) * 7
    c, o, s = mc.emul(L, el, P, model, pr, se, jd, fr, w, 0.5, 12, 0, seeds, record=12)
    perm = np.random.default_rng(1).permutation(np.concatenate([np.arange(len(pr)), [0, 3]]))
    c2, o2, s2 = mc.emul(L, el, P, model, pr[perm], se[perm], jd[perm], fr[perm], w[perm], 0.5, 12, 0, seeds[perm],
                         record=12)
    assert np.array_equal(c[perm], c2) and np.array_equal(s[perm], s2)
    assert o[perm].tobytes() == o2.tobytes()


def test_statuses(L):
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    P = P.copy()
    P[pr[0]] = _P(_pair(1 + 2e-12))
    bad = el.copy()
    bad[2, se[1]] = 1.5          # e > 1: the nominal set cannot be built
    c, o, s = mc.emul(L, bad, P, model, [pr[0], pr[1], pr[2], 0, pr[2]], [se[0], se[1], se[2], 0, 10 ** 6], jd[0],
                      fr[0], 1.0, 0.5, 8, 0, 0, record=4)
    assert list(s) == [6, 1, 0, 5, 5]
    assert (c[[0, 1, 3, 4]] == 0).all() and np.isnan(o[[0, 1, 3, 4]]).all()


# ---- 5. the C ABI's refusals and the wrapper ------------------------------------------------------------------------
def _abi_inputs():
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    m = len(pr)
    return dict(el=np.ascontiguousarray(el), P=P, model=model, pr=pr.astype(np.uint32), se=se.astype(np.uint32),
                jd=jd, fr=fr, w=w, r=np.full(m, 0.01), ns=np.full(m, 100, np.uint64), first=np.zeros(m, np.uint64),
                seed=np.zeros(m, np.uint64))


def _call(a, grav=1, device=0, record=2, out=True):
    from astroz_b200 import _lib

    m = len(a["pr"])
    counts = np.full((m, 3), 7, np.uint64)
    so = np.full((m, record, 2), 7.0) if out else None
    st = np.full(m, 9, np.uint8)
    p = lambda x: None if x is None else C.c_void_p(x.ctypes.data)  # noqa: E731
    rc = _lib.lib().astroz_cuda_conjunction_mc(p(a["el"]), a["el"].shape[1], grav, p(a["P"]), p(a["model"]),
                                               p(a["pr"]), p(a["se"]), p(a["jd"]), p(a["fr"]), p(a["w"]), p(a["r"]),
                                               p(a["ns"]), p(a["first"]), p(a["seed"]), m, record, device, p(counts),
                                               p(so), p(st))
    return rc, counts, so, st


REFUSALS = {
    "device": ({"device": -1}, "runs on one device"), "grav": ({"grav": 7}, "grav must be"),
    "row": ("se", "outside the catalogue"), "self": ("self", "with itself"), "window": ("w", "half windows"),
    "radius": ("r", "hard-body radii"), "model": ("model", "model byte"), "nan_el": ("nan_el", "elements must be"),
    "nan_P": ("nan_P", "covariance words"), "nan_time": ("fr", "guess times"), "overflow": ("first", "2^64"),
    "no_sample_out": ({"out": False}, "needs sample_out"),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_c_abi_refusals(case):
    from astroz_b200 import _lib
    from astroz_b200._abi import DEFINES as D

    a = _abi_inputs()
    how, text = REFUSALS[case]
    kw = how if isinstance(how, dict) else {}
    if how == "se":
        a["se"][1] = a["el"].shape[1]
    elif how == "self":
        a["se"][2] = a["pr"][2]
    elif how == "w":
        a["w"][0] = 0.0
    elif how == "r":
        a["r"][3] = -1e-3
    elif how == "model":
        a["model"] = a["model"].copy()
        a["model"][0] = 2
    elif how == "nan_el":
        a["el"][2, 1] = np.nan
    elif how == "nan_P":
        a["P"][1, 3] = np.inf
    elif how == "fr":
        a["fr"][1] = np.nan
    elif how == "first":
        a["first"][2] = np.uint64(2 ** 64 - 50)
    rc, counts, so, st = _call(a, **kw)
    assert rc == D["ASTROZ_VALUE_ERROR"]
    assert text in _lib.lib().astroz_cuda_last_error().decode()
    assert (counts == 7).all() and (st == 9).all() and (so is None or (so == 7.0).all())


def test_valid_input_without_a_device_writes_nothing():
    from astroz_b200 import _lib
    from astroz_b200._abi import DEFINES as D

    if _lib.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    rc, counts, so, st = _call(_abi_inputs())
    assert rc == D["ASTROZ_NO_DEVICE"] and (counts == 7).all() and (st == 9).all() and (so == 7.0).all()
    b = C.c_uint64(5)
    assert _lib.lib().astroz_cuda_conjunction_mc_scratch_bytes(4, C.byref(b)) == D["ASTROZ_NO_DEVICE"]
    assert b.value == 5
    assert _lib.lib().astroz_cuda_conjunction_mc_scratch_bytes(4, None) == D["ASTROZ_NULL_POINTER"]
    a = _abi_inputs()
    p = lambda x: C.c_void_p(x.ctypes.data)  # noqa: E731
    args = [p(a["el"]), a["el"].shape[1], 1, p(a["P"]), p(a["model"]), p(a["pr"]), p(a["se"]), p(a["jd"]),
            p(a["fr"]), p(a["w"]), p(a["r"]), p(a["ns"]), None, None, len(a["pr"]), 0]
    dev = _lib.lib().astroz_cuda_conjunction_mc_device
    assert dev(*args, -1, p(counts), None, p(st), p(counts), None) == D["ASTROZ_VALUE_ERROR"]
    assert dev(*args, 0, p(counts), None, None, p(counts), None) == D["ASTROZ_NULL_POINTER"]
    assert dev(*args, 0, p(counts), None, p(st), p(counts), None) == D["ASTROZ_NO_DEVICE"]
    assert (counts == 7).all() and (st == 9).all()


def test_wrapper_order_broadcasting_and_interval(monkeypatch):
    """monte_carlo() passes candidates in the caller's order with scalars broadcast, and its Pc and Wilson interval are
    the closed forms (scipy's binomial interval at 0 and n hits as a check of the edges)"""
    from astroz_b200 import collision

    seen = {}

    class Fake:
        def astroz_cuda_conjunction_mc(self, el, n, grav, cov, md, pr, se, jd, fr, w, r, ns, fi, sd, m, record, dev,
                                       counts, out, stat):
            arr = lambda ptr, t: np.ctypeslib.as_array(C.cast(ptr, C.POINTER(t)), (m,)).copy()  # noqa: E731
            seen.update(pr=arr(pr, C.c_uint32), ns=arr(ns, C.c_uint64), fi=arr(fi, C.c_uint64), sd=arr(sd, C.c_uint64),
                        w=arr(w, C.c_double), record=record)
            c = np.ctypeslib.as_array(C.cast(counts, C.POINTER(C.c_uint64)), (m, 3))
            c[:, 0] = seen["pr"]
            c[:, 2] = 1
            o = np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_double)), (m, record, 2))
            o[:, :, 0] = seen["pr"][:, None]
            return 0

    monkeypatch.setattr(collision, "lib", lambda: Fake())
    el, model, _ = cc.catalogue()
    n = el.shape[1]
    pr = np.array([5, 0, 3, 9, 2])
    res = collision.monte_carlo(el, pr, (pr + 1) % n, 2460000.5, 0.25, window_min=1.0, hbr_km=0.01, samples=11,
                                seed=[1, 2, 3, 4, 5], first=100, record=3, covariance=np.zeros((n, 28)), model=model)
    assert (seen["pr"] == pr).all() and (seen["ns"] == 11).all() and (seen["fi"] == 100).all()
    assert (seen["sd"] == [1, 2, 3, 4, 5]).all() and (seen["w"] == 1.0).all() and seen["record"] == 3
    assert (res.hits == pr).all() and (res.sample_dt == pr[:, None]).all() and res.sample_miss.shape == (5, 3)
    assert np.allclose(res.pc, pr / 10.0)
    lo, hi = res.interval()
    for h, a, b in zip(pr, lo, hi):
        p, z, N = h / 10, 1.96, 10
        c = (p + z * z / (2 * N)) / (1 + z * z / N)
        d = z * np.sqrt(p * (1 - p) / N + z * z / (4 * N * N)) / (1 + z * z / N)
        assert np.isclose(a, max(c - d, 0)) and np.isclose(b, min(c + d, 1))
    assert lo[1] == 0.0 and hi[1] > 0.0         # 0 hits: [0, z^2 / (n + z^2)]
    assert np.isclose(hi[1], 1.96 ** 2 / (10 + 1.96 ** 2))
    empty = collision.MonteCarloResult(*(np.zeros(1, np.uint64),) * 4, np.zeros(1, np.uint8), None, None)
    assert np.isnan(empty.pc).all() and np.isnan(empty.interval()[0]).all()
    with pytest.raises(ValueError):
        collision.monte_carlo(el, [0], [1], 2460000.5, 0.0, window_min=1.0, hbr_km=0.01, samples=-1,
                              covariance=np.zeros((n, 28)))
