"""K15 importance-sampled collision probability (az_conjunction_is.cuh, az_conjunction_is.cu) on the CPU.

The host build of the device source (tests/host_emul/emul_conjunction_is.cu) against the independent numpy statement
(tests/fit_oracle/conjunction_is.py): the linear proposal on the engineered cases and a LEO ladder, the log weights and
the 256-bit words, the zero-shift identity with K14's host build, the estimator on the linear model for Pc 1e-4 to 1e-12
under good and poor shifts, each drawn pair against the C restatement of K11, the split-range and batch invariants, the
C ABI's refusals and the Python wrapper.  The device runs are in tests/test_gpu_conjunction_is.py."""
import ctypes as C

import numpy as np
import pytest

from tests.fit_oracle import conjunction as cj
from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import conjunction_is as ci
from tests.fit_oracle import conjunction_mc as mc


@pytest.fixture(scope="module")
def L():
    lib = ci.emul_library()
    if lib is None or cj.emul_library() is None:
        pytest.skip("nvcc unavailable")
    return lib


def _guess(el, p):
    jd = np.floor(el[0, p] - 0.5) + 0.5
    return jd, el[0, p] - jd


def _scenes():
    """(label, elements, model, P, (p, s, window), hbr): the engineered cases and the LEO ladder (miss at 3 .. 7 sigma)"""
    el, P, hbr = cc.high_pc_leo(lambda el, P, hbr: ci.emul_assess(el, P, hbr))
    out = [("high-Pc LEO", el, np.zeros(2, np.uint8), P, (0, 1, 1.0), hbr)]
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], scale=300.0, deep=model.astype(bool))
    for p, s, w, label in cands:
        if label in ("LEO-Molniya", "LEO-GTO"):
            out.append((label, el, model, P, (p, s, w), 1.0))
    out.append(("GEO slow pair", cc.pair(cc.geo(), 0.05), np.ones(2, np.uint8),
                cc.P_words(2, scale=0.2, bstar=False, deep=np.ones(2, bool)), (0, 1, 30.0), 0.05))
    base = cc.pair(cc.leo(), 40.0, dnode=0.0005)
    P0 = cc.P_words(2, scale=1.0, bstar=False)
    rec = ci.emul_assess(base, P0, 0.01)
    xx, xy, yy = rec[9:12]
    k0 = rec[1] * np.sqrt(yy / (xx * yy - xy * xy))
    for k in (3, 4, 5, 6, 7):
        out.append((f"LEO ladder {k} sigma", base, np.zeros(2, np.uint8), P0 * (k0 / k) ** 2, (0, 1, 1.0), 0.2))
    return out


SAMPLES = 256


@pytest.fixture(scope="module")
def scenes(L):
    res = []
    for label, el, model, P, (p, s, w), hbr in _scenes():
        jd, fr = _guess(el, p)
        r = ci.emul(L, el, P, model, [p], [s], jd, fr, w, hbr, SAMPLES, 0, 5, record=SAMPLES)
        res.append((label, el, model, P, (p, s, w), hbr, jd, fr, r))
    return res


# ---- 1. the proposal --------------------------------------------------------------------------------------------------
def test_linear_proposal_matches_the_statement(scenes):
    """Statuses and kinds; |d + G c| <= 1e-9 |d|; c against the numpy statement (J from the C restatement of K10) within
    2e-6 of |c|; |c|^2 against d^T C2^-1 d from K11's own record within 1e-6 relative"""
    for label, el, model, P, (p, s, w), hbr, jd, fr, r in scenes:
        assert r["status"][0] == 0 and r["k11"][0] in (0, 3), label
        assert r["kind"][0] == ci.LINEAR, label
        c = r["proposal"][0, :14]
        G = r["G"][0]
        E, d = ci.plane(r["states"][0])
        res = np.linalg.norm(d + G @ c) / np.linalg.norm(d)
        ref = ci.linear_shift(el, P, model, p, s, jd, fr, r["record"][0, 0], r["states"][0])
        assert ref is not None, label
        dc = np.abs(c - ref[0]).max() / np.abs(ref[0]).max()
        xx, xy, yy = r["record"][0, 9:12]
        C2 = np.array([[xx, xy], [xy, yy]])
        maha = d @ np.linalg.solve(C2, d)
        cc2 = c @ c
        print(f"{label}: |c|^2 {cc2:.6g}, d^T C2^-1 d {maha:.6g}, |d + Gc| / |d| {res:.1e}, c vs statement {dc:.1e}")
        assert res <= 1e-9, label
        assert dc <= 2e-6, label
        assert abs(cc2 - maha) <= 1e-6 * maha, label
        seq = 0.0
        for x in c:                               # |c|^2 summed in the shift's order
            seq += x * x
        assert r["proposal"][0, 14] == 0.0 - 0.5 * seq


# ---- 2. the weights ---------------------------------------------------------------------------------------------------
def test_log_weights_and_words(scenes):
    """log w of every recorded sample against numpy on the Philox normals within 1e-12 (1 + |log w|); the 256-bit words
    equal the Python-integer sums of the hits' rounded v and v^2 exactly"""
    total_hits = 0
    for label, el, model, P, (p, s, w), hbr, jd, fr, r in scenes:
        c = r["proposal"][0, :14]
        lw = ci.log_weights(5, np.arange(SAMPLES, dtype=np.uint64), c)
        ok = ~np.isnan(r["out"][0, :, 2])
        err = (np.abs(r["out"][0, ok, 2] - lw[ok]) / (1.0 + np.abs(lw[ok]))).max()
        assert err <= 1e-12, label
        hit = ok & (r["out"][0, :, 1] < hbr)
        V, V2, ov = ci.sums(r["v"][0, hit])
        assert np.array_equal(r["counts"][0, 4:8], V) and np.array_equal(r["counts"][0, 8:12], V2), label
        assert int(r["counts"][0, 3]) == ov and int(r["counts"][0, 0]) == hit.sum(), label
        total_hits += hit.sum()
    assert total_hits > 100


def test_zero_shift_is_k14(L):
    """A given shift of 0 reproduces K14's host build bit for bit: hits, edge, failed and the (dt, miss) words; V_hit and
    V2_hit are hits 2^128 and log w is 0"""
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], scale=300.0, deep=model.astype(bool))
    pr, se, w = (np.array([c[q] for c in cands]) for q in range(3))
    jd = np.floor(el[0][pr] - 0.5) + 0.5
    fr = el[0][pr] - jd
    Lm = mc.emul_library()
    k14 = mc.emul(Lm, el, P, model, pr, se, jd, fr, w, 1.0, 64, 0, 3, record=64)
    r = ci.emul(L, el, P, model, pr, se, jd, fr, w, 1.0, 64, 0, 3, shift=np.zeros(14), record=64)
    assert np.array_equal(r["counts"][:, :3], k14[0]) and np.array_equal(r["status"], k14[2])
    assert r["out"][:, :, :2].tobytes() == k14[1].tobytes()
    assert (r["kind"] == ci.GIVEN).all() and (r["proposal"] == 0.0).all()
    hits = [int(h) for h in k14[0][:, 0]]
    for lo in (4, 8):
        assert [sum(int(x) << (64 * q) for q, x in enumerate(row)) for row in r["counts"][:, lo:lo + 4]] == \
            [h << 128 for h in hits]
    ok = ~np.isnan(r["out"][:, :, 2])
    assert (r["out"][:, :, 2][ok] == 0.0).all() and k14[0][:, 0].sum() > 0


# ---- 3. the estimator -------------------------------------------------------------------------------------------------
def _linear_estimate(L, c, G, d, R, n, seed=11):
    """the IS estimate and its standard error when the host build's draws z = u + c are scored by d + G z"""
    u = mc.emul_normals(L, seed, np.arange(n, dtype=np.uint64))
    z = u + c[None, :]
    hit = np.linalg.norm(d[None, :] + z @ G.T, axis=1) < R
    wgt = np.exp(-(u[:, :7] @ c[:7] + u[:, 7:] @ c[7:]) - 0.5 * (c @ c)) * hit
    return wgt.mean(), wgt.std() / np.sqrt(n), hit.mean()


@pytest.mark.parametrize("target", [1e-4, 1e-6, 1e-8, 1e-10, 1e-12])
def test_estimator_is_unbiased_on_the_linear_model(L, target):
    """On the linear model d + G z the estimate of 20,000 draws lies within 4 sigma_IS of the 30-digit 2-D Pc of N(d, C),
    C = G G^T, for the host build's shift and, down to Pc 1e-8 (|c| ~ 6), for poor given shifts (0.5 c, 1.5 c, c
    turned by 30 deg in 14-space): the weight variance of a shift off by b grows like exp(|b|^2), so at 1e-10 and 1e-12
    those need far more draws than the test spends"""
    el, P, R = ci.leo_at_pc(ci.emul_assess, target)
    jd, fr = _guess(el, 0)
    r = ci.emul(L, el, P, np.zeros(2, np.uint8), [0], [1], jd, fr, 1.0, R, 0)
    assert r["kind"][0] == ci.LINEAR
    c, G = r["proposal"][0, :14], r["G"][0]
    _, d = ci.plane(r["states"][0])
    Cm = G @ G.T
    ref = cj.pc_reference(Cm[0, 0], Cm[0, 1], Cm[1, 1], np.linalg.norm(d), R)
    rng = np.random.default_rng(1)
    q = rng.standard_normal(14)
    q -= (q @ c) / (c @ c) * c
    turned = np.cos(np.pi / 6) * c + np.sin(np.pi / 6) * np.linalg.norm(c) * q / np.linalg.norm(q)
    shifts = [("linear", c)]
    if target >= 1e-8:   # further out a shift |c| / 2 off the collision point needs far more than 20,000 draws
        shifts += [("0.5 c", 0.5 * c), ("1.5 c", 1.5 * c), ("turned 30 deg", turned)]
    for label, shift in shifts:
        est, se, frac = _linear_estimate(L, shift, G, d, R, 20000)
        print(f"Pc {ref:.4e} ({label}): estimate {est:.4e} +- {se:.2e}, hit fraction {frac:.4f}")
        assert se > 0 and abs(est - ref) <= 4.0 * se, label


# ---- 4. each drawn pair against the restatement ---------------------------------------------------------------------------
def test_nonlinear_draws_match_the_restatement(scenes):
    """Each shifted draw's pair assessed by the C restatement of K11 with P = 0: failed and edge classes equal, dt |dv|
    and the miss within K14's 1e-7 km, hits equal where no miss lies within 1e-6 km of the radius"""
    for label, el, model, P, (p, s, w), hbr, jd, fr, r in scenes:
        if not label.startswith(("high-Pc", "LEO-Molniya", "GEO", "LEO ladder 5")):
            continue
        c = r["proposal"][0, :14]
        k = np.arange(SAMPLES, dtype=np.uint64)
        u = mc.normals(5, k)
        cols = []
        for o, row in enumerate((p, s)):
            sd, Lm, _ = mc.factor(P[row])
            x = mc.vars_of(el[:, row], bool(model[row]))[None, :] + ((u[:, 7 * o:7 * o + 7] + c[7 * o:7 * o + 7]) @
                                                                     Lm.T) * sd[None, :]
            cols.append(mc.elements_of(x, el[0, row], bool(model[row])))
        sel = np.empty((8, 2 * SAMPLES))
        sel[:, 0::2], sel[:, 1::2] = cols
        md = np.repeat(np.asarray(model)[[p, s]][None], SAMPLES, axis=0).reshape(-1)
        dt, st, _, rs = cj.restated(sel, np.zeros((2 * SAMPLES, 28)), md, np.arange(0, 2 * SAMPLES, 2),
                                    np.arange(1, 2 * SAMPLES, 2), jd, fr, np.full(SAMPLES, w))
        miss = np.linalg.norm(st[:, 1, :3] - st[:, 0, :3], axis=1)
        speed = np.linalg.norm(st[:, 1, 3:] - st[:, 0, 3:], axis=1)
        out = r["out"][0]
        failed = np.isnan(out[:, 0])
        assert np.array_equal(failed, ~np.isin(rs, (0, 3))), label
        assert int(r["counts"][0, 1]) == (rs == 3).sum(), label
        ok = ~failed
        e_dt = (np.abs(out[ok, 0] - dt[ok]) * 60.0 * speed[ok]).max(initial=0.0)
        e_miss = np.abs(out[ok, 1] - miss[ok]).max(initial=0.0)
        near = np.abs(miss[ok] - hbr) <= 1e-6
        print(f"{label}: hits {r['counts'][0, 0]}, edge {r['counts'][0, 1]}, failed {r['counts'][0, 2]}; "
              f"|d dt| |dv| {e_dt:.1e} km, miss {e_miss:.1e} km")
        assert e_dt <= 1e-7 and e_miss <= 1e-7, label
        assert ((out[ok, 1] < hbr) == (miss[ok] < hbr))[~near].all(), label


# ---- 5. bookkeeping ---------------------------------------------------------------------------------------------------
def _catalogue_inputs():
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], scale=300.0, deep=model.astype(bool))
    pr, se, w = (np.array([c[q] for c in cands]) for q in range(3))
    jd = np.floor(el[0][pr] - 0.5) + 0.5
    return el, model, P, pr, se, jd, el[0][pr] - jd, w


def test_split_ranges_add_exactly(L):
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    a = ci.emul(L, el, P, model, pr, se, jd, fr, w, 1.0, 40, 0, 9, record=40)
    b = ci.emul(L, el, P, model, pr, se, jd, fr, w, 1.0, 17, 0, 9, record=17)
    c = ci.emul(L, el, P, model, pr, se, jd, fr, w, 1.0, 23, 17, 9, record=23)
    tot = lambda x, lo: [sum(int(v) << (64 * q) for q, v in enumerate(row)) for row in x[:, lo:lo + 4]]  # noqa
    assert np.array_equal(a["counts"][:, :4], b["counts"][:, :4] + c["counts"][:, :4])
    for lo in (4, 8):
        assert tot(a["counts"], lo) == [x + y for x, y in zip(tot(b["counts"], lo), tot(c["counts"], lo))]
    assert np.array_equal(a["out"][:, :17], b["out"], equal_nan=True)
    assert np.array_equal(a["out"][:, 17:], c["out"], equal_nan=True)
    assert np.array_equal(a["proposal"], b["proposal"])


def test_batch_order_and_duplicates_change_no_byte(L):
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    seeds = np.arange(len(pr), dtype=np.uint64) * 7
    a = ci.emul(L, el, P, model, pr, se, jd, fr, w, 1.0, 12, 0, seeds, record=12)
    perm = np.random.default_rng(1).permutation(np.concatenate([np.arange(len(pr)), [0, 3]]))
    b = ci.emul(L, el, P, model, pr[perm], se[perm], jd[perm], fr[perm], w[perm], 1.0, 12, 0, seeds[perm], record=12)
    for key in ("counts", "proposal", "kind", "status", "out"):
        assert a[key][perm].tobytes() == b[key].tobytes(), key


def test_statuses_and_plain_proposals(L):
    """Candidates that are not OK: zero counts and proposal words, PLAIN, NaN samples.  A zero-covariance row pair is
    OK but C = 0: PLAIN"""
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    bad = el.copy()
    bad[2, se[1]] = 1.5
    Pz = P.copy()
    Pz[pr[2]] = 0.0
    Pz[se[2]] = 0.0
    r = ci.emul(L, bad, Pz, model, [pr[0], pr[1], pr[2], 0], [se[0], se[1], se[2], 0], jd[0], fr[0], 1.0, 0.5, 8,
                record=4)
    assert list(r["status"]) == [0, 1, 0, 5]
    assert list(r["kind"]) == [ci.LINEAR, ci.PLAIN, ci.PLAIN, ci.PLAIN]
    for i in (1, 3):
        assert (r["counts"][i] == 0).all() and (r["proposal"][i] == 0).all() and np.isnan(r["out"][i]).all()
    assert (r["proposal"][2] == 0).all()


# ---- 6. the C ABI's refusals and the wrapper ---------------------------------------------------------------------------
def _abi_inputs():
    el, model, P, pr, se, jd, fr, w = _catalogue_inputs()
    m = len(pr)
    return dict(el=np.ascontiguousarray(el), P=P, model=model, pr=pr.astype(np.uint32), se=se.astype(np.uint32),
                jd=jd, fr=fr, w=w, r=np.full(m, 0.01), ns=np.full(m, 100, np.uint64), first=np.zeros(m, np.uint64),
                seed=np.zeros(m, np.uint64), shift=np.zeros((m, 14)))


def _call(a, grav=1, device=0, record=2, out=True, shift=True):
    from astroz_b200 import _lib

    m = len(a["pr"])
    counts = np.full((m, 12), 7, np.uint64)
    prop = np.full((m, 15), 7.0)
    kind = np.full(m, 9, np.uint8)
    so = np.full((m, record, 3), 7.0) if out else None
    st = np.full(m, 9, np.uint8)
    p = lambda x: None if x is None else C.c_void_p(x.ctypes.data)  # noqa: E731
    rc = _lib.lib().astroz_cuda_conjunction_is(p(a["el"]), a["el"].shape[1], grav, p(a["P"]), p(a["model"]),
                                               p(a["pr"]), p(a["se"]), p(a["jd"]), p(a["fr"]), p(a["w"]), p(a["r"]),
                                               p(a["ns"]), p(a["first"]), p(a["seed"]),
                                               p(a["shift"]) if shift else None, m, record, device, p(counts), p(prop),
                                               p(kind), p(so), p(st))
    return rc, (counts, prop, kind, so, st)


REFUSALS = {
    "device": ({"device": -1}, "runs on one device"), "grav": ({"grav": 7}, "grav must be"),
    "row": ("se", "outside the catalogue"), "self": ("self", "with itself"), "window": ("w", "half windows"),
    "radius": ("r", "hard-body radii"), "model": ("model", "model byte"), "nan_el": ("nan_el", "elements must be"),
    "nan_P": ("nan_P", "covariance words"), "nan_time": ("fr", "guess times"), "overflow": ("first", "2^64"),
    "no_sample_out": ({"out": False}, "needs sample_out"), "nan_shift": ("shift", "shift words"),
    "inf_shift": ("shift_inf", "shift words"),
}


def _untouched(outs):
    counts, prop, kind, so, st = outs
    return (counts == 7).all() and (prop == 7.0).all() and (kind == 9).all() and (st == 9).all() and \
        (so is None or (so == 7.0).all())


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
    elif how == "shift":
        a["shift"][3, 9] = np.nan
    elif how == "shift_inf":
        a["shift"][0, 0] = -np.inf
    rc, outs = _call(a, **kw)
    assert rc == D["ASTROZ_VALUE_ERROR"]
    assert text in _lib.lib().astroz_cuda_last_error().decode()
    assert _untouched(outs)


def test_valid_input_without_a_device_writes_nothing():
    from astroz_b200 import _lib
    from astroz_b200._abi import DEFINES as D

    if _lib.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    for shift in (True, False):
        rc, outs = _call(_abi_inputs(), shift=shift)
        assert rc == D["ASTROZ_NO_DEVICE"] and _untouched(outs)
    b = C.c_uint64(5)
    assert _lib.lib().astroz_cuda_conjunction_is_scratch_bytes(4, C.byref(b)) == D["ASTROZ_NO_DEVICE"]
    assert b.value == 5
    assert _lib.lib().astroz_cuda_conjunction_is_scratch_bytes(4, None) == D["ASTROZ_NULL_POINTER"]
    a = _abi_inputs()
    counts, st = np.full((len(a["pr"]), 12), 7, np.uint64), np.full(len(a["pr"]), 9, np.uint8)
    p = lambda x: C.c_void_p(x.ctypes.data)  # noqa: E731
    args = [p(a["el"]), a["el"].shape[1], 1, p(a["P"]), p(a["model"]), p(a["pr"]), p(a["se"]), p(a["jd"]),
            p(a["fr"]), p(a["w"]), p(a["r"]), p(a["ns"]), None, None, None, len(a["pr"]), 0]
    dev = _lib.lib().astroz_cuda_conjunction_is_device
    assert dev(*args, -1, p(counts), None, None, None, p(st), p(counts), None) == D["ASTROZ_VALUE_ERROR"]
    assert dev(*args, 0, p(counts), None, None, None, None, p(counts), None) == D["ASTROZ_NULL_POINTER"]
    assert dev(*args, 0, p(counts), None, None, None, p(st), None, None) == D["ASTROZ_NULL_POINTER"]
    assert dev(*args, 0, p(counts), None, None, None, p(st), p(counts), None) == D["ASTROZ_NO_DEVICE"]
    assert (counts == 7).all() and (st == 9).all()


def _words(x):
    return [(x >> (64 * q)) & (2 ** 64 - 1) for q in range(4)]


def test_wrapper(monkeypatch):
    """importance_sampling() passes candidates in the caller's order with scalars and a (14,) shift broadcast; pc,
    std_error, interval and combine are the closed forms of the words"""
    from astroz_b200 import collision

    seen = {}
    V = [3 << 128, 5 << 120, 0, 2 ** 200 + 12345]
    V2 = [3 << 128, 7 << 110, 0, 2 ** 230 + 99]

    class Fake:
        def astroz_cuda_conjunction_is(self, el, n, grav, cov, md, pr, se, jd, fr, w, r, ns, fi, sd, sh, m, record,
                                       dev, counts, prop, kind, out, stat):
            arr = lambda ptr, t, shape: np.ctypeslib.as_array(C.cast(ptr, C.POINTER(t)), shape)  # noqa: E731
            seen.update(pr=arr(pr, C.c_uint32, (m,)).copy(), ns=arr(ns, C.c_uint64, (m,)).copy(),
                        sh=arr(sh, C.c_double, (m, 14)).copy(), record=record)
            c = arr(counts, C.c_uint64, (m, 12))
            c[:, 0] = [3, 2, 0, 4]
            for i in range(m):
                c[i, 4:8] = _words(V[i])
                c[i, 8:12] = _words(V2[i])
            p = arr(prop, C.c_double, (m, 15))
            p[:, 14] = [0.0, -1.0, 0.0, -2.0]
            arr(kind, C.c_uint8, (m,))[:] = [1, 1, 2, 1]
            arr(out, C.c_double, (m, record, 3))[:, :, 2] = -0.5
            return 0

    monkeypatch.setattr(collision, "lib", lambda: Fake())
    el, model, _ = cc.catalogue()
    n = el.shape[1]
    pr = np.array([5, 0, 3, 9])
    shift = np.arange(14.0)
    res = collision.importance_sampling(el, pr, (pr + 1) % n, 2460000.5, 0.25, window_min=1.0, hbr_km=0.01,
                                        samples=10, seed=1, record=2, shift=shift, covariance=np.zeros((n, 28)),
                                        model=model)
    assert (seen["pr"] == pr).all() and (seen["ns"] == 10).all() and (seen["sh"] == shift).all()
    assert seen["record"] == 2 and (res.sample_log_weight == -0.5).all() and (res.kind == [1, 1, 2, 1]).all()
    N = 10
    m1 = np.array([np.exp(l0) * v / 2 ** 128 / N for v, l0 in zip(V, res.log_scale)])
    m2 = np.array([np.exp(2 * l0) * v / 2 ** 128 / N for v, l0 in zip(V2, res.log_scale)])
    assert np.allclose(res.pc, m1, rtol=1e-15, atol=0)
    assert np.allclose(res.std_error, np.sqrt(np.maximum(m2 - m1 ** 2, 0) / (N - 1)), rtol=1e-12, atol=0)
    lo, hi = res.interval(2.0)
    assert np.isnan(lo[2]) and np.isnan(hi[2])                      # no hit
    assert lo[0] == max(m1[0] - 2 * res.std_error[0], 0.0) and np.isclose(hi[3], m1[3] + 2 * res.std_error[3])
    assert np.allclose(res.proposal_hit_fraction, [0.3, 0.2, 0.0, 0.4])
    both = res.combine(res)
    assert (both.samples == 20).all() and (both.hits == 2 * res.hits).all()
    for i in range(4):
        assert sum(int(x) << (64 * q) for q, x in enumerate(both.counts[i, 4:8])) == 2 * V[i]
    assert np.allclose(both.pc, res.pc, rtol=1e-15)
    with pytest.raises(ValueError):
        res.combine(collision.ImportanceResult(res.counts, res.samples, res.shift + 1.0, res.log_scale, res.kind,
                                               res.status, None, None, None))
