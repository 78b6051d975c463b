"""K16 collision-avoidance manoeuvre trials (az_avoid.cuh, az_avoid.cu) on the CPU.

The host build of the device source (tests/host_emul/emul_avoid.cu, composed with the host builds of K10, K8 and K11)
on the engineered crossings of tests/fit_oracle/conjunction_cases.py and a LEO Pc ladder: the zero burn against K11's
host build, continuity of the new set through the oracle's SGP4 / SDP4, Clohessy-Wiltshire on a near-circular LEO, the
covariance transport against the numpy statement (tests/fit_oracle/avoid.py) and a Monte Carlo through the C
restatement of the fit, the composition with K11, the statuses and invariants, the C ABI's refusals and the planner.
The device runs are in tests/test_gpu_avoid.py."""
import ctypes as C
import os

import numpy as np
import pytest

import tests.fit_oracle as fo
from tests.fit_oracle import avoid as av
from tests.fit_oracle import conjunction as cj
from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import covariance as K
from tests.fit_oracle import deep as fd
from tests.fit_oracle.conjunction_mc import vars_of


@pytest.fixture(scope="module")
def L():
    lib = av.emul_library()
    if lib is None or cj.emul_library() is None:
        pytest.skip("nvcc unavailable")
    return lib


@pytest.fixture(scope="module")
def LC(L):
    return cj.emul_library()


def _catalogue():
    """(elements, model, P, primary, secondary, jd, fr, window): the engineered crossings, guess at the first epoch"""
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], scale=300.0, deep=model.astype(bool))
    pr = np.array([c[0] for c in cands])
    se = np.array([c[1] for c in cands])
    w = np.array([c[2] for c in cands], np.float64)
    jd = np.floor(el[0, pr] - 0.5) + 0.5
    return el, model, P, pr, se, jd, el[0, pr] - jd, w


def _burn(el, pr, jd, fr, orbits):
    """burn times `orbits` primary periods before the guesses"""
    return jd, fr - orbits / el[1, pr]


def _oracle_state(el, jd, fr):
    """the oracle's TEME state (6,) of a set under its class (SGP4 or SDP4)"""
    deep = 1440.0 / el[1] > 225.0
    pos, vel = (fd.observe if deep else fo.observe)(el, np.array([jd]), np.array([fr]))
    return np.r_[pos[0], vel[0]]


def _ladder():
    """a LEO crossing and its P scaled so that the nominal miss sits at 1.7 sigma: with a 0.2 km radius Pc 1.8e-4"""
    base = cc.pair(cc.leo(), 40.0, dnode=0.0005)
    P0 = cc.P_words(2, scale=1.0, bstar=False)
    jd = np.floor(base[0, 0] - 0.5) + 0.5
    fr = base[0, 0] - jd + 3.0 / 1440.0
    LC = cj.emul_library()
    rec = cj.emul(LC, base, P0, None, [0], [1], jd, fr, 5.0, 0.02)[0][0]
    xx, xy, yy = rec[9:12]
    k0 = rec[1] * np.sqrt(yy / (xx * yy - xy * xy))
    return base, P0 * (k0 / 1.7) ** 2, jd, fr


# ---- 1. the zero burn -------------------------------------------------------------------------------------------------
def test_zero_burn_is_the_nominal_assessment(L, LC):
    """dv = 0: record and status equal K11's host build bit for bit, the row is the primary's words and P' = P; with
    sigma > 0 only P' (and so C2 and Pc) changes"""
    el, model, P, pr, se, jd, fr, w = _catalogue()
    m = len(pr)
    bj, bf = _burn(el, pr, jd, fr, 2.0)
    rec0, _, _, st0 = cj.emul(LC, el, P, model, pr, se, jd, fr, w, 0.01)
    rec, ne, nc, res, st = av.emul(L, el, P, model, pr, se, jd, fr, w, 0.01, np.arange(m), bj, bf, np.zeros(3))
    assert np.array_equal(st, st0) and np.array_equal(rec.view(np.uint64), rec0.view(np.uint64))
    assert np.array_equal(ne, el[:, pr].T) and np.array_equal(nc, P[pr]) and (res == 0).all()
    rec1, ne1, nc1, res1, st1 = av.emul(L, el, P, model, pr, se, jd, fr, w, 0.01, np.arange(m), bj, bf, np.zeros(3),
                                        dv_sigma=[1e-4, 2e-4, 5e-5])
    assert np.array_equal(ne1, ne) and (res1 == 0).all() and np.array_equal(st1, st)
    assert not np.array_equal(nc1, nc) and np.array_equal(rec1[:, :9], rec[:, :9])


# ---- 2. continuity ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mag", [1e-6, 1e-4, 1e-2])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_new_set_meets_the_post_burn_state(L, axis, mag):
    """The returned set propagated by the ORACLE's SGP4 / SDP4 to t_b gives x(t_b) + [0; R dv] within 1e-6 km and
    1e-9 km/s, near-earth and deep-space primaries, 1 mm/s to 10 m/s on each RTN axis"""
    el, model, P, pr, se, jd, fr, w = _catalogue()
    m = len(pr)
    bj, bf = _burn(el, pr, jd, fr, 1.5)
    dv = np.zeros(3)
    dv[axis] = mag
    rec, ne, nc, res, st = av.emul(L, el, P, model, pr, se, jd, fr, w, 0.01, np.arange(m), bj, bf, dv)
    checked = 0
    for k in range(m):
        assert st[k] in (av.OK, av.WINDOW_EDGE), (k, st[k])
        x0 = _oracle_state(el[:, pr[k]], bj[k], bf[k])
        x1 = _oracle_state(ne[k], bj[k], bf[k])
        R = av.rtn(x0)
        assert np.abs(x1[:3] - x0[:3]).max() <= 1e-6, k
        assert np.abs(x1[3:] - (x0[3:] + R.T @ dv)).max() <= 1e-9, k
        assert ne[k, 0] == el[0, pr[k]]                   # the epoch is kept
        checked += 1
    assert checked == m and model[pr].any()


# ---- 3. physics -------------------------------------------------------------------------------------------------------
# Measured on the host build: over 1-5 orbits and 1-10 mm/s, the primary's RTN displacement at the TCA differs from
# Clohessy-Wiltshire by at most 2.2 % of the along-track displacement (J2 and SGP4's short-period terms, and the
# orbit's 0.0012 eccentricity, which CW ignores).  The bound below keeps a margin.
CW_REL = 0.05


def test_tangential_burns_follow_clohessy_wiltshire(L):
    base = cc.pair(cc.leo(), 40.0, dnode=0.0005)
    P = cc.P_words(2, scale=1.0, bstar=False)
    n = base[1, 0] * 2 * np.pi / 86400.0
    jd = np.floor(base[0, 0] - 0.5) + 0.5
    fr = base[0, 0] - jd + 5.5 / base[1, 0]
    worst = 0.0
    for orbits in (1.0, 2.0, 3.5, 5.0):
        for dvt in (1e-6, 5e-6, 1e-5):
            bj, bf = jd, fr - orbits / base[1, 0]
            out = []
            for d in (dvt, 2 * dvt):
                rec, ne, nc, res, st = av.emul(L, base, P, None, [0], [1], jd, fr, 5.0, 0.01, [0], bj, bf, [0, d, 0])
                assert st[0] == av.OK
                x0 = _oracle_state(base[:, 0], jd, fr)
                x1 = _oracle_state(ne[0], jd, fr)
                R = av.rtn(x0)
                out.append(R @ (x1[:3] - x0[:3]))
            t = orbits / base[1, 0] * 86400.0
            rad, along = av.cw(dvt, n, t)
            scale = abs(along)
            worst = max(worst, abs(out[0][0] - rad) / scale, abs(out[0][1] - along) / scale)
            # doubling dv doubles the displacement to second order
            assert np.abs(out[1] - 2 * out[0]).max() <= 1e-3 * np.abs(out[0]).max()
    assert worst <= CW_REL, worst


# ---- 4. covariance through the burn -----------------------------------------------------------------------------------
def _jacobians(el_old, el_new, P, model, bj, bf):
    off = np.array([0, 1], np.uint32)
    md = None if model is None else np.array([model], np.uint8)
    out = []
    for e in (el_old, el_new):
        st, _, jac, status = K.restated(e[:, None], P[None], md, off, np.array([bj]), np.array([bf]))
        assert status[0] == 0
        out.append((st[0], jac[0]))
    return out


@pytest.mark.parametrize("sigma", [None, [2e-5, 1e-5, 3e-5]])
def test_transport_matches_the_statement(L, sigma):
    """P' of the host build against A P A^T (+ the execution term) with J, J' from the C restatement of K10"""
    el, model, P, pr, se, jd, fr, w = _catalogue()
    m = len(pr)
    bj, bf = _burn(el, pr, jd, fr, 2.0)
    for dv in ([0, 1e-3, 0], [2e-4, 0, 5e-4]):
        rec, ne, nc, res, st = av.emul(L, el, P, model, pr, se, jd, fr, w, 0.01, np.arange(m), bj, bf, dv,
                                       dv_sigma=sigma)
        for k in range(m):
            p = pr[k]
            (x, J), (_, Jp) = _jacobians(el[:, p], ne[k], P[p], model[p], bj[k], bf[k])
            ref = av.transport(J, Jp, K.unpack7(P[p]), x, sigma)
            got = K.unpack7(nc[k])
            scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
            assert np.abs(got - ref).max() <= 1e-4 * scale.max(), k
            assert np.all(np.abs(got - ref) <= 5e-3 * scale + 1e-30), k   # two propagators' forward differences


def test_execution_error_alone(L):
    """P = 0, sigma > 0: K10's Sigma (its host build) of the new row at t_b, in RTN, is diag(0, sigma^2) within 1e-7 of
    its scale on near-earth primaries (measured 4.5e-9 to 5.9e-8) and 2e-5 on deep-space ones (measured 1.0e-5 on the
    GEO row): Sigma = J'' P' J''^T with J'' the new set's own forward differences, whose noise P' = J'6^-1 Q J'6^-T
    does not cancel"""
    el, model, P, pr, se, jd, fr, w = _catalogue()
    m = len(pr)
    bj, bf = _burn(el, pr, jd, fr, 2.0)
    Z = np.zeros_like(P)
    sigma = np.array([3e-5, 1e-5, 2e-5])
    rec, ne, nc, res, st = av.emul(L, el, Z, model, pr, se, jd, fr, w, 0.01, np.arange(m), bj, bf, [0, 5e-4, 0],
                                   dv_sigma=sigma)
    KL = K.emul_library()
    for k in range(m):
        off = np.array([0, 1], np.uint32)
        _, sig, _, status = K.emul(KL, ne[k][:, None], nc[k][None], model[pr[k]:pr[k] + 1], off, np.array([bj[k]]),
                                   np.array([bf[k]]), frame=1)
        S = K.unpack6(sig[0])
        ref = np.zeros((6, 6))
        ref[3:, 3:] = np.diag(sigma ** 2)
        bound = 2e-5 if model[pr[k]] else 1e-7
        assert status[0] == 0 and np.abs(S - ref).max() <= bound * sigma.max() ** 2, (k, np.abs(S - ref).max())


def test_transport_against_monte_carlo(L):
    """20,000 draws from N(x^, P) of a fitted-scale P on the LEO ladder's primary, each propagated by the oracle to t_b,
    burnt and converted by the C restatement of the fit under the same rules: the sample covariance of the converted
    variables against P' within 5 sigma of its chi-square spread (per variance) and 5 sqrt(2 / N) (whitened)"""
    base, P, jd, fr = _ladder()
    bj, bf = jd, fr - 2.0 / base[1, 0]
    dv = np.array([0.0, 2e-3, 0.0])
    rec, ne, nc, res, st = av.emul(L, base, P, None, [0], [1], jd, fr, 5.0, 0.2, [0], bj, bf, dv)
    assert st[0] == av.OK
    N = 20000
    rng = np.random.default_rng(11)
    P7 = K.unpack7(P[0])[:6, :6]
    x0 = vars_of(base[:, 0], False)
    draws = x0[None, :6] + rng.multivariate_normal(np.zeros(6), P7, N)
    els = K.elements_of(np.c_[draws, np.full(N, base[7, 0])], base[0, 0], False)
    pos, vel = np.zeros((N, 3)), np.zeros((N, 3))
    for i in range(N):
        s = _oracle_state(els[:, i], bj, bf)
        R = av.rtn(s)
        pos[i], vel[i] = s[:3], s[3:] + R.T @ dv
    off = np.arange(N + 1, dtype=np.uint32)
    init = np.repeat(base[:, :1], N, axis=1)
    fitted, rms, _, status = fo.fit(init, off, np.full(N, bj), np.full(N, bf), pos, vel, fit_bstar=False, max_iter=50,
                                    threads=os.cpu_count() or 1)
    ok = (status == 0) & (rms[:, 0] <= 1e-6) & (rms[:, 1] <= 1e-9)
    assert ok.mean() > 0.999
    xs = np.stack([vars_of(fitted[:, i], False)[:6] for i in np.nonzero(ok)[0]])
    ref = K.unpack7(nc[0])[:6, :6]
    S = np.cov(xs.T)
    d = np.diag(ref)
    assert np.all(np.abs(np.diag(S) - d) <= 5 * np.sqrt(2.0 / len(xs)) * d)
    Lc = np.linalg.cholesky(ref)
    W = np.linalg.solve(Lc, np.linalg.solve(Lc, S).T)
    assert np.abs(W - np.eye(6)).max() <= 5 * np.sqrt(2.0 / len(xs))


# ---- 5. composition ---------------------------------------------------------------------------------------------------
def test_returned_row_composes_with_k11(L, LC):
    """K11 on the returned row appended to the catalogue gives the trial's record bit for bit"""
    el, model, P, pr, se, jd, fr, w = _catalogue()
    m = len(pr)
    bj, bf = _burn(el, pr, jd, fr, 2.0)
    rec, ne, nc, res, st = av.emul(L, el, P, model, pr, se, jd, fr, w, 0.01, np.arange(m), bj, bf, [1e-4, 2e-3, -5e-4],
                                   dv_sigma=[1e-5, 1e-5, 1e-5])
    n = el.shape[1]
    el2 = np.concatenate([el, ne.T], axis=1)
    P2 = np.concatenate([P, nc])
    md2 = np.concatenate([model, model[pr]])
    rec2, _, _, st2 = cj.emul(LC, el2, P2, md2, n + np.arange(m), se, jd, fr, w, 0.01)
    assert np.array_equal(st2, st) and np.array_equal(rec2.view(np.uint64), rec.view(np.uint64))


# ---- 6. statuses and invariants ---------------------------------------------------------------------------------------
def test_statuses(L):
    """BAD_TRIAL (burn inside the window, candidate index >= m), BAD_PAIR, CONVERSION_FAILED (a burn that takes a
    224-minute orbit across 225 minutes), every output zero for each"""
    el, model, P, pr, se, jd, fr, w = _catalogue()
    m = len(pr)
    bj, bf = _burn(el, pr, jd, fr, 2.0)
    # a near-earth primary just under 225 min and a crossing partner
    near = np.array([2460000.25, 1440.0 / 224.0, 0.001, 30.0, 10.0, 0.0, 0.0, 0.0])
    pair = cc.pair(near, 20.0, dnode=0.001)
    el2 = np.concatenate([el, pair], axis=1)
    P2 = np.concatenate([P, cc.P_words(2, scale=1.0, bstar=False)])
    md2 = np.concatenate([model, [0, 0]]).astype(np.uint8)
    n = el.shape[1]
    pr2, se2 = np.r_[pr, n, 0], np.r_[se, n + 1, 0]
    jd2, fr2, w2 = np.r_[jd, jd[0], jd[0]], np.r_[fr, fr[0], fr[0]], np.r_[w, 1.0, 1.0]
    cand = np.array([0, 0, m, m + 1, m + 2])
    bjd = np.r_[bj[0], jd[0], bj[0], jd[0] - 1.0, bj[0]]
    bfr = np.r_[bf[0], fr[0], bf[0], fr2[m], bf[0]]
    dv = np.array([[0, 1e-3, 0], [0, 1e-3, 0], [0, 0.5, 0], [0, 1e-3, 0], [0, 1e-3, 0]])
    rec, ne, nc, res, st = av.emul(L, el2, P2, md2, pr2, se2, jd2, fr2, w2, 0.01, cand, bjd, bfr, dv)
    assert list(st) == [av.OK, av.BAD_TRIAL, av.CONVERSION_FAILED, av.BAD_PAIR, av.BAD_TRIAL], st
    for k in (1, 2, 3, 4):
        assert (rec[k] == 0).all() and (ne[k] == 0).all() and (nc[k] == 0).all() and (res[k] == 0).all()
    rec, *_, st = av.emul(L, el2, P2, md2, pr2, se2, jd2, fr2, w2, 0.01, [m + 3], bjd[:1], bfr[:1], dv[:1])
    assert st[0] == av.BAD_TRIAL and (rec == 0).all()


def test_batch_order_and_duplicates_change_no_byte(L):
    el, model, P, pr, se, jd, fr, w = _catalogue()
    m = len(pr)
    bj, bf = _burn(el, pr, jd, fr, 2.0)
    rng = np.random.default_rng(3)
    t = 40
    cand = rng.integers(0, m, t)
    dv = rng.normal(0, 1e-3, (t, 3))
    dv[::7] = 0.0
    sg = np.abs(rng.normal(0, 1e-5, (t, 3)))
    full = av.emul(L, el, P, model, pr, se, jd, fr, w, 0.01, cand, bj[cand], bf[cand], dv, sg)
    perm = rng.permutation(t)
    shuf = av.emul(L, el, P, model, pr, se, jd, fr, w, 0.01, cand[perm], bj[cand][perm], bf[cand][perm], dv[perm],
                   sg[perm])
    for a, b in zip(full, shuf):
        assert np.array_equal(a[perm].view(np.uint8), b.view(np.uint8))
    for k in (0, 13, 39):
        one = av.emul(L, el, P, model, pr, se, jd, fr, w, 0.01, cand[k:k + 1].repeat(2), bj[cand[k:k + 1]].repeat(2),
                      bf[cand[k:k + 1]].repeat(2), np.repeat(dv[k:k + 1], 2, 0), np.repeat(sg[k:k + 1], 2, 0))
        for a, b in zip(full, one):
            assert np.array_equal(a[k].view(np.uint8), b[0].view(np.uint8))
            assert np.array_equal(b[0].view(np.uint8), b[1].view(np.uint8))


def _abi_inputs():
    el, model, P, pr, se, jd, fr, w = _catalogue()
    m = len(pr)
    bj, bf = _burn(el, pr, jd, fr, 2.0)
    return dict(el=np.ascontiguousarray(el), P=P, model=model, pr=pr.astype(np.uint32), se=se.astype(np.uint32), jd=jd,
                fr=fr, w=w, r=np.full(m, 0.01), cand=np.arange(m, dtype=np.uint32), bj=np.array(bj),
                bf=np.array(bf), dv=np.full((m, 3), 1e-3), sg=np.full((m, 3), 1e-5))


def _call(a, grav=1, device=0):
    from astroz_b200 import _lib

    m, t = len(a["pr"]), len(a["cand"])
    rec, ne, nc, res = np.full((t, 13), 7.0), np.full((t, 8), 7.0), np.full((t, 28), 7.0), np.full((t, 2), 7.0)
    st = np.full(t, 9, np.uint8)
    p = lambda x: None if x is None else C.c_void_p(x.ctypes.data)  # noqa: E731
    rc = _lib.lib().astroz_cuda_conjunction_maneuver(
        p(a["el"]), a["el"].shape[1], grav, p(a["P"]), p(a["model"]), p(a["pr"]), p(a["se"]), p(a["jd"]), p(a["fr"]),
        p(a["w"]), p(a["r"]), m, p(a["cand"]), p(a["bj"]), p(a["bf"]), p(a["dv"]), p(a["sg"]), t, device, p(rec),
        p(ne), p(nc), p(res), p(st))
    return rc, (rec, ne, nc, res, st)


REFUSALS = {
    "device": ({"device": -1}, "on one device"), "grav": ({"grav": 7}, "grav must be"),
    "row": ("se", "outside the catalogue"), "self": ("self", "with itself"), "window": ("w", "half windows"),
    "radius": ("r", "hard-body radii"), "model": ("model", "model byte"), "nan_el": ("nan_el", "elements must be"),
    "nan_P": ("nan_P", "covariance words"), "nan_time": ("fr", "guess times"), "candidate": ("cand", "candidate index"),
    "burn_in_window": ("late", "before its candidate's window"), "nan_burn": ("bj", "burn times"),
    "nan_dv": ("dv", "dv words"), "inf_sigma": ("sg_inf", "execution sigmas"), "negative_sigma": ("sg_neg", "sigmas"),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_c_abi_refusals(case):
    from astroz_b200 import _lib
    from astroz_b200._abi import DEFINES as D

    a = _abi_inputs()
    how, text = REFUSALS[case]
    kw = how if isinstance(how, dict) else {}
    edits = {
        "se": lambda: a["se"].__setitem__(1, a["el"].shape[1]), "self": lambda: a["se"].__setitem__(2, a["pr"][2]),
        "w": lambda: a["w"].__setitem__(0, 0.0), "r": lambda: a["r"].__setitem__(3, -1e-3),
        "nan_el": lambda: a["el"].__setitem__((2, 1), np.nan), "nan_P": lambda: a["P"].__setitem__((1, 3), np.inf),
        "fr": lambda: a["fr"].__setitem__(1, np.nan), "cand": lambda: a["cand"].__setitem__(4, len(a["pr"])),
        "late": lambda: a["bf"].__setitem__(2, a["fr"][2]), "bj": lambda: a["bj"].__setitem__(0, np.nan),
        "dv": lambda: a["dv"].__setitem__((3, 1), np.nan), "sg_inf": lambda: a["sg"].__setitem__((0, 2), np.inf),
        "sg_neg": lambda: a["sg"].__setitem__((5, 0), -1e-6),
    }
    if how == "model":
        a["model"] = a["model"].copy()
        a["model"][0] = 2
    elif not kw:
        edits[how]()
    rc, outs = _call(a, **kw)
    assert rc == D["ASTROZ_VALUE_ERROR"]
    assert text in _lib.lib().astroz_cuda_last_error().decode()
    assert all((o == 7.0).all() if o.dtype == np.float64 else (o == 9).all() for o in outs)


def test_scratch_bytes_and_device_call_scalars():
    from astroz_b200 import _lib
    from astroz_b200._abi import DEFINES as D

    b = C.c_uint64(0)
    assert _lib.lib().astroz_cuda_conjunction_maneuver_scratch_bytes(1000, C.byref(b)) == D["ASTROZ_OK"]
    assert b.value == av.emul_library().emul_avoid_scratch_bytes(1000)
    assert _lib.lib().astroz_cuda_conjunction_maneuver_scratch_bytes(4, None) == D["ASTROZ_NULL_POINTER"]
    dev = _lib.lib().astroz_cuda_conjunction_maneuver_device
    args = [None, 0, 1] + [None] * 8 + [0] + [None] * 5 + [4]
    assert dev(*args, -1, *[None] * 7) == D["ASTROZ_VALUE_ERROR"]
    assert dev(*args[:-1], 2 ** 31, 0, *[None] * 7) == D["ASTROZ_VALUE_ERROR"]
    assert dev(*args, 0, *[None] * 7) == D["ASTROZ_NULL_POINTER"]


def test_wrapper_broadcasts(monkeypatch):
    """maneuver_trials() broadcasts a scalar candidate, burn time and one dv over the trials and returns catalogue rows
    in the fit's layout"""
    from astroz_b200 import collision

    seen = {}

    class Fake:
        def astroz_cuda_conjunction_maneuver(self, el, n, grav, cov, md, pr, se, jd, fr, w, r, m, ca, bj, bf, dv, sg,
                                             t, dev, rec, ne, nc, res, st):
            arr = lambda ptr, ty, shape: np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ty)), shape)  # noqa: E731
            seen.update(ca=arr(ca, C.c_uint32, (t,)).copy(), dv=arr(dv, C.c_double, (t, 3)).copy(),
                        bj=arr(bj, C.c_double, (t,)).copy(), sg=sg, t=t)
            arr(ne, C.c_double, (t, 8))[:] = np.arange(8.0)
            return 0

    monkeypatch.setattr(collision, "lib", lambda: Fake())
    el, model, _ = cc.catalogue()
    n = el.shape[1]
    res = collision.maneuver_trials(el, [0, 2], [1, 3], 2460000.5, 0.25, window_min=1.0, hbr_km=0.01, candidate=1,
                                    burn_jd=2460000.5, burn_fr=[0.1, 0.2, 0.3], dv_rtn=[0, 1e-3, 0],
                                    covariance=np.zeros((n, 28)), model=model)
    assert seen["t"] == 3 and (seen["ca"] == 1).all() and (seen["dv"] == [0, 1e-3, 0]).all() and seen["sg"] is None
    e, P, md = res.catalogue_rows()
    assert e.shape == (8, 3) and (e[:, 0] == np.arange(8.0)).all() and P.shape == (3, 28) and (md == model[2]).all()


# ---- 7. the planner ---------------------------------------------------------------------------------------------------
def _host_run(L, el, P, md, pr, se, jd, fr, w, hbr):
    def run(cand, bjd, bfr, dv, sg):
        rec, ne, nc, res, st = av.emul(L, el, P, md, pr, se, jd, fr, w, hbr, cand, bjd, bfr, dv, sg)
        return rec, st
    return run


def test_planner_on_the_ladder(L):
    """pc_max 1e-6 on the 1.7-sigma LEO crossing: the returned dv meets it, dv (1 - 2 * 2^-rounds) does not, and a
    brute-force scan of 2,000 magnitudes finds the same first crossing within the bisection width"""
    from astroz_b200.collision import _avoidance

    base, P, jd, fr = _ladder()
    run = _host_run(L, base, P, None, np.array([0]), np.array([1]), jd, fr, 5.0, 0.2)
    rounds, dv_max = 20, 0.05
    r = _avoidance(run, 1, np.array([jd]), np.array([fr]), [30.0, 120.0], (0, 1, 0), 1e-6, dv_max, 32, rounds, None)
    assert r.pc.shape == (1, 2, 2, 32) and r.pc_nominal[0] > 1e-6
    for li in range(2):
        for s in range(2):
            dv = r.dv_kms[0, li, s]
            assert np.isfinite(dv), (li, s)
            assert r.record[0, li, s, 12] <= 1e-6 and r.status[0, li, s] == av.OK
            u = np.array([0, (-1.0, 1.0)[s], 0])
            below = dv * (1 - 2 * 2.0 ** -rounds)
            rec, st = run([0], [r.burn_jd[0, li]], [r.burn_fr[0, li]], (below * u)[None], None)
            assert rec[0, 12] > 1e-6
            # brute force from 0 to the ladder step above dv
            top = r.ladder_kms[np.searchsorted(r.ladder_kms, dv)]
            mags = np.linspace(top / 2000, top, 2000)
            rec, st = run(np.zeros(2000, np.int64), np.full(2000, r.burn_jd[0, li]), np.full(2000, r.burn_fr[0, li]),
                          mags[:, None] * u[None], None)
            feas = (st == av.OK) & (rec[:, 12] <= 1e-6)
            first = mags[np.argmax(feas)]
            width = top / 2 / 2.0 ** rounds + top / 2000
            assert abs(first - dv) <= width, (li, s, first, dv)


def _engineered():
    """A LEO crossing at 40 deg whose secondary trails the primary along track (its mean anomaly 0.01 deg on, no node
    offset), P scaled so that the nominal miss sits at 2 sigma, radius 0.2 km; the guess at the TCA"""
    base = cc.pair(cc.leo(), 40.0, dnode=0.0, dm=0.01)
    P0 = cc.P_words(2, scale=1.0, bstar=False)
    jd = np.floor(base[0, 0] - 0.5) + 0.5
    fr = base[0, 0] - jd + 3.0 / 1440.0
    rec = cj.emul(cj.emul_library(), base, P0, None, [0], [1], jd, fr, 5.0, 0.02)[0][0]
    xx, xy, yy = rec[9:12]
    k0 = rec[1] * np.sqrt(yy / (xx * yy - xy * xy))
    return base, P0 * (k0 / 2.0) ** 2, jd, fr + rec[0] / 1440.0, rec


def test_planner_with_a_non_monotone_pc(L):
    """On the engineered crossing the secondary trails the primary along track (dr_T < 0), so by Clohessy-Wiltshire
    (along-track -3 dv t after whole orbits) a +T burn first moves the primary back towards it: Pc rises above the
    nominal, then falls below pc_max.  The planner returns the least feasible dv of a brute-force scan on that sign
    (and on the monotone -T sign) within the bisection width"""
    from astroz_b200.collision import _avoidance

    base, P, jd, fr, rec = _engineered()
    assert rec[4] < 0                                  # dr_T: the secondary trails
    run = _host_run(L, base, P, None, np.array([0]), np.array([1]), jd, fr, 5.0, 0.2)
    lead = 2.0 / base[1, 0] * 1440.0                    # two orbits
    rounds, pc_max = 20, 1e-4
    r = _avoidance(run, 1, np.array([jd]), np.array([fr]), [lead], (0, 1, 0), pc_max, 2e-3, 16, rounds, None)
    up = r.pc[0, 0, 1]
    assert r.pc_nominal[0] > pc_max and np.nanmax(up) > 1.2 * r.pc_nominal[0], (r.pc_nominal, up)
    peak = r.ladder_kms[np.nanargmax(up)]
    for s in range(2):
        dv = r.dv_kms[0, 0, s]
        assert np.isfinite(dv) and r.status[0, 0, s] == av.OK and r.record[0, 0, s, 12] <= pc_max
        top = r.ladder_kms[np.searchsorted(r.ladder_kms, dv)]
        mags = np.linspace(top / 2000, top, 2000)
        u = np.array([0, (-1.0, 1.0)[s], 0])
        rc, st = run(np.zeros(2000, np.int64), np.full(2000, r.burn_jd[0, 0]), np.full(2000, r.burn_fr[0, 0]),
                     mags[:, None] * u[None], None)
        feas = (st == av.OK) & (rc[:, 12] <= pc_max)
        first = mags[np.argmax(feas)]
        assert abs(first - dv) <= top / 2 / 2.0 ** rounds + top / 2000, (s, first, dv)
    assert r.dv_kms[0, 0, 1] > peak > r.dv_kms[0, 0, 0]


def test_planner_rejects_a_burn_that_leaves_the_window(L):
    """With a half window of 0.004 min about the TCA, -T burns of 0.13 m/s and more move the TCA out of it: those
    trials are WINDOW_EDGE with a Pc taken at the window end, below pc_max from 0.25 m/s on.  The planner does not
    count them, so -T finds nothing; with a 0.5 min window the same burns are OK and it finds one"""
    from astroz_b200.collision import NOT_FOUND, _avoidance

    base, P, jd, fr, _ = _engineered()
    lead = 2.0 / base[1, 0] * 1440.0
    args = (1, np.array([jd]), np.array([fr]), [lead], (0, -1, 0), 1e-4, 1e-3, 8, 20, None)
    narrow = _host_run(L, base, P, None, np.array([0]), np.array([1]), jd, fr, 0.004, 0.2)
    steps = 1e-3 * 2.0 ** (np.arange(8) - 7)
    rc, st = narrow(np.zeros(8, np.int64), np.full(8, jd), np.full(8, fr - lead / 1440.0),
                    -steps[:, None] * np.array([0, 1.0, 0])[None], None)
    edge = (st == av.WINDOW_EDGE) & (rc[:, 12] <= 1e-4)
    assert edge.any() and not ((st == av.OK) & (rc[:, 12] <= 1e-4)).any(), (st, rc[:, 12])
    r = _avoidance(narrow, *args)
    assert np.isnan(r.dv_kms).all() and (r.status == NOT_FOUND).all() and (r.record == 0).all()
    assert np.isnan(r.pc[0, 0, 1][st == av.WINDOW_EDGE]).all()   # sign 1: +direction, -T
    wide = _avoidance(_host_run(L, base, P, None, np.array([0]), np.array([1]), jd, fr, 0.5, 0.2), *args)
    assert np.isfinite(wide.dv_kms).all() and (wide.status == av.OK).all()


def test_a_failed_reassessment_zeroes_every_output(L):
    """A secondary that K11 cannot build (a near-earth set under model byte 1): the burn and the conversion succeed,
    K11 answers INIT_FAILED, and the trial's record, row, P' and residual are all zero"""
    base = cc.pair(cc.leo(), 40.0, dnode=0.0005)
    P = cc.P_words(2, scale=1.0, bstar=False)
    jd = np.floor(base[0, 0] - 0.5) + 0.5
    fr = base[0, 0] - jd
    rec, ne, nc, res, st = av.emul(L, base, P, np.array([0, 1], np.uint8), [0], [1], jd, fr, 1.0, 0.01, [0, 0], jd,
                                   fr - 2.0 / base[1, 0], [[0, 1e-3, 0], [0, 0, 0]])
    assert (st == av.INIT_FAILED).all()
    assert (rec == 0).all() and (ne == 0).all() and (nc == 0).all() and (res == 0).all()
