"""K11 conjunction assessment (az_conjunction.cuh, az_conjunction.cu) on the CPU.

The host build of the device source (tests/host_emul/emul_conjunction.cu): its Pc integrator against a 30-digit mpmath
value, the closed form of an isotropic C2, the degenerate limits and the scale rule; its TCA, states and Sigma against
the independent C restatement on the oracle's SGP4 / SDP4 (tests/fit_oracle/conjunction.c) on engineered crossings;
the window rules, symmetry and zero-P rule; a Monte Carlo through the oracle; the C ABI's refusals and the Python
wrapper's order.  The device runs are in tests/test_gpu_conjunction.py."""
import ctypes as C

import numpy as np
import pytest

from tests.fit_oracle import conjunction as cj
from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import covariance as K


@pytest.fixture(scope="module")
def L():
    lib = cj.emul_library()
    if lib is None:
        pytest.skip("nvcc unavailable")
    return lib


def _c2(sigma, ratio, angle):
    """C2 words (xx, xy, yy) of major semi-axis sigma, minor sigma / ratio, major axis at `angle` from the miss"""
    c, s = np.cos(angle), np.sin(angle)
    l1, l2 = sigma ** 2, (sigma / ratio) ** 2
    return l1 * c * c + l2 * s * s, (l1 - l2) * c * s, l1 * s * s + l2 * c * c


# ---- 1. the Pc integrator -------------------------------------------------------------------------------------------
GRID = [(dsig, sr, ratio, k) for dsig in (0.0, 1.0, 4.0, 15.0) for sr in (1e-2, 1.0, 1e2, 1e4)
        for ratio in (1.0, 1e2, 1e4) for k in range(8)]


def _grid_case(case):
    dsig, sr, ratio, k = case
    xx, xy, yy = _c2(sr, ratio, k * np.pi / 8)
    return (xx, xy, yy, dsig * sr), cj.pc_reference(xx, xy, yy, dsig * sr, 1.0)


def test_pc_against_the_30_digit_reference(L):
    """d / sigma 0 .. 15, sigma / R 1e-2 .. 1e4, axis ratio 1 .. 1e4, 8 orientations (384 cases, the references on a
    process pool): within 1e-6 relative wherever the reference is above 1e-60, and below 1e-55 elsewhere.  The
    reference integrates along the minor axis with mpmath's own error control, the device along the major axis by
    fixed panels."""
    import os
    from concurrent.futures import ProcessPoolExecutor

    with ProcessPoolExecutor(max_workers=os.cpu_count() or 1) as ex:
        refs = list(ex.map(_grid_case, GRID, chunksize=4))
    worst, n = 0.0, 0
    for (args, ref), case in zip(refs, GRID):
        got = cj.emul_pc(L, *args, 1.0)
        if ref > 1e-60:
            worst = max(worst, abs(got - ref) / ref)
            n += 1
            assert abs(got - ref) <= 1e-6 * ref, (case, got, ref)
        else:
            assert got <= 1e-55, (case, got, ref)
    print(f"Pc vs 30-digit reference: {n} of {len(GRID)} cases above 1e-60, worst relative {worst:.2e}")
    assert n > 250


def test_isotropic_pc_is_the_noncentral_chi_square():
    from scipy.stats import ncx2

    L_ = cj.emul_library()
    worst = 0.0
    for sr in np.geomspace(1e-2, 1e4, 13):
        for dsig in np.linspace(0.0, 15.0, 16):
            s, R = sr, 1.0
            ref = ncx2.cdf(R * R / (s * s), 2, (dsig * dsig))
            got = cj.emul_pc(L_, s * s, 0.0, s * s, dsig * s, R)
            if ref > 1e-300 and ref < 1.0 - 1e-12:
                worst = max(worst, abs(got - ref) / ref)
    print(f"isotropic Pc vs ncx2: worst relative {worst:.2e}")
    assert worst < 1e-6


def test_degenerate_limits(L):
    # C2 = 0: the indicator d < R
    assert cj.emul_pc(L, 0.0, 0.0, 0.0, 0.5, 1.0) == 1.0
    assert cj.emul_pc(L, 0.0, 0.0, 0.0, 1.5, 1.0) == 0.0
    assert cj.emul_pc(L, 0.0, 0.0, 0.0, 1.0, 1.0) == 0.0
    # one eigenvalue 0: a 1-D normal difference over the chord the line of the mean cuts from the disk
    from scipy.stats import norm

    s, d, R = 0.7, 0.4, 1.0
    ref = norm.cdf((R - d) / s) - norm.cdf((-R - d) / s)   # major axis along the miss: chord [-R, R]
    assert abs(cj.emul_pc(L, s * s, 0.0, 0.0, d, R) - ref) < 1e-15
    h = np.sqrt(R * R - d * d)                             # major axis across the miss: chord half-length h
    ref = norm.cdf(h / s) - norm.cdf(-h / s)
    assert abs(cj.emul_pc(L, 0.0, 0.0, s * s, d, R) - ref) < 1e-15
    assert cj.emul_pc(L, 0.0, 0.0, s * s, 1.2, R) == 0.0


def test_scale_rule(L):
    """Pc(k C2, sqrt(k) R, sqrt(k) d) = Pc(C2, R, d) within 1e-9 relative: the panel edges are rounded anew at each
    scale, which moves the quadrature's own error by ~1e-11"""
    rng = np.random.default_rng(1)
    for _ in range(40):
        xx, xy, yy = _c2(10 ** rng.uniform(-2, 3), 10 ** rng.uniform(0, 3), rng.uniform(0, np.pi))
        d, R = 10 ** rng.uniform(-1, 2), 1.0
        base = cj.emul_pc(L, xx, xy, yy, d, R)
        for k in (1e-6, 4.0, 1e8):
            got = cj.emul_pc(L, k * xx, k * xy, k * yy, np.sqrt(k) * d, np.sqrt(k) * R)
            assert abs(got - base) <= 1e-9 * base + 1e-300


# ---- 2. the host build against the restatement ----------------------------------------------------------------------
def _run(L, el, model, P, cands, jd=None, fr=None, hbr=0.01, frame=0):
    pr = np.array([c[0] for c in cands])
    se = np.array([c[1] for c in cands])
    w = np.array([c[2] for c in cands])
    if jd is None:
        jd = np.floor(el[0][pr] - 0.5) + 0.5
        fr = el[0][pr] - jd
    return cj.emul(L, el, P, model, pr, se, jd, fr, w, hbr, frame), (pr, se, jd, fr, w)


@pytest.mark.parametrize("frame", [0, 1])
def test_host_build_matches_the_restatement(L, frame):
    """Engineered crossings (LEO-LEO di 0.5 .. 170 deg, LEO-Molniya, LEO-GTO, GEO-GEO): equal statuses,
    |dTCA| |dv| <= 1e-7 km (measured 2.4e-8), miss within 1e-7 km (6e-11), each Sigma within K10's 6e-6 of its scale
    (3.5e-7), C2 within 1e-6 of its scale against a numpy plane on the restatement's states and Sigma, and Pc within
    1e-6 relative (or 1e-60) of the 30-digit value on the host build's own plane.  The Pc of the restatement's plane
    is printed, not asserted: the two Sigma differ by ~3e-7 of scale, which (d / sigma)^2 amplifies in a tail Pc
    (measured 2.5e-5 relative at d / sigma ~ 9)."""
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], scale=30.0, deep=model.astype(bool))
    (rec, st, sig, status), (pr, se, jd, fr, w) = _run(L, el, model, P, cands, frame=frame, hbr=0.05)
    dt, rst, rsig, rstatus = cj.restated(el, P, model, pr, se, jd, fr, w, frame=frame)
    assert (status == rstatus).all()
    worst = {"tca": 0.0, "miss": 0.0, "sig": 0.0, "c2": 0.0, "pc": 0.0, "pc_restated_plane": 0.0}
    for k, c in enumerate(cands):
        miss, speed, d, c2 = cj.plane(rst[k], rsig[k], frame)
        worst["tca"] = max(worst["tca"], abs(rec[k, 0] - dt[k]) * 60.0 * speed)
        worst["miss"] = max(worst["miss"], abs(rec[k, 1] - miss))
        for o in range(2):
            worst["sig"] = max(worst["sig"], np.abs(sig[k, o] - rsig[k, o]).max() / np.abs(rsig[k, o]).max())
        worst["c2"] = max(worst["c2"], np.abs(rec[k, 9:12] - c2).max() / np.abs(c2).max())
        own = cj.plane(st[k], sig[k], frame)
        ref = cj.pc_reference(*rec[k, 9:12], own[2], 0.05)
        rref = cj.pc_reference(*c2, d, 0.05)
        if ref > 1e-60:
            worst["pc"] = max(worst["pc"], abs(rec[k, 12] - ref) / ref)
            worst["pc_restated_plane"] = max(worst["pc_restated_plane"], abs(rec[k, 12] - rref) / rref)
        else:
            assert rec[k, 12] < 1e-55
    print("host build vs restatement: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    assert worst["tca"] <= 1e-7 and worst["miss"] <= 1e-7 and worst["sig"] <= 6e-6
    assert worst["c2"] <= 1e-6 and worst["pc"] <= 1e-6


# ---- 3. window rules, symmetry, zero P ------------------------------------------------------------------------------
def _leo_pair():
    el = cc.pair(cc.leo(), 60.0, dnode=0.003, dm=0.0)
    return el, np.zeros(2, np.uint8), cc.P_words(2, scale=30.0)


def test_window_rules(L):
    el, model, P = _leo_pair()
    jd0 = np.floor(el[0, 0] - 0.5) + 0.5
    fr0 = el[0, 0] - jd0
    (rec, _, _, status), _ = _run(L, el, model, P, [(0, 1, 1.0, "")], np.array([jd0]), np.array([fr0]))
    assert status[0] == 0
    tca = rec[0, 0]
    # moving the guess inside the window does not move the TCA beyond the tolerance
    t_abs = lambda fr, dt: ((jd0 + fr) - el[0, 0]) * 1440.0 + dt   # noqa: E731  (the guess's tsince, as K10 forms it)
    for shift in (-0.6, -0.2, 0.3, 0.7):
        fr = fr0 + shift / 1440
        (r2, _, _, s2), _ = _run(L, el, model, P, [(0, 1, 1.0, "")], np.array([jd0]), np.array([fr]))
        assert s2[0] == 0
        assert abs(t_abs(fr, r2[0, 0]) - t_abs(fr0, tca)) * 60.0 * rec[0, 2] < 1e-7
        assert abs(r2[0, 1] - rec[0, 1]) < 1e-7
    # a minimum outside the window: WINDOW_EDGE at the nearer end, the outputs filled
    (r3, _, _, s3), _ = _run(L, el, model, P, [(0, 1, 0.5, "")], np.array([jd0]), np.array([fr0 + 2.0 / 1440]))
    assert s3[0] == 3 and r3[0, 0] == -0.5 and r3[0, 1] > rec[0, 1] and r3[0, 12] >= 0.0
    # two minima half an orbit apart (both orbits cross at both nodes): the deeper one is returned
    period = 1440.0 / el[1, 0]
    (r4, _, _, s4), _ = _run(L, el, model, P, [(0, 1, 0.8 * period, "")], np.array([jd0]),
                             np.array([fr0 + 0.3 * period / 1440]))
    (ra, _, _, _), _ = _run(L, el, model, P, [(0, 1, 2.0, "")], np.array([jd0]), np.array([fr0]))
    (rb, _, _, _), _ = _run(L, el, model, P, [(0, 1, 2.0, "")], np.array([jd0]), np.array([fr0 + 0.5 * period / 1440]))
    assert s4[0] == 0
    assert abs(r4[0, 1] - min(ra[0, 1], rb[0, 1])) < 1e-6


def test_swap_symmetry(L):
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], scale=30.0, deep=model.astype(bool))
    (rec, _, _, status), _ = _run(L, el, model, P, cands, hbr=0.05)
    swapped = [(c[1], c[0], c[2], c[3]) for c in cands]
    pr = np.array([c[0] for c in cands])
    jd = np.floor(el[0][pr] - 0.5) + 0.5
    (rs, _, _, ss), _ = _run(L, el, model, P, swapped, jd=jd, fr=el[0][pr] - jd, hbr=0.05)
    assert (status == ss).all()
    for k in range(len(cands)):
        for q in (0, 1, 2):
            assert abs(rs[k, q] - rec[k, q]) <= 1e-12 * max(1.0, abs(rec[k, q])) * (100 if q == 0 else 1)
        e1 = np.linalg.eigvalsh(np.array([[rec[k, 9], rec[k, 10]], [rec[k, 10], rec[k, 11]]]))
        e2 = np.linalg.eigvalsh(np.array([[rs[k, 9], rs[k, 10]], [rs[k, 10], rs[k, 11]]]))
        assert np.allclose(e1, e2, rtol=1e-9, atol=0)
        assert abs(rs[k, 12] - rec[k, 12]) <= 1e-9 * rec[k, 12] + 1e-300


def test_zero_P_gives_the_indicator(L):
    el, model, cands = cc.catalogue()
    P = np.zeros((el.shape[1], 28))
    (rec, st, sig, status), _ = _run(L, el, model, P, cands, hbr=1.0)
    assert (status == 0).all() and (sig == 0).all() and (rec[:, 9:12] == 0).all()
    assert ((rec[:, 12] == 1.0) == (rec[:, 1] < 1.0)).all() and set(np.unique(rec[:, 12])) <= {0.0, 1.0}


# ---- 4. Monte Carlo through the oracle ------------------------------------------------------------------------------
def _monte_carlo(L, el, model, P, cand, hbr, draws, seed):
    """`draws` samples N(x, P) of both rows' variables.  Returns the host build's record, the fraction of drawn pairs
    whose miss at their own TCA (the restatement's) is below hbr, the same fraction under the linear model (each draw's
    relative position at the nominal TCA mapped by J, projected on the nominal encounter plane), and the draws
    counted.  The two fractions share their draws, so their difference is the linearisation effect with little
    sampling noise."""
    from tests.fit_oracle.covariance import elements_of, unpack7

    rng = np.random.default_rng(seed)
    p, s, w = cand
    jd = np.floor(el[0, p] - 0.5) + 0.5
    fr = el[0, p] - jd
    (rec, _, _, status), _ = _run(L, el, model, P, [(p, s, w, "")], np.array([jd]), np.array([fr]), hbr=hbr)
    # J of both rows at the nominal TCA (covariance.c) and the nominal plane
    two = np.ascontiguousarray(el[:, [p, s]])
    f0, _, J, _ = K.restated(two, P[[p, s]], model[[p, s]], np.array([0, 1, 2]), np.full(2, jd),
                             np.full(2, fr + rec[0, 0] / 1440.0))
    dr0 = f0[1, :3] - f0[0, :3]
    z = (f0[1, 3:] - f0[0, 3:]) / np.linalg.norm(f0[1, 3:] - f0[0, 3:])
    xh = dr0 - (dr0 @ z) * z
    xh /= np.linalg.norm(xh)
    E = np.stack([xh, np.cross(z, xh)])
    cols, lin = [], dr0.copy()[None, :]
    for k, o in enumerate((p, s)):
        deep = bool(model[o])
        e = el[:, o]
        if not deep:
            wr = np.radians(e[5])
            x = np.array([e[1], e[2] * np.cos(wr), e[2] * np.sin(wr), np.radians(e[3]), np.radians(e[4]),
                          np.radians(e[6]) + wr, e[7]])
        else:
            node, peri, ti = np.radians(e[4]), np.radians(e[5] + e[4]), np.tan(np.radians(e[3]) / 2)
            x = np.array([e[1], e[2] * np.cos(peri), e[2] * np.sin(peri), ti * np.cos(node), ti * np.sin(node),
                          np.radians(e[6]) + peri, e[7]])
        draws_x = rng.multivariate_normal(x, unpack7(P[o]), size=draws, method="eigh")
        cols.append(elements_of(draws_x, e[0], deep))
        lin = lin + (1.0 if k else -1.0) * (draws_x - x) @ J[k, :3].T
    sel = np.empty((8, 2 * draws))
    sel[:, 0::2], sel[:, 1::2] = cols[0], cols[1]
    md = np.repeat(model[[p, s]][None], draws, axis=0).reshape(-1)
    pr, se = np.arange(0, 2 * draws, 2), np.arange(1, 2 * draws, 2)
    dt, st, _, rstatus = cj.restated(sel, np.zeros((2 * draws, 28)), md, pr, se, jd, fr, np.full(draws, w))
    miss = np.linalg.norm(st[:, 1, :3] - st[:, 0, :3], axis=1)
    ok = np.isin(rstatus, (0, 3))
    lin_hit = np.linalg.norm(lin @ E.T, axis=1) < hbr
    return rec[0], (miss[ok] < hbr).mean(), lin_hit[ok].mean(), ok.sum()


def test_monte_carlo_high_pc_leo(L):
    """20,000 draws of a LEO crossing at Pc 0.26 (conjunction_cases.high_pc_leo).  The hit fraction must lie within 4
    binomial sigma of the linear Pc plus a linearisation allowance of 0.01.  The allowance is measured here: the
    fraction under the linear model from the same draws differs from the nonlinear one by the linearisation effect
    alone, and that difference must stay below 0.01 (measured 1.5e-4); the linear model's own fraction must lie within 4
    sigma of Pc."""
    el, P, hbr = cc.high_pc_leo(lambda el, P, hbr: _run(L, el, np.zeros(2, np.uint8), P, [(0, 1, 1.0, "")],
                                                           hbr=hbr)[0][0][0])
    model = np.zeros(2, np.uint8)
    rec, frac, frac_lin, n = _monte_carlo(L, el, model, P, (0, 1, 1.0), hbr, 20000, seed=11)
    pc = rec[12]
    sig = np.sqrt(pc * (1 - pc) / n)
    print(f"LEO Monte Carlo: Pc {pc:.4f}, hit fraction {frac:.4f}, linear-model fraction {frac_lin:.4f} over {n} "
          f"draws, 4 sigma {4 * sig:.4f}, measured linearisation effect {abs(frac - frac_lin):.1e}")
    assert 0.1 < pc < 0.3
    assert abs(frac_lin - pc) <= 4 * sig
    assert abs(frac - frac_lin) <= 0.01
    assert abs(frac - pc) <= 4 * sig + 0.01


def test_monte_carlo_slow_geo_ratio_is_printed(L):
    """The short-encounter model's known limit: a GEO pair at ~3 m/s stays close for tens of minutes, so the hit
    fraction over the window and the 2-D Pc can differ.  The ratio is printed, not asserted."""
    el = cc.pair(cc.geo(), 0.05, dnode=0.0, dm=0.0)
    model = np.ones(2, np.uint8)
    P = cc.P_words(2, scale=0.2, bstar=False, deep=np.ones(2, bool))
    rec, frac, frac_lin, n = _monte_carlo(L, el, model, P, (0, 1, 30.0), 0.05, 4000, seed=12)
    print(f"GEO Monte Carlo: Pc {rec[12]:.3e}, hit fraction {frac:.3e} (linear model {frac_lin:.3e}) over {n} draws, "
          f"ratio {frac / rec[12] if rec[12] > 0 else float('nan'):.3f}")


# ---- 5. the C ABI's refusals and the wrapper's order ----------------------------------------------------------------
def _abi_inputs():
    el, model, cands = cc.catalogue()
    P = cc.P_words(el.shape[1], deep=model.astype(bool))
    m = len(cands)
    pr = np.array([c[0] for c in cands], np.uint32)
    se = np.array([c[1] for c in cands], np.uint32)
    jd = np.floor(el[0][pr] - 0.5) + 0.5
    return dict(el=np.ascontiguousarray(el), P=P, model=model, pr=pr, se=se, jd=jd, fr=el[0][pr] - jd,
                w=np.ones(m), r=np.full(m, 0.01))


def _call(a, grav=1, frame=0, device=0):
    from astroz_b200 import _lib

    m = len(a["pr"])
    rec = np.full((m, 13), 7.0)
    st = np.full(m, 9, np.uint8)
    p = lambda x: None if x is None else C.c_void_p(x.ctypes.data)  # noqa: E731
    rc = _lib.lib().astroz_cuda_conjunction(p(a["el"]), a["el"].shape[1], grav, p(a["P"]), p(a["model"]), p(a["pr"]),
                                            p(a["se"]), p(a["jd"]), p(a["fr"]), p(a["w"]), p(a["r"]), m, frame, device,
                                            p(rec), None, None, p(st))
    return rc, rec, st


@pytest.mark.parametrize("case", ["device", "grav", "frame", "row", "self", "window", "radius", "model", "nan_el",
                                  "nan_P", "nan_time", "nan_window", "inf_radius"])
def test_c_abi_refusals(case):
    from astroz_b200._abi import DEFINES as D

    a = _abi_inputs()
    kw = {}
    if case == "device":
        kw["device"] = -1
    elif case == "grav":
        kw["grav"] = 7
    elif case == "frame":
        kw["frame"] = 2
    elif case == "row":
        a["se"][1] = a["el"].shape[1]
    elif case == "self":
        a["se"][2] = a["pr"][2]
    elif case == "window":
        a["w"][0] = 0.0
    elif case == "radius":
        a["r"][3] = -1e-3
    elif case == "model":
        a["model"] = a["model"].copy()
        a["model"][0] = 2
    elif case == "nan_el":
        a["el"][2, 1] = np.nan
    elif case == "nan_P":
        a["P"][1, 3] = np.inf
    elif case == "nan_time":
        a["fr"][1] = np.nan
    elif case == "nan_window":
        a["w"][1] = np.nan
    elif case == "inf_radius":
        a["r"][1] = np.inf
    rc, rec, st = _call(a, **kw)
    assert rc == D["ASTROZ_VALUE_ERROR"]
    assert (rec == 7.0).all() and (st == 9).all()


def test_wrapper_keeps_candidate_order(monkeypatch):
    """conjunctions() passes candidates through in the caller's order and splits the TCA into (jd, fr + dt / 1440)"""
    from astroz_b200 import collision

    seen = {}

    class Fake:
        def astroz_cuda_conjunction(self, el, n, grav, cov, md, pr, se, jd, fr, w, r, m, frame, dev, rec, st, sig,
                                    stat):
            prv = np.ctypeslib.as_array(C.cast(pr, C.POINTER(C.c_uint32)), (m,)).copy()
            seen["pr"] = prv
            out = np.ctypeslib.as_array(C.cast(rec, C.POINTER(C.c_double)), (m, 13))
            out[:, 0] = prv * 0.5
            out[:, 12] = prv / 100.0
            return 0

    monkeypatch.setattr(collision, "lib", lambda: Fake())
    el, model, _ = cc.catalogue()
    n = el.shape[1]
    pr = np.array([5, 0, 3, 9, 2])
    se = (pr + 1) % n
    res = collision.conjunctions(el, pr, se, 2460000.5, 0.25, window_min=1.0, hbr_km=0.01,
                                 covariance=np.zeros((n, 28)), model=model)
    assert (seen["pr"] == pr).all()
    assert np.allclose(res.pc, pr / 100.0) and np.allclose(res.tca_fr, 0.25 + pr * 0.5 / 1440.0)
    assert (res.tca_jd == 2460000.5).all()
    with pytest.raises(ValueError):
        collision.conjunctions(el, [0, n], [1, 2], 2460000.5, 0.0, window_min=1.0, hbr_km=0.01,
                               covariance=np.zeros((n, 28)))
