"""Deep-space element fits on the CPU: the independent restatement (tests/fit_oracle/fit_oracle_deep.c,
fitref_fit_mixed on the oracle's SDP4) recovers config-3 GEO, Molniya and GPS-like sets from perturbed guesses; the fit's
own source (az_fit.cuh's FitDeepSpace with fit_deep_kernel's pass, run by tests/host_emul/emul_fit_deep.cu) agrees with
it; the resonance lattice gives the bits of stepping fresh from atime = 0; the statuses of the mixed entry point; the C
ABI refusals of the _mixed exports.  The device runs are in tests/test_gpu_fit_deep.py."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import fit_oracle as R
from tests.fit_oracle import deep as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "host_emul")
LYDDANE = np.degrees(0.2)   # dpper switches to its low-inclination form below 0.2 rad


def deep_cases():
    """Config-3 deep-space sets: 4 GEO (irez 1), then GEO variants at i = 0, i = 1e-3 deg, e = 0 and i just either side
    of 0.2 rad, then 4 GPS-like (irez 0) and 4 Molniya (irez 2).  Returns (elements (8, 17), held) where held marks
    the GEO and GPS-like sets, whose B* is held: a day says nothing about their drag."""
    from astroz_b200 import synth

    el = synth.elements_from_tles(synth.mixed_catalog(13478))
    deep = el[:, 1440.0 / el[1] > 225.0]
    geo = deep[:, np.abs(deep[1] - 1.0027) < 0.001][:, :4]
    gps = deep[:, (np.abs(deep[1] - 2.0056) < 0.001) & (deep[2] < 0.05)][:, :4]
    mol = deep[:, deep[2] > 0.5][:, :4]
    extra = np.repeat(geo[:, :1], 5, axis=1)
    extra[3] = [0.0, 1e-3, 5.0, LYDDANE - 0.01, LYDDANE + 0.01]
    extra[2, 2] = 0.0
    cases = np.concatenate([geo, extra, gps, mol], axis=1)
    held = np.arange(cases.shape[1]) < 13
    return cases, held


def observations(el, jd, fr):
    """Oracle TEME observations of every (deep-space) column of el at the same epochs: (jd, fr, pos, vel, offsets)."""
    n, m = el.shape[1], len(jd)
    pos, vel = np.zeros((n, m, 3)), np.zeros((n, m, 3))
    for s in range(n):
        pos[s], vel[s] = D.observe(el[:, s], jd, fr)
    return np.tile(jd, n), np.tile(fr, n), pos.reshape(-1, 3), vel.reshape(-1, 3), \
        np.arange(n + 1, dtype=np.uint32) * m


def guesses(el, held):
    g = R.perturbed(el, seed=1)
    g[3] = np.abs(g[3])          # i = 0 +- 0.05 deg: keep the guess's inclination non-negative
    g[7, held] = el[7, held]
    return g


def equinoctial(f):
    """(k, h, q, p, lambda) of element columns: the deep-space fit's variables, defined at i = 0 and e = 0"""
    d = np.pi / 180.0
    node = f[4] * d
    P = f[5] * d + node
    ti = np.tan(0.5 * f[3] * d)
    return np.array([f[2] * np.cos(P), f[2] * np.sin(P), ti * np.cos(node), ti * np.sin(node),
                     np.mod(f[6] * d + P, 2 * np.pi)])


def wrapped(a, b, period):
    return np.abs(np.mod(a - b + 0.5 * period, period) - 0.5 * period)


@pytest.fixture(scope="module")
def emul():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = os.path.join(EMUL_DIR, "libemul_fit_deep.so")
    srcs = [os.path.join(EMUL_DIR, f) for f in ("emul_fit_deep.cu", "emul_fit.cu")]
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = srcs + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, *srcs], check=True,
                       capture_output=True)
    return C.CDLL(so)


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def emul_fit(L, entry, elements, offsets, jd, fr, pos, vel=None, fit_bstar=True, max_iter=25):
    el = np.ascontiguousarray(elements, dtype=np.float64)
    n = el.shape[1]
    arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (jd, fr, pos)]
    v = None if vel is None else np.ascontiguousarray(vel, dtype=np.float64)
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    fitted, rms = np.zeros((8, n)), np.zeros((n, 2))
    iters, status = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
    getattr(L, entry)(_p(el), C.c_uint32(n), 1, _p(off), *[_p(a) for a in arrs], _p(v), C.c_double(1.0),
                      C.c_double(1e-3), int(bool(fit_bstar)), C.c_uint32(max_iter), _p(fitted), _p(rms), _p(iters),
                      _p(status))
    return fitted, rms, iters, status


def _arcs():
    from astroz_b200 import synth

    el, held = deep_cases()
    jd0 = float(el[0].min())
    day = synth.time_grid(1440, jd0=jd0)                                   # 1 day at 1 min from the first epoch
    week = (np.full(1008, jd0 - 2.0), np.arange(1008) * 10.0 / 1440.0)    # 7 days at 10 min, from 2 days before
    return el, held, {"1d": (day, 1440), "7d": (week, 1008)}


def _groups(el, held, g, obs, m):
    """The held-B* and free-B* groups as separate fits: (mask, fit_bstar, guess, offsets, jd, fr, pos, vel)."""
    J, F, P, V, off = obs
    for mask, fb in ((held, False), (~held, True)):
        idx = np.flatnonzero(mask)
        rows = np.concatenate([np.arange(off[s], off[s + 1]) for s in idx])
        yield mask, fb, g[:, idx], np.arange(len(idx) + 1, dtype=np.uint32) * m, J[rows], F[rows], P[rows], V[rows]


@pytest.fixture(scope="module")
def restated():
    el, held, arcs = _arcs()
    g = guesses(el, held)
    out = {}
    for arc, ((jd, fr), m) in arcs.items():
        obs = observations(el, jd, fr)
        out[arc] = [(grp, D.fit_mixed(*grp[2:], fit_bstar=grp[1], threads=os.cpu_count() or 1))
                    for grp in _groups(el, held, g, obs, m)]
    return el, held, out


I0, E0 = 4, 6   # the i = 0 and e = 0 cases


def test_restatement_recovers_config3_deep_space_elements(restated):
    el, held, out = restated
    for arc, groups in out.items():
        for (mask, fb, *_), (f, rms, iters, status) in groups:
            e = el[:, mask]
            cols = np.flatnonzero(mask)
            ok = cols != I0
            assert (status[ok] == R.CONVERGED).all(), (arc, status, iters)
            assert (rms[ok, 0] < 1e-6).all(), (arc, rms[:, 0])
            assert np.abs(f[1, ok] - e[1, ok]).max() < 1e-9                       # n [rev/day]
            # SDP4 raises a mean eccentricity below 1e-6 to 1e-6, so e = 0 is recovered only to that order
            ecc = ok & (cols != E0)
            assert np.abs(f[2, ecc] - e[2, ecc]).max() < 1e-8                     # e
            assert (f[2, cols == E0] < 2e-6).all()
            de = wrapped(equinoctial(f), equinoctial(e), 2 * np.pi)
            assert de[:2, ecc].max() < 1e-8 and de[2:, ok].max() < 1e-8, de.max(axis=1)   # k, h; q, p, lambda [rad]
            assert (f[0] == e[0]).all()
            if not fb:
                assert (f[7] == e[7]).all()
            if mask[I0]:
                # At i = 0 exactly SDP4's inclination periodics carry i through zero and flip node and argument of
                # perigee by 180 deg (dpper): the model is not smooth there and the fit stops at the step limit some
                # 12 m away.  i = 1e-3 deg already converges.
                j = int(np.flatnonzero(cols == I0)[0])
                assert status[j] == R.ITERATION_LIMIT and rms[j, 0] < 0.05, (status[j], rms[j])


def test_host_emulation_matches_restatement(restated, emul):
    """The fit's own source on the CPU against the restatement.  Measured over these cases (1-day and 7-day arcs):
    n within 2e-12 relative, the equinoctial elements within 4e-11, RMS within 1.7e-8 km and 7e-12 km/s, B* of the
    Molniya sets within 7e-8 (7e-4 relative: a day of observations hardly constrains it), iterations within one.  The
    bounds below are those with a factor of about 5: both fits stop at the rounding floor of their own SDP4 (the
    library's and the oracle's), which differ by ~1e-8 km, so that is where the RMS and the last digits part."""
    el, held, out = restated
    for arc, groups in out.items():
        for (mask, fb, g, off, jd, fr, pos, vel), (rf, rrms, riters, rstatus) in groups:
            f, rms, iters, status = emul_fit(emul, "emul_fit_mixed", g, off, jd, fr, pos, vel, fit_bstar=fb)
            assert status.tolist() == rstatus.tolist(), arc
            assert np.abs(f[1] - rf[1]).max() <= 1e-11 * np.abs(rf[1]).max()
            assert wrapped(equinoctial(f), equinoctial(rf), 2 * np.pi).max() <= 2e-10
            assert np.abs(rms[:, 0] - rrms[:, 0]).max() <= 1e-7 and np.abs(rms[:, 1] - rrms[:, 1]).max() <= 5e-11
            assert (np.abs(f[7] - rf[7]) <= 5e-3 * np.abs(rf[7]) + 1e-15).all(), (f[7], rf[7])
            assert np.abs(iters.astype(int) - riters.astype(int)).max() <= 1
            assert (f[0] == rf[0]).all()


def test_lattice_equals_fresh_stepping(emul):
    """Every observation of the 1-day and 7-day arcs: the query through fit_deep_kernel's lattice gives the bits of
    stepping the resonance integrator from atime = 0 (a lattice of node 0 alone)."""
    el, held, arcs = _arcs()
    resonant = 0
    for (jd, fr), m in arcs.values():
        jd, fr = np.ascontiguousarray(jd), np.ascontiguousarray(fr)
        for s in range(el.shape[1]):
            e = np.ascontiguousarray(el[:, s])
            a, b = np.zeros((m, 6)), np.zeros((m, 6))
            sa, sb = np.zeros(m, np.uint8), np.zeros(m, np.uint8)
            assert emul.emul_deep_states(_p(e), 1, _p(jd), _p(fr), C.c_uint32(m), 0, _p(a), _p(sa)) == 0
            assert emul.emul_deep_states(_p(e), 1, _p(jd), _p(fr), C.c_uint32(m), 1, _p(b), _p(sb)) == 0
            assert a.tobytes() == b.tobytes() and (sa == 0).all() and (sb == 0).all(), s
            resonant += abs(e[1] - 1.0027) < 0.001 or e[2] > 0.5
    assert resonant == 2 * 13   # the 9 GEO and 4 Molniya cases, on both arcs


def test_mixed_statuses(emul):
    """Init failure, too few observations and a near-earth row on the mixed entry point; the near-earth row's bytes are
    emul_fit's."""
    from astroz_b200 import synth

    el, held = deep_cases()
    near = synth.elements_from_tles(synth.near_earth_catalog(1))
    jd, fr = synth.time_grid(60, jd0=float(el[0, 0]))
    p_geo, _ = D.observe(el[:, 0], jd, fr)
    p_near, _ = R.observe(near[:, 0], jd, fr)
    bad = el[:, [0]].copy()
    bad[2] = 1.5                               # not an orbit
    cols = np.concatenate([el[:, [0]], bad, el[:, [0]], near], axis=1)
    P = np.concatenate([p_geo, p_geo, p_geo[:2], p_near])
    J = np.concatenate([jd, jd, jd[:2], jd])
    F = np.concatenate([fr, fr, fr[:2], fr])
    off = np.array([0, 60, 120, 122, 182], dtype=np.uint32)   # set 2: two positions, 6 residuals < 7 variables
    f, rms, iters, status = emul_fit(emul, "emul_fit_mixed", cols, off, J, F, P)
    assert status.tolist() == [R.CONVERGED, R.INIT_FAILED, R.TOO_FEW, R.CONVERGED]
    assert (f[:, 1:3] == cols[:, 1:3]).all() and (rms[1:3] == 0).all() and (iters[1:3] == 0).all()
    nf, nrms, niters, nstatus = emul_fit(emul, "emul_fit", cols, off, J, F, P)
    assert nstatus.tolist() == [R.DEEP_SPACE, R.INIT_FAILED, R.DEEP_SPACE, R.CONVERGED]
    assert f[:, 3].tobytes() == nf[:, 3].tobytes() and rms[3].tobytes() == nrms[3].tobytes()
    assert iters[3] == niters[3]
    # the restatement gives the same statuses
    assert D.fit_mixed(cols, off, J, F, P)[3].tolist() == status.tolist()


# ---- C ABI: argument checks of the _mixed exports (every refusal comes before the device is looked for) -------------
def _abi_args(n=2, m=4):
    el = np.tile(np.array([[2460437.0], [1.0027], [1e-4], [3.0], [10.0], [20.0], [30.0], [0.0]]), (1, n))
    off = np.array([0, 2, m], dtype=np.uint32)[: n + 1]
    jd, fr, pos = np.full(m, 2460437.0), np.zeros(m), np.full((m, 3), 42164.0)
    out = [np.full((8, n), -7.0), np.full((n, 2), -7.0), np.full(n, 7, dtype=np.uint32), np.full(n, 9, dtype=np.uint8)]
    return el, off, jd, fr, pos, out


def _untouched(out):
    return (out[0] == -7).all() and (out[1] == -7).all() and (out[2] == 7).all() and (out[3] == 9).all()


def _call(el, off, jd, fr, pos, out, *, n=2, m=4, grav=1, ps=1.0, vs=1e-3, max_iter=25, device=0, vel=None):
    from astroz_b200 import _lib

    return _lib.lib().astroz_cuda_fit_elements_mixed(_p(el), n, grav, _p(off), _p(jd), _p(fr), _p(pos), _p(vel), m,
                                                     ps, vs, 1, max_iter, device, *[_p(o) for o in out])


def test_cabi_mixed_value_errors_write_nothing():
    pytest.importorskip("astroz_b200")
    for kw in [dict(device=-1), dict(ps=0.0), dict(vs=-1.0), dict(ps=float("nan")), dict(max_iter=0), dict(grav=7),
               dict(m=5)]:
        args = _abi_args()
        assert _call(*args, **kw) == -20, kw
        assert _untouched(args[-1]), kw
    el, off, jd, fr, pos, out = _abi_args()
    off[1], off[2] = 3, 2                        # decreasing
    assert _call(el, off, jd, fr, pos, out) == -20 and _untouched(out)
    el, off, jd, fr, pos, out = _abi_args()
    pos[1, 2] = np.nan
    assert _call(el, off, jd, fr, pos, out) == -20 and _untouched(out)
    el, off, jd, fr, pos, out = _abi_args()
    assert _call(el, off, jd, fr, pos, out, n=0) == 0 and _untouched(out)
    assert _lib_null(el, off, jd, fr, pos, out) == -101 and _untouched(out)


def _lib_null(el, off, jd, fr, pos, out):
    from astroz_b200 import _lib

    return _lib.lib().astroz_cuda_fit_elements_mixed(_p(el), 2, 1, _p(off), _p(jd), _p(fr), _p(pos), None, 4, 1.0,
                                                     1e-3, 1, 25, 0, None, *[_p(o) for o in out[1:]])


def test_cabi_mixed_device_refusals():
    from astroz_b200 import _lib

    el, off, jd, fr, pos, out = _abi_args()
    dev = _lib.lib().astroz_cuda_fit_elements_mixed_device
    assert dev(_p(el), 2, 1, _p(off), _p(jd), _p(fr), _p(pos), None, 1.0, 1e-3, 1, 25, -1, *[_p(o) for o in out],
               None) == -20
    assert dev(_p(el), 2, 1, _p(off), _p(jd), _p(fr), _p(pos), None, 0.0, 1e-3, 1, 25, 0, *[_p(o) for o in out],
               None) == -20
    assert dev(_p(el), 0, 1, _p(off), _p(jd), _p(fr), _p(pos), None, 1.0, 1e-3, 1, 25, 0, *[_p(o) for o in out],
               None) == 0
    assert dev(None, 2, 1, _p(off), _p(jd), _p(fr), _p(pos), None, 1.0, 1e-3, 1, 25, 0, *[_p(o) for o in out],
               None) == -101
    assert _untouched(out)


def test_deep_space_fit_renders_as_tle_pairs(restated):
    """FitResult.to_tle_pairs on deep-space output: GEO, GPS-like and Molniya columns read back by the library's
    parser."""
    from astroz_b200 import frontend
    from astroz_b200.fit import FitResult, parse_tle

    el, held, out = restated
    fitted = np.concatenate([f for _, (f, *_r) in out["1d"]], axis=1)
    n = fitted.shape[1]
    res = FitResult(fitted, np.zeros(n), np.zeros(n), np.zeros(n, np.uint32), np.zeros(n, np.uint8))
    for (l1, l2), s in zip(res.to_tle_pairs(satnums=range(40000, 40000 + n)), range(n)):
        assert len(l1) == 69 and len(l2) == 69
        assert l1[68] == frontend._checksum(l1[:68]) and l2[68] == frontend._checksum(l2[:68])
        back = parse_tle(l1, l2)
        e = fitted[:, s]
        assert abs(back[0] - e[0]) < 1e-8 and abs(back[1] - e[1]) < 1e-8 and abs(back[2] - e[2]) < 1e-7
        for c in (3, 4, 5, 6):
            assert wrapped(back[c], e[c], 360.0) < 1e-4


def test_implied_decimal_field_carries_into_the_exponent():
    """A B* whose five digits round up to the next power of ten (a fitted 9.999995e-5) keeps its 8-column field."""
    from astroz_b200 import frontend

    assert frontend._implied_decimal(9.99999511e-05) == " 10000-3"
    assert frontend._implied_decimal(-9.999996e-3) == "-10000-1"
    assert frontend._implied_decimal(1.2345e-4) == " 12345-3"
