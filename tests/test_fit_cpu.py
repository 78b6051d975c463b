"""The element fit of K8 on the CPU: an independent restatement on the oracle's SGP4 (tests/fit_oracle) recovers known
config-2 elements from perturbed guesses; the fit's own source (az_fit.cuh) run on the CPU by the test-only harness
tests/host_emul/emul_fit.cu agrees with it; the C ABI's argument checks; TLE rendering of fitted columns.  The device
runs are in tests/test_gpu_fit.py."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import fit_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "host_emul")
RE_KM = 6378.135


@pytest.fixture(scope="module")
def emul_fit():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = os.path.join(EMUL_DIR, "libemul_fit.so")
    src = os.path.join(EMUL_DIR, "emul_fit.cu")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)

    def run(elements, offsets, jd, fr, pos, vel=None, pos_sigma=1.0, vel_sigma=1e-3, fit_bstar=True, max_iter=25):
        el = np.ascontiguousarray(elements, dtype=np.float64)
        n = el.shape[1]
        p = lambda a: None if a is None else C.c_void_p(np.ascontiguousarray(a).ctypes.data)  # noqa: E731
        arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (jd, fr, pos)]
        v = None if vel is None else np.ascontiguousarray(vel, dtype=np.float64)
        off = np.ascontiguousarray(offsets, dtype=np.uint32)
        fitted, rms = np.zeros((8, n)), np.zeros((n, 2))
        iters, status = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
        L.emul_fit(p(el), C.c_uint32(n), 1, p(off), *[p(a) for a in arrs], p(v), C.c_double(pos_sigma),
                   C.c_double(vel_sigma), int(bool(fit_bstar)), C.c_uint32(max_iter), p(fitted), p(rms), p(iters),
                   p(status))
        return fitted, rms, iters, status

    return run


def _round_trip_cases():
    """Config-2 element sets (seed 13478) covering the shell mix: low-perigee isimp sets, the 2 % eccentric sets, the
    smallest eccentricities, and a few ordinary shells; 1 day of oracle observations at 1 min."""
    from astroz_b200 import synth

    el = synth.elements_from_tles(synth.near_earth_catalog(600))
    a = (398600.8 / (el[1] * 2 * np.pi / 86400.0) ** 2) ** (1.0 / 3.0)
    perigee = a * (1.0 - el[2]) - RE_KM
    isimp = np.flatnonzero(perigee < 220.0)[:3]
    ecc = np.flatnonzero(el[2] > 0.02)[:3]
    low_e = np.argsort(el[2])[:3]
    pick = np.unique(np.concatenate([isimp, ecc, low_e, [0, 1, 2]]))
    assert len(isimp) == 3 and len(ecc) == 3 and el[2, low_e].max() < 2e-5
    el = el[:, pick]
    jd, fr = synth.time_grid(1440)
    n = el.shape[1]
    pos, vel = np.zeros((n, 1440, 3)), np.zeros((n, 1440, 3))
    for s in range(n):
        pos[s], vel[s] = R.observe(el[:, s], jd, fr)
    offsets = np.arange(n + 1, dtype=np.uint32) * 1440
    return el, offsets, np.tile(jd, n), np.tile(fr, n), pos.reshape(-1, 3), vel.reshape(-1, 3)


@pytest.fixture(scope="module")
def round_trip():
    el, off, jd, fr, pos, vel = _round_trip_cases()
    guess = R.perturbed(el, seed=1)
    ref = R.fit(guess, off, jd, fr, pos, vel, threads=os.cpu_count() or 1)
    return el, guess, off, jd, fr, pos, vel, ref


def test_restatement_recovers_config2_elements(round_trip):
    el, guess, off, jd, fr, pos, vel, (fitted, rms, iters, status) = round_trip
    assert (status == R.CONVERGED).all(), (status, iters)
    assert (rms[:, 0] < 1e-6).all(), rms[:, 0]
    assert (rms[:, 1] < 1e-9).all(), rms[:, 1]
    # the recovered elements are the generating ones: to 1e-9 rev/day in n, 1e-9 in e, 1e-7 deg in the angles
    assert np.abs(fitted[1] - el[1]).max() < 1e-9
    assert np.abs(fitted[2] - el[2]).max() < 1e-9
    for c in (3, 4):
        assert np.abs((fitted[c] - el[c] + 180.0) % 360.0 - 180.0).max() < 1e-7
    arg_lat = lambda e: (e[5] + e[6]) % 360.0  # noqa: E731  (w and M alone are ill-conditioned as e -> 0)
    assert np.abs((arg_lat(fitted) - arg_lat(el) + 180.0) % 360.0 - 180.0).max() < 1e-7
    assert (fitted[0] == el[0]).all()


def test_host_emulation_matches_restatement(round_trip, emul_fit):
    el, guess, off, jd, fr, pos, vel, (rf, rrms, riters, rstatus) = round_trip
    f, rms, iters, status = emul_fit(guess, off, jd, fr, pos, vel)
    assert (status == R.CONVERGED).all(), status
    # converged elements within 1e-9 relative (angles: 1e-9 of a turn).  RMS within 5e-9 km: both fits stop at the
    # rounding floor, where each RMS is what separates its own SGP4 (the library's, the oracle's) from the oracle's
    # observations -- a few 1e-9 km for the library, zero to rounding for the restatement
    assert np.abs(f[1] - rf[1]).max() <= 1e-9 * np.abs(rf[1]).max()
    assert np.abs(f[2] - rf[2]).max() <= 1e-9 * max(np.abs(rf[2]).max(), 1e-5)
    for c in (3, 4):
        assert np.abs((f[c] - rf[c] + 180.0) % 360.0 - 180.0).max() <= 360.0 * 1e-9
    assert np.abs((f[5] + f[6] - rf[5] - rf[6] + 180.0) % 360.0 - 180.0).max() <= 360.0 * 1e-9
    assert np.abs(rms[:, 0] - rrms[:, 0]).max() <= 5e-9 and np.abs(rms[:, 1] - rrms[:, 1]).max() <= 5e-12
    # iteration counts may differ by one where a cost decrease lands within rounding of the stopping tolerance
    assert np.abs(iters.astype(int) - riters.astype(int)).max() <= 1


def test_host_emulation_positions_only_and_held_bstar(round_trip, emul_fit):
    el, guess, off, jd, fr, pos, vel, _ = round_trip
    g = guess.copy()
    g[7] = el[7]
    f, rms, iters, status = emul_fit(g, off, jd, fr, pos, None, fit_bstar=False)
    rf, rrms, riters, rstatus = R.fit(g, off, jd, fr, pos, None, fit_bstar=False)
    assert (status == R.CONVERGED).all() and (rstatus == R.CONVERGED).all()
    assert (f[7] == g[7]).all() and (rms[:, 1] == 0).all()
    assert (rms[:, 0] < 1e-6).all() and np.abs(rms[:, 0] - rrms[:, 0]).max() <= 5e-9


def test_host_emulation_statuses(emul_fit):
    from astroz_b200 import synth

    el = synth.elements_from_tles(synth.near_earth_catalog(4))
    jd, fr = synth.time_grid(60)
    pos, vel = R.observe(el[:, 0], jd, fr)
    guess = el.copy()
    guess[1, 1] = 1.0027       # geostationary mean motion: deep space
    guess[2, 2] = 1.5          # not an orbit: init fails
    off = np.array([0, 60, 60, 60, 61], dtype=np.uint32)   # satellite 3: one position, 3 residuals < 7 variables
    P = np.concatenate([pos, pos[:1]])
    J = np.concatenate([jd, jd[:1]])
    F = np.concatenate([fr, fr[:1]])
    f, rms, iters, status = emul_fit(guess, off, J, F, P)
    assert status.tolist() == [R.CONVERGED, R.DEEP_SPACE, R.INIT_FAILED, R.TOO_FEW]
    assert (f[:, 1:] == guess[:, 1:]).all() and (rms[1:] == 0).all() and (iters[1:] == 0).all()
    # the statuses of the restatement are the same
    assert R.fit(guess, off, J, F, P)[3].tolist() == status.tolist()


# ---- C ABI: argument checks (no device needed: every refusal comes before the device is looked for) ----------------
def _abi_args(n=2, m=4):
    import ctypes as C

    el = np.tile(np.array([[2460437.0], [15.5], [1e-3], [53.0], [10.0], [20.0], [30.0], [1e-4]]), (1, n))
    off = np.array([0, 2, m], dtype=np.uint32)[: n + 1]
    jd, fr, pos = np.full(m, 2460437.0), np.zeros(m), np.full((m, 3), 7000.0)
    out = [np.full((8, n), -7.0), np.full((n, 2), -7.0), np.full(n, 7, dtype=np.uint32), np.full(n, 9, dtype=np.uint8)]
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    return el, off, jd, fr, pos, out, p


def _call(el, off, jd, fr, pos, out, p, *, n=2, m=4, grav=1, ps=1.0, vs=1e-3, max_iter=25, device=0, vel=None):
    from astroz_b200 import _lib

    return _lib.lib().astroz_cuda_fit_elements(p(el), n, grav, p(off), p(jd), p(fr), p(pos), p(vel), m, ps, vs, 1,
                                               max_iter, device, *[p(o) for o in out])


def _untouched(out):
    return (out[0] == -7).all() and (out[1] == -7).all() and (out[2] == 7).all() and (out[3] == 9).all()


def test_cabi_value_errors_write_nothing():
    pytest.importorskip("astroz_b200")
    cases = [dict(device=-1), dict(ps=0.0), dict(vs=-1.0), dict(ps=float("nan")), dict(vs=float("inf")),
             dict(max_iter=0), dict(grav=7), dict(m=5)]
    for kw in cases:
        el, off, jd, fr, pos, out, p = _abi_args()
        assert _call(el, off, jd, fr, pos, out, p, **kw) == -20, kw
        assert _untouched(out), kw
    el, off, jd, fr, pos, out, p = _abi_args()
    off[1] = 3
    off[2] = 2                                   # decreasing
    assert _call(el, off, jd, fr, pos, out, p) == -20 and _untouched(out)
    for arr, idx in (("el", (3, 1)), ("jd", 2), ("fr", 0), ("pos", (1, 2))):
        el, off, jd, fr, pos, out, p = _abi_args()
        {"el": el, "jd": jd, "fr": fr, "pos": pos}[arr][idx] = np.nan
        assert _call(el, off, jd, fr, pos, out, p) == -20 and _untouched(out), arr
    el, off, jd, fr, pos, out, p = _abi_args()
    vel = np.zeros((4, 3))
    vel[3, 0] = np.inf
    assert _call(el, off, jd, fr, pos, out, p, vel=vel) == -20 and _untouched(out)


def test_cabi_empty_batch_and_no_device():
    from astroz_b200 import _lib

    el, off, jd, fr, pos, out, p = _abi_args()
    assert _call(el, off, jd, fr, pos, out, p, n=0) == 0 and _untouched(out)
    rc = _call(el, off, jd, fr, pos, out, p)
    if _lib.device_count() > 0:
        assert rc == 0
    else:
        assert rc == -201 and _untouched(out)


# ---- TLE rendering -----------------------------------------------------------------------------------------------------
def test_fitted_columns_render_as_tle_pairs():
    from astroz_b200 import frontend, synth
    from astroz_b200.fit import FitResult, parse_tle

    tles = synth.near_earth_catalog(40)
    el = synth.elements_from_tles(tles)
    el[1] += 3.3e-9                     # beyond the column precision: rendering rounds
    res = FitResult(el, np.zeros(40), np.zeros(40), np.zeros(40, np.uint32), np.zeros(40, np.uint8))
    pairs = res.to_tle_pairs(satnums=range(10000, 10040))
    for (l1, l2), ref, s in zip(pairs, tles, range(40)):
        assert len(l1) == 69 and len(l2) == 69
        assert l1[68] == frontend._checksum(l1[:68]) and l2[68] == frontend._checksum(l2[:68])
        back = parse_tle(l1, l2)
        assert abs(back[0] - el[0, s]) < 1e-8                                    # epoch: 1e-8 day
        assert abs(back[1] - el[1, s]) < 1e-8 and abs(back[2] - el[2, s]) < 1e-7  # n, e
        for c in (3, 4, 5, 6):
            assert abs((back[c] - el[c, s] + 180.0) % 360.0 - 180.0) < 1e-4
        assert abs(back[7] - el[7, s]) <= 1e-5 * abs(el[7, s]) + 1e-12
        assert l2[8:63] == ref[1][8:63]                                          # the catalogue's own columns


def test_omm_rendering_is_unchanged_by_the_shared_helper():
    """The formatting omm_to_tle_pairs and FitResult.to_tle_pairs share gives the bytes it gave before it was shared."""
    import json

    from astroz_b200 import frontend

    recs = [{"OBJECT_NAME": "ISS (ZARYA)", "OBJECT_ID": "1998-067A", "EPOCH": "2024-05-06T19:53:05.000000",
             "MEAN_MOTION": 15.50957674, "ECCENTRICITY": 0.000358, "INCLINATION": 51.6393, "RA_OF_ASC_NODE": 160.4574,
             "ARG_OF_PERICENTER": 140.6673, "MEAN_ANOMALY": 205.725, "EPHEMERIS_TYPE": 0, "CLASSIFICATION_TYPE": "U",
             "NORAD_CAT_ID": 25544, "ELEMENT_SET_NO": 999, "REV_AT_EPOCH": 45212, "BSTAR": 0.0002731,
             "MEAN_MOTION_DOT": 0.00015698, "MEAN_MOTION_DDOT": 0},
            {"OBJECT_ID": "DEB", "EPOCH": "2023-12-31T23:59:59.123456", "MEAN_MOTION": 1.00271,
             "ECCENTRICITY": 0.1234567, "INCLINATION": 98.7, "RA_OF_ASC_NODE": 359.99, "ARG_OF_PERICENTER": 0.01,
             "MEAN_ANOMALY": 12.5, "NORAD_CAT_ID": 7, "BSTAR": -1.5e-5, "MEAN_MOTION_DOT": -1e-6,
             "MEAN_MOTION_DDOT": 1.2e-9}]
    assert frontend.omm_to_tle_pairs(json.dumps(recs)) == [
        ("1 25544U 98067A   24127.82853009  .00015698  00000+0  27310-3 0  9995",
         "2 25544  51.6393 160.4574 0003580 140.6673 205.7250 15.50957674452123"),
        ("1 00007U DEB      23365.99998985 -.00000100  12000-8 -15000-4 0    09",
         "2 00007  98.7000 359.9900 1234567   0.0100  12.5000  1.00271000    06")]
