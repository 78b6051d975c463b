"""The propagation cores through the series paths the synthetic catalogues never reach, on crafted element sets, against
the scalar oracle: heavy drag (every drag-angle series of sgp4_cell), the 1e-6 eccentricity floor, eccentric near-earth
orbits (the Newton loop's full rotations), inclinations of exactly 0, 90 and 180 degrees, each perigee band of the
initialisation, the 12-hour resonance across its e <= 0.65 / e < 0.7 coefficient splits, the one-day resonance below
0.2 rad (Lyddane), and resonant objects decades from epoch, past the 16384-node resonance lattice.

Every fixture proves that it reaches its path with a check made here, from the quantities that select the path
(tests/host_emul/emul.cu, emul_regimes), so a fixture that drifts out of its regime fails instead of silently testing the
usual path.  The same fixtures run through the host emulation of the cores (CPU) and on the device (gpu mark), through
host and device element initialisation, the grid in both layouts and propagate_pairs.

Tolerances are the suite's: 1e-6 km and 1e-9 km/s against the oracle.  Near-earth cells whose oracle radius is below one
Earth radius (or not finite) are skipped: the object has decayed there, and near-earth status semantics are not tested
here.  Deep-space status bytes are compared exactly.
"""
import ctypes as C

import numpy as np
import pytest

from astroz_b200 import synth
from tests.test_kernel_cores_host_emulation import emul  # noqa: F401  (module fixture: the host emulation build)

POS_TOL = 1e-6   # km
VEL_TOL = 1e-9   # km/s
RE_KM = 6378.135  # WGS72
EPOCH_DOY = 128.0     # 2024-05-07 00:00 UTC
EPOCH_JD = 2460437.5
LATTICE_CAP = 16384   # ensure_lattice (az_capi.cu): nodes of 720 minutes, about 22.4 years
YEAR_DAYS = 365.25


def _axis(days):
    days = np.asarray(days, dtype=np.float64)
    return np.full(len(days), EPOCH_JD), days.copy()


def _near(satnum, n_rev_day, ecc, bstar, incl=51.6, argp=0.0, raan=0.0, ma=40.0):
    return synth.tle_lines(satnum, 24, EPOCH_DOY, incl, raan, ecc, argp, ma, n_rev_day, bstar)


def _n_for_perigee(h_km, ecc):
    return float(synth._rev_per_day((RE_KM + h_km) / (1.0 - ecc)))


# name -> (tles, jd, fr).  Regime checks are in _reach below.
FIXTURES = {
    # sgp4_cell's drag angle tho: micro (<= 2e-3), tiny (<= 0.05), quarter (<= 0.78) and full; bstar 0.01 .. 0.5
    "drag_angle": ([_near(31001, 11.0, 1e-3, 0.1), _near(31002, 12.0, 1.2e-4, 0.5), _near(31003, 14.0, 3e-4, 0.5),
                    _near(31004, 14.0, 1.2e-4, 0.5), _near(31005, 15.5, 1e-3, 1e-2, argp=30.0),
                    _near(31006, 15.0, 1e-3, 0.3, argp=30.0, raan=30.0)], *_axis(np.linspace(0.0, 14.0, 57))),
    # eccentricity 0 and 1e-7 exactly, and drag that drives ecco - tempe below the 1e-6 floor
    "em_floor": ([_near(31101, 14.5, 0.0, 0.05), _near(31102, 14.5, 1e-7, 0.05), _near(31103, 15.2, 0.0, 0.5),
                  _near(31104, 13.8, 1e-7, 0.2, incl=97.6), _near(31105, 14.0, 1.2e-4, 0.5)],
                 *_axis(np.linspace(0.0, 5.0, 41))),
    # near-earth e 0.3 .. 0.46 (period <= 225 min): Newton steps beyond 0.05 rad take the loop's full rotations
    "eccentric": ([_near(31201, 7.9, 0.30, 1e-4, argp=10.0), _near(31202, 7.2, 0.38, 1e-4, incl=63.0, argp=200.0),
                   _near(31203, 6.6, 0.46, 1e-4, incl=28.5, argp=95.0, ma=170.0),
                   _near(31204, 6.5, 0.45, 5e-4, incl=98.0, argp=270.0, ma=300.0)],
                  *_axis(np.linspace(0.0, 3.0, 73))),
    # inclination exactly 0, 90 and 180 degrees (tle_lines reduces the angle mod 180, so 180 is written as the value
    # that prints as 180.0000); at 180 the xlcof guard on 1 + cos i is taken
    "inclination": ([_near(31301, 15.5, 1e-3, 1e-4, incl=0.0), _near(31302, 15.5, 1e-3, 1e-4, incl=90.0),
                     _near(31303, 15.5, 1e-3, 1e-4, incl=179.99999), _near(31304, 13.0, 0.05, 1e-4, incl=179.99999),
                     _near(31305, 12.0, 0.02, 1e-4, incl=90.0)],
                    *_axis(np.linspace(-1.0, 2.0, 61))),
    # perigee in each initialisation band: < 98 km, 98 .. 156, 156 .. 220, and just either side of 220 km
    "perigee": ([_near(31400 + i, _n_for_perigee(h, 0.02), 0.02, 1e-4, argp=40.0 * i)
                 for i, h in enumerate((80.0, 120.0, 150.0, 180.0, 218.0, 222.0, 240.0))],
                *_axis(np.linspace(0.0, 1.0, 49))),
    # 12-hour resonance with e on both sides of 0.65 (and below 0.7); one-day resonance below 0.2 rad (Lyddane)
    "resonance": ([synth.tle_lines(32000 + i, 24, EPOCH_DOY, 63.4, 40.0 * i, e, 270.0, 30.0 * i, 2.006, 1e-4)
                   for i, e in enumerate((0.50, 0.56, 0.62, 0.65, 0.66, 0.68, 0.695))]
                  + [synth.tle_lines(32100 + i, 24, EPOCH_DOY, inc, 75.0 * i, 2e-4, 10.0, 50.0 * i, 1.0027, 0.0)
                     for i, inc in enumerate((0.0, 0.05, 2.0, 5.0, 11.0))],
                  *_axis(np.linspace(-40.0, 60.0, 51))),
}


def _decade_tles():
    """GEO, Molniya and 12-hour (e in the 0.5 .. 0.65 band) objects for the decades past the lattice cap."""
    return [synth.tle_lines(33001, 24, EPOCH_DOY, 0.05, 80.0, 3e-4, 10.0, 20.0, 1.0027, 0.0),
            synth.tle_lines(33002, 24, EPOCH_DOY, 8.0, 120.0, 1e-4, 200.0, 300.0, 1.00272, 0.0),
            synth.tle_lines(33003, 24, EPOCH_DOY, 63.4, 30.0, 0.72, 270.0, 10.0, 2.006, 1e-5),
            synth.tle_lines(33004, 24, EPOCH_DOY, 63.4, 150.0, 0.60, 270.0, 200.0, 2.0058, 0.0),
            synth.tle_lines(33005, 24, EPOCH_DOY, 55.0, 10.0, 0.01, 20.0, 30.0, 2.0056, 0.0)]


def _decade_days(years):
    """Epochs around +-`years`, a few days apart, plus one on an exact resonance node either side of the cap."""
    d = np.concatenate([years * YEAR_DAYS + np.linspace(0.0, 6.0, 9), -(years * YEAR_DAYS + np.linspace(0.0, 6.0, 9))])
    return d


FIXTURES["decades"] = (_decade_tles(), *_axis(np.concatenate([_decade_days(25), _decade_days(30),
                                                               [(LATTICE_CAP - 1) * 0.5, LATTICE_CAP * 0.5,
                                                                -(LATTICE_CAP + 1) * 0.5]])))
# the multi-decade cells: tens of thousands of resonance steps and angles of ~1e5 rad (the suite's multi-year bound)
POS_TOL_DECADES = 1e-5


def _regimes(emul, tles, jd, fr):
    L = emul.lib
    n, nt = len(tles), len(jd)
    a1 = (C.c_char_p * n)(*[t[0].encode() for t in tles])
    a2 = (C.c_char_p * n)(*[t[1].encode() for t in tles])
    out = np.zeros((n, nt, 4))
    ecco = np.zeros(n)
    inclo = np.zeros(n)
    dp = C.POINTER(C.c_double)
    rc = L.emul_regimes(a1, a2, n, 1, jd.ctypes.data_as(dp), fr.ctypes.data_as(dp), nt, out.ctypes.data_as(dp),
                        ecco.ctypes.data_as(dp), inclo.ctypes.data_as(dp))
    assert rc == 0
    return out, ecco, inclo


def _valid(po, klass):
    """Cells compared: every deep-space cell (its status is compared too), near-earth cells above the surface."""
    r = np.linalg.norm(po, axis=-1) / RE_KM
    ok = np.isfinite(r) & (r >= 1.0)
    ok[klass > 0] = True
    return ok


def _reach(name, emul, oracle, tles, jd, fr, klass, ok):
    """Assert that the fixture reaches the path it is named for."""
    reg, ecco, inclo = _regimes(emul, tles, jd, fr)
    near = klass == 0
    if name == "drag_angle":
        tho = np.abs(reg[..., 0])[ok & near[:, None]]
        for lo, hi in ((0.0, 2e-3), (2e-3, 0.05), (0.05, 0.78), (0.78, np.inf)):
            assert np.any((tho > lo) & (tho <= hi)), (name, lo, hi)
    elif name == "em_floor":
        assert {0.0, 1e-7} <= set(ecco.tolist())
        assert np.min(reg[..., 1][ok & near[:, None]]) < 1e-6
    elif name == "eccentric":
        assert near.all() and ecco.min() >= 0.3 and ecco.max() <= 0.46
        assert np.max(np.abs(reg[..., 2])) > 0.05     # a first Newton step the loop rotates by with sincos_full
    elif name == "inclination":
        assert near.all()
        assert np.allclose(sorted(set(np.round(inclo, 9).tolist())), [0.0, np.pi / 2, np.pi], atol=1e-12)
    elif name == "perigee":
        hp = np.array([(oracle.Sgp4(*t).el["a"] * (1.0 - oracle.Sgp4(*t).el["ecco"]) - 1.0) * RE_KM for t in tles])
        for lo, hi in ((-np.inf, 98.0), (98.0, 156.0), (156.0, 220.0), (215.0, 220.0), (220.0, 225.0)):
            assert np.any((hp >= lo) & (hp < hi)), (lo, hi, hp)
    elif name == "resonance":
        half_day = klass == 3
        assert np.any(half_day & (ecco >= 0.5) & (ecco <= 0.65))
        assert np.any(half_day & (ecco > 0.65) & (ecco < 0.7))
        assert np.any((klass == 2) & (inclo < 0.2))
    elif name == "decades":
        assert {2, 3} <= set(klass.tolist())
        ts = np.abs((jd + fr) - EPOCH_JD) * 1440.0
        assert np.any(ts // 720.0 > LATTICE_CAP) and np.any((ts // 720.0 == LATTICE_CAP - 1))
    else:
        raise AssertionError(name)


def _tols(name):
    return (POS_TOL_DECADES if name == "decades" else POS_TOL), VEL_TOL


def _compare(name, p, v, st, po, vo, err, klass):
    ok = _valid(po, klass)
    ptol, vtol = _tols(name)
    dr = float(np.max(np.abs(p - po)[ok])) if ok.any() else 0.0
    dv = float(np.max(np.abs(v - vo)[ok])) if ok.any() else 0.0
    assert dr < ptol and dv < vtol, (name, dr, dv)
    if st is not None:
        deep = klass > 0
        assert np.array_equal(st[deep], err[deep]), name
    return dr, dv


# ---------------------------------------------------------------------------------------------- host emulation (CPU)
@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_cold_paths_host_emulation(emul, oracle, name):
    tles, jd, fr = FIXTURES[name]
    po, vo, err, klass = oracle.constellation_propagate(tles, jd, fr)
    _reach(name, emul, oracle, tles, jd, fr, klass, _valid(po, klass))
    for lanes in (1, 2, 3):
        emul.lib.emul_set_lanes(lanes)
        pe, ve, st = emul(tles, jd, fr)
        _compare(name, pe, ve, st, po, vo, err, klass)
    emul.lib.emul_set_lanes(1)


# ---------------------------------------------------------------------------------------------- device
@pytest.fixture(scope="module")
def az():
    import astroz_b200

    astroz_b200.lib()
    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return astroz_b200


def _device_grid(az, c, jd, fr, layout):
    import torch

    n, nt = c.numSatellites, len(jd)
    shape = (n, nt, 3) if layout == 0 else (nt, n, 3)
    pos = torch.empty(shape, dtype=torch.float64, device="cuda")
    vel = torch.empty_like(pos)
    st = torch.full((n, nt), 255, dtype=torch.uint8, device="cuda")
    c.propagate_device(jd, fr, pos, vel, st, layout=layout)
    c.synchronize()
    p, v = pos.cpu().numpy(), vel.cpu().numpy()
    if layout == 1:
        p, v = p.transpose(1, 0, 2), v.transpose(1, 0, 2)
    return p, v, st.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_cold_paths_on_device(az, emul, oracle, name):
    """Each fixture on the device: host and device element initialisation, the grid in both layouts and
    propagate_pairs, against the oracle (positions, velocities, deep-space status bytes)."""
    import torch

    tles, jd, fr = FIXTURES[name]
    po, vo, err, klass = oracle.constellation_propagate(tles, jd, fr)
    _reach(name, emul, oracle, tles, jd, fr, klass, _valid(po, klass))
    worst = [0.0, 0.0]
    handles = [az.Constellation(tles),
               az.Constellation.from_device_elements(torch.from_numpy(synth.elements_from_tles(tles)).cuda())]
    for c in handles:
        assert list(c.classes) == list(klass)
        for layout in (0, 1):
            p, v, st = _device_grid(az, c, jd, fr, layout)
            for k, e in enumerate(_compare(name, p, v, st, po, vo, err, klass)):
                worst[k] = max(worst[k], e)
        n, nt = len(tles), len(jd)
        sat = np.repeat(np.arange(n, dtype=np.int64), nt)
        pj, pf = np.tile(jd, n), np.tile(fr, n)
        pp, pv, pst = c.propagate_pairs(sat, pj, pf)
        for k, e in enumerate(_compare(name, pp.reshape(n, nt, 3), pv.reshape(n, nt, 3), pst.reshape(n, nt), po, vo, err,
                                       klass)):
            worst[k] = max(worst[k], e)
    print(f"\n{name}: max |dr| = {worst[0]:.3e} km, max |dv| = {worst[1]:.3e} km/s vs oracle")


@pytest.mark.gpu
def test_lattice_growth_is_invisible(az):
    """Short, then decades, then short again on one handle: every call is bit-identical to a fresh handle's, through
    the grid (both layouts) and propagate_pairs.  Growing the lattice to its cap, and stepping on past it, must not
    change the cells the smaller lattice already served."""
    tles, jd_long, fr_long = FIXTURES["decades"]
    jd_short, fr_short = _axis(np.linspace(-3.0, 9.0, 37))
    n = len(tles)

    def run(c, jd, fr):
        out = [c.propagate(jd, fr, layout=layout) for layout in (0, 1)]
        sat = np.repeat(np.arange(n, dtype=np.int64), len(jd))
        out.append(c.propagate_pairs(sat, np.tile(jd, n), np.tile(fr, n)))
        return out

    def same(a, b):
        return all(np.array_equal(x, y) for u, w in zip(a, b) for x, y in zip(u, w))

    reused = az.Constellation(tles)
    short1 = run(reused, jd_short, fr_short)
    long1 = run(reused, jd_long, fr_long)
    short2 = run(reused, jd_short, fr_short)
    assert same(short1, run(az.Constellation(tles), jd_short, fr_short))
    assert same(long1, run(az.Constellation(tles), jd_long, fr_long))
    assert same(short2, short1)
