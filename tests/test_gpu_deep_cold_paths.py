"""The deep-space cell (sdp4_cell_n, az_device.cuh) on the orbits the synthetic catalogues never make, and through every
branch of the cell.

* Transfer and highly eccentric orbits: GTO rocket bodies at 0.5 .. 51.6 degrees with real drag, a super-synchronous
  GTO, HEO at e = 0.8 .. 0.97 up to a lunar-transfer apogee, and cells whose first Kepler step needs the +-0.95 clamp.
* Retrograde deep space at 170 .. 179.9999 degrees, synchronous and non-resonant: xlcof = -j3/j2 sin i (3 + 5 cos i) /
  (4 (1 + cos i)) is recomputed per cell with a guard at 1 + cos i = 1.5e-12, and near 180 degrees 1 + cos i cancels.
* The cold branches: a large inclination excursion (sincos_full(inclm)), the inclm < 0 flip, the Lyddane node wrap, the
  general cube root for a libration |x| > 3e-3, and each status the cell sets.

Every fixture proves that it reaches its regime with the quantities that select it (tests/host_emul/emul_deep.cu,
emul_deep_regimes), so a fixture that drifts out of its regime fails instead of silently testing the usual path.

Two references.  The oracle (oracle/astroz_oracle.c) is the scalar restatement in doubles; sdp4_statement below restates
the same steps at 40 digits from the oracle's exported init record, solving Kepler's equation to convergence.  Where the
problem is well conditioned the suite's bounds against the oracle hold (1e-6 km, 1e-9 km/s; status bytes equal).  Near
180 degrees the double inputs leave the result undetermined by what moving inclo and the perturbed inclination by one
ulp moves the 40-digit value; there both the cells and the oracle are held to that value within 1e-6 km plus twice that
spread.  The oracle forms 1 + cos i as 1 + cos(inclm) and loses up to 1.1e-16 / (1 + cos i) of it; a retrograde cell
forms it as sin^2 / (1 - cos) from the small rotation of the element set's sin/cos, which keeps its digits.  The cell
meets the bound at every cell; the oracle misses it by up to a kilometre where 1 + cos i is below 1e-8, and that is
asserted as the oracle's own limit.  (Before the cell took the identity it missed the bound like the oracle, by up to
4.8 km at 179.999 degrees.)
"""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from astroz_b200 import synth
from tests.golden import tles as G

mpmath = pytest.importorskip("mpmath")
mp = mpmath.mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "astroz_b200", "csrc")
POS_TOL = 1e-6    # km
VEL_TOL = 1e-9    # km/s
REL_POS_TOL = 1e-12  # of |r|, where |r| > 1e6 km (none of the fixtures here goes that far; see _pos_tol)
RE_KM = 6378.135  # WGS72
EPOCH_DOY = 128.0     # 2024-05-07 00:00 UTC
EPOCH_JD = 2460437.5
(X, DINCL, INCLM, OPC, NODDIFF, R2, EM_PRE, EM_POST, AM, NM, KEP1, STATUS, MRT) = range(13)  # emul_deep.cu, DeepRegime
NREG = 13


# ------------------------------------------------------------------------------------- the 40-digit statement
# WGS72 as the oracle holds it (oracle/astroz_oracle.c, azo_gravity): the doubles are the inputs of the statement
J2, J3OJ2, XKE, RE = 0.001082616, -0.00234506972242078, 0.0743669161331734132, 6378.135
ZES, ZEL, ZNS, ZNL, RPTIM = 0.01675, 0.05490, 1.19459e-5, 1.5835218e-4, 4.37526908801129966e-3
G22, G32, G44, G52, G54 = 5.7686396, 0.95240898, 1.8014998, 1.0508330, 4.4108898
FASX2, FASX4, FASX6 = 0.13130908, 2.8843198, 0.37448087


def _mod2pi(x):
    return x - 2 * mp.pi * mpmath.floor(x / (2 * mp.pi))


def _resonance_accel(el, xli, xni, atime):
    f = {k: mp.mpf(el[k]) for k in ("d2201", "d2211", "d3210", "d3222", "d4410", "d4422", "d5220", "d5232", "d5421",
                                    "d5433", "del1", "del2", "del3")}
    xldot = xni + mp.mpf(el["xfact"])
    if el["irez"] == 2:
        w = mp.mpf(el["argpo"]) + mp.mpf(el["argpdot"]) * atime
        terms = [("d2201", 2 * w + xli - G22, 1), ("d2211", xli - G22, 1), ("d3210", w + xli - G32, 1),
                 ("d3222", -w + xli - G32, 1), ("d4410", 2 * w + 2 * xli - G44, 2), ("d4422", 2 * xli - G44, 2),
                 ("d5220", w + xli - G52, 1), ("d5232", -w + xli - G52, 1), ("d5421", w + 2 * xli - G54, 2),
                 ("d5433", -w + 2 * xli - G54, 2)]
    else:
        terms = [("del1", xli - FASX2, 1), ("del2", 2 * (xli - FASX4), 2), ("del3", 3 * (xli - FASX6), 3)]
    xndt = sum(f[k] * mpmath.sin(a) for k, a, _ in terms)
    xnddt = sum(m * f[k] * mpmath.cos(a) for k, a, m in terms) * xldot
    return xndt, xnddt, xldot


def _dpper_terms(el, t):
    out = [0, 0, 0, 0, 0]
    for body, zm0, zn, ze in (("solar_", el["zmos"], ZNS, ZES), ("lunar_", el["zmol"], ZNL, ZEL)):
        zm = mp.mpf(zm0) + mp.mpf(zn) * t
        zf = zm + 2 * mp.mpf(ze) * mpmath.sin(zm)
        sz = mpmath.sin(zf)
        f2 = sz * sz / 2 - mp.mpf(1) / 4
        f3 = -sz * mpmath.cos(zf) / 2
        c = {k: mp.mpf(el[body + k]) for k in ("e2", "e3", "i2", "i3", "l2", "l3", "l4", "gh2", "gh3", "gh4", "h2",
                                               "h3")}
        for i, v in enumerate((c["e2"] * f2 + c["e3"] * f3, c["i2"] * f2 + c["i3"] * f3,
                               c["l2"] * f2 + c["l3"] * f3 + c["l4"] * sz,
                               c["gh2"] * f2 + c["gh3"] * f3 + c["gh4"] * sz, c["h2"] * f2 + c["h3"] * f3)):
            out[i] += v
    return out  # pe, pinc, pl, pgh, ph


def sdp4_statement(el, tsince, inclo_ulps=0, inclm_ulps=0):
    """SDP4 at one tsince (minutes), at mp.dps digits, from the oracle's init record `el` (oracle.Sdp4(...).el):
    dspace from atime = 0 in 720-minute steps, the final partial step, dpper (Lyddane below 0.2 rad), the
    inclination-dependent terms, Kepler's equation solved to convergence (the reference's Newton loop with its +-0.95
    clamp, run until the step is below 1e-30) and the short-period terms.  inclo_ulps / inclm_ulps move inclo / the
    perturbed inclination by that many ulps of their double.
    Returns (status, r km, v km/s) like oracle.Sdp4.propagate."""
    mpf = mp.mpf
    t = mpf(float(tsince))
    inclo = float(el["inclo"])
    if inclo_ulps:
        inclo = float(np.nextafter(inclo, np.inf if inclo_ulps > 0 else -np.inf))
    no = mpf(el["noUnkozai"])
    t2 = t * t
    tempa = 1 - mpf(el["cc1"]) * t
    tempe = mpf(el["bstar"]) * mpf(el["cc4"]) * t
    templ = mpf(el["t2cof"]) * t2
    mm = mpf(el["mo"]) + mpf(el["mdot"]) * t + mpf(el["dmdt"]) * t
    argpm = mpf(el["argpo"]) + mpf(el["argpdot"]) * t + mpf(el["domdt"]) * t
    nodem = mpf(el["nodeo"]) + mpf(el["nodedot"]) * t + mpf(el["xnodcf"]) * t2 + mpf(el["dnodt"]) * t
    em = mpf(el["ecco"]) + mpf(el["dedt"]) * t
    inclm = mpf(inclo) + mpf(el["didt"]) * t
    nm = no
    if el["irez"] != 0:
        atime, xli, xni = mpf(0), mpf(el["xlamo"]), no
        delt = mpf(720) if tsince > 0 else mpf(-720)
        while abs(t - atime) >= 720:
            xndt, xnddt, xldot = _resonance_accel(el, xli, xni, atime)
            xli += xldot * delt + xndt * 259200
            xni += xndt * delt + xnddt * 259200
            atime += delt
        ft = t - atime
        xndt, xnddt, xldot = _resonance_accel(el, xli, xni, atime)
        nm = xni + xndt * ft + xnddt * ft * ft / 2
        xl = xli + xldot * ft + xndt * ft * ft / 2
        theta = mpf(el["gsto"]) + t * mpf(RPTIM)
        mm = xl - 2 * nodem + 2 * theta if el["irez"] == 2 else xl - nodem - argpm + theta
    if nm <= 0:
        return 1, None, None
    am = (mpf(XKE) / nm) ** (mpf(2) / 3) * tempa * tempa
    nm = mpf(XKE) / am ** mpf(1.5)
    em -= tempe
    if em >= 1 or em < mpf(-0.001):
        return 2, None, None
    em = max(em, mpf(1e-6))
    if am < mpf(0.95):
        return 1, None, None
    mm += no * templ

    pe, pinc, pl, pgh, ph = _dpper_terms(el, t)
    inclm += pinc
    if inclm_ulps:
        u = float(inclm)
        inclm += mpf(float(np.spacing(abs(u)))) * inclm_ulps
    em += pe
    sinip, cosip = mpmath.sin(inclm), mpmath.cos(inclm)
    if inclm >= mpf(0.2):
        ph /= sinip
        argpm += pgh - cosip * ph
        nodem += ph
        mm += pl
    else:
        nod = _mod2pi(nodem)
        sinop, cosop = mpmath.sin(nod), mpmath.cos(nod)
        alfdp = sinip * sinop + ph * cosop + pinc * cosip * sinop
        betdp = sinip * cosop - ph * sinop + pinc * cosip * cosop
        xls = mm + argpm + cosip * nod
        dls = pl + pgh - pinc * nod * sinip
        nn = mpmath.atan2(alfdp, betdp)
        if abs(nod - nn) > mp.pi:
            nn += 2 * mp.pi if nn < nod else -2 * mp.pi
        nodem = nn
        mm += pl
        argpm = xls + dls - mm - cosip * nn
    if inclm < 0:
        inclm, nodem, argpm = -inclm, nodem + mp.pi, argpm - mp.pi
    em = max(em, mpf(1e-6))
    if em >= 1:
        return 2, None, None
    sinip, cosip = mpmath.sin(inclm), mpmath.cos(inclm)
    opc = 2 * mpmath.cos(inclm / 2) ** 2  # 1 + cos(inclm)
    xlcof = -mpf(J3OJ2) / 4 * sinip * (3 + 5 * cosip) / (opc if opc > mpf(1.5e-12) else mpf(1.5e-12))
    aycof = -mpf(J3OJ2) / 2 * sinip

    # Kepler (src/Sgp4.zig:495-546), solved to convergence
    temp = 1 / (am * (1 - em * em))
    axnl = em * mpmath.cos(argpm)
    aynl = em * mpmath.sin(argpm) + temp * aycof
    u = _mod2pi(mm + argpm + temp * xlcof * axnl)
    eo1 = u
    for _ in range(200):
        s, c = mpmath.sin(eo1), mpmath.cos(eo1)
        step = (u - aynl * c + axnl * s - eo1) / (1 - c * axnl - s * aynl)
        step = max(min(step, mpf(0.95)), mpf(-0.95))
        eo1 += step
        if abs(step) < mpf(1e-30):
            break
    else:
        raise AssertionError("Kepler's equation did not converge")
    s, c = mpmath.sin(eo1), mpmath.cos(eo1)
    ecose = axnl * c + aynl * s
    esine = axnl * s - aynl * c
    el2 = axnl * axnl + aynl * aynl
    pl_ = am * (1 - el2)
    betal = mpmath.sqrt(1 - el2)
    rl = am * (1 - ecose)
    rdotl = mpmath.sqrt(am) * esine / rl
    rvdotl = mpmath.sqrt(pl_) / rl
    aor = am / rl
    est = esine / (1 + betal)
    sinu = aor * (s - aynl - axnl * est)
    cosu = aor * (c - axnl + aynl * est)
    su = mpmath.atan2(sinu, cosu)
    sin2u, cos2u = 2 * sinu * cosu, 1 - 2 * sinu * sinu
    cosip2 = cosip * cosip
    con41, x1mth2, x7thm1 = 3 * cosip2 - 1, 1 - cosip2, 7 * cosip2 - 1
    temp1 = mpf(J2) / 2 / pl_
    temp2 = temp1 / pl_
    mrt = rl * (1 - mpf(1.5) * temp2 * betal * con41) + temp1 / 2 * x1mth2 * cos2u
    su -= temp2 / 4 * x7thm1 * sin2u
    xnode = nodem + mpf(1.5) * temp2 * cosip * sin2u
    xinc = inclm + mpf(1.5) * temp2 * cosip * sinip * cos2u
    mvt = rdotl - nm * temp1 * x1mth2 * sin2u / mpf(XKE)
    rvdot = rvdotl + nm * temp1 * (x1mth2 * cos2u + mpf(1.5) * con41) / mpf(XKE)
    if mrt < 1:
        return 1, None, None
    sinsu, cossu = mpmath.sin(su), mpmath.cos(su)
    snod, cnod = mpmath.sin(xnode), mpmath.cos(xnode)
    sini, cosi = mpmath.sin(xinc), mpmath.cos(xinc)
    xmx, xmy = -snod * cosi, cnod * cosi
    ux, uy, uz = xmx * sinsu + cnod * cossu, xmy * sinsu + snod * cossu, sini * sinsu
    vx, vy, vz = xmx * cossu - cnod * sinsu, xmy * cossu - snod * sinsu, sini * cossu
    vk = mpf(el["vkmpersec"])
    r = np.array([float(mrt * RE * w) for w in (ux, uy, uz)])
    v = np.array([float((mvt * a + rvdot * b) * vk) for a, b in ((ux, vx), (uy, vy), (uz, vz))])
    return 0, r, v


@pytest.fixture(autouse=True)
def _forty_digits():
    with mpmath.workdps(40):
        yield


# ------------------------------------------------------------------------------------- fixtures
def _axis(days):
    days = np.asarray(days, dtype=np.float64)
    return np.full(len(days), EPOCH_JD), days.copy()


def _rev_day(rp_km, ra_km):
    return float(synth._rev_per_day(0.5 * (rp_km + ra_km)))


def _deep(satnum, incl, ecc, n_rev_day, bstar=1e-5, raan=10.0, argp=20.0, ma=30.0):
    return synth.tle_lines(satnum, 24, EPOCH_DOY, incl, raan, ecc, argp, ma, n_rev_day, bstar)


def _apsides(satnum, hp_km, ha_km, incl, bstar, argp=180.0, ma=10.0, raan=30.0):
    rp, ra = RE_KM + hp_km, RE_KM + ha_km
    return _deep(satnum, incl, (ra - rp) / (ra + rp), _rev_day(rp, ra), bstar, raan, argp, ma)


def _ecc_perigee(satnum, hp_km, ecc, incl, bstar, argp=0.0, ma=5.0, raan=0.0):
    a = (RE_KM + hp_km) / (1.0 - ecc)
    return _deep(satnum, incl, ecc, float(synth._rev_per_day(a)), bstar, raan, argp, ma)


RETRO_INCL = (170.0, 179.0, 179.9, 179.99, 179.999, 179.9999)

# name -> (tles, jd, fr).  Regime checks are in _reach below.
FIXTURES = {
    # GTO rocket bodies (perigee 250 km, apogee 35,786 km, e ~ 0.73, ~630 min, irez 0) with real drag
    "gto": ([_apsides(44001 + i, 250.0, 35786.0, inc, b, argp=argp, ma=ma)
             for i, (inc, b, argp, ma) in enumerate(((0.5, 1e-4, 0.0, 0.0), (6.0, 5e-4, 178.0, 200.0),
                                                      (27.0, 1e-3, 180.0, 10.0), (51.6, 2e-3, 90.0, 350.0)))]
            + [_apsides(44005, 300.0, 60000.0, 28.5, 1e-4, argp=270.0, ma=120.0)],   # super-synchronous
            *_axis(np.linspace(-5.0, 30.0, 281))),
    # HEO at e = 0.8 .. 0.97 and a lunar-transfer apogee (380,000 km); cells near perigee need the +-0.95 clamp
    "heo": ([_ecc_perigee(44101, 500.0, 0.80, 63.4, 1e-5, argp=270.0), _ecc_perigee(44102, 1000.0, 0.90, 28.5, 1e-5),
             _ecc_perigee(44103, 2000.0, 0.95, 57.0, 1e-5, argp=120.0, raan=80.0),
             _ecc_perigee(44104, 8000.0, 0.97, 40.0, 0.0, argp=300.0, raan=200.0),
             _apsides(44105, 250.0, 380000.0, 28.5, 1e-5, argp=200.0, ma=0.5)],
            *_axis(np.concatenate([np.linspace(-5.0, 30.0, 141), np.linspace(-0.02, 0.02, 41)]))),
    # retrograde, synchronous (irez 1) and non-resonant; the dense axis puts cells on both sides of xlcof's guard and
    # beyond 180 degrees once the luni-solar inclination terms carry inclm across pi
    "retrograde": ([_deep(44200 + 10 * k + i, inc, 0.01, n) for k, n in enumerate((1.0027, 3.0))
                    for i, inc in enumerate(RETRO_INCL)], *_axis(np.linspace(-2.0, 28.0, 2161))),
    # the large inclination excursion (years from epoch), the inclm < 0 flip (inclination 0) and the Lyddane node wrap
    # (nodes past 180 degrees)
    "inclination": ([_deep(44301, 0.0, 2e-4, 1.0027, 0.0, raan=250.0), _deep(44302, 0.0, 0.01, 3.0, 0.0, raan=200.0),
                     _deep(44303, 1.5, 3e-4, 1.0027, 0.0, raan=300.0), _deep(44304, 15.0, 1e-3, 1.0027, 0.0),
                     _deep(44305, 100.0, 0.01, 2.5, 0.0)],
                    *_axis(np.concatenate([np.linspace(-30.0, 30.0, 121), 365.25 * np.linspace(-8.0, 8.0, 17)]))),
}
# Every check the cell makes on the way to a status (regimes below); the GTO with a 120 km perigee and bstar 0.5 crosses
# e = 1 about 0.436 days before epoch, where the dense run puts cells that pass the drag check and fail after dpper; the
# GTO with a 150 km perigee first dips below the surface 40,656 minutes before epoch, where one-second steps put cells
# within 6 km of it on both sides
FIXTURES["status"] = ([_apsides(44401, 120.0, 35786.0, 27.0, 0.5, argp=90.0, raan=120.0),
                       _ecc_perigee(44402, 150.0, 0.73, 27.0, 0.05)],
                      *_axis(np.concatenate([np.linspace(-30.0, 30.0, 1201), np.linspace(-0.4364, -0.4360, 41),
                                             (-40656.0 + np.linspace(0.0, 1.0, 61)) / 1440.0])))
# where 1 + cos(inclm) is below this the oracle's cancellation exceeds the suite's bound; the 40-digit statement decides
ILL_OPC = 1e-6


# ------------------------------------------------------------------------------------- harnesses
def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    return nvcc


def _build(src, so, flags):
    deps = [src] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".hpp", ".inc"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([_nvcc()] + flags + ["-std=c++17", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared",
                                            "-I" + CSRC, "-o", so, src], check=True, capture_output=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def deep():
    """tests/host_emul/emul_deep.cu: the regime probe and the host build of sdp4_cell."""
    d = os.path.join(ROOT, "tests", "host_emul")
    return _build(os.path.join(d, "emul_deep.cu"), os.path.join(d, "libemul_deep.so"),
                  ["-O2", "-Wno-deprecated-gpu-targets"])


@pytest.fixture(scope="module")
def probe():
    """tests/device_probe/probe_deep.cu (probe_sdp4_cell), with the flags tests/test_math_primitives.py builds probe.cu
    with."""
    d = os.path.join(ROOT, "tests", "device_probe")
    return _build(os.path.join(d, "probe_deep.cu"), os.path.join(d, "libprobe_deep.so"),
                  ["-gencode", "arch=compute_90a,code=sm_90a", "-O3"])


from tests.test_kernel_cores_host_emulation import emul  # noqa: E402,F401  (module fixture: the host emulation build)

_dp = C.POINTER(C.c_double)


def _lines(tles):
    n = len(tles)
    return (C.c_char_p * n)(*[t[0].encode() for t in tles]), (C.c_char_p * n)(*[t[1].encode() for t in tles])


def _regimes(deep, tles, jd, fr):
    n, nt = len(tles), len(jd)
    out = np.zeros((n, nt, NREG))
    assert deep.emul_deep_regimes(*_lines(tles), n, 1, jd.ctypes.data_as(_dp), fr.ctypes.data_as(_dp), nt,
                                  out.ctypes.data_as(_dp)) == 0
    return out


def _reach(name, reg, klass):
    """Assert that the fixture reaches the regime it is named for, from the quantities that select it."""
    assert (klass > 0).all(), name                     # every fixture here is deep space
    st = reg[..., STATUS]
    ok = st == 0
    kep = np.abs(reg[..., KEP1])
    if name == "gto":
        assert (klass == 1).all()
        e = np.array([reg[s, 0, EM_PRE] for s in range(len(klass))])
        assert np.all((e > 0.72) & (e < 0.83))
        assert np.any(kep[ok] > 0.95)                  # first Newton steps the +-0.95 clamp cuts
    elif name == "heo":
        e0 = reg[:, np.argmin(np.abs(FIXTURES[name][2])), EM_PRE]
        for lo in (0.8, 0.9, 0.95, 0.97):
            assert np.any(np.abs(e0 - lo) < 5e-3), (lo, e0)
        assert np.any(kep[ok] > 0.95)
    elif name == "retrograde":
        assert {1, 2} <= set(klass.tolist())
        opc, inclm = reg[..., OPC], reg[..., INCLM]
        assert np.any(opc < 1.5e-12) and np.any((opc > 1.5e-12) & (opc < 3e-12))  # both sides of xlcof's guard
        assert np.any(inclm > np.pi)
        for k in (1, 2):                               # below the guard for a synchronous and a non-resonant set
            assert np.any(opc[klass == k] < 1.5e-12), k
    elif name == "inclination":
        assert np.any(np.abs(reg[..., DINCL]) > 0.05)  # sincos_full(inclm)
        assert np.any(reg[..., INCLM] < 0.0)           # the flip
        nd = reg[..., NODDIFF]
        assert np.any(np.abs(nd[np.isfinite(nd)]) > np.pi)  # the Lyddane wrap
        assert np.any(reg[..., INCLM] >= 0.2) and np.any(reg[..., INCLM] < 0.2)
    elif name == "status":
        em0, em1, am = reg[..., EM_PRE], reg[..., EM_POST], reg[..., AM]
        drag_ok = (em0 < 1.0) & (em0 >= -0.001)
        cases = {"em >= 1 before dpper": (em0 >= 1.0) & (st == 2), "em < -0.001": (em0 < -0.001) & (st == 2),
                 "am < 0.95": drag_ok & (am < 0.95) & (st == 1),
                 "em >= 1 after dpper": drag_ok & (am >= 0.95) & (em1 >= 1.0) & (st == 2),
                 "mrt < 1": drag_ok & (am >= 0.95) & (em1 < 1.0) & (st == 1),
                 "mrt just below 1": (st == 1) & (reg[..., MRT] >= 0.999) & (reg[..., MRT] < 1.0),
                 "mrt just above 1": (st == 0) & (reg[..., MRT] >= 1.0) & (reg[..., MRT] < 1.001)}
        for what, hit in cases.items():
            assert hit.any(), what
    else:
        raise AssertionError(name)
    # no element set here reaches the general cube root of the resonance libration (|x| > 3e-3): it is driven through
    # the direct cell entry instead (test_libration_cube_root_and_nm_status)
    assert np.all(np.abs(reg[..., X]) <= 3e-3)


def _valid(po):
    return np.isfinite(po).all(axis=-1)


def _pos_tol(po):
    """The suite's 1e-6 km, or 1e-12 |r| where |r| is above 1e6 km (fp64 keeps ~16 digits of the radius)."""
    return np.maximum(POS_TOL, REL_POS_TOL * np.linalg.norm(po, axis=-1))


def _compare(name, p, v, st, po, vo, err, mask):
    """Cells in `mask` against the oracle at the suite's bounds; status bytes everywhere."""
    assert np.array_equal(st, err), name
    dr = np.max(np.abs(p - po), axis=-1)
    dv = np.max(np.abs(v - vo), axis=-1)
    m = mask & (err == 0)
    assert np.all(dr[m] < _pos_tol(po)[m]) and np.all(dv[m] < VEL_TOL), (name, dr[m].max(), dv[m].max())
    return float(dr[m].max()), float(dv[m].max())


def _well_conditioned(name, reg):
    if name != "retrograde":
        return np.ones(reg.shape[:2], dtype=bool)
    return reg[..., OPC] > ILL_OPC


# ------------------------------------------------------------------------------------- the 40-digit cells
_STATEMENT = {}


def _statement_cells(name, oracle, deep):
    """(sat, epoch) cells where the problem is ill conditioned, their 40-digit (r, v), and the +-1-ulp spread of each.
    Retrograde: per satellite with 1 + cos(inclm) below ILL_OPC, the six cells nearest 180 degrees, the two either side
    of the guard, and the two where the oracle's cancellation moves it most.  HEO: the cells nearest perigee."""
    if name in _STATEMENT:
        return _STATEMENT[name]
    tles, jd, fr = FIXTURES[name]
    reg = _regimes(deep, tles, jd, fr)
    cells = []
    for s in range(len(tles)):
        if name == "retrograde":
            opc = reg[s, :, OPC]
            if opc.min() > ILL_OPC:
                continue
            order = np.argsort(opc)
            above, below = np.nonzero(opc > 1.5e-12)[0], np.nonzero(opc <= 1.5e-12)[0]
            pick = list(order[:6]) + list(above[np.argsort(opc[above])[:2]]) + list(below[np.argsort(-opc[below])[:2]])
            cond = np.where(opc < ILL_OPC, 1.0 / np.maximum(opc, 1.5e-12), 0.0)  # the oracle's loss ~ 1 / (1 + cos i)
            pick += list(np.argsort(-cond * (opc > 1.5e-12))[:2])
        else:
            rr = np.linalg.norm(oracle.constellation_propagate([tles[s]], jd, fr)[0][0], axis=-1)
            pick = list(np.argsort(rr)[:4])
        for k in sorted(set(int(i) for i in pick)):
            cells.append((s, k))
    out = []
    for s, k in cells:
        sat = oracle.Sdp4(*tles[s])
        t = (jd[k] + fr[k] - sat.epochJd) * 1440.0
        st, r0, v0 = sdp4_statement(sat.el, t)
        assert st == 0, (name, s, k)
        sr = sv = 0.0
        for a, b in ((1, 0), (-1, 0), (0, 1), (0, -1)):
            _, r1, v1 = sdp4_statement(sat.el, t, inclo_ulps=a, inclm_ulps=b)
            sr, sv = max(sr, np.abs(r1 - r0).max()), max(sv, np.abs(v1 - v0).max())
        out.append((s, k, r0, v0, sr, sv))
    _STATEMENT[name] = out
    return out


def _against_statement(name, p, v, cells):
    """Max |dr|, |dv| of (p, v) from the 40-digit value, and whether every cell is within 1e-6 km (1e-9 km/s) plus
    twice the +-1-ulp spread."""
    dr = np.array([np.abs(p[s, k] - r0).max() for s, k, r0, _, _, _ in cells])
    dv = np.array([np.abs(v[s, k] - v0).max() for s, k, _, v0, _, _ in cells])
    br = np.array([POS_TOL + 2.0 * sr for *_, sr, _ in cells])
    bv = np.array([VEL_TOL + 2.0 * sv for *_, sv in cells])
    return dr, dv, (dr < br) & (dv < bv)


def _check_ill(name, p, v, po, vo, oracle, deep, who):
    if name not in ("retrograde", "heo"):
        return ""
    cells = _statement_cells(name, oracle, deep)
    dr, dv, ok = _against_statement(name, p, v, cells)
    assert ok.all(), (name, who, [(c[0], c[1], dr[i], c[4]) for i, c in enumerate(cells) if not ok[i]])
    odr, odv, ook = _against_statement(name, po, vo, cells)
    if name == "heo":
        assert ook.all(), (name, "oracle", odr.max())
    else:
        # the oracle's own limit: where it misses the bound, 1 + cos(inclm) is small enough that its rounding of
        # cos(inclm) (1.1e-16 absolute) is what moves it
        opc = _regimes(deep, *FIXTURES[name])[..., OPC]
        miss = [opc[s, k] for i, (s, k, *_) in enumerate(cells) if not ook[i]]
        assert all(o < 1e-8 for o in miss), miss
    spread = max(c[4] for c in cells)
    return (f"; 40-digit value over {len(cells)} cells: {who} max |dr| = {dr.max():.3e} km, |dv| = {dv.max():.3e} km/s; "
            f"oracle max |dr| = {odr.max():.3e} km ({int((~ook).sum())} cells outside the bound); "
            f"+-1-ulp spread up to {spread:.3e} km")


# ------------------------------------------------------------------------------------- CPU
def test_statement_matches_oracle_on_golden_sets(oracle):
    """The 40-digit statement against the oracle on the reference's golden GPS (non-resonant), GEO (synchronous,
    Lyddane) and HEO (half-day resonance) sets, from epoch to 30 days: rounding level of the oracle's doubles."""
    for tle in (G.GPS20413, G.GEO28626, G.HEO09880):
        sat = oracle.Sdp4(*tle)
        for t in (0.0, 720.0, 1440.0, -3000.0, 10000.0, 43200.0):
            rc, r, v = sat.propagate(t)
            st, rm, vm = sdp4_statement(sat.el, t)
            assert rc == st == 0
            assert np.abs(r - rm).max() < 5e-8 and np.abs(v - vm).max() < 5e-12, (tle[1][:7], t)


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_deep_cold_paths_host_emulation(emul, deep, oracle, name):
    """Each fixture through the host emulation of the grid core at 1, 2 and 3 lanes: the oracle's bounds where the
    problem is well conditioned, the 40-digit value where it is not, status bytes everywhere."""
    tles, jd, fr = FIXTURES[name]
    po, vo, err, klass = oracle.constellation_propagate(tles, jd, fr)
    reg = _regimes(deep, tles, jd, fr)
    _reach(name, reg, klass)
    assert np.array_equal(reg[..., STATUS].astype(np.uint8), err), name  # the probe's status is the oracle's
    wc = _well_conditioned(name, reg)
    for lanes in (1, 2, 3):
        emul.lib.emul_set_lanes(lanes)
        pe, ve, st = emul(tles, jd, fr)
        dr, dv = _compare(name, pe, ve, st, po, vo, err, wc)
        extra = _check_ill(name, pe, ve, po, vo, oracle, deep, "host emulation")
    emul.lib.emul_set_lanes(1)
    print(f"\n{name}: host emulation max |dr| = {dr:.3e} km, |dv| = {dv:.3e} km/s vs oracle{extra}")


def _direct_cases(oracle):
    """A synchronous GEO and a half-day Molniya at a carried node (atime = +-720 n, the oracle honours such a carry):
    librations x = (xni - no) / no on both sides of 3e-3 and far beyond it, and xni <= 0 (nm <= 0)."""
    cases = []
    for tle in (G.GEO28626, G.HEO09880):
        sat = oracle.Sdp4(*tle)
        no = sat.el["noUnkozai"]
        for x in (2.9e-3, -2.9e-3, 3.1e-3, -3.1e-3, 1e-2, -2e-2, 0.1, -1.0, -1.5):
            for t, atime in ((1000.0, 720.0), (-2000.0, -1440.0), (30000.0, 29520.0)):
                cases.append((tle, sat, t, sat.el["xlamo"] + 0.01, no * (1.0 + x), atime, x))
    return cases


def _direct(lib_call, cases):
    out = []
    for tle, _, t, xli, xni, atime, _ in cases:
        out.append(lib_call(tle, t, xli, xni, atime))
    return out


def _check_direct(cases, results, oracle):
    hit = set()
    for (tle, sat, t, xli, xni, atime, x), (st, r, v) in zip(cases, results):
        sat._carry = np.array([atime, xli, xni])
        rc, ro, vo = sat.propagate_carry(t)
        assert st == rc, (tle[1][:7], t, x, st, rc)
        if rc == 0:
            assert np.abs(r - ro).max() < POS_TOL and np.abs(v - vo).max() < VEL_TOL, (tle[1][:7], t, x)
            hit.add("cbrt" if abs(x) > 3e-3 else "series")
        elif xni <= 0.0:
            hit.add("nm <= 0")
    assert hit == {"cbrt", "series", "nm <= 0"}, hit


def test_libration_cube_root_and_nm_status(deep, oracle):
    """The general cube root (|x| > 3e-3) and the nm <= 0 status, which no catalogued element set reaches (every
    fixture above asserts |x| <= 3e-3), driven through sdp4_cell with a caller-supplied (xli, xni, atime) against the
    oracle started from the same carried state."""
    cases = _direct_cases(oracle)

    def call(tle, t, xli, xni, atime):
        a = [np.array([v]) for v in (t, xli, xni, atime)]
        p, v, st = np.zeros(3), np.zeros(3), np.zeros(1, dtype=np.int32)
        assert deep.emul_deep_cell(tle[0].encode(), tle[1].encode(), 1, *[x.ctypes.data_as(_dp) for x in a], 1,
                                   p.ctypes.data_as(_dp), v.ctypes.data_as(_dp),
                                   st.ctypes.data_as(C.POINTER(C.c_int32))) == 0
        return int(st[0]), p, v

    _check_direct(cases, _direct(call, cases), oracle)


# ------------------------------------------------------------------------------------- device
@pytest.fixture(scope="module")
def az():
    import astroz_b200

    astroz_b200.lib()
    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return astroz_b200


def _device_grid(c, jd, fr, layout):
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
def test_deep_cold_paths_on_device(az, deep, oracle, name):
    """Each fixture on the device: host- and K5-initialised handles, the grid in both layouts and propagate_pairs, with
    the host-emulation test's bounds."""
    import torch

    tles, jd, fr = FIXTURES[name]
    po, vo, err, klass = oracle.constellation_propagate(tles, jd, fr)
    reg = _regimes(deep, tles, jd, fr)
    _reach(name, reg, klass)
    wc = _well_conditioned(name, reg)
    worst = [0.0, 0.0]
    extra = ""
    handles = [az.Constellation(tles),
               az.Constellation.from_device_elements(torch.from_numpy(synth.elements_from_tles(tles)).cuda())]
    n, nt = len(tles), len(jd)
    for c in handles:
        assert list(c.classes) == list(klass)
        runs = [_device_grid(c, jd, fr, layout) for layout in (0, 1)]
        sat = np.repeat(np.arange(n, dtype=np.int64), nt)
        pp, pv, pst = c.propagate_pairs(sat, np.tile(jd, n), np.tile(fr, n))
        runs.append((pp.reshape(n, nt, 3), pv.reshape(n, nt, 3), pst.reshape(n, nt)))
        for p, v, st in runs:
            for k, e in enumerate(_compare(name, p, v, st, po, vo, err, wc)):
                worst[k] = max(worst[k], e)
            extra = _check_ill(name, p, v, po, vo, oracle, deep, "device") or extra
    print(f"\n{name}: device max |dr| = {worst[0]:.3e} km, |dv| = {worst[1]:.3e} km/s vs oracle{extra}")


@pytest.mark.gpu
def test_libration_cube_root_and_nm_status_on_device(probe, oracle):
    """The direct-entry cases of test_libration_cube_root_and_nm_status through sdp4_cell in a device kernel."""
    cases = _direct_cases(oracle)

    def call(tle, t, xli, xni, atime):
        a = [np.array([v]) for v in (t, xli, xni, atime)]
        out, st = np.zeros(6), np.zeros(1, dtype=np.int32)
        rc = probe.probe_sdp4_cell(tle[0].encode(), tle[1].encode(), 1, *[x.ctypes.data_as(_dp) for x in a], 1,
                                   out.ctypes.data_as(_dp), st.ctypes.data_as(C.POINTER(C.c_int32)), 1)
        assert rc == 0, rc
        ok = st[0] == 0
        return int(st[0]), out[:3] if ok else np.zeros(3), out[3:] if ok else np.zeros(3)

    _check_direct(cases, _direct(call, cases), oracle)
