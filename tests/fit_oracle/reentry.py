"""K19 reentry prediction for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

An independent numpy / scipy statement of the definition: Vallado's Table 8-4 atmosphere, the WGS-84 geodetic height
by fixed-point iteration on the latitude, the force (two-body, textbook J2, quadratic co-rotating drag), the GMST of the
ECEF output mode, and a trajectory integrated by scipy's DOP853 with a height event.
emul_library(): the host build of the device source (tests/host_emul/emul_reentry.cu) and thin wrappers of its entry
points."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731

H0 = np.array([0, 25, 30, 40, 50, 60, 70, 80, 90, 100, 110, 120, 130, 140, 150, 180, 200, 250, 300, 350, 400, 450, 500,
               600, 700, 800, 900, 1000], dtype=np.float64)
RHO0 = np.array([1.225, 3.899e-2, 1.774e-2, 3.972e-3, 1.057e-3, 3.206e-4, 8.770e-5, 1.905e-5, 3.396e-6, 5.297e-7,
                 9.661e-8, 2.438e-8, 8.484e-9, 3.845e-9, 2.070e-9, 5.464e-10, 2.789e-10, 7.248e-11, 2.418e-11,
                 9.518e-12, 3.725e-12, 1.585e-12, 6.967e-13, 1.454e-13, 3.614e-14, 1.170e-14, 5.245e-15, 3.019e-15])
HS = np.array([7.249, 6.349, 6.682, 7.554, 8.382, 7.714, 6.549, 5.799, 5.382, 5.877, 7.263, 9.473, 12.636, 16.149,
               22.523, 29.740, 37.105, 45.546, 53.628, 53.298, 58.515, 60.828, 63.822, 71.835, 88.667, 124.64, 181.05,
               268.00])
OMEGA = 7.292115e-5
BSTAR_TO_B = 12.741621
WGS72 = dict(mu=398600.8, req=6378.135, j2=0.001082616)
A_WGS84, F_WGS84 = 6378.137, 1.0 / 298.257223563


def density(h):
    h = np.asarray(h, dtype=np.float64)
    j = np.clip(np.searchsorted(H0, h, side="right") - 1, 0, len(H0) - 1)
    return RHO0[j] * np.exp(-(h - H0[j]) / HS[j])


def geodetic(r):
    """(lat rad, lon rad, h km) of positions r (..., 3) on WGS-84, latitude iterated to convergence"""
    r = np.asarray(r, dtype=np.float64)
    e2 = 2 * F_WGS84 - F_WGS84 ** 2
    x, y, z = r[..., 0], r[..., 1], r[..., 2]
    p = np.hypot(x, y)
    lat = np.arctan2(z, p * (1 - e2))
    for _ in range(30):
        N = A_WGS84 / np.sqrt(1 - e2 * np.sin(lat) ** 2)
        lat = np.arctan2(z + e2 * N * np.sin(lat), p)
    N = A_WGS84 / np.sqrt(1 - e2 * np.sin(lat) ** 2)
    h = p * np.cos(lat) + z * np.sin(lat) - A_WGS84 * np.sqrt(1 - e2 * np.sin(lat) ** 2)
    return lat, np.arctan2(y, x), h


def accel(s, mu, req, j2, omega, bf):
    s = np.asarray(s, dtype=np.float64)
    r, v = s[..., :3], s[..., 3:]
    rn = np.linalg.norm(r, axis=-1, keepdims=True)
    z2 = (r[..., 2:3] / rn) ** 2
    k = -1.5 * j2 * mu * req ** 2 / rn ** 5
    aj2 = k * r * np.concatenate([1 - 5 * z2, 1 - 5 * z2, 3 - 5 * z2], axis=-1)
    vrel = v - np.cross(np.array([0.0, 0.0, omega]), r)
    h = geodetic(r)[2][..., None]
    drag = -0.5 * bf * density(h) * np.linalg.norm(vrel, axis=-1, keepdims=True) * vrel * 1e3
    return -mu * r / rn ** 3 + aj2 + drag


def gmst(jd):
    """julian_to_gmst of the ECEF output mode [rad]"""
    d = jd - 2451545.0
    t = d / 36525.0
    g = 280.46061837 + 360.98564736629 * d + 0.000387933 * t * t - t ** 3 / 38710000.0
    return np.radians(np.mod(g, 360.0))


def footprint(r, jd):
    """(lat deg, east lon deg) of TEME position r at jd"""
    g = gmst(jd)
    x = np.cos(g) * r[0] + np.sin(g) * r[1]
    y = -np.sin(g) * r[0] + np.cos(g) * r[1]
    lat, lon, _ = geodetic(np.array([x, y, r[2]]))
    return np.degrees(lat), np.degrees(lon)


def integrate(y0, B, hi, horizon_s, mu, req, j2, omega=OMEGA, scale=1.0, rtol=1e-12):
    """(t_cross s or inf, state at the crossing) by DOP853 with a height event"""
    from scipy.integrate import solve_ivp

    bf = B * scale
    f = lambda t, s: np.r_[s[3:], accel(s, mu, req, j2, omega, bf)]  # noqa: E731
    ev = lambda t, s: geodetic(s[:3])[2] - hi  # noqa: E731
    ev.terminal, ev.direction = True, -1
    sol = solve_ivp(f, (0.0, horizon_s), np.asarray(y0, dtype=np.float64), method="DOP853", rtol=rtol, atol=1e-9,
                    events=ev)
    if len(sol.t_events[0]) == 0:
        return np.inf, None
    return sol.t_events[0][0], sol.y_events[0][0]


# ---- the host build ---------------------------------------------------------------------------------------------------
def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_reentry.so")
    src = os.path.join(emul_dir, "emul_reentry.cu")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    d, u32, u64, i = C.c_double, C.c_uint32, C.c_uint64, C.c_int
    vp = C.c_void_p
    L.emul_reentry_density.argtypes = [vp, u32, vp]
    L.emul_reentry_height.argtypes = [vp, u32, vp]
    L.emul_reentry_accel.argtypes = [vp, u32, d, d, d, d, d, vp]
    L.emul_reentry_locate.argtypes = [vp, vp, d, d]
    L.emul_reentry_locate.restype = d
    L.emul_reentry_hermite.argtypes = [vp, vp, d, d, vp]
    L.emul_reentry_integrate.argtypes = [vp, d, d, d, d, d, d, d, d, d, d, d, vp]
    L.emul_reentry_draw.argtypes = [vp, i, vp, vp, d, u64, vp, u32, i, vp, vp, vp, vp, vp]
    L.emul_reentry.argtypes = [vp, u32, i, vp, vp, vp, vp, vp, vp, vp, u32, d, d, d, d, d, u32, vp, vp, vp, vp, vp, vp,
                               i]
    return L


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def emul_density(L, h):
    h = f64(np.atleast_1d(h))
    out = np.zeros_like(h)
    L.emul_reentry_density(_p(h), len(h), _p(out))
    return out


def emul_height(L, r):
    r = f64(np.reshape(r, (-1, 3)))
    out = np.zeros(len(r))
    L.emul_reentry_height(_p(r), len(r), _p(out))
    return out


def emul_accel(L, s, mu, req, j2, omega, bf):
    s = f64(np.reshape(s, (-1, 6)))
    out = np.zeros((len(s), 3))
    L.emul_reentry_accel(_p(s), len(s), mu, req, j2, omega, bf, _p(out))
    return out


def emul_integrate(L, y0, B, hi, horizon_s, mu, req, j2, omega=OMEGA, epoch=2460000.5, f=1.0, step=60.0, scale=1.0):
    """dict of the trajectory's words"""
    y0 = f64(y0)
    out = np.zeros(15)
    L.emul_reentry_integrate(_p(y0), epoch, B, f, hi, horizon_s, step, scale, omega, mu, req, j2, _p(out))
    return dict(dt=out[0], lat=out[1], lon=out[2], speed=out[3], fpa=out[4], y=out[5:11], acc=int(out[11]),
                rej=int(out[12]), status=int(out[13]))


def emul_locate(L, a, b, dt, hi):
    a, b = f64(a), f64(b)
    return L.emul_reentry_locate(_p(a), _p(b), dt, hi)


def emul_draw(L, el, model, P, seed, k, sigma=0.0, ballistic=None, grav=1):
    k = np.ascontiguousarray(k, np.uint64)
    n = len(k)
    x, B, f, y, built = np.zeros((n, 7)), np.zeros(n), np.zeros(n), np.zeros((n, 6)), np.zeros(n, np.uint8)
    bc = None if ballistic is None else f64([ballistic])
    el, P = f64(el), f64(P)
    st = L.emul_reentry_draw(_p(el), int(model), _p(P), _p(bc), sigma, seed, _p(k), n, grav, _p(x), _p(B),
                             _p(f), _p(y), _p(built))
    return st, x, B, f, y, built


def emul(L, el, cov, model, rows, *, ballistic=None, samples=0, first=0, seed=0, hi=80.0, horizon_days=30.0,
         step=60.0, scale=1.0, sigma=0.0, record=0, grav=1, threads=8):
    """the host build's (record (m, 8), states (m, 6), nominal status, counts (m, 3), sample words (m, record, 4),
    status)"""
    el = f64(el)
    n = el.shape[1]
    cov = f64(cov)
    md = None if model is None else np.ascontiguousarray(model, np.uint8)
    rows = np.ascontiguousarray(rows, np.uint32)
    m = len(rows)
    u64 = lambda a: np.ascontiguousarray(np.broadcast_to(np.asarray(a, np.uint64), (m,)))  # noqa: E731
    bc = None if ballistic is None else f64(np.broadcast_to(ballistic, (m,)))
    rec, states, nst = np.zeros((m, 8)), np.zeros((m, 6)), np.zeros(m, np.uint8)
    counts, out, status = np.zeros((m, 3), np.uint64), np.zeros((m, record, 4)), np.zeros(m, np.uint8)
    ns, fi, sd = u64(samples), u64(first), u64(seed)   # held: the pointers must outlive the call
    L.emul_reentry(_p(el), n, grav, _p(cov), _p(md), _p(rows), _p(bc), _p(ns), _p(fi), _p(sd), m, hi, horizon_days, step, scale, sigma, record, _p(rec), _p(states), _p(nst),
                   _p(counts), _p(out), _p(status), threads)
    return rec, states, nst, counts, out, status
