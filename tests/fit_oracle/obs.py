"""An independent numpy statement of the observation kinds of the element fit (astroz_b200/csrc/az_obs.cuh), for the
observation-fit tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.  Written from the definitions
(GMST polynomial, WGS84 geodetic station, horizon frame, topocentric angles), not from the device source."""
from __future__ import annotations

import numpy as np

TEME, ECEF, RADAR, OPTICAL = 0, 1, 2, 3
COUNTS = {TEME: 6, ECEF: 6, RADAR: 4, OPTICAL: 2}
OMEGA = np.deg2rad(360.98564736629) / 86400.0      # rad/s, the GMST polynomial's rate
A84, F84 = 6378.137, 1.0 / 298.257223563


def gmst(jd_full):
    d = np.asarray(jd_full, dtype=np.float64) - 2451545.0
    t = d / 36525.0
    g = 280.46061837 + 360.98564736629 * d + 0.000387933 * t * t - t ** 3 / 38710000.0
    return np.deg2rad(np.mod(g, 360.0))


def station_ecef(llh):
    lat, lon, h = np.deg2rad(llh[0]), np.deg2rad(llh[1]), llh[2]
    e2 = F84 * (2.0 - F84)
    N = A84 / np.sqrt(1.0 - e2 * np.sin(lat) ** 2)
    return np.array([(N + h) * np.cos(lat) * np.cos(lon), (N + h) * np.cos(lat) * np.sin(lon),
                     (N * (1.0 - e2) + h) * np.sin(lat)])


def enu_basis(llh):
    lat, lon = np.deg2rad(llh[0]), np.deg2rad(llh[1])
    east = np.array([-np.sin(lon), np.cos(lon), 0.0])
    north = np.array([-np.sin(lat) * np.cos(lon), -np.sin(lat) * np.sin(lon), np.cos(lat)])
    up = np.array([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)])
    return east, north, up


def rot(theta):
    """Rz(theta): TEME -> Earth-fixed for theta = GMST, one 3 x 3 per epoch"""
    c, s = np.cos(theta), np.sin(theta)
    R = np.zeros(np.shape(theta) + (3, 3))
    R[..., 0, 0], R[..., 0, 1], R[..., 1, 0], R[..., 1, 1], R[..., 2, 2] = c, s, -s, c, 1.0
    return R


def ecef_state(states, jd_full):
    states = np.asarray(states, dtype=np.float64).reshape(-1, 6)
    R = rot(gmst(jd_full) * np.ones(len(states)))
    r = np.einsum("nij,nj->ni", R, states[:, :3])
    v = np.einsum("nij,nj->ni", R, states[:, 3:]) - np.cross([0.0, 0.0, OMEGA], r)
    return r, v


def observe(kind, states, jd_full, llh=None):
    """values (m, 6) of one kind, TEME states (m, 6) at jd_full (m,), one station (lat deg, lon deg, h km)"""
    states = np.asarray(states, dtype=np.float64).reshape(-1, 6)
    jd_full = np.asarray(jd_full, dtype=np.float64) * np.ones(len(states))
    out = np.zeros((len(states), 6))
    if kind == TEME:
        return states.copy()
    r, v = ecef_state(states, jd_full)
    if kind == ECEF:
        out[:, :3], out[:, 3:] = r, v
        return out
    rs = station_ecef(llh)
    if kind == RADAR:
        e, n, u = enu_basis(llh)
        rho = r - rs
        E, N, U = rho @ e, rho @ n, rho @ u
        rng = np.linalg.norm(rho, axis=1)
        out[:, 0] = rng
        out[:, 1] = np.mod(np.arctan2(E, N), 2 * np.pi)
        out[:, 2] = np.arctan2(U, np.hypot(E, N))
        out[:, 3] = np.einsum("ni,ni->n", rho, v) / rng
        return out
    R = rot(gmst(jd_full))
    rho = states[:, :3] - np.einsum("nji,j->ni", R, rs)      # station in TEME: R^T r_station
    out[:, 0] = np.mod(np.arctan2(rho[:, 1], rho[:, 0]), 2 * np.pi)
    out[:, 1] = np.arctan2(rho[:, 2], np.hypot(rho[:, 0], rho[:, 1]))
    return out


def elevation(states, jd_full, llh):
    return observe(RADAR, states, jd_full, llh)[:, 2]


# ---- tracks and the host emulation of the observation fits ----------------------------------------------------------
RADAR_SITES = np.array([[42.6, -71.5, 0.12], [9.4, 167.5, 0.01], [-31.0, 136.0, 0.15], [69.3, 16.0, 0.05],
                        [36.0, 139.0, 0.2], [-22.0, -47.0, 0.7]])
RADAR_SIGMA = np.array([0.01, np.deg2rad(0.01), np.deg2rad(0.01), 1e-5])     # 10 m, 36", 36", 1 cm/s
OPTICAL_SIGMA = np.array([np.deg2rad(1.0 / 3600), np.deg2rad(1.0 / 3600)])   # 1"


def states_of(el, jd, fr):
    """oracle TEME states (m, 6) of one element set (SGP4 or SDP4 by its period)"""
    from tests import fit_oracle as R
    from tests.fit_oracle import deep as D

    obs = D.observe if 1440.0 / el[1] > 225.0 else R.observe
    p, v = obs(el, jd, fr)
    return np.concatenate([p, v], axis=1)


def tracks(el, kind, sites, jd, fr, min_el_deg=10.0, sigma=None):
    """Noise-free observations of one set: every (site, epoch) with the satellite above min_el_deg (all epochs for
    the state kinds, which take no site).  Returns jd, fr, kind, value (m, 6), sigma (m, 6), station (m,)."""
    st = states_of(el, jd, fr)
    jdf = jd + fr
    rows = []
    if kind in (TEME, ECEF):
        sig = np.array([1e-3] * 3 + [1e-6] * 3) if sigma is None else sigma
        rows.append((np.arange(len(jd)), 0, observe(kind, st, jdf)))
    else:
        sig = (RADAR_SIGMA if kind == RADAR else OPTICAL_SIGMA) if sigma is None else sigma
        for k, site in enumerate(sites):
            keep = np.flatnonzero(elevation(st, jdf, site) > np.deg2rad(min_el_deg))
            rows.append((keep, k, observe(kind, st[keep], jdf[keep], site)))
    idx = np.concatenate([r[0] for r in rows])
    val = np.concatenate([r[2] for r in rows])
    station = np.concatenate([np.full(len(r[0]), r[1], dtype=np.uint32) for r in rows])
    sigma6 = np.full((len(idx), 6), np.inf)
    sigma6[:, :len(sig)] = sig
    return jd[idx], fr[idx], np.full(len(idx), kind, dtype=np.uint8), val, sigma6, station


def concat(per_sat):
    """[(jd, fr, kind, value, sigma, station), ...] per satellite -> one batch grouped by satellite + offsets"""
    cols = [np.concatenate([t[c] for t in per_sat]) for c in range(6)]
    offsets = np.concatenate([[0], np.cumsum([len(t[0]) for t in per_sat])]).astype(np.uint32)
    return (*cols, offsets)


def emul_library():
    import ctypes as C
    import os
    import shutil
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    emul_dir = os.path.join(root, "tests", "host_emul")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_fit_obs.so")
    src = os.path.join(emul_dir, "emul_fit_obs.cu")
    csrc = os.path.join(root, "astroz_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    return C.CDLL(so)


def _p(a):
    import ctypes as C

    return None if a is None else C.c_void_p(a.ctypes.data)


def emul_fit(L, elements, jd, fr, kind, value, sigma, station, offsets, stations, *, fit_bstar=True, max_iter=25,
             mixed=True, grav=1):
    """The host emulation of astroz_cuda_fit_observations[_mixed]: (fitted, wrms, n_residuals, covariance,
    iterations, status)"""
    import ctypes as C

    el = np.ascontiguousarray(elements, dtype=np.float64)
    n = el.shape[1]
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (jd, fr, value, sigma)]
    sta = np.ascontiguousarray(station, dtype=np.uint32)
    kd = np.ascontiguousarray(kind, dtype=np.uint8)
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    st = np.ascontiguousarray(stations, dtype=np.float64).reshape(-1, 3)
    fitted, wrms, nres = np.zeros((8, n)), np.zeros(n), np.zeros(n, dtype=np.uint32)
    cov, iters, status = np.zeros((n, 28)), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
    f = L.emul_fit_obs_mixed if mixed else L.emul_fit_obs
    f(_p(el), C.c_uint32(n), grav, _p(off), *[_p(x) for x in a[:2]], _p(a[2]), _p(a[3]), _p(sta), _p(kd), _p(st),
      int(bool(fit_bstar)), C.c_uint32(max_iter), _p(fitted), _p(wrms), _p(nres), _p(cov), _p(iters), _p(status))
    return fitted, wrms, nres, cov, iters, status


def emul_observe(L, states, jd, fr, kind, station, stations):
    import ctypes as C

    s = np.ascontiguousarray(states, dtype=np.float64).reshape(-1, 6)
    m = len(s)
    a = [np.ascontiguousarray(np.broadcast_to(x, (m,)), dtype=np.float64) for x in (jd, fr)]
    kd = np.ascontiguousarray(np.broadcast_to(kind, (m,)), dtype=np.uint8)
    sta = np.ascontiguousarray(np.broadcast_to(station, (m,)), dtype=np.uint32)
    st = np.ascontiguousarray(stations, dtype=np.float64).reshape(-1, 3)
    out = np.zeros((m, 6))
    L.emul_observe(_p(s), _p(a[0]), _p(a[1]), _p(kd), _p(sta), C.c_uint32(m), _p(st), _p(out))
    return out


def fit_vars(el, deep):
    """the fit's variables (7,) of element columns el (8,): near-earth or equinoctial"""
    d = np.pi / 180.0
    node, w = el[4] * d, el[5] * d
    if not deep:
        return np.array([el[1], el[2] * np.cos(w), el[2] * np.sin(w), el[3] * d, node, el[6] * d + w, el[7]])
    P, t = w + node, np.tan(0.5 * el[3] * d)
    return np.array([el[1], el[2] * np.cos(P), el[2] * np.sin(P), t * np.cos(node), t * np.sin(node),
                     el[6] * d + P, el[7]])


def restated_library():
    """fit_oracle_obs.c with the oracle's SGP4 / SDP4 (gcc -ffp-contract=off), built next to its source on first use"""
    import ctypes as C
    import os
    import subprocess

    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(os.path.dirname(here))
    srcs = [os.path.join(here, "fit_oracle_obs.c"), os.path.join(root, "oracle", "astroz_oracle.c"),
            os.path.join(root, "oracle", "astroz_oracle.h")]
    so = os.path.join(here, "libfit_oracle_obs.so")
    if not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(s) for s in srcs):
        subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-shared", "-o", so, *srcs[:2],
                        "-lm", "-lpthread"], check=True, capture_output=True)
    return C.CDLL(so)


def restated_fit(elements, jd, fr, kind, value, sigma, station, offsets, stations, *, fit_bstar=True, max_iter=25,
                 mixed=True, grav=1, threads=None):
    """The independent C restatement of astroz_cuda_fit_observations[_mixed]: (fitted, wrms, n_residuals, covariance,
    iterations, status)"""
    import ctypes as C
    import os

    L = restated_library()
    el = np.ascontiguousarray(elements, dtype=np.float64)
    n = el.shape[1]
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (jd, fr, value, sigma)]
    sta = np.ascontiguousarray(station, dtype=np.uint32)
    kd = np.ascontiguousarray(kind, dtype=np.uint8)
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    st = np.ascontiguousarray(stations, dtype=np.float64).reshape(-1, 3)
    fitted, wrms, nres = np.zeros((8, n)), np.zeros(n), np.zeros(n, dtype=np.uint32)
    cov, iters, status = np.zeros((n, 28)), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
    L.fitref_fit_obs(_p(el), C.c_uint32(n), grav, _p(off), _p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(sta), _p(kd),
                     _p(st), int(bool(fit_bstar)), C.c_uint32(max_iter), int(bool(mixed)),
                     int(threads or os.cpu_count() or 1), _p(fitted), _p(wrms), _p(nres), _p(cov), _p(iters),
                     _p(status))
    return fitted, wrms, nres, cov, iters, status
