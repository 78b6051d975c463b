"""K11 conjunction assessment for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

pc_reference(): a 30-digit mpmath value of the short-encounter 2-D Pc, written independently of the device quadrature:
    the outer integral runs along C2's MINOR principal axis (the device's runs along the major one), by mpmath's
    tanh-sinh rule with its own error control, and the inner one is a normal-CDF difference along the major axis.
restated(): the independent C restatement (conjunction.c: bisection TCA on the oracle's SGP4 / SDP4, Sigma from
    covariance.c).
emul(), emul_pc(): the host build of the device source (tests/host_emul/emul_conjunction.cu)."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import mpmath as mp
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731

RECORD_WORDS = 13


def pc_reference(xx, xy, yy, d, R, dps: int = 30) -> float:
    """Pc = integral over u^2 + v^2 <= R^2 of N((u, v); (d, 0), [[xx, xy], [xy, yy]]), to `dps` digits"""
    with mp.workdps(dps + 10):
        xx, xy, yy, d, R = (mp.mpf(v) for v in (xx, xy, yy, d, R))
        if xx == 0 and xy == 0 and yy == 0:
            return 1.0 if d < R else 0.0
        half, q = (xx + yy) / 2, mp.sqrt(((xx - yy) / 2) ** 2 + xy ** 2)
        l1, l2 = half + q, (xx * yy - xy ** 2) / (half + q)
        phi = mp.atan2(2 * xy, xx - yy) / 2
        c, s = mp.cos(phi), mp.sin(phi)
        # disk centre relative to the mean, in the principal axes (u1 major, u2 minor)
        a1, a2 = d * c, -d * s
        s1, s2 = mp.sqrt(l1), mp.sqrt(l2)

        def phidiff(lo, hi):   # Phi(hi) - Phi(lo) without cancelling in a far tail
            k = 1 / mp.sqrt(2)
            if lo >= 0:
                return (mp.erfc(lo * k) - mp.erfc(hi * k)) / 2
            if hi <= 0:
                return (mp.erfc(-hi * k) - mp.erfc(-lo * k)) / 2
            return 1 - (mp.erfc(hi * k) + mp.erfc(-lo * k)) / 2

        def f(t):   # u2 = R sin t, chord half-length along u1 = R cos t
            u2, h = R * mp.sin(t), R * mp.cos(t)
            dens = mp.exp(-((u2 - a2) / s2) ** 2 / 2) / (s2 * mp.sqrt(2 * mp.pi))
            return R * mp.cos(t) * dens * phidiff((-h - a1) / s1, (h - a1) / s1)

        pts = {-mp.pi / 2, mp.pi / 2}
        for k in range(-12, 13):   # the minor-axis density's centre and sigma steps, and the chord ends over the major
            for v in (a2 + k * s2 / 2,):
                if abs(v) < R:
                    pts.add(mp.asin(v / R))
            for v in (abs(a1) + k * s1 / 2,):
                if 0 < v < R:
                    pts.add(mp.acos(v / R))
                    pts.add(-mp.acos(v / R))
        pts = sorted(pts)
        fine = []
        for lo, hi in zip(pts[:-1], pts[1:]):   # a uniform floor of 64 panels over the half turn
            n = max(1, int(mp.ceil((hi - lo) / (mp.pi / 64))))
            fine += [lo + (hi - lo) * j / n for j in range(n)]
        fine.append(pts[-1])
        return float(mp.quad(f, fine))


def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_conjunction.so")
    src = os.path.join(emul_dir, "emul_conjunction.cu")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    L.emul_conj_pc.restype = C.c_double
    L.emul_conj_pc.argtypes = [C.c_double] * 5
    return L


def emul_pc(L, xx, xy, yy, d, R) -> float:
    return float(L.emul_conj_pc(xx, xy, yy, d, R))


def _inputs(elements, cov, model, primary, secondary, jd, fr, window, hbr):
    el = np.ascontiguousarray(elements, dtype=np.float64)
    n = el.shape[1]
    cv = np.ascontiguousarray(cov, dtype=np.float64).reshape(n, 28)
    md = None if model is None else np.ascontiguousarray(model, dtype=np.uint8)
    pr = np.ascontiguousarray(primary, dtype=np.uint32)
    m = len(pr)
    f64 = lambda a: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (m,)))  # noqa: E731
    return el, cv, md, pr, np.ascontiguousarray(secondary, dtype=np.uint32), f64(jd), f64(fr), f64(window), f64(hbr)


def emul(L, elements, cov, model, primary, secondary, jd, fr, window, hbr, frame=0, grav=1):
    """the host build's (record (m, 13), states (m, 2, 6), state covariance (m, 2, 21), status (m,))"""
    el, cv, md, pr, se, jd_, fr_, w_, r_ = _inputs(elements, cov, model, primary, secondary, jd, fr, window, hbr)
    m = len(pr)
    rec, st, sig, status = np.zeros((m, RECORD_WORDS)), np.zeros((m, 2, 6)), np.zeros((m, 2, 21)), np.zeros(m, np.uint8)
    L.emul_conjunction(_p(el), C.c_uint32(el.shape[1]), grav, _p(cv), _p(md), _p(pr), _p(se), _p(jd_), _p(fr_), _p(w_),
                       _p(r_), C.c_uint32(m), int(frame), _p(rec), _p(st), _p(sig), _p(status))
    return rec, st, sig, status


def _restated_lib() -> C.CDLL:
    srcs = [os.path.join(_HERE, "conjunction.c"), os.path.join(_HERE, "covariance.c"),
            os.path.join(_HERE, "fit_oracle_obs.c"), os.path.join(_ROOT, "oracle", "astroz_oracle.c"),
            os.path.join(_ROOT, "oracle", "astroz_oracle.h")]
    so = os.path.join(_HERE, "libconjunction_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(s) for s in srcs):
        subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-Wno-unused-function",
                        "-shared", "-o", so, srcs[0], srcs[3], "-lm", "-lpthread"], check=True, capture_output=True)
    return C.CDLL(so)


def restated(elements, cov, model, primary, secondary, jd, fr, window, frame=0, grav=1, threads=None):
    """(dt_tca (m,), states (m, 2, 6), state covariance (m, 2, 21), status (m,)) of the C restatement; the plane and
    Pc are formed from these by the caller (plane_pc)"""
    el, cv, md, pr, se, jd_, fr_, w_, _ = _inputs(elements, cov, model, primary, secondary, jd, fr, window, 0.0)
    m = len(pr)
    dt, st, sig, status = np.zeros(m), np.zeros((m, 2, 6)), np.zeros((m, 2, 21)), np.zeros(m, np.uint8)
    _restated_lib().conjref_assess(_p(el), C.c_uint32(el.shape[1]), grav, _p(cv), _p(md), _p(pr), _p(se), _p(jd_),
                                   _p(fr_), _p(w_), C.c_uint32(m), int(frame), int(threads or os.cpu_count() or 1),
                                   _p(dt), _p(st), _p(sig), _p(status))
    return dt, st, sig, status


def plane(states, sig, frame=0):
    """numpy statement of the encounter plane: (miss, speed, d, C2 (3,)) from TEME states (2, 6) and Sigma words (2, 21)"""
    from tests.fit_oracle.covariance import rtn, unpack6
    dr, dv = states[1, :3] - states[0, :3], states[1, 3:] - states[0, 3:]
    z = dv / np.linalg.norm(dv)
    x = dr - (dr @ z) * z
    d = np.linalg.norm(x)
    x = x / d
    y = np.cross(z, x)
    E = np.stack([x, y])
    C2 = np.zeros((2, 2))
    for o in range(2):
        S = unpack6(sig[o])[:3, :3]
        if frame == 1:
            R = rtn(states[o][None])[0]
            S = R.T @ S @ R
        C2 += E @ S @ E.T
    return np.linalg.norm(dr), np.linalg.norm(dv), d, np.array([C2[0, 0], C2[0, 1], C2[1, 1]])
