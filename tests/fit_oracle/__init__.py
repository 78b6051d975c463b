"""ctypes loader for the scalar C restatement of the element fit (fit_oracle.c, on the CPU oracle's SGP4) -- TEST
INFRASTRUCTURE ONLY; the product package never imports it.  The library is compiled with gcc -ffp-contract=off together
with oracle/astroz_oracle.c on first use, next to its source."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRCS = [os.path.join(_HERE, "fit_oracle.c"), os.path.join(_ROOT, "oracle", "astroz_oracle.c"),
         os.path.join(_ROOT, "oracle", "astroz_oracle.h")]
_SO = os.path.join(_HERE, "libfit_oracle.so")
_lib = None

CONVERGED, ITERATION_LIMIT, INIT_FAILED, DEEP_SPACE, TOO_FEW = 0, 1, 2, 3, 4


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in _SRCS):
            subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-shared", "-o", _SO,
                            *_SRCS[:2], "-lm", "-lpthread"], check=True, capture_output=True)
        L = C.CDLL(_SO)
        vp, d, u32, i32 = C.c_void_p, C.c_double, C.c_uint32, C.c_int
        L.fitref_fit.argtypes = [vp, u32, i32, vp, vp, vp, vp, vp, d, d, i32, u32, i32, vp, vp, vp, vp]
        L.fitref_fit.restype = i32
        L.fitref_observe.argtypes = [vp, i32, vp, vp, u32, vp, vp]
        L.fitref_observe.restype = i32
        _lib = L
    return _lib


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def csr(n, sat):
    """offsets[n + 1] of observations already grouped by satellite"""
    return np.searchsorted(np.asarray(sat), np.arange(n + 1)).astype(np.uint32)


def fit(elements, offsets, jd, fr, pos, vel=None, *, pos_sigma=1.0, vel_sigma=1e-3, fit_bstar=True, max_iter=25,
        grav=1, threads=1):
    """elements (8, n); observations grouped by satellite with offsets[n + 1].  Returns (fitted (8, n), rms (n, 2),
    iterations (n,), status (n,))."""
    el = np.ascontiguousarray(elements, dtype=np.float64)
    n = el.shape[1]
    arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (jd, fr, pos)]
    v = None if vel is None else np.ascontiguousarray(vel, dtype=np.float64)
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    fitted, rms = np.zeros((8, n)), np.zeros((n, 2))
    iters, status = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
    lib().fitref_fit(_p(el), n, grav, _p(off), *[_p(a) for a in arrs], _p(v), float(pos_sigma), float(vel_sigma),
                     int(bool(fit_bstar)), int(max_iter), int(threads), _p(fitted), _p(rms), _p(iters), _p(status))
    return fitted, rms, iters, status


def observe(el, jd, fr, grav=1):
    """TEME (pos, vel) of one numeric element set (8,) at jd + fr, tsince = ((jd + fr) - epoch) * 1440."""
    el = np.ascontiguousarray(el, dtype=np.float64)
    jd = np.ascontiguousarray(jd, dtype=np.float64)
    fr = np.ascontiguousarray(fr, dtype=np.float64)
    pos, vel = np.zeros((len(jd), 3)), np.zeros((len(jd), 3))
    rc = lib().fitref_observe(_p(el), grav, _p(jd), _p(fr), len(jd), _p(pos), _p(vel))
    if rc != 0:
        raise ValueError(f"oracle init failed rc={rc}")
    return pos, vel


def perturbed(elements, seed=0):
    """The round-trip guesses: n + 1e-4 rev/day, e + 1e-4, +-0.05 deg on each angle, B* x 2 (signs drawn per
    satellite)."""
    rng = np.random.default_rng(seed)
    g = np.array(elements, dtype=np.float64, copy=True)
    n = g.shape[1]
    sign = lambda: rng.choice([-1.0, 1.0], n)  # noqa: E731
    g[1] += 1e-4 * sign()
    g[2] = np.abs(g[2] + 1e-4 * sign())
    for c in (3, 4, 5, 6):
        g[c] += 0.05 * sign()
    g[4:7] %= 360.0
    g[7] *= 2.0
    return g
