"""ctypes loader for the deep-space restatement fit_oracle_deep.c (fitref_fit_mixed, fitref_observe_deep) -- TEST
INFRASTRUCTURE ONLY; the product package never imports it.  Compiled with gcc -ffp-contract=off together with
fit_oracle.c (the near-earth rows) and oracle/astroz_oracle.c on first use, next to its source."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from tests.fit_oracle import _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRCS = [os.path.join(_HERE, "fit_oracle_deep.c"), os.path.join(_HERE, "fit_oracle.c"),
         os.path.join(_ROOT, "oracle", "astroz_oracle.c"), os.path.join(_ROOT, "oracle", "astroz_oracle.h")]
_SO = os.path.join(_HERE, "libfit_oracle_deep.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in _SRCS):
            subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-shared", "-o", _SO,
                            *_SRCS[:3], "-lm", "-lpthread"], check=True, capture_output=True)
        L = C.CDLL(_SO)
        vp, d, u32, i32 = C.c_void_p, C.c_double, C.c_uint32, C.c_int
        L.fitref_fit_mixed.argtypes = [vp, u32, i32, vp, vp, vp, vp, vp, d, d, i32, u32, i32, vp, vp, vp, vp]
        L.fitref_fit_mixed.restype = i32
        L.fitref_observe_deep.argtypes = [vp, i32, vp, vp, u32, vp, vp]
        L.fitref_observe_deep.restype = i32
        _lib = L
    return _lib


def fit_mixed(elements, offsets, jd, fr, pos, vel=None, *, pos_sigma=1.0, vel_sigma=1e-3, fit_bstar=True,
              max_iter=25, grav=1, threads=1):
    """tests.fit_oracle.fit with the deep-space sets fitted too (fitref_fit_mixed).  Same arguments and returns."""
    el = np.ascontiguousarray(elements, dtype=np.float64)
    n = el.shape[1]
    arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (jd, fr, pos)]
    v = None if vel is None else np.ascontiguousarray(vel, dtype=np.float64)
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    fitted, rms = np.zeros((8, n)), np.zeros((n, 2))
    iters, status = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
    lib().fitref_fit_mixed(_p(el), n, grav, _p(off), *[_p(a) for a in arrs], _p(v), float(pos_sigma),
                           float(vel_sigma), int(bool(fit_bstar)), int(max_iter), int(threads), _p(fitted), _p(rms),
                           _p(iters), _p(status))
    return fitted, rms, iters, status


def observe(el, jd, fr, grav=1):
    """TEME (pos, vel) of one deep-space element set (8,) at jd + fr, from the oracle's SDP4."""
    el = np.ascontiguousarray(el, dtype=np.float64)
    jd = np.ascontiguousarray(jd, dtype=np.float64)
    fr = np.ascontiguousarray(fr, dtype=np.float64)
    pos, vel = np.zeros((len(jd), 3)), np.zeros((len(jd), 3))
    rc = lib().fitref_observe_deep(_p(el), grav, _p(jd), _p(fr), len(jd), _p(pos), _p(vel))
    if rc != 0:
        raise ValueError(f"not a deep-space set, or the oracle's propagation failed: rc={rc}")
    return pos, vel
