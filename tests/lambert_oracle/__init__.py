"""ctypes loader for the scalar C statement of the Lambert solver (lambert.c) -- TEST INFRASTRUCTURE ONLY; the product
package never imports it.  The library is compiled with gcc -ffp-contract=off on first use, next to its source."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "lambert.c")
_SO = os.path.join(_HERE, "liblambert_oracle.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
            subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-shared", "-o", _SO, _SRC,
                            "-lm", "-lpthread"], check=True, capture_output=True)
        L = C.CDLL(_SO)
        vp, d = C.c_void_p, C.c_double
        L.lam_batch.argtypes = [vp, vp, vp, vp, C.c_size_t, d, C.c_uint32, vp, vp, vp, vp, C.c_int]
        L.lam_tmin.argtypes = [d, C.c_int]
        L.lam_tmin.restype = d
        L.lam_tof.argtypes = [d, d, C.c_int]
        L.lam_tof.restype = d
        L.lam_geometry.argtypes = [vp, vp, d, d, vp, vp]
        L.lam_geometry.restype = C.c_int
        _lib = L
    return _lib


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def solve(r1, r2, tof, mu, *, max_revs=0, normal=None, threads=1):
    """lambert_batch's outputs for n problems: v1, v2 (n, S, 3), status, iterations (n, S)."""
    r1 = np.ascontiguousarray(np.asarray(r1, dtype=np.float64).reshape(-1, 3))
    n = len(r1)
    r2 = np.ascontiguousarray(np.asarray(r2, dtype=np.float64).reshape(n, 3))
    tof = np.ascontiguousarray(np.broadcast_to(np.asarray(tof, dtype=np.float64), (n,)))
    nrm = None if normal is None else np.ascontiguousarray(np.broadcast_to(np.asarray(normal, dtype=np.float64), (n, 3)))
    S = 2 * max_revs + 1
    v1, v2 = np.zeros((n, S, 3)), np.zeros((n, S, 3))
    st, it = np.zeros((n, S), dtype=np.uint8), np.zeros((n, S), dtype=np.uint8)
    lib().lam_batch(_p(r1), _p(r2), _p(tof), _p(nrm), n, float(mu), max_revs, _p(v1), _p(v2), _p(st), _p(it),
                    int(threads))
    return v1, v2, st, it


def geometry(r1, r2, tof, mu, normal=(0.0, 0.0, 1.0)):
    """(lambda, T) of a problem, or None when the whole problem has a non-OK status"""
    out = np.zeros(18)
    a = [np.ascontiguousarray(x, dtype=np.float64) for x in (r1, r2, normal)]
    if lib().lam_geometry(_p(a[0]), _p(a[1]), float(tof), float(mu), _p(a[2]), _p(out)):
        return None
    return out[0], out[1]


def t_min(lam, M):
    return lib().lam_tmin(float(lam), int(M))


def tof_of_x(x, lam, M):
    return lib().lam_tof(float(x), float(lam), int(M))
