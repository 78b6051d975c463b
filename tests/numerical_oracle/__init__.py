"""ctypes loader for the scalar C restatement of the reference's numerical propagation (numerical_oracle.c) -- TEST
INFRASTRUCTURE ONLY; the product package never imports it.  The library is compiled with gcc -ffp-contract=off on first
use, next to its source."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "numerical_oracle.c")
_SO = os.path.join(_HERE, "libnumerical_oracle.so")
FORCE_J2, FORCE_DRAG = 1, 2
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
            subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-shared", "-o", _SO, _SRC,
                            "-lm", "-lpthread"], check=True, capture_output=True)
        L = C.CDLL(_SO)
        vp, d = C.c_void_p, C.c_double
        L.azn_tableau.argtypes = [vp, vp, vp, vp]
        L.azn_times.argtypes = [d, d, d, vp, C.c_uint64, C.POINTER(C.c_uint64)]
        L.azn_times.restype = C.c_int
        L.azn_propagate_batch.argtypes = [vp, C.c_size_t, d, d, d, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp,
                                          C.c_int]
        L.azn_propagate_batch.restype = C.c_uint64
        _lib = L
    return _lib


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def tableau():
    c, a, b8, b7 = np.zeros(13), np.zeros((13, 12)), np.zeros(13), np.zeros(13)
    lib().azn_tableau(_p(c), _p(a), _p(b8), _p(b7))
    return c, a, b8, b7


def times(t0, duration, dt, max_samples=1 << 32):
    n = C.c_uint64()
    if lib().azn_times(float(t0), float(duration), float(dt), None, max_samples, C.byref(n)) != 0:
        raise ValueError("the sampling loop does not end")
    out = np.zeros(n.value)
    lib().azn_times(float(t0), float(duration), float(dt), _p(out), max_samples, C.byref(n))
    return out


def propagate(states, t0, duration, dt, mu, *, j2=None, r_eq=None, drag_cd=None, drag_area=None, drag_mass=None,
              integrator="dp87", rtol=1e-9, atol=1e-12, threads=1, k7_step_factor=False):
    """The reference's propagate_numerical for each row of states (n, 6): (times, traj[n, samples, 6], status[n],
    steps[n, 2]).  threads > 1 deals states to pthreads; the arithmetic per state does not change.  k7_step_factor forms
    the DP87 step factor errNorm^(-1/8) as K7 does (three square roots) instead of with pow: the one place where K7's
    operations differ from the reference's, so this isolates what that difference does to a trajectory."""
    states = np.ascontiguousarray(np.atleast_2d(states), dtype=np.float64)
    n = states.shape[0]
    forces = (FORCE_J2 if j2 is not None else 0) | (FORCE_DRAG if drag_cd is not None else 0)
    drag = [None] * 3
    if drag_cd is not None:
        drag = [np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (n,))) for x in
                (drag_cd, drag_area, drag_mass)]
    par = np.array([mu, j2 or 0.0, r_eq or 0.0, rtol, atol, 1.0 if k7_step_factor else 0.0], dtype=np.float64)
    t = times(t0, duration, dt)
    out = np.zeros((n, len(t), 6))
    status = np.zeros(n, dtype=np.uint8)
    steps = np.zeros((n, 2), dtype=np.uint64)
    k = lib().azn_propagate_batch(_p(states), n, float(t0), float(duration), float(dt), _p(par), forces, *map(_p, drag),
                                  {"rk4": 0, "dp87": 1}[integrator], _p(out), _p(status), _p(steps), int(threads))
    assert k == len(t)
    return t, out, status, steps
