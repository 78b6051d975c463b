"""ctypes loader for the maneuver restatement maneuvers.c (azn_propagate_maneuvers, azn_apply_burn) -- TEST
INFRASTRUCTURE ONLY.  The library is compiled with gcc -ffp-contract=off on first use, next to its source.  Schedules
are the product's (astroz_b200.numerical.pack_schedules), model lists its descriptors."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from astroz_b200 import numerical as P
from tests.numerical_oracle import models as M

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, f) for f in ("maneuvers.c", "numerical_oracle_models.c", "numerical_oracle.c")]
_SO = os.path.join(_HERE, "libnumerical_oracle_maneuvers.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in _SRCS):
            subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-shared", "-o", _SO,
                            _SRCS[0], "-lm", "-lpthread"], check=True, capture_output=True)
        L = C.CDLL(_SO)
        vp, d, sz = C.c_void_p, C.c_double, C.c_size_t
        L.azn_propagate_maneuvers.argtypes = [vp, sz, d, d, d, d, vp, vp, vp, C.c_int, C.c_int, d, d, C.c_int, sz, vp,
                                              vp, vp, vp, vp, C.c_int]
        L.azn_propagate_maneuvers.restype = None
        L.azn_apply_burn.argtypes = [vp, sz, C.c_int32, vp, d, C.c_int, vp]
        L.azn_apply_burn.restype = None
        _lib = L
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data) if a.size else None


def propagate(states, t0, duration, h, models, schedules, *, mu=P.EARTH_MU, integrator="rk4", rtol=1e-9, atol=1e-12,
              max_samples=None, k7_forms=False, threads=1):
    """Spacecraft.propagate of each row of states (n, 6) with its schedule: (times[n, S], traj[n, S, 6], n_samples[n],
    status[n], steps[n, 2]).  max_samples None: rows as long as the longest trajectory (found by a first pass).
    k7_forms forms pow and errNorm^(-1/8) as the device cores do."""
    states = np.ascontiguousarray(np.atleast_2d(states), dtype=np.float64)
    n = states.shape[0]
    offsets, imp = P.pack_schedules(schedules, n)
    descs, keep = M.descriptors(models, n, 1)

    def run(cap):
        times = np.zeros((n, cap))
        out = np.zeros((n, cap, 6))
        count = np.zeros(n, dtype=np.uint64)
        status = np.zeros(n, dtype=np.uint8)
        steps = np.zeros((n, 2), dtype=np.uint64)
        lib().azn_propagate_maneuvers(_p(states), n, float(t0), float(duration), float(h), float(mu), _p(offsets),
                                      _p(imp), C.cast(descs, C.c_void_p), len(descs),
                                      {"rk4": 0, "dp87": 1}[integrator], float(rtol), float(atol),
                                      1 if k7_forms else 0, cap, _p(times), _p(out), _p(count), _p(status), _p(steps),
                                      int(threads))
        return times, out, count, status, steps

    if max_samples is None:
        probe = run(1)
        max_samples = max(1, int(probe[2].max(initial=1)))
    res = run(int(max_samples))
    del keep
    return res


def apply_burn(y, burn, mu=P.EARTH_MU, k7_forms=False):
    """The restatement's burn `burn` (a phasing burn: its first half) applied to states y (m, 6)"""
    y = np.ascontiguousarray(np.atleast_2d(y), dtype=np.float64)
    out = np.zeros_like(y)
    p = np.ascontiguousarray(burn.p, dtype=np.float64)
    lib().azn_apply_burn(_p(y), len(y), burn.kind, _p(p), float(mu), 1 if k7_forms else 0, _p(out))
    return out
