"""ctypes loader for the model-list restatement numerical_oracle_models.c (azn_propagate_models, azn_models_accel) --
TEST INFRASTRUCTURE ONLY.  The library is compiled with gcc -ffp-contract=off on first use, next to its source.  Model
lists are the product's descriptors (astroz_b200.numerical's TwoBody ... ThirdBody packed as astroz_force_model_t), which
the restatement reads with its own layout of the same fields."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from astroz_b200 import numerical as P
from tests import numerical_oracle as N

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, f) for f in ("numerical_oracle_models.c", "numerical_oracle.c")]
_SO = os.path.join(_HERE, "libnumerical_oracle_models.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in _SRCS):
            subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-shared", "-o", _SO,
                            _SRCS[0], "-lm", "-lpthread"], check=True, capture_output=True)
        L = C.CDLL(_SO)
        vp, d = C.c_void_p, C.c_double
        L.azn_models_accel.argtypes = [vp, C.c_int, vp, vp, C.c_uint64, C.c_size_t, vp]
        L.azn_models_accel.restype = None
        L.azn_propagate_models.argtypes = [vp, C.c_size_t, d, d, d, vp, C.c_int, C.c_int, d, d, C.c_int, vp, vp, vp,
                                           C.c_int]
        L.azn_propagate_models.restype = C.c_uint64
        _lib = L
    return _lib


def descriptors(models, n, K):
    """(astroz_force_model_t array, arrays to keep alive) for `models` over n states and K intervals"""
    return P._descriptors(models, n, K, P._host_array)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def accel(models, s, items=None, k=0):
    """The list's acceleration (one model as it is, several through Composite) at states s (m, 6) for batch items
    `items` (default 0..m-1) during interval k.  Per-state arrays must cover the largest item, tables row k."""
    s = np.ascontiguousarray(np.atleast_2d(s), dtype=np.float64)
    items = np.arange(len(s), dtype=np.uint64) if items is None else np.ascontiguousarray(items, dtype=np.uint64)
    n = int(items.max()) + 1 if len(items) else 1
    K = max(k + 1, max((len(m._pos) for m in models if m._pos is not None and np.ndim(m._pos) == 2), default=1))
    descs, keep = descriptors(models, _per_state_len(models, n), K)
    out = np.zeros((len(s), 3))
    lib().azn_models_accel(C.cast(descs, C.c_void_p), len(descs), _p(s), _p(items), k, len(s), _p(out))
    del keep
    return out


def _per_state_len(models, default):
    for m in models:
        for v in m._coefs.values():
            if np.ndim(v) == 1:
                return len(v)
    return default


def propagate(states, t0, duration, dt, models, *, integrator="dp87", rtol=1e-9, atol=1e-12, k7_step_factor=False,
              threads=1):
    """Propagator.propagate of each row of states (n, 6) under the list: (times, traj[n, samples, 6], status[n],
    steps[n, 2]).  k7_step_factor forms errNorm^(-1/8) as K7 does (three square roots)."""
    states = np.ascontiguousarray(np.atleast_2d(states), dtype=np.float64)
    n = states.shape[0]
    t = N.times(t0, duration, dt)
    descs, keep = descriptors(models, n, len(t) - 1)
    out = np.zeros((n, len(t), 6))
    status = np.zeros(n, dtype=np.uint8)
    steps = np.zeros((n, 2), dtype=np.uint64)
    k = lib().azn_propagate_models(_p(states), n, float(t0), float(duration), float(dt), C.cast(descs, C.c_void_p),
                                   len(descs), {"rk4": 0, "dp87": 1}[integrator], float(rtol), float(atol),
                                   1 if k7_step_factor else 0, _p(out), _p(status), _p(steps), int(threads))
    del keep
    assert k == len(t)
    return t, out, status, steps
