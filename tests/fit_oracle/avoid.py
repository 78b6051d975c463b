"""K16 manoeuvre trials for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

transport(): an independent numpy statement of the covariance through the burn: A from J and J' (numpy's solve), P' =
    A P A^T plus the execution term, the held-B* and zero-burn rules.
cw(): the Clohessy-Wiltshire displacement of a tangential burn.
emul_library(), emul(): the host build of the device source (tests/host_emul/emul_avoid.cu, linked with the host builds
    of K10, K8 and K11)."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from tests.fit_oracle import covariance as K

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731

OK, INIT_FAILED, CELL_FAILED, WINDOW_EDGE, NO_PLANE, BAD_PAIR = 0, 1, 2, 3, 4, 5
CONVERSION_FAILED, BAD_TRIAL = 7, 8


def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_avoid.so")
    srcs = [os.path.join(emul_dir, f) for f in ("emul_avoid.cu", "emul_fit.cu", "emul_fit_deep.cu",
                                                "emul_covariance.cu", "emul_conjunction.cu")]
    deps = srcs + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, *srcs], check=True,
                       capture_output=True)
    L = C.CDLL(so)
    L.emul_avoid_scratch_bytes.restype = C.c_uint64
    L.emul_avoid_scratch_bytes.argtypes = [C.c_uint32]
    return L


def emul(L, elements, cov, model, primary, secondary, jd, fr, window, hbr, candidate, burn_jd, burn_fr, dv,
         dv_sigma=None, grav=1):
    """the host build's (record (t, 13), elements (t, 8), covariance (t, 28), residual (t, 2), status (t,))"""
    el = np.ascontiguousarray(elements, dtype=np.float64)
    n = el.shape[1]
    cv = np.ascontiguousarray(cov, dtype=np.float64).reshape(n, 28)
    md = None if model is None else np.ascontiguousarray(model, dtype=np.uint8)
    pr = np.ascontiguousarray(primary, dtype=np.uint32).reshape(-1)
    m = len(pr)
    f64m = lambda a: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (m,)))  # noqa: E731
    se = np.ascontiguousarray(secondary, dtype=np.uint32).reshape(-1)
    ca = np.ascontiguousarray(candidate, dtype=np.uint32).reshape(-1)
    t = len(ca)
    f64t = lambda a: np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (t,)))  # noqa: E731
    d = np.ascontiguousarray(np.broadcast_to(np.asarray(dv, dtype=np.float64), (t, 3)))
    sg = None if dv_sigma is None else np.ascontiguousarray(np.broadcast_to(np.asarray(dv_sigma, np.float64), (t, 3)))
    rec, ne, nc = np.zeros((t, 13)), np.zeros((t, 8)), np.zeros((t, 28))
    res, st = np.zeros((t, 2)), np.zeros(t, np.uint8)
    args = [f64m(jd), f64m(fr), f64m(window), f64m(hbr)]
    bj, bf = f64t(burn_jd), f64t(burn_fr)   # held until the call returns
    L.emul_avoid(_p(el), C.c_uint32(n), grav, _p(cv), _p(md), _p(pr), _p(se), *[_p(a) for a in args], C.c_uint32(m),
                 _p(ca), _p(bj), _p(bf), _p(d), _p(sg), C.c_uint32(t), _p(rec), _p(ne), _p(nc), _p(res), _p(st))
    return rec, ne, nc, res, st


def emul_transport(L, J, Jp, P, x, sigma, zero):
    """the host build's P' words (28,), or None when J'6 is singular"""
    arr = [np.ascontiguousarray(a, np.float64) for a in (J, Jp, P, x)]
    sg = None if sigma is None else np.ascontiguousarray(sigma, np.float64)
    out = np.zeros(28)
    rc = L.emul_avoid_covariance(*[_p(a) for a in arr], _p(sg), int(bool(zero)), _p(out))
    return None if rc else out


def rtn(x):
    """(3, 3) rows R, T, N of TEME state x (6,)"""
    return K.rtn(np.asarray(x, np.float64)[None])[0]


def transport(J, Jp, P, x, sigma=None, zero=False):
    """numpy statement of P' (7, 7) from J, J' (6, 7), P (7, 7), the pre-burn state x and sigma (3,) or None"""
    A = np.eye(7)
    if not zero:
        B = J.copy()
        B[:, 6] -= Jp[:, 6]
        A[:6] = np.linalg.solve(Jp[:, :6], B)
    Pn = A @ P @ A.T
    if sigma is not None and np.any(np.asarray(sigma) != 0):
        R = rtn(x)
        Q = np.zeros((6, 6))
        Q[3:, 3:] = R.T @ np.diag(np.asarray(sigma, np.float64) ** 2) @ R
        Ji = np.linalg.inv(Jp[:, :6])
        Pn[:6, :6] += Ji @ Q @ Ji.T
    return Pn


def cw(dv_t, n, t):
    """Clohessy-Wiltshire (radial, along-track) displacement [km] at t [s] after a tangential burn dv_t [km/s] on a
    circular orbit of mean motion n [rad/s]"""
    return (2.0 / n) * dv_t * (1.0 - np.cos(n * t)), (4.0 / n) * dv_t * np.sin(n * t) - 3.0 * dv_t * t
