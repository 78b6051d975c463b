"""K15 importance-sampled collision probability for the tests -- TEST INFRASTRUCTURE ONLY; the product package never
imports it.

An independent numpy statement of the proposal and the weights: the plane and in-plane miss from K11's states, J from
the C restatement of K10 (tests/fit_oracle/covariance.c) at K11's TCA, the factor of tests/fit_oracle/conjunction_mc.py,
G, the pseudo-inverse by numpy's eigh and c = -G^T C+ d; log w = -u . c - |c|^2 / 2 on the numpy Philox normals; the
256-bit sums as Python integers.
emul_library(), emul(): the host build of the device source (tests/host_emul/emul_conjunction_is.cu), with K11's
nominal assessment from K11's host build."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np

from tests.fit_oracle import conjunction as cj
from tests.fit_oracle import conjunction_mc as mc
from tests.fit_oracle import covariance as K

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731

LINEAR, GIVEN, PLAIN = 0, 1, 2
EIGEN_ZERO = 1e-14
V_MAX = 2.0 ** 31


# ---- the proposal ----------------------------------------------------------------------------------------------------
def plane(states):
    """(E (2, 3) rows x, y, d (2,)) of K11's TEME states (2, 6) at the TCA"""
    dr, dv = states[1, :3] - states[0, :3], states[1, 3:] - states[0, 3:]
    z = dv / np.linalg.norm(dv)
    x = dr - (dr @ z) * z
    x = x / np.linalg.norm(x)
    E = np.stack([x, np.cross(z, x)])
    return E, E @ dr


def jacobians(el, P, model, p, s, jd, fr, dt):
    """(J_p, J_s) (6, 7) TEME Jacobians of the C restatement at jd + fr + dt / 1440, and their statuses"""
    rows = [p, s]
    J, st = [], []
    for r in rows:
        off = np.array([0, 1], np.uint32)
        _, _, jac, status = K.restated(el[:, r:r + 1], P[r][None], None if model is None else model[r:r + 1], off,
                                       np.array([jd]), np.array([fr + dt / 1440.0]))
        J.append(jac[0])
        st.append(status[0])
    return J, st


def linear_shift(el, P, model, p, s, jd, fr, dt, states):
    """(c (14,), G (2, 14), d (2,), C (2, 2)) of the linear proposal, or None for PLAIN"""
    E, d = plane(states)
    J, st = jacobians(el, P, model, p, s, jd, fr, dt)
    if any(st):
        return None
    G = np.zeros((2, 14))
    for o, r in enumerate((p, s)):
        sd, L, ok = mc.factor(P[r])
        if not ok:
            return None
        G[:, 7 * o:7 * o + 7] = (-1.0 if o == 0 else 1.0) * (E @ J[o][:3]) @ (sd[:, None] * L)
    Cm = G @ G.T
    tr = np.trace(Cm)
    if not tr > 0:
        return None
    lam, U = np.linalg.eigh(Cm)
    inv = np.where(lam > EIGEN_ZERO * tr, 1.0 / np.where(lam > 0, lam, 1.0), 0.0)
    Cp = (U * inv) @ U.T
    return -G.T @ (Cp @ d), G, d, Cm


def log_weights(seed, k, c):
    """log w of samples k (n,) under seed with shift c (14,): -u . c - |c|^2 / 2 on the numpy normals"""
    u = mc.normals(seed, k)
    return -(u[:, :7] @ c[:7] + u[:, 7:] @ c[7:]) - 0.5 * (c @ c)


def fixed(x) -> int:
    """the nearest integer to x 2^128, ties to even (Python's round of a Fraction)"""
    return round(Fraction(float(x)) * 2 ** 128)


def words(total: int) -> np.ndarray:
    return np.array([(total >> (64 * q)) & (2 ** 64 - 1) for q in range(4)], np.uint64)


def sums(v):
    """(V, V2, overflow) of the hits' weight factors v as the 256-bit words and the overflow count"""
    V = V2 = ov = 0
    for x in v:
        if not x < V_MAX:
            ov += 1
            continue
        V += fixed(x)
        V2 += fixed(float(x) * float(x))
    return words(V), words(V2), ov


# ---- the host build ---------------------------------------------------------------------------------------------------
def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_conjunction_is.so")
    src = os.path.join(emul_dir, "emul_conjunction_is.cu")
    deps = [src, os.path.join(emul_dir, "emul_conjunction_mc.cu")] + \
        [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    L.emul_normals.argtypes = [C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p]
    return L


def emul(L, elements, cov, model, primary, secondary, jd, fr, window, hbr, samples, first=None, seed=None, shift=None,
         record=0, grav=1):
    """the host build's dict: counts (m, 12) uint64, proposal (m, 15), kind (m,), out (m, record, 3), status (m,),
    G (m, 2, 14), v (m, record), and K11's record and states of the nominal pairs"""
    a = mc.mc_inputs(elements, cov, model, primary, secondary, jd, fr, window, hbr, samples, first, seed)
    el = a[0]
    m = len(a[3])
    rec, st, _, k11 = cj.emul(cj.emul_library(), el, a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8])
    sh = None if shift is None else np.ascontiguousarray(np.broadcast_to(np.asarray(shift, np.float64), (m, 14)))
    r = dict(counts=np.zeros((m, 12), np.uint64), proposal=np.zeros((m, 15)), kind=np.zeros(m, np.uint8),
             out=np.zeros((m, record, 3)), status=np.zeros(m, np.uint8), G=np.zeros((m, 2, 14)),
             v=np.zeros((m, record)), record=rec, states=st, k11=k11)
    L.emul_conjunction_is(_p(el), C.c_uint32(el.shape[1]), grav, *[_p(x) for x in a[1:]], _p(sh), _p(rec),
                          _p(np.ascontiguousarray(st)), _p(k11), C.c_uint32(m), C.c_uint32(record), _p(r["counts"]),
                          _p(r["proposal"]), _p(r["kind"]), _p(r["out"]), _p(r["status"]), _p(r["G"]), _p(r["v"]))
    return r


# ---- engineered cases -------------------------------------------------------------------------------------------------
def leo_at_pc(assess, target):
    """(elements (8, 2), P words (2, 28), hbr): conjunction_cases' LEO crossing at di = 40 deg (miss d ~ 3.9 km), radius
    R = d / 10, both covariances scaled (by bisection on the Mahalanobis distance k of the nominal miss under K11's C2,
    over [1, 10], where Pc falls with k) until K11's Pc is `target`.  assess(el, P, hbr) returns the record of candidate
    (0, 1) over +-1 min from the first set's epoch."""
    from tests.fit_oracle import conjunction_cases as cc

    el = cc.pair(cc.leo(), 40.0, dnode=0.0005)
    P0 = cc.P_words(2, scale=1.0, bstar=False)
    rec = assess(el, P0, 0.01)
    d, (xx, xy, yy) = rec[1], rec[9:12]
    k0 = d * np.sqrt(yy / (xx * yy - xy * xy))   # the miss lies along x
    R = d / 10.0
    lo, hi = 1.0, 10.0
    for _ in range(50):
        mid = 0.5 * (lo + hi)
        if assess(el, P0 * (k0 / mid) ** 2, R)[12] > target:
            lo = mid
        else:
            hi = mid
    return el, P0 * (k0 / lo) ** 2, R


def emul_assess(el, P, hbr, model=None, w=1.0):
    """K11's host-build record of candidate (0, 1) over +-w min from the first set's epoch"""
    jd = np.floor(el[0, 0] - 0.5) + 0.5
    md = np.zeros(2, np.uint8) if model is None else model
    return cj.emul(cj.emul_library(), el, P, md, [0], [1], jd, el[0, 0] - jd, w, hbr)[0][0]
