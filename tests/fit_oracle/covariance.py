"""K10 state covariance for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

restated(): the independent C restatement (covariance.c, on the oracle's SGP4 / SDP4, gcc -ffp-contract=off).
emul(): the host build of the device source (tests/host_emul/emul_covariance.cu) with a chosen chunk.
elements_of(): a numpy statement of the fit's variables -> element columns map, near-earth and equinoctial."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731


def _restated_lib() -> C.CDLL:
    srcs = [os.path.join(_HERE, "covariance.c"), os.path.join(_HERE, "fit_oracle_obs.c"),
            os.path.join(_ROOT, "oracle", "astroz_oracle.c"), os.path.join(_ROOT, "oracle", "astroz_oracle.h")]
    so = os.path.join(_HERE, "libcovariance_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(s) for s in srcs):
        subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-Wno-unused-function",
                        "-shared", "-o", so, srcs[0], srcs[2], "-lm", "-lpthread"], check=True, capture_output=True)
    return C.CDLL(so)


def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_covariance.so")
    src = os.path.join(emul_dir, "emul_covariance.cu")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    L.emul_cov_chunk.restype = C.c_uint32
    L.emul_cov_chunk.argtypes = [C.c_uint32]
    return L


def _inputs(elements, cov, model, offsets, jd, fr):
    el = np.ascontiguousarray(elements, dtype=np.float64)
    cv = np.ascontiguousarray(cov, dtype=np.float64).reshape(el.shape[1], 28)
    md = None if model is None else np.ascontiguousarray(model, dtype=np.uint8)
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    return el, cv, md, off, np.ascontiguousarray(jd, dtype=np.float64), np.ascontiguousarray(fr, dtype=np.float64)


def _outputs(m):
    return np.zeros((m, 6)), np.zeros((m, 21)), np.zeros((m, 6, 7)), np.zeros(m, dtype=np.uint8)


def restated(elements, cov, model, offsets, jd, fr, frame=0, grav=1, threads=None):
    """(state (m, 6), Sigma words (m, 21), J (m, 6, 7), status (m,)) of the C restatement"""
    el, cv, md, off, jd_, fr_ = _inputs(elements, cov, model, offsets, jd, fr)
    st, sig, jac, status = _outputs(len(jd_))
    _restated_lib().covref_propagate(_p(el), C.c_uint32(el.shape[1]), grav, _p(cv), _p(md), _p(off), _p(jd_),
                                     _p(fr_), int(frame), int(threads or os.cpu_count() or 1), _p(st), _p(sig),
                                     _p(jac), _p(status))
    return st, sig, jac, status


def emul(L, elements, cov, model, offsets, jd, fr, frame=0, grav=1, chunk=None):
    """the host build's (state, Sigma words, J, status); chunk None = the library's cov_chunk(m)"""
    el, cv, md, off, jd_, fr_ = _inputs(elements, cov, model, offsets, jd, fr)
    st, sig, jac, status = _outputs(len(jd_))
    m = len(jd_)
    L.emul_propagate_covariance(_p(el), C.c_uint32(el.shape[1]), grav, _p(cv), _p(md), _p(off), _p(jd_), _p(fr_),
                                C.c_uint32(m), int(frame), C.c_uint32(chunk or L.emul_cov_chunk(m)), _p(st), _p(sig),
                                _p(jac), _p(status))
    return st, sig, jac, status


TRIU6 = np.triu_indices(6)
TRIU7 = np.triu_indices(7)


def unpack6(words):
    """(..., 21) upper-triangle words -> (..., 6, 6)"""
    words = np.asarray(words)
    S = np.zeros(words.shape[:-1] + (6, 6))
    S[..., TRIU6[0], TRIU6[1]] = words
    S[..., TRIU6[1], TRIU6[0]] = words
    return S


def pack7(P):
    """(7, 7) -> 28 words"""
    return np.asarray(P)[TRIU7]


def unpack7(words):
    P = np.zeros((7, 7))
    P[TRIU7] = words
    return P + np.triu(P, 1).T


def rtn(state):
    """(m, 3, 3) rows R, T, N of TEME states (m, 6)"""
    r, v = state[:, :3], state[:, 3:]
    R = r / np.linalg.norm(r, axis=1)[:, None]
    h = np.cross(r, v)
    N = h / np.linalg.norm(h, axis=1)[:, None]
    return np.stack([R, np.cross(N, R), N], axis=1)


def elements_of(x, epoch, deep):
    """the fit's variables x (..., 7) -> element columns (8, ...): near-earth or equinoctial, node / w / M in [0, 360)"""
    x = np.asarray(x, dtype=np.float64)
    r2d = 180.0 / np.pi
    out = np.zeros((8,) + x.shape[:-1])
    out[0] = epoch
    out[1] = x[..., 0]
    out[2] = np.hypot(x[..., 1], x[..., 2])
    P = np.arctan2(x[..., 2], x[..., 1])
    if not deep:
        out[3] = x[..., 3] * r2d
        out[4] = np.mod(x[..., 4] * r2d, 360.0)
        out[5] = np.mod(P * r2d, 360.0)
    else:
        node = np.arctan2(x[..., 4], x[..., 3])
        out[3] = 2.0 * np.arctan(np.hypot(x[..., 3], x[..., 4])) * r2d
        out[4] = np.mod(node * r2d, 360.0)
        out[5] = np.mod((P - node) * r2d, 360.0)
    out[6] = np.mod((x[..., 5] - P) * r2d, 360.0)
    out[7] = x[..., 6]
    return out
