"""K14 Monte Carlo collision probability for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

An independent numpy statement of the draws: Philox4x32-10 (Salmon et al., SC 2011) on uint64 arrays, the uniforms and
Box-Muller normals, the unit-diagonal semidefinite Cholesky by its textbook column recurrence, and x_k = x^ + D^1/2 L z.
restated(): each sample's drawn sets fed as element columns with P = 0 to the C restatement of K11
(tests/fit_oracle/conjunction.c), so the TCA and the miss of every sample come from the oracle's SGP4 / SDP4.
emul_library(), emul(): the host build of the device source (tests/host_emul/emul_conjunction_mc.cu)."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from tests.fit_oracle import conjunction as cj
from tests.fit_oracle.covariance import elements_of, unpack7

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)
PIVOT_ZERO = 1e-12
NOT_PSD, INIT_FAILED = 6, 1


# ---- the generator --------------------------------------------------------------------------------------------------
def philox(ctr, key):
    """ctr (n, 4), key (n, 2) uint32 -> (n, 4) uint32: ten rounds of Philox4x32"""
    c = [np.asarray(ctr, np.uint64)[:, q].copy() for q in range(4)]
    k0, k1 = (np.asarray(key, np.uint64)[:, q].copy() for q in range(2))
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(W0)) & MASK
            k1 = (k1 + np.uint64(W1)) & MASK
        p0, p1 = M0 * c[0], M1 * c[2]          # < 2^64: exact in uint64
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & MASK, p1 >> np.uint64(32), p1 & MASK
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, axis=1).astype(np.uint32)


def uniforms(a, b):
    u = (np.asarray(a, np.uint64) << np.uint64(21)) + (np.asarray(b, np.uint64) >> np.uint64(11))
    return (u.astype(np.float64) + 0.5) * 2.0 ** -53


def normals(seed, k):
    """(n, 14) normals of samples k (n,) under seed: block j of counter (j, k lo, k hi, 0), key (seed lo, seed hi)"""
    k = np.asarray(k, np.uint64).reshape(-1)
    n = len(k)
    key = np.tile(np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint64), (n, 1))
    out = np.empty((n, 14))
    for j in range(7):
        ctr = np.stack([np.full(n, j, np.uint64), k & MASK, k >> np.uint64(32), np.zeros(n, np.uint64)], axis=1)
        w = philox(ctr, key)
        u1, u2 = uniforms(w[:, 0], w[:, 1]), uniforms(w[:, 2], w[:, 3])
        r, t = np.sqrt(-2.0 * np.log(u1)), 2.0 * np.pi * u2
        out[:, 2 * j], out[:, 2 * j + 1] = r * np.cos(t), r * np.sin(t)
    return out


# ---- the factor and the draws ---------------------------------------------------------------------------------------
def nvar_of(P_words):
    return 7 if np.any(unpack7(P_words)[6] != 0.0) else 6


def factor(P_words):
    """(sd (7,), L (7, 7) lower, ok): S = D^-1/2 P D^-1/2 over nvar variables, the semidefinite Cholesky of S with
    pivots in [-1e-12, 1e-12] zeroing their column and one below -1e-12 (or a negative variance) not PSD"""
    P = unpack7(P_words)
    nv = nvar_of(P_words)
    d = np.where(np.arange(7) < nv, np.diag(P), 0.0)
    if (d < 0).any():
        return np.zeros(7), np.zeros((7, 7)), False
    sd = np.sqrt(d)
    live = sd > 0
    S = np.zeros((7, 7))
    ix = np.flatnonzero(live)
    S[np.ix_(ix, ix)] = P[np.ix_(ix, ix)] / np.outer(sd[ix], sd[ix])
    L = np.zeros((7, 7))
    for j in range(nv):
        if not live[j]:
            continue
        piv = S[j, j] - L[j, :j] @ L[j, :j]
        if piv < -PIVOT_ZERO:
            return sd, L, False
        if piv <= PIVOT_ZERO:
            continue
        L[j, j] = np.sqrt(piv)
        for a in range(j + 1, nv):
            if live[a]:
                L[a, j] = (S[a, j] - L[a, :j] @ L[j, :j]) / L[j, j]
    return sd, L, True


def vars_of(e, deep):
    e = np.asarray(e, dtype=np.float64)
    if not deep:
        wr = np.radians(e[5])
        return np.array([e[1], e[2] * np.cos(wr), e[2] * np.sin(wr), np.radians(e[3]), np.radians(e[4]),
                         np.radians(e[6]) + wr, e[7]])
    node, peri, ti = np.radians(e[4]), np.radians(e[5]) + np.radians(e[4]), np.tan(0.5 * np.radians(e[3]))
    return np.array([e[1], e[2] * np.cos(peri), e[2] * np.sin(peri), ti * np.cos(node), ti * np.sin(node),
                     np.radians(e[6]) + peri, e[7]])


def draws(e, deep, P_words, seed, o, k):
    """(n, 7) drawn variables of row o (element column e (8,)) for samples k, or None when the factor is not PSD"""
    sd, L, ok = factor(P_words)
    if not ok:
        return None
    z = normals(seed, k)[:, 7 * o:7 * o + 7]
    return vars_of(e, deep)[None, :] + (z @ L.T) * sd[None, :]


# ---- the per-sample restatement ---------------------------------------------------------------------------------------
def restated(el, P, model, p, s, jd, fr, w, samples, first=0, seed=0, threads=None):
    """(dt (samples,), miss (samples,), status (samples,)) of one candidate, each sample's drawn sets assessed by the
    C restatement with P = 0 (status 0 / 3 scored, 1 a set that cannot be built, 2 a failed cell)"""
    k = np.arange(first, first + samples, dtype=np.uint64)
    cols = []
    for o, row in enumerate((p, s)):
        x = draws(el[:, row], bool(model[row]), P[row], seed, o, k)
        cols.append(elements_of(x, el[0, row], bool(model[row])))
    sel = np.empty((8, 2 * samples))
    sel[:, 0::2], sel[:, 1::2] = cols[0], cols[1]
    md = np.repeat(np.asarray(model)[[p, s]][None], samples, axis=0).reshape(-1)
    pr, se = np.arange(0, 2 * samples, 2), np.arange(1, 2 * samples, 2)
    dt, st, _, status = cj.restated(sel, np.zeros((2 * samples, 28)), md, pr, se, jd, fr, np.full(samples, w),
                                    threads=threads)
    miss = np.linalg.norm(st[:, 1, :3] - st[:, 0, :3], axis=1)
    return dt, miss, status


# ---- the host build ---------------------------------------------------------------------------------------------------
def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_conjunction_mc.so")
    src = os.path.join(emul_dir, "emul_conjunction_mc.cu")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    L.emul_draw.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p,
                            C.c_int]
    L.emul_normals.argtypes = [C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p]
    return L


def emul_philox(L, ctr, key):
    ctr = np.ascontiguousarray(ctr, np.uint32)
    key = np.ascontiguousarray(key, np.uint32)
    out = np.zeros_like(ctr)
    L.emul_philox(_p(ctr), _p(key), C.c_uint32(len(ctr)), _p(out))
    return out


def emul_normals(L, seed, k):
    k = np.ascontiguousarray(k, np.uint64)
    z = np.zeros((len(k), 14))
    L.emul_normals(seed, _p(k), len(k), _p(z))
    return z


def emul_factor(L, P_words):
    P = np.ascontiguousarray(P_words, np.float64)
    sd, Lm = np.zeros(7), np.zeros((7, 7))
    ok = L.emul_factor(_p(P), _p(sd), _p(Lm))
    return sd, Lm, bool(ok)


def emul_draw(L, e, deep, P_words, seed, o, k, grav=1):
    e = np.ascontiguousarray(e, np.float64)
    P = np.ascontiguousarray(P_words, np.float64)
    k = np.ascontiguousarray(k, np.uint64)
    x = np.zeros((len(k), 7))
    st = L.emul_draw(_p(e), int(deep), _p(P), seed, o, _p(k), len(k), _p(x), grav)
    return x, st


def mc_inputs(elements, cov, model, primary, secondary, jd, fr, window, hbr, samples, first, seed):
    el, cv, md, pr, se, jd_, fr_, w_, r_ = cj._inputs(elements, cov, model, primary, secondary, jd, fr, window, hbr)
    m = len(pr)
    u64 = lambda a: None if a is None else np.ascontiguousarray(np.broadcast_to(np.asarray(a, np.uint64), (m,)))  # noqa
    return el, cv, md, pr, se, jd_, fr_, w_, r_, u64(samples), u64(first), u64(seed)


def emul(L, elements, cov, model, primary, secondary, jd, fr, window, hbr, samples, first=None, seed=None, record=0,
         grav=1):
    """the host build's (counts (m, 3) uint64, sample words (m, record, 2), status (m,))"""
    a = mc_inputs(elements, cov, model, primary, secondary, jd, fr, window, hbr, samples, first, seed)
    el = a[0]
    m = len(a[3])
    counts = np.zeros((m, 3), np.uint64)
    out = np.zeros((m, record, 2))
    status = np.zeros(m, np.uint8)
    L.emul_conjunction_mc(_p(el), C.c_uint32(el.shape[1]), grav, *[_p(x) for x in a[1:]], C.c_uint32(m),
                          C.c_uint32(record), _p(counts), _p(out), _p(status))
    return counts, out, status
