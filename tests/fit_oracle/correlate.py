"""K12 track correlation for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

emul(), emul_pair(), emul_fit_sums(): the host build of the device source (tests/host_emul/emul_correlate.cu).
restated_pair(): the independent C restatement of one pair on the oracle's SGP4 / SDP4 (correlate.c), on the stacked form.
base_rows(), track_of(): a small catalogue and oracle tracks of every kind; device_tracks(): many tracks from
propagate_pairs states, for the device tests and the timing tool."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import obs as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
EMPTY = 0xFFFFFFFF


def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_correlate.so")
    src = os.path.join(emul_dir, "emul_correlate.cu")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    L.emul_chi2_quantile.restype = C.c_double
    L.emul_chi2_quantile.argtypes = [C.c_uint32, C.c_double]
    L.emul_corr_pair.restype = C.c_double
    L.emul_corr_scratch_bytes.restype = C.c_size_t
    return L


def _restated_lib() -> C.CDLL:
    srcs = [os.path.join(_HERE, "correlate.c"), os.path.join(_HERE, "covariance.c"),
            os.path.join(_HERE, "fit_oracle_obs.c"), os.path.join(_ROOT, "oracle", "astroz_oracle.c"),
            os.path.join(_ROOT, "oracle", "astroz_oracle.h")]
    so = os.path.join(_HERE, "libcorrelate_ref.so")
    if not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(s) for s in srcs):
        subprocess.run(["gcc", "-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-Wall", "-Wno-unused-function",
                        "-shared", "-o", so, srcs[0], srcs[3], "-lm", "-lpthread"], check=True, capture_output=True)
    return C.CDLL(so)


class Tracks:
    """observations grouped by track: jd, fr, kind, value (m, 6), sigma (m, 6), station (m,), offsets (t + 1,)"""

    def __init__(self, per_track, stations):
        jd, fr, kind, value, sigma, station, offsets = O.concat(per_track)
        self.jd, self.fr = np.ascontiguousarray(jd, np.float64), np.ascontiguousarray(fr, np.float64)
        self.kind = np.ascontiguousarray(kind, np.uint8)
        self.value, self.sigma = np.ascontiguousarray(value, np.float64), np.ascontiguousarray(sigma, np.float64)
        self.station = np.ascontiguousarray(station, np.uint32)
        self.offsets = np.ascontiguousarray(offsets, np.uint32)
        self.stations = np.ascontiguousarray(stations, np.float64).reshape(-1, 3)
        self.t = len(self.offsets) - 1

    def track_ids(self):
        return np.repeat(np.arange(self.t), np.diff(self.offsets))

    def obs_args(self):
        return (_p(self.jd), _p(self.fr), _p(self.kind), _p(self.value), _p(self.sigma), _p(self.station),
                _p(self.stations))


def _cat(el, cov, model):
    el = np.ascontiguousarray(el, np.float64)
    cv = None if cov is None else np.ascontiguousarray(cov, np.float64).reshape(el.shape[1], 28)
    md = None if model is None else np.ascontiguousarray(model, np.uint8)
    return el, cv, md


def emul(L, el, cov, model, tr: Tracks, gate_probability=0.999, best=4, grav=1, full=False):
    """the host build's (rows (t, best), d2, used, n_gate, n_failed, status, row_status[, d2_all (t, n)])"""
    el, cv, md = _cat(el, cov, model)
    n, t = el.shape[1], tr.t
    rows, d2 = np.zeros((t, best), np.uint32), np.zeros((t, best))
    used, ng, nf = (np.zeros(t, np.uint32) for _ in range(3))
    status, rs = np.zeros(t, np.uint8), np.zeros(n, np.uint8)
    d2all = np.zeros((t, n)) if full else None
    L.emul_correlate(_p(el), C.c_uint32(n), grav, _p(cv), _p(md), _p(tr.offsets), C.c_uint32(t), *tr.obs_args(),
                     C.c_double(gate_probability), C.c_uint32(best), _p(rows), _p(d2), _p(used), _p(ng), _p(nf),
                     _p(status), _p(rs), _p(d2all))
    out = (rows, d2, used, ng, nf, status, rs)
    return out + (d2all,) if full else out


def emul_pair(L, el, cov, model, tr: Tracks, s, j, grav=1):
    """(z (L, 6), G (L, 7, 6), sums (43,), f0 (L, 6), d2 unclamped) of pair (track j, row s)"""
    el, cv, md = _cat(el, cov, model)
    b, e = int(tr.offsets[j]), int(tr.offsets[j + 1])
    z, G, sums, f0 = np.zeros((e - b, 6)), np.zeros((e - b, 7, 6)), np.zeros(43), np.zeros((e - b, 6))
    d2 = L.emul_corr_pair(_p(el), C.c_uint32(el.shape[1]), grav, _p(cv), _p(md), C.c_uint32(s), C.c_uint32(b),
                          C.c_uint32(e), *tr.obs_args(), _p(z), _p(G), _p(sums), _p(f0))
    return z, G, sums, f0, d2


def emul_fit_sums(L, el, cov, model, tr: Tracks, s, j, grav=1):
    el, cv, md = _cat(el, cov, model)
    b, e = int(tr.offsets[j]), int(tr.offsets[j + 1])
    sums = np.zeros(43)
    rc = L.emul_fit_obs_sums(_p(el), C.c_uint32(el.shape[1]), grav, _p(cv), _p(md), C.c_uint32(s), C.c_uint32(b),
                             C.c_uint32(e), *tr.obs_args(), _p(sums))
    return rc, sums


def restated_pair(el, cov, model, tr: Tracks, s, j, grav=1):
    """(rc, z (L, 6), G (L, 6, 7), d2) of the C restatement"""
    el, cv, md = _cat(el, cov, model)
    b, e = int(tr.offsets[j]), int(tr.offsets[j + 1])
    z, G, d2 = np.zeros((e - b, 6)), np.zeros((e - b, 6, 7)), C.c_double()
    rc = _restated_lib().corrref_pair(_p(el), C.c_uint32(el.shape[1]), grav, _p(cv), _p(md), C.c_uint32(s),
                                      C.c_uint32(b), C.c_uint32(e), *tr.obs_args(), _p(z), _p(G), C.byref(d2))
    return rc, z, G, d2.value


def restated_sweep(el, cov, model, tr: Tracks, grav=1, threads=None):
    """d2 (t, n) of every pair by the C restatement on `threads` pthreads (NaN: a row not built or a failed cell)"""
    el, cv, md = _cat(el, cov, model)
    d2 = np.zeros((tr.t, el.shape[1]))
    _restated_lib().corrref_sweep(_p(el), C.c_uint32(el.shape[1]), grav, _p(cv), _p(md), _p(tr.offsets),
                                  C.c_uint32(tr.t), *tr.obs_args(), int(threads or os.cpu_count() or 1), _p(d2))
    return d2


def subset(tr: Tracks, picks):
    """the tracks `picks` of tr, in that order"""
    return Tracks([tuple(a[tr.offsets[j]:tr.offsets[j + 1]] for a in (tr.jd, tr.fr, tr.kind, tr.value, tr.sigma,
                                                                       tr.station)) for j in picks], tr.stations)


def emul_threaded(L, el, cov, model, tr: Tracks, chunks=None, **kw):
    """emul over chunks of tracks on a thread pool (the host build holds no state between calls), concatenated"""
    from concurrent.futures import ThreadPoolExecutor

    chunks = chunks or os.cpu_count() or 1
    parts = [p for p in np.array_split(np.arange(tr.t), chunks) if len(p)]
    with ThreadPoolExecutor(len(parts)) as ex:
        outs = list(ex.map(lambda p: emul(L, el, cov, model, subset(tr, p), **kw), parts))
    return tuple(np.concatenate([o[q] for o in outs]) for q in range(6)) + (outs[0][6],)


def stacked(z, G, P, nvar=7):
    """the used rows of a pair stacked: (z (k,), G (k, 7)) from z (L, 6) and G (L, 7, 6)"""
    zs, gs = [], []
    for i in range(len(z)):
        for c in range(6):
            if z[i, c] != 0.0 or np.any(G[i, :, c] != 0.0):
                zs.append(z[i, c])
                gs.append(G[i, :, c])
    return np.array(zs), np.array(gs).reshape(-1, 7)


# ---- a small scene --------------------------------------------------------------------------------------------------
def base_rows():
    """(elements (8, 4), model (4,)): a LEO, a sun-synchronous LEO, a GEO and a Molniya orbit"""
    sso = cc.leo().copy()
    sso[1], sso[3], sso[4] = 14.3, 98.2, 30.0
    mol = cc.molniya_at_perigee().copy()
    mol[6] = 40.0
    return np.stack([cc.leo(), sso, cc.geo(), mol], axis=1), np.array([0, 0, 1, 1], np.uint8)


def track_of(el, kind, t0, minutes, step_s, sites=O.RADAR_SITES, sigma=None, rng=None, noise=True):
    """one track of set el: samples every step_s over `minutes` from t0 (JD), the kind's sites above 10 deg elevation
    (first site that sees it), Gaussian noise at the kind's sigma"""
    k = np.arange(0.0, minutes * 60.0 + 1e-9, step_s) / 86400.0
    jd = np.full(len(k), np.floor(t0 - 0.5) + 0.5)
    fr = (t0 - jd) + k
    if kind in (O.TEME, O.ECEF):
        out = O.tracks(el, kind, sites, jd, fr, sigma=sigma)
    else:
        out = None
        for q, site in enumerate(sites):
            cand = O.tracks(el, kind, site[None], jd, fr, sigma=sigma)
            if len(cand[0]):
                out = cand[:5] + (np.full(len(cand[0]), q, np.uint32),)
                break
        if out is None:
            return None
    jd_, fr_, kd, val, sg, st = out
    val = val.copy()
    if noise:
        rng = rng or np.random.default_rng(0)
        fin = np.isfinite(sg)
        val[fin] += rng.standard_normal(fin.sum()) * sg[fin]
        if kind == O.RADAR:
            val[:, 1] %= 2 * np.pi
        if kind == O.OPTICAL:
            val[:, 0] %= 2 * np.pi
    return jd_, fr_, kd, val, sg, st


def device_tracks(el, rows, kind, L, step_s, seed, start=0.0, span=1.0):
    """Tracks of L observations of each of `rows`, starting at a uniform time in [epoch + start, epoch + start + span)
    days, one random station each, from propagate_pairs states (the device
    model) through the numpy statement of the kinds, with noise at the kind's sigma; geometric, so visibility is not
    modelled.  Returns (track ids (m,), jd, fr, kind, value (m, 6), sigma (m, 6), station)."""
    from astroz_b200.constellation import Constellation

    rng = np.random.default_rng(seed)
    t = len(rows)
    sat = np.repeat(rows, L)
    t0 = el[0][rows] + start + rng.uniform(0.0, span, t)
    jd = np.repeat(np.floor(t0 - 0.5) + 0.5, L)
    fr = np.repeat(t0, L) - jd + np.tile(np.arange(L) * step_s / 86400.0, t)
    c = Constellation.from_elements(*el)
    p, v, _ = c.propagate_pairs(sat, jd, fr)
    c.deinit()
    states = np.concatenate([np.asarray(p), np.asarray(v)], axis=1)
    station = np.repeat(rng.integers(0, len(O.RADAR_SITES), t), L).astype(np.uint32)
    value = np.zeros((len(sat), 6))
    for q in range(len(O.RADAR_SITES)):
        sel = station == q
        value[sel] = O.observe(kind, states[sel], jd[sel] + fr[sel], O.RADAR_SITES[q])
    sig = O.RADAR_SIGMA if kind == O.RADAR else O.OPTICAL_SIGMA
    sigma = np.full((len(sat), 6), np.inf)
    sigma[:, :len(sig)] = sig
    value[:, :len(sig)] += rng.standard_normal((len(sat), len(sig))) * sig
    return np.repeat(np.arange(t), L), jd, fr, np.full(len(sat), kind, np.uint8), value, sigma, station
