"""K17 track linking for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

emul_library(), emul(), emul_hypotheses(), emul_anchor(): the host build of the device source
(tests/host_emul/emul_link.cu, linked with the host emulation of the mixed element fit).  The rest is an independent
numpy restatement written from the definition in az_link.cuh, not from the device source: the range bounds as numpy
polynomial roots, the hypotheses' Lambert transfers by K9's scalar C statement (tests/lambert_oracle), their two-body
propagation by Kepler's equation (tests.fit_oracle.iod.kepler) and the probe residuals by the numpy observation model
(tests.fit_oracle.obs.observe); and the exact two-body optical and radar tracks the CPU tests link."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from tests.fit_oracle import correlate as cr
from tests.fit_oracle import iod as I
from tests.fit_oracle import obs as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
RANGES, SEEDS = 32, 4
OK, TOO_FEW, NO_CANDIDATE, CONVERSION_FAILED, BAD_TRACK, BAD_PAIR = 0, 1, 2, 3, 4, 5
RETROGRADE, RIGHT_BRANCH = 1, 2


def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_link.so")
    srcs = [os.path.join(emul_dir, f) for f in ("emul_link.cu", "emul_fit.cu", "emul_fit_deep.cu")]
    deps = srcs + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, *srcs], check=True,
                       capture_output=True)
    L = C.CDLL(so)
    L.emul_link_range.restype = C.c_double
    L.emul_link_range.argtypes = [C.c_double, C.c_double, C.c_uint32, C.c_uint32]
    return L


def emul(L, tr, pairs, r_min, r_max, max_revs=1, bstar=None, grav=1):
    """the host build's outputs over the grouped, time-ordered tracks tr (tests.fit_oracle.correlate.Tracks): a dict of
    elements (8, p), state (p, 6), rho (p, 2), revs, flags, wrms, used, hypotheses, conv (p, 2), deep, status, and the
    seeds seed_F / seed_key (p, SEEDS), and converged (p,): the winner's refinement ended on its step tolerance"""
    pairs = np.ascontiguousarray(np.asarray(pairs, np.uint32).reshape(-1, 2))
    p = len(pairs)
    o = dict(elements=np.zeros((8, p)), state=np.zeros((p, 6)), rho=np.zeros((p, 2)), revs=np.zeros(p, np.uint8),
             flags=np.zeros(p, np.uint8), wrms=np.zeros(p), used=np.zeros(p, np.uint32),
             hypotheses=np.zeros(p, np.uint32), conv=np.zeros((p, 2)), deep=np.zeros(p, np.uint8),
             status=np.zeros(p, np.uint8), seed_F=np.zeros((p, SEEDS)), seed_key=np.zeros((p, SEEDS), np.uint32),
             converged=np.zeros(p, np.uint8))
    bs = None if bstar is None else np.ascontiguousarray(np.broadcast_to(bstar, (p,)), np.float64)
    L.emul_link(_p(tr.offsets), C.c_uint32(tr.t), *tr.obs_args(), _p(pairs), C.c_uint32(p), _p(bs),
                C.c_double(r_min), C.c_double(r_max), C.c_uint32(max_revs), grav,
                *[_p(o[k]) for k in ("elements", "state", "rho", "revs", "flags", "wrms", "used", "hypotheses", "conv",
                                     "deep", "status", "seed_F", "seed_key", "converged")])
    return o


def emul_anchor(L, tr, j, r_min, r_max):
    """(index, t, R, L, lo, hi, n) of track j's anchor, or None"""
    out = np.zeros(11)
    if not L.emul_link_anchor(C.c_uint32(tr.offsets[j]), C.c_uint32(tr.offsets[j + 1]), *tr.obs_args(),
                              C.c_double(r_min), C.c_double(r_max), _p(out)):
        return None
    return int(out[0]), out[1], out[2:5], out[5:8], out[8], out[9], int(out[10])


def emul_hypotheses(L, tr, a, b, r_min, r_max, max_revs=1, grav=1, cap=200000):
    """(keys, F_probe, epoch states (k, 6), probe observation indices) of every admissible state of pair (a, b), or the
    pair's status when it is not OK"""
    keys, F, states = np.zeros(cap, np.uint32), np.zeros(cap), np.zeros((cap, 6))
    probes, n_probe = np.zeros(6, np.uint32), C.c_int()
    n = L.emul_link_hypotheses(_p(tr.offsets), C.c_uint32(tr.t), *tr.obs_args(), C.c_uint32(a), C.c_uint32(b),
                               C.c_double(r_min), C.c_double(r_max), C.c_uint32(max_revs), grav, C.c_uint32(cap),
                               _p(keys), _p(F), _p(states), _p(probes), C.byref(n_probe))
    if n < 0:
        return -1 - n
    return keys[:n], F[:n], states[:n], probes[:n_probe.value]


# ---- the restatement -------------------------------------------------------------------------------------------------
def range_roots(R, L, r):
    """the positive root of |R + rho L| = r, by numpy's polynomial roots"""
    rts = np.roots([1.0, 2.0 * (R @ L), R @ R - r * r])
    return float(np.max(rts.real))


def key(M, retro, right, i1, i2):
    return M << 18 | retro << 17 | right << 16 | i1 << 8 | i2


def residuals(tr, i, s, t_ref, mu):
    """the weighted residuals (6,) of observation i of tr for the state s at jdFull t_ref, two-body (restated)"""
    jdf = tr.jd[i] + tr.fr[i]
    st = I.kepler(s, (jdf - t_ref) * 86400.0, mu)
    kind = int(tr.kind[i])
    llh = tr.stations[tr.station[i]] if kind >= O.RADAR else None
    h = O.observe(kind, st[None], np.array([jdf]), llh)[0]
    v, sg = tr.value[i], tr.sigma[i]
    count = {O.TEME: 6, O.ECEF: 6, O.RADAR: 4, O.OPTICAL: 2}[kind]
    wrapped = {O.RADAR: 1, O.OPTICAL: 0}.get(kind, -1)
    partner = {O.RADAR: 2, O.OPTICAL: 1}.get(kind, -1)
    r = np.zeros(6)
    for c in range(count):
        if not np.isfinite(sg[c]):
            continue
        d = v[c] - h[c]
        w = 1.0 / sg[c]
        if c == wrapped:
            d = (d + np.pi) % (2 * np.pi) - np.pi
            w *= np.cos(v[partner])
        r[c] = d * w
    return r


def restated_hypotheses(tr, a, b, r_min, r_max, anchors, max_revs=1, grav=1):
    """{key: F_probe} of every admissible state of pair (a, b), restated.  anchors[j] = (index, R, L, known range or
    None) of the host build's anchor geometry; the range grid, the transfers, the admissibility and the probe scores are
    the restatement's."""
    from tests import lambert_oracle as K9

    mu, rE = I.MU[grav], I.RE[grav]
    t = {j: tr.jd[anchors[j][0]] + tr.fr[anchors[j][0]] for j in (a, b)}
    one, two = (a, b) if t[a] < t[b] else (b, a)
    grids = []
    for j in (one, two):
        _, R, Lv, known = anchors[j]
        if known is not None:
            grids.append(np.array([known]))
        else:
            lo, hi = range_roots(R, Lv, r_min), range_roots(R, Lv, r_max)
            g = lo * (hi / lo) ** (np.arange(RANGES) / (RANGES - 1))
            g[0], g[-1] = lo, hi
            grids.append(g)
    probes = []
    for j in (one, two):
        b0, e0 = int(tr.offsets[j]), int(tr.offsets[j + 1])
        for i in (b0, anchors[j][0], e0 - 1):
            if i not in probes:
                probes.append(i)
    t_ref = t[two]
    tof = (t[two] - t[one]) * 86400.0
    out = {}
    for i1, x1 in enumerate(grids[0]):
        for i2, x2 in enumerate(grids[1]):
            r1 = anchors[one][1] + x1 * anchors[one][2]
            r2 = anchors[two][1] + x2 * anchors[two][2]
            for retro, nz in ((0, 1.0), (1, -1.0)):
                _, v2, st, _ = K9.solve(r1[None], r2[None], np.array([tof]), mu, max_revs=max_revs,
                                        normal=np.array([[0.0, 0.0, nz]]))
                for slot in range(2 * max_revs + 1):
                    if st[0, slot] != 0:
                        continue
                    s = np.concatenate([r2, v2[0, slot]])
                    if not I.admissible(s, mu, rE):
                        continue
                    M = (slot + 1) // 2
                    F = sum(float(np.sum(residuals(tr, i, s, t_ref, mu) ** 2)) for i in probes)
                    out[key(M, retro, int(M > 0 and slot % 2 == 0), i1, i2)] = F
    return out


# ---- exact two-body tracks -------------------------------------------------------------------------------------------
def two_body_track(s0, t0_jd, kind, site, seconds, t_state=None, grav=1, jd0=2460000.5):
    """one noise-free track of the exact two-body orbit s0 (TEME state at jdFull t_state, default t0_jd) observed from
    site (lat, lon, h) at t0_jd + seconds: (per-track tuple for correlate.Tracks with station 0, true states (k, 6))"""
    mu = I.MU[grav]
    t_state = t0_jd if t_state is None else t_state
    fr = (t0_jd - jd0) + np.asarray(seconds, float) / 86400.0
    jd = np.full(len(fr), jd0)
    S = np.array([I.kepler(s0, (jd0 + f - t_state) * 86400.0, mu) for f in fr])
    val = O.observe(kind, S, jd + fr, site)
    sig = np.full((len(fr), 6), np.inf)
    sg = O.RADAR_SIGMA if kind == O.RADAR else O.OPTICAL_SIGMA if kind == O.OPTICAL else np.array([1e-3] * 3)
    sig[:, :len(sg)] = sg
    return (jd, fr, np.full(len(fr), kind, np.uint8), val, sig, np.zeros(len(fr), np.uint32)), S


def tracks_with_sites(per, sites):
    """correlate.Tracks of per-track tuples each observed from its own site: station q of tuple q"""
    per = [tuple(x if k < 5 else np.full(len(x), q, np.uint32) for k, x in enumerate(tp)) for q, tp in enumerate(per)]
    return cr.Tracks(per, np.asarray(sites, float).reshape(-1, 3))


# ---- workloads of the device tests and the timing tool ---------------------------------------------------------------
def closed_loop_tracks(n_objects, n_distractors, seed, nights=(1.0, 2.0)):
    """Optical tracks in K13's failing shape (12 observations at 300 s, 55 min) of deep-space objects outside the
    catalogue (the synthetic catalogue's rows with the mean anomaly moved by 0.5 deg), one per night in `nights` (days
    after the row's epoch, starting up to 0.3 days later), from the oracle's SDP4 with 1" noise, plus single tracks of
    other deep-space objects.  Returns (tracks, owner object per track (t,), the objects' true element columns (8, k),
    the owner's column of each track)."""
    from astroz_b200 import synth

    truth = synth.elements_from_tles(synth.mixed_catalog(4000, n_geo=400, n_molniya=100, n_gps=100))
    deep = np.flatnonzero(1440.0 / truth[1] > 225.0)
    rng = np.random.default_rng(seed)
    rows = rng.choice(deep, n_objects + n_distractors, replace=False)
    per, owner = [], []
    for q, s in enumerate(rows):
        el = truth[:, s].copy()
        el[6] = (el[6] + 0.5) % 360.0
        for night in (nights if q < n_objects else nights[:1]):
            for _ in range(20):
                trk = cr.track_of(el, O.OPTICAL, truth[0, s] + night + rng.uniform(0.0, 0.3), 55, 300.0, rng=rng)
                if trk is not None and len(trk[0]) == 12:
                    per.append(trk)
                    owner.append(q)
                    break
    el_true = truth[:, rows].copy()
    el_true[6] = (el_true[6] + 0.5) % 360.0
    return cr.Tracks(per, O.RADAR_SITES), np.array(owner), el_true


def mixed_pairs_tracks(seed):
    """Tracks of a mixed scene for the device-against-host comparison: pairs of optical tracks of GEO, GPS and Molniya
    objects on consecutive nights, radar tracks of LEO objects on two passes, TEME position tracks, and a radar track
    followed by an optical one of GPS objects; every pair of them within 1.5 days is a test pair"""
    from astroz_b200 import synth

    truth = synth.elements_from_tles(synth.mixed_catalog(600, n_geo=48, n_molniya=8, n_gps=8))
    deep = np.flatnonzero(1440.0 / truth[1] > 225.0)
    near = np.setdiff1d(np.arange(truth.shape[1]), deep)
    rng = np.random.default_rng(seed)
    per = []

    def add(el, kind, t0, minutes, step):
        trk = cr.track_of(el, kind, t0, minutes, step, rng=rng)
        if trk is not None and len(trk[0]) >= 3:
            per.append(trk)

    for s in rng.choice(deep, 34, replace=False):
        for night in (0.0, 1.0):
            add(truth[:, s], O.OPTICAL, truth[0, s] + night + rng.uniform(0.0, 0.3), 55, 300.0)
    for s in rng.choice(near, 16, replace=False):
        for k in range(2):
            add(truth[:, s], O.RADAR, truth[0, s] + 0.05 * k + rng.uniform(0.0, 0.01), 8, 30.0)
    for s in rng.choice(near, 8, replace=False):
        add(truth[:, s], O.TEME, truth[0, s] + rng.uniform(0.0, 0.5), 3, 60.0)
    for s in rng.choice(deep, 8, replace=False):
        add(truth[:, s], O.RADAR, truth[0, s] + 0.2, 10, 60.0)
        add(truth[:, s], O.OPTICAL, truth[0, s] + 0.4, 55, 300.0)
    return cr.Tracks(per, O.RADAR_SITES)


def geo_tracks(n_objects, seed):
    """2 n_objects optical tracks (12 at 300 s) of GEO rows of a synthetic catalogue, one in each of the two days
    after the row's epoch (starting up to 0.3 days in), from propagate_pairs states with 1" noise (cr.device_tracks:
    geometric, visibility not modelled)"""
    from astroz_b200 import synth

    truth = synth.elements_from_tles(synth.mixed_catalog(max(4 * n_objects, 400), n_geo=n_objects, n_molniya=0,
                                                         n_gps=0))
    geo = np.flatnonzero(np.abs(truth[1] - 1.0027) < 0.01)[:n_objects]
    per = []
    for day in (0, 1):
        ids, jd, fr, kind, value, sigma, station = cr.device_tracks(truth, geo, O.OPTICAL, 12, 300.0, seed + day,
                                                                    start=0.2 + day, span=0.3)
        off = np.searchsorted(ids, np.arange(len(geo) + 1))
        per += [tuple(a[off[j]:off[j + 1]] for a in (jd, fr, kind, value, sigma, station)) for j in range(len(geo))]
    return cr.Tracks(per, O.RADAR_SITES), np.tile(np.arange(len(geo)), 2)
