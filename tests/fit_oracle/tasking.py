"""K18 sensor tasking for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

emul(), emul_slot(), emul_update(): the host build of the device source (tests/host_emul/emul_tasking.cu).
greedy(): a brute-force statement of the schedule driven by emul_slot's per-cell scores.
visibility(): a numpy statement of the visibility rules on given TEME states, with each cell's margin to its nearest
threshold.  scene(): a small mixed catalogue, radar and optical sensors and slots."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
from dataclasses import dataclass

import numpy as np

from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import correlate as cr
from tests.fit_oracle import obs as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
IDLE = 0xFFFFFFFF
CELL = 36
R_EARTH = 6378.137


def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_tasking.so")
    src = os.path.join(emul_dir, "emul_tasking.cu")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    L.emul_task_scratch_bytes.restype = C.c_size_t
    return L


@dataclass
class Scene:
    el: np.ndarray        # (8, n)
    model: np.ndarray     # (n,) uint8
    P: np.ndarray         # (n, 28)
    kind: np.ndarray      # (S,) uint8
    station: np.ndarray   # (S,) uint32
    sigma: np.ndarray     # (S, 4)
    limits: np.ndarray    # (S, 4)
    stations: np.ndarray  # (k, 3)
    jd: np.ndarray        # (T,)
    fr: np.ndarray        # (T,)
    sun: np.ndarray       # (T, 3)

    @property
    def n(self):
        return self.el.shape[1]

    @property
    def S(self):
        return len(self.kind)

    @property
    def T(self):
        return len(self.jd)

    def sensor_args(self):
        return (_p(self.kind), _p(self.station), _p(self.sigma), _p(self.limits), C.c_uint32(self.S),
                _p(self.stations))


def sensors(radar_sites, optical_sites, el_min=10.0, sun_el_max=-12.0, exclusion=40.0, range_max=np.inf):
    """(kind, station, sigma, limits, stations): one sensor per site, radars first"""
    sites = np.concatenate([np.reshape(radar_sites, (-1, 3)), np.reshape(optical_sites, (-1, 3))])
    nr = len(np.reshape(radar_sites, (-1, 3)))
    S = len(sites)
    kind = np.array([O.RADAR] * nr + [O.OPTICAL] * (S - nr), np.uint8)
    sigma = np.full((S, 4), np.inf)
    sigma[:nr] = O.RADAR_SIGMA
    sigma[nr:, :2] = O.OPTICAL_SIGMA
    limits = np.tile([np.deg2rad(el_min), range_max, np.deg2rad(sun_el_max), np.deg2rad(exclusion)], (S, 1))
    return kind, np.arange(S, dtype=np.uint32), sigma, limits, np.ascontiguousarray(sites, np.float64)


OPTICAL_SITES = np.array([[32.4, -110.7, 2.5], [-30.2, -70.8, 2.7], [28.8, -17.9, 2.4]])


def scene(n_per=10, T=60, step_min=2.0, t0=2460000.25 + 0.3, seed=3, radar=O.RADAR_SITES[:2],
          optical=OPTICAL_SITES[:1], scale=1.0, **limits):
    """n_per copies of base_rows (LEO, SSO, GEO, Molniya) spread in mean anomaly and node, P at a radar fit's scale"""
    from astroz_b200.tasking import sun_direction

    el0, md0 = cr.base_rows()
    rng = np.random.default_rng(seed)
    el = np.repeat(el0, n_per, axis=1).copy()
    model = np.repeat(md0, n_per).astype(np.uint8)
    el[6] = rng.uniform(0.0, 360.0, el.shape[1])
    el[4] = (el[4] + rng.uniform(-60.0, 60.0, el.shape[1])) % 360.0
    P = cc.P_words(el.shape[1], scale=scale, seed=seed + 1, deep=model == 1)
    kind, station, sigma, lim, stations = sensors(radar, optical, **limits)
    k = np.arange(T) * step_min / 1440.0
    jd = np.full(T, np.floor(t0 - 0.5) + 0.5)
    fr = (t0 - jd) + k
    return Scene(np.ascontiguousarray(el), model, P, kind, station, sigma, lim, stations, jd, fr,
                 np.ascontiguousarray(sun_direction(jd, fr)))


def emul(L, sc: Scene, gain_min=0.0, grav=1, cov="P"):
    """the host build's outputs as a dict"""
    n, S, T = sc.n, sc.S, sc.T
    P = sc.P if isinstance(cov, str) else cov
    P = None if P is None else np.ascontiguousarray(P, np.float64)
    out = dict(task_row=np.zeros((S, T), np.uint32), task_gain=np.zeros((S, T)), task_value=np.zeros((S, T, 4)),
               task_spread=np.zeros((S, T, 4)), n_candidates=np.zeros((S, T), np.uint32),
               posterior=np.zeros((n, 28)), n_tasks=np.zeros(n, np.uint32), n_visible=np.zeros(n, np.uint32),
               n_failed=np.zeros(n, np.uint32), row_status=np.zeros(n, np.uint8))
    L.emul_tasking(_p(sc.el), C.c_uint32(n), grav, _p(P), _p(sc.model), *sc.sensor_args(), _p(sc.jd), _p(sc.fr),
                   C.c_uint32(T), _p(sc.sun), C.c_double(gain_min), *[_p(out[k]) for k in out])
    return out


def emul_slot(L, sc: Scene, t, P, grav=1, cov="P"):
    """(gain (S, n), cell (S, n, 36), visible (n,) masks, failed (n,), f0 (n, 6), row_status (n,)) of slot t under
    covariances P (n, 28); the rows' sets are built under `cov` (default the scene's P)"""
    n, S = sc.n, sc.S
    C0 = sc.P if isinstance(cov, str) else cov
    C0 = None if C0 is None else np.ascontiguousarray(C0, np.float64)
    gain, cell = np.zeros((S, n)), np.zeros((S, n, CELL))
    vis, fail, f0, rs = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros((n, 6)), np.zeros(n, np.uint8)
    L.emul_task_slot(_p(sc.el), C.c_uint32(n), grav, _p(C0), _p(sc.model), *sc.sensor_args(),
                     C.c_double(sc.jd[t]), C.c_double(sc.fr[t]), _p(np.ascontiguousarray(sc.sun[t])),
                     _p(np.ascontiguousarray(P, np.float64)), _p(gain), _p(cell), _p(vis), _p(fail), _p(f0), _p(rs))
    return gain, cell, vis, fail, f0, rs


def emul_update(L, G, P, sigma):
    """(rc, gain, spread (4,), P+ (28,)) of one cell: G (4, 7), P (28,), sigma (4,)"""
    g, spread, Pp = C.c_double(), np.zeros(4), np.zeros(28)
    rc = L.emul_task_update(_p(np.ascontiguousarray(G, np.float64)), _p(np.ascontiguousarray(P, np.float64)),
                            _p(np.ascontiguousarray(sigma, np.float64)), C.byref(g), _p(spread), _p(Pp))
    return rc, g.value, spread, Pp


def greedy(L, sc: Scene, gain_min=0.0):
    """The schedule by its statement: per slot, score every cell under the current P (emul_slot), let sensors pick in
    order, replace each taken row's P by the posterior of its cell (emul_update).  Returns (task_row, task_gain,
    n_candidates, posterior)."""
    n, S, T = sc.n, sc.S, sc.T
    P = sc.P.copy()
    rows, gains, cands = np.full((S, T), IDLE, np.uint32), np.zeros((S, T)), np.zeros((S, T), np.uint32)
    for t in range(T):
        gain, cell, _, _, _, _ = emul_slot(L, sc, t, P)
        taken = set()
        for k in range(S):
            ok = [s for s in range(n) if gain[k, s] > gain_min and s not in taken]
            cands[k, t] = len(ok)
            if not ok:
                continue
            s = min(ok, key=lambda r: (-gain[k, r], r))
            rows[k, t], gains[k, t] = s, gain[k, s]
            taken.add(s)
        for k in range(S):
            s = rows[k, t]
            if s != IDLE:
                rc, _, _, Pp = emul_update(L, cell[k, s, 8:].reshape(4, 7), P[s], sc.sigma[k])
                assert rc == 0
                P[s] = Pp
    return rows, gains, cands, P


def visibility(states, jd_full, llh, kind, limits, sun):
    """(visible, margin) of TEME states (m, 6) at jd_full (m,) from one sensor, by the rules' own statement: margin is
    the least distance (rad or km) of the cell to a threshold of the rules it was decided by"""
    h = O.observe(O.RADAR, states, jd_full, llh)
    el, rng = h[:, 2], h[:, 0]
    vis = (el >= limits[0]) & (rng <= limits[1])
    margin = np.minimum(np.abs(el - limits[0]), np.abs(rng - limits[1]))
    if kind == O.OPTICAL:
        u = sun / np.linalg.norm(sun, axis=-1, keepdims=True) * np.ones((len(states), 1))
        r = states[:, :3]
        rs = np.einsum("ni,ni->n", r, u)
        perp = np.linalg.norm(r - rs[:, None] * u, axis=1)
        lit = (rs >= 0) | (perp > R_EARTH)
        up = O.enu_basis(llh)[2]
        ue = np.einsum("nij,nj->ni", O.rot(O.gmst(jd_full)), u)
        sun_el = np.arcsin(np.clip(ue @ up, -1, 1))
        rho = r - np.einsum("nji,j->ni", O.rot(O.gmst(jd_full)), O.station_ecef(llh))
        ang = np.arctan2(np.linalg.norm(np.cross(rho, u), axis=1), np.einsum("ni,ni->n", rho, u))
        vis &= lit & (sun_el <= limits[2]) & (ang >= limits[3])
        m_lit = np.where(rs >= 0, np.abs(rs), np.abs(perp - R_EARTH))
        margin = np.minimum.reduce([margin, m_lit, np.abs(sun_el - limits[2]), np.abs(ang - limits[3])])
    return vis, margin
