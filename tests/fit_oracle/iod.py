"""K13 initial orbits for the tests -- TEST INFRASTRUCTURE ONLY; the product package never imports it.

emul_library(), emul(): the host build of the device source (tests/host_emul/emul_iod.cu, linked with the host
emulation of the mixed element fit).  The rest is an independent numpy / scipy restatement written from the textbook
definitions, not from the device source: two-body propagation by Kepler's equation in the eccentric anomaly (elliptic
orbits only), Gibbs and Herrick-Gibbs, Gauss' method with np.roots for the octic and its own universal-variable
refinement, and rv2coe."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
MU = {1: 398600.8, 2: 398600.5}              # WGS72, WGS84 (the gravity models' mu)
RE = {1: 6378.135, 2: 6378.137}
STATE, GIBBS, HERRICK_GIBBS, LAMBERT, GAUSS, NONE = 0, 1, 2, 3, 4, 255


def emul_library():
    emul_dir = os.path.join(_ROOT, "tests", "host_emul")
    csrc = os.path.join(_ROOT, "astroz_b200", "csrc")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(emul_dir, "libemul_iod.so")
    srcs = [os.path.join(emul_dir, f) for f in ("emul_iod.cu", "emul_fit.cu", "emul_fit_deep.cu")]
    deps = srcs + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        if not os.path.exists(nvcc):
            return None
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, *srcs], check=True,
                       capture_output=True)
    L = C.CDLL(so)
    L.emul_iod_admissible.restype = C.c_int
    return L


def emul(L, tr, bstar=None, grav=1):
    """the host build's (elements (8, t), state (t, 6), wrms, method, candidates, conv (t, 2), deep, status, init
    (8, t), fit_status) over the grouped, time-ordered tracks tr (tests.fit_oracle.correlate.Tracks)"""
    t = tr.t
    el, state, wrms = np.zeros((8, t)), np.zeros((t, 6)), np.zeros(t)
    method, cand = np.zeros(t, np.uint8), np.zeros(t, np.uint32)
    conv, deep, status = np.zeros((t, 2)), np.zeros(t, np.uint8), np.zeros(t, np.uint8)
    init, fit_status = np.zeros((8, t)), np.zeros(t, np.uint8)
    bs = None if bstar is None else np.ascontiguousarray(bstar, np.float64)
    L.emul_iod(_p(tr.offsets), C.c_uint32(t), *tr.obs_args(), _p(bs), grav, _p(el), _p(state), _p(wrms), _p(method),
               _p(cand), _p(conv), _p(deep), _p(status), _p(init), _p(fit_status))
    return el, state, wrms, method, cand, conv, deep, status, init, fit_status


def emul_gauss(L, Ls, Rs, ts, grav=1):
    """(octic roots above 1 ER, refined states (k, 6), their root indices) of the host build on one triplet"""
    Ls, Rs, ts = (np.ascontiguousarray(a, np.float64) for a in (Ls, Rs, ts))
    states, roots, refined = np.zeros((3, 6)), np.zeros(3, np.int32), C.c_int()
    nr = L.emul_iod_gauss(_p(Ls), _p(Rs), _p(ts), C.c_double(MU[grav]), C.c_double(RE[grav]), _p(states), _p(roots),
                          C.byref(refined))
    return nr, states[:refined.value], roots[:refined.value]


# ---- the restatement ---------------------------------------------------------------------------------------------------
def kepler(s0, dt, mu):
    """two-body state after dt seconds from s0, by Kepler's equation in the eccentric anomaly (elliptic orbits)"""
    r0, v0 = np.asarray(s0[:3], float), np.asarray(s0[3:], float)
    rn = np.linalg.norm(r0)
    a = 1.0 / (2.0 / rn - v0 @ v0 / mu)
    n = np.sqrt(mu / a ** 3)
    sig = r0 @ v0 / np.sqrt(mu * a)        # e sin E0
    ec = 1.0 - rn / a                      # e cos E0
    dM = n * dt
    x = dM                                 # dE
    for _ in range(100):
        f = x - ec * np.sin(x) + sig * (1.0 - np.cos(x)) - dM
        d = f / (1.0 - ec * np.cos(x) + sig * np.sin(x))
        x -= d
        if abs(d) < 1e-15 * max(1.0, abs(x)):
            break
    F = 1.0 - a / rn * (1.0 - np.cos(x))
    G = dt - (x - np.sin(x)) / n
    r = F * r0 + G * v0
    r1 = np.linalg.norm(r)
    Fd = -np.sqrt(mu * a) / (r1 * rn) * np.sin(x)
    Gd = 1.0 - a / r1 * (1.0 - np.cos(x))
    return np.concatenate([r, Fd * r0 + Gd * v0])


def gibbs(r1, r2, r3, mu):
    a, b, c = (np.linalg.norm(r) for r in (r1, r2, r3))
    N = a * np.cross(r2, r3) + b * np.cross(r3, r1) + c * np.cross(r1, r2)
    D = np.cross(r1, r2) + np.cross(r2, r3) + np.cross(r3, r1)
    S = (b - c) * r1 + (c - a) * r2 + (a - b) * r3
    return np.sqrt(mu / (np.linalg.norm(N) * np.linalg.norm(D))) * (np.cross(D, r2) / b + S)


def herrick_gibbs(r1, r2, r3, t1, t2, t3, mu):
    d31, d32, d21 = t3 - t1, t3 - t2, t2 - t1
    a, b, c = (np.linalg.norm(r) for r in (r1, r2, r3))
    return (-d32 * (1 / (d21 * d31) + mu / (12 * a ** 3)) * r1 + (d32 - d21) * (1 / (d21 * d32) + mu / (12 * b ** 3)) * r2
            + d21 * (1 / (d32 * d31) + mu / (12 * c ** 3)) * r3)


def _fg(r2, v2, tau, mu):
    """Lagrange f and g of a flight of tau seconds from (r2, v2), from the restated propagation"""
    s = kepler(np.concatenate([r2, v2]), tau, mu)
    # r(tau) = f r2 + g v2: solve in the orbit plane
    A = np.stack([r2, v2], axis=1)
    f, g = np.linalg.lstsq(A, s[:3], rcond=None)[0]
    return f, g


def gauss(Ls, Rs, ts, mu, rE, d0_min=1e-12, tol=1e-10, iters=200):
    """(roots above rE, [(root index, state at t2)] of the refined roots); Curtis Algorithms 5.5 / 5.6 with np.roots"""
    L1, L2, L3 = (np.asarray(x, float) for x in Ls)
    R1, R2, R3 = (np.asarray(x, float) for x in Rs)
    tau1, tau3 = ts[0] - ts[1], ts[2] - ts[1]
    tau = tau3 - tau1
    p1, p2, p3 = np.cross(L2, L3), np.cross(L1, L3), np.cross(L1, L2)
    D0 = L1 @ p1
    if abs(D0) < d0_min:
        return np.zeros(0), []
    D = np.array([[R @ p for p in (p1, p2, p3)] for R in (R1, R2, R3)])
    A = (-D[0, 1] * tau3 / tau + D[1, 1] + D[2, 1] * tau1 / tau) / D0
    B = (D[0, 1] * (tau3 ** 2 - tau ** 2) * tau3 / tau + D[2, 1] * (tau ** 2 - tau1 ** 2) * tau1 / tau) / (6 * D0)
    E, R22 = L2 @ R2, R2 @ R2
    a, b, c = -(A * A + 2 * A * E + R22), -2 * mu * B * (A + E), -mu * mu * B * B
    rts = np.roots([1, 0, a, 0, 0, b, 0, 0, c])
    rts = np.sort(rts[(np.abs(rts.imag) <= 1e-9 * np.abs(rts)) & (rts.real > rE)].real)
    out = []
    for q, x in enumerate(rts):
        x3 = x ** 3
        rho = np.array([
            ((6 * (D[2, 0] * tau1 / tau3 + D[1, 0] * tau / tau3) * x3 + mu * D[2, 0] * (tau ** 2 - tau1 ** 2) * tau1 / tau3)
             / (6 * x3 + mu * (tau ** 2 - tau3 ** 2)) - D[0, 0]) / D0,
            A + mu * B / x3,
            ((6 * (D[0, 2] * tau3 / tau1 - D[1, 2] * tau / tau1) * x3 + mu * D[0, 2] * (tau ** 2 - tau3 ** 2) * tau3 / tau1)
             / (6 * x3 + mu * (tau ** 2 - tau1 ** 2)) - D[2, 2]) / D0])
        f1, f3 = 1 - 0.5 * mu * tau1 ** 2 / x3, 1 - 0.5 * mu * tau3 ** 2 / x3
        g1, g3 = tau1 - mu * tau1 ** 3 / (6 * x3), tau3 - mu * tau3 ** 3 / (6 * x3)

        def geom(rho, f1, f3, g1, g3):
            r1, r2, r3 = R1 + rho[0] * L1, R2 + rho[1] * L2, R3 + rho[2] * L3
            return r1, r2, r3, (-f3 * r1 + f1 * r3) / (f1 * g3 - f3 * g1)

        r1, r2, r3, v2 = geom(rho, f1, f3, g1, g3)
        ok, done = bool(np.all(rho > 0)), False
        for _ in range(iters):
            if not ok or done:
                break
            if not (2 / np.linalg.norm(r2) - v2 @ v2 / mu > 0):
                ok = False
                break
            F1, G1 = _fg(r2, v2, tau1, mu)
            F3, G3 = _fg(r2, v2, tau3, mu)
            f1, g1, f3, g3 = (f1 + F1) / 2, (g1 + G1) / 2, (f3 + F3) / 2, (g3 + G3) / 2
            den = f1 * g3 - f3 * g1
            c1, c3 = g3 / den, -g1 / den
            nrho = np.array([(-D[0, 0] + D[1, 0] / c1 - c3 / c1 * D[2, 0]) / D0,
                             (-c1 * D[0, 1] + D[1, 1] - c3 * D[2, 1]) / D0,
                             (-c1 / c3 * D[0, 2] + D[1, 2] / c3 - D[2, 2]) / D0])
            done = bool(np.all(np.abs(nrho - rho) <= tol * np.abs(nrho)))
            rho = nrho
            ok = bool(np.all(rho > 0))
            r1, r2, r3, v2 = geom(rho, f1, f3, g1, g3)
        if ok and done:
            out.append((q, np.concatenate([r2, v2])))
    return rts, out


def rv2coe(s, mu):
    """(a, e, i, RAAN, w, M) in km and rad of a TEME state"""
    r, v = np.asarray(s[:3], float), np.asarray(s[3:], float)
    h = np.cross(r, v)
    rn = np.linalg.norm(r)
    ev = ((v @ v - mu / rn) * r - (r @ v) * v) / mu
    a = 1.0 / (2.0 / rn - v @ v / mu)
    e = np.linalg.norm(ev)
    i = np.arccos(h[2] / np.linalg.norm(h))
    nvec = np.array([-h[1], h[0], 0.0])
    node = np.arctan2(nvec[1], nvec[0]) % (2 * np.pi)
    w = np.arctan2(ev @ np.cross(h / np.linalg.norm(h), nvec / np.linalg.norm(nvec)), ev @ nvec / np.linalg.norm(nvec))
    nu = np.arctan2(np.cross(ev, r) @ h / (e * np.linalg.norm(h)), ev @ r / e)
    E = 2 * np.arctan(np.sqrt((1 - e) / (1 + e)) * np.tan(nu / 2))
    return a, e, i, node, w % (2 * np.pi), (E - e * np.sin(E)) % (2 * np.pi)


def coe2rv(a, e, i, node, w, M, mu):
    """TEME state of classical elements (elliptic), for building exact two-body truth"""
    E = M
    for _ in range(50):
        E -= (E - e * np.sin(E) - M) / (1 - e * np.cos(E))
    nu = 2 * np.arctan2(np.sqrt(1 + e) * np.sin(E / 2), np.sqrt(1 - e) * np.cos(E / 2))
    p = a * (1 - e * e)
    rpf = p / (1 + e * np.cos(nu)) * np.array([np.cos(nu), np.sin(nu), 0.0])
    vpf = np.sqrt(mu / p) * np.array([-np.sin(nu), e + np.cos(nu), 0.0])
    cO, sO, ci, si, cw, sw = np.cos(node), np.sin(node), np.cos(i), np.sin(i), np.cos(w), np.sin(w)
    Q = np.array([[cO * cw - sO * sw * ci, -cO * sw - sO * cw * ci, sO * si],
                  [sO * cw + cO * sw * ci, -sO * sw + cO * cw * ci, -cO * si],
                  [sw * si, cw * si, ci]])
    return np.concatenate([Q @ rpf, Q @ vpf])


# ---- a track's candidates, restated -----------------------------------------------------------------------------------
def triplet_table(c):
    """the triplets of a method with c observations: 30 fractional entries in sixteenths (whole span; halves, quarters
    and eighths with the middle at the midpoint; four long spans with an off-centre middle), rounded half up onto
    0 .. c - 1; entries that collapse or repeat an earlier one are skipped"""
    fr = [(0, 8, 16)] + [(s, s + 4, s + 8) for s in (0, 4, 8)] + [(s, s + 2, s + 4) for s in range(0, 13, 2)] + \
         [(s, s + 1, s + 2) for s in range(15)] + [(0, m, 16) for m in (4, 12, 2, 14)]
    out = []
    for q, u in enumerate(fr):
        ix = tuple((x * (c - 1) + 8) // 16 for x in u)
        if c >= 3 and ix[0] < ix[1] < ix[2] and ix not in [o for _, o in out]:
            out.append((q, ix))
    return out


def admissible(s, mu, rE):
    s = np.asarray(s, float)
    if not np.all(np.isfinite(s)):
        return False
    r, v = s[:3], s[3:]
    rn = np.linalg.norm(r)
    alpha = 2.0 / rn - v @ v / mu
    e = np.linalg.norm(((v @ v - mu / rn) * r - (r @ v) * v) / mu)
    return bool(alpha > 0 and e < 1 and (1 - e) / alpha >= rE)


def O_rot(jdf):
    from tests.fit_oracle import obs as O

    return O.rot(O.gmst(jdf))


def candidates(tr, j, grav=1):
    """(built, admissible) candidate counts of track j of tr (time-ordered): every state observation, Gibbs and
    Herrick-Gibbs on every radar triplet, the zero-revolution Lambert transfer for normals +z and -z between exactly two
    radar positions (K9's scalar C statement, tests/lambert_oracle), Gauss on every optical triplet with every refined
    root, from the restated geometry and methods"""
    from tests.fit_oracle import obs as O

    mu, rE = MU[grav], RE[grav]
    b, e = int(tr.offsets[j]), int(tr.offsets[j + 1])
    geo = {1: [], 2: [], 3: []}
    for i in range(b, e):
        k, v, sg = int(tr.kind[i]), tr.value[i], tr.sigma[i]
        need = 6 if k <= 1 else 3 if k == 2 else 2
        if not np.all(np.isfinite(sg[:need])):
            continue
        jdf = tr.jd[i] + tr.fr[i]
        R = O_rot(jdf)
        if k == 0:
            geo[1].append((jdf, v.copy()))
        elif k == 1:
            vv = v[3:] + np.cross([0.0, 0.0, O.OMEGA], v[:3])
            geo[1].append((jdf, np.concatenate([R.T @ v[:3], R.T @ vv])))
        else:
            llh = tr.stations[tr.station[i]]
            st = O.station_ecef(llh)
            if k == 2:
                E, N, U = O.enu_basis(llh)
                los = np.cos(v[2]) * np.sin(v[1]) * E + np.cos(v[2]) * np.cos(v[1]) * N + np.sin(v[2]) * U
                geo[2].append((jdf, R.T @ (st + v[0] * los)))
            else:
                geo[3].append((jdf, np.array([np.cos(v[1]) * np.cos(v[0]), np.cos(v[1]) * np.sin(v[0]), np.sin(v[1])]),
                               R.T @ st))
    built = ok = 0

    def offer(s):
        nonlocal built, ok
        built += 1
        ok += admissible(s, mu, rE)

    for _, s in geo[1]:
        offer(s)
    if len(geo[2]) == 2:
        from tests import lambert_oracle as K9

        (t1, r1), (t2, r2) = geo[2]
        for nz in (1.0, -1.0):
            v1, _, st, _ = K9.solve(r1[None], r2[None], np.array([(t2 - t1) * 86400.0]), mu,
                                    normal=np.array([[0.0, 0.0, nz]]))
            if st[0, 0] == 0:
                offer(np.concatenate([r1, v1[0, 0]]))
    for _, ix in triplet_table(len(geo[2])):
        (t1, r1), (t2, r2), (t3, r3) = (geo[2][q] for q in ix)
        offer(np.concatenate([r2, gibbs(r1, r2, r3, mu)]))
        offer(np.concatenate([r2, herrick_gibbs(r1, r2, r3, 0.0, (t2 - t1) * 86400, (t3 - t1) * 86400, mu)]))
    for _, ix in triplet_table(len(geo[3])):
        obs = [geo[3][q] for q in ix]
        ts = [(o[0] - obs[1][0]) * 86400 for o in obs]
        _, refined = gauss([o[1] for o in obs], [o[2] for o in obs], ts, mu, rE)
        for _, s in refined:
            offer(s)
    return built, ok


# ---- workloads of the device tests and the timing tool ----------------------------------------------------------------
def mixed_tracks(n_tracks, seed):
    """radar tracks of the near-earth rows (10 observations at 30 s; every 20th cut to its first and last, a Lambert
    pair 270 s apart), optical tracks of the deep-space rows (12 at 300 s) and TEME-state tracks (3 at 60 s) of a
    synthetic mixed catalogue, from propagate_pairs states with noise"""
    from astroz_b200 import synth
    from tests.fit_oracle import correlate as cr
    from tests.fit_oracle import obs as O

    truth = synth.elements_from_tles(synth.mixed_catalog(4000, n_geo=400, n_molniya=100, n_gps=100))
    deep = np.flatnonzero(1440.0 / truth[1] > 225.0)
    near = np.setdiff1d(np.arange(truth.shape[1]), deep)
    rng = np.random.default_rng(seed)
    n_opt, n_state = n_tracks // 4, n_tracks // 10
    parts = [cr.device_tracks(truth, rng.choice(near, n_tracks - n_opt - n_state), O.RADAR, 10, 30.0, seed),
             cr.device_tracks(truth, rng.choice(deep, n_opt), O.OPTICAL, 12, 300.0, seed + 1)]
    per = []
    for p, (ids, jd, fr, kind, value, sigma, station) in enumerate(parts):
        off = np.searchsorted(ids, np.arange(ids.max() + 2))
        for j in range(len(off) - 1):
            take = [off[j], off[j + 1] - 1] if p == 0 and j % 20 == 0 else slice(off[j], off[j + 1])
            per.append(tuple(a[take] for a in (jd, fr, kind, value, sigma, station)))
    rows = rng.integers(0, truth.shape[1], n_state)
    jd0 = np.floor(truth[0, rows] - 0.5) + 0.5
    for s, j0 in zip(rows, jd0):
        fr = truth[0, s] - j0 + 0.3 + np.arange(3) * 60.0 / 86400.0
        st = O.states_of(truth[:, s], np.full(3, j0), fr)
        noise = rng.standard_normal((3, 6)) * np.array([1e-3] * 3 + [1e-6] * 3)
        per.append((np.full(3, j0), fr, np.zeros(3, np.uint8), st + noise, np.tile([1e-3] * 3 + [1e-6] * 3, (3, 1)),
                    np.zeros(3, np.uint32)))
    return cr.Tracks(per, O.RADAR_SITES)
