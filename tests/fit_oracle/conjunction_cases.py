"""Engineered conjunctions for the K11 tests -- TEST INFRASTRUCTURE ONLY.

A crossing is built from a copy of a set: both sets sit at their ascending node at epoch (argument of latitude 0, where
orbits of any inclination on a common node meet), the copy's inclination is changed by di, and small node and
mean-anomaly offsets set the miss."""
from __future__ import annotations

import numpy as np

from tests.fit_oracle import covariance as K


def at_node(el):
    """el (8,) with M = -w: the set is at its ascending node at epoch (to its eccentricity)"""
    el = np.array(el, dtype=np.float64)
    el[6] = (-el[5]) % 360.0
    return el


def pair(base, di, dnode=0.0, dm=0.0, other=None):
    """(8, 2) element columns: base at its node, and `other` (default: base) with i + di, node + dnode, M + dm at the
    same node and epoch"""
    a = at_node(base)
    b = at_node(base if other is None else other)
    b[0] = a[0]
    b[4] = a[4] + dnode
    b[3] = np.clip(a[3] + di, 0.01, 179.9) if other is None else b[3]
    b[6] = (b[6] + dm) % 360.0
    return np.stack([a, b], axis=1)


def leo():
    return np.array([2460000.25, 15.2, 0.0012, 51.6, 120.0, 80.0, 0.0, 2e-5])


def geo():
    return np.array([2460000.25, 1.0027, 0.0002, 0.05, 80.0, 10.0, 0.0, 0.0])


def molniya_at_perigee():
    """a Molniya orbit with its perigee on the ascending node (w = 0), at perigee at epoch"""
    return np.array([2460000.25, 2.006, 0.72, 63.4, 120.0, 0.0, 0.0, 0.0])


def gto_at_perigee():
    return np.array([2460000.25, 2.26, 0.73, 27.0, 120.0, 0.0, 0.0, 0.0])


def leo_under(deep, incl):
    """a circular LEO on deep's node whose radius is deep's perigee radius, inclination incl"""
    n_deep = deep[1]
    a_deep = (398600.8 * (86400.0 / (2 * np.pi * n_deep)) ** 2) ** (1.0 / 3.0)
    rp = a_deep * (1.0 - deep[2])
    n = 86400.0 / (2 * np.pi) * np.sqrt(398600.8 / rp ** 3)
    return np.array([deep[0], n, 0.0005, incl, deep[4], 0.0, 0.0, 1e-5])


def P_words(n, scale=1.0, seed=5, bstar=True, deep=None):
    """PSD covariances in the fit's variables at a radar fit's scale times `scale` (as the K10 tests make them)"""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 28))
    for s in range(n):
        dd = deep is not None and deep[s]
        d = np.array([1e-7, 1e-6, 1e-6, 1e-5, 1e-5, 1e-5, 1e-5 if bstar and not dd else 0.0]) * scale
        A = rng.standard_normal((7, 7))
        Cm = A @ A.T / 7.0 + 0.3 * np.eye(7)
        Cm /= np.sqrt(np.outer(np.diag(Cm), np.diag(Cm)))
        out[s] = K.pack7(Cm * np.outer(d, d))
    return out


def catalogue():
    """(elements (8, n), model (n,), candidates [(p, s, window_min, label)]): LEO-LEO at di from 0.5 to 170 deg,
    LEO against Molniya and GTO near their perigees, GEO-GEO"""
    cols, model, cands = [], [], []

    def add(el2, m2, w, label):
        k = sum(c.shape[1] for c in cols)
        cols.append(el2)
        model.extend(m2)
        cands.append((k, k + 1, w, label))

    for j, di in enumerate([0.5, 2.0, 10.0, 45.0, 90.0, 130.0, 170.0]):
        add(pair(leo(), di, dnode=0.002 * (j + 1), dm=0.001), [0, 0], 1.0, f"LEO-LEO di {di}")
    mol, gto = molniya_at_perigee(), gto_at_perigee()
    for deep, label in ((mol, "LEO-Molniya"), (gto, "LEO-GTO")):
        lo = leo_under(deep, 98.0 if label == "LEO-Molniya" else 51.6)
        add(np.stack([lo, deep], axis=1), [0, 1], 2.0, label)
    add(pair(geo(), 0.05, dnode=0.0, dm=0.0005), [1, 1], 30.0, "GEO-GEO")
    return np.concatenate(cols, axis=1), np.array(model, np.uint8), cands


def high_pc_leo(assess):
    """(elements (8, 2), P words (2, 28), hbr): a LEO crossing at di = 40 deg whose covariance is scaled so that the
    encounter-plane sigma is 1.4 times the miss and the radius equals the miss: Pc 0.26.  assess(el, P, hbr)
    returns the record of candidate (0, 1) over +-1 min from the first set's epoch."""
    el = pair(leo(), 40.0, dnode=0.0005, dm=0.0)
    P = P_words(2, scale=1.0, bstar=False)
    rec = assess(el, P, 0.01)
    miss, c2 = rec[1], rec[9:12]
    sigma = np.sqrt(0.5 * (c2[0] + c2[2]))
    k = (1.4 * miss / sigma) ** 2
    return el, P * k, miss


def crossings(el, rows, di):
    """Engineered partners of catalogue rows: a copy of each row el[:, rows] with its inclination changed by di [deg]
    (toward 90 deg).  Row and copy share their argument of latitude at every time to the eccentricity, so they meet
    near the node (u = 0).  Returns (partner columns (8, k), the guess time: the row's first node crossing after
    its epoch as (jd, fr))."""
    cp = el[:, rows].copy()
    cp[3] = np.clip(cp[3] + di * np.where(cp[3] > 90.0, -1.0, 1.0), 0.01, 179.9)
    u0 = np.radians(el[5, rows] + el[6, rows]) % (2 * np.pi)
    t_node = el[0, rows] + ((2 * np.pi - u0) / (2 * np.pi)) / el[1, rows]
    jd = np.floor(t_node - 0.5) + 0.5
    return cp, jd, t_node - jd


def leo_deep_partner(leo_el, jd, fr):
    """A deep-space (Molniya-like, 12 h) set whose perigee lies on the LEO row's node, at the LEO's radius, with the
    object at perigee at the LEO's node crossing jd + fr: a LEO-deep crossing at high relative speed"""
    mu = 398600.8
    n_leo = leo_el[1] * 2 * np.pi / 86400.0
    a_leo = (mu / n_leo ** 2) ** (1.0 / 3.0)
    n_d = 2.006
    a_d = (mu / (n_d * 2 * np.pi / 86400.0) ** 2) ** (1.0 / 3.0)
    dtd = (jd + fr) - leo_el[0]
    return np.array([leo_el[0], n_d, 1.0 - a_leo / a_d, 63.4, leo_el[4], 0.0, (-n_d * dtd * 360.0) % 360.0, 0.0])
