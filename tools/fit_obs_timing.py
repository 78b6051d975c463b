"""Time the element fit from sensor observations (astroz_b200/csrc/az_fit_obs.cu) on two workloads; print one JSON line.

    python tools/fit_obs_timing.py [--sats 13478] [--cpu-sample 32]

OT1: the config-2 catalogue refitted from radar tracks of six stations over two days.  The tracks are made by the
     library itself: propagate_pairs TEME states at 2 min, then observe, keeping samples above 10 deg elevation.
     Perturbed guesses (n + 1e-4 rev/day, e + 1e-4, 0.05 deg on each angle), B* held at its generating value.
OT2: config 3's GEO objects (n within 0.001 rev/day of 1.0027) from optical angles over three 10-hour nights at 5 min,
     six stations around the equator at +-30 deg latitude, deep_space=True, B* held.
Reported per workload: device ms (one call of the _device entry point, CUDA events, after a warm-up; best of 3 and the
spread), host-call ms (pageable buffers), the iteration and status histograms, SGP4 / SDP4 evaluations per second
((1 + variables) x observations per pass), and the threaded CPU restatement (tests/fit_oracle/fit_oracle_obs.c, on the
oracle's SGP4 / SDP4) on a sample of satellites scaled to the whole batch, on the same host.  Card name, power limit and
maximum SM clock are read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.fit_timing import _card  # noqa: E402


def _tracks(el, kind, sites, jd, fr, chunk=1000):
    """library-made tracks of every column of el above 10 deg at any of the sites: per satellite (jd, fr, kind,
    value, sigma, station)"""
    from astroz_b200.constellation import Constellation
    from astroz_b200.fit import observe
    from tests.fit_oracle import obs as O

    sig = O.RADAR_SIGMA if kind == O.RADAR else O.OPTICAL_SIGMA
    n, t = el.shape[1], len(jd)
    c = Constellation.from_elements(*el)
    per = []
    for s0 in range(0, n, chunk):
        k = min(chunk, n - s0)
        p, v, st = c.propagate_pairs(np.repeat(np.arange(s0, s0 + k), t), np.tile(jd, k), np.tile(fr, k))
        states = np.concatenate([np.asarray(p), np.asarray(v)], axis=1)
        ok = np.asarray(st) == 0
        rows, vals, stas = [], [], []
        for q in range(len(sites)):
            h = observe(states, np.tile(jd, k), np.tile(fr, k), O.RADAR, q, sites)
            keep = np.flatnonzero(ok & (h[:, 2] > np.deg2rad(10.0)))
            rows.append(keep)
            vals.append(h[keep] if kind == O.RADAR else observe(states[keep], np.tile(jd, k)[keep],
                                                                 np.tile(fr, k)[keep], kind, q, sites))
            stas.append(np.full(len(keep), q, np.uint32))
        rows, vals, stas = np.concatenate(rows), np.concatenate(vals), np.concatenate(stas)
        sat = rows // t
        for j in range(k):
            m = np.flatnonzero(sat == j)
            m = m[np.argsort(rows[m] % t, kind="stable")]
            sig6 = np.full((len(m), 6), np.inf)
            sig6[:, :len(sig)] = sig
            per.append((jd[rows[m] % t], fr[rows[m] % t], np.full(len(m), kind, np.uint8), vals[m], sig6, stas[m]))
    c.deinit()
    return per


def _run(name, el, guess, per, sites, cpu_sample, deep_space):
    import torch

    from astroz_b200.fit import fit_observations, fit_observations_device
    from tests.fit_oracle import obs as O

    jd, fr, kd, val, sig, sta, off = O.concat(per)
    n, m = el.shape[1], len(jd)
    dev = torch.device("cuda", 0)
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a)).to(dev, dt)  # noqa: E731
    args = [t(guess), t(off, torch.int32), t(jd), t(fr), t(kd, torch.uint8), t(val), t(sig), t(sta, torch.int32),
            t(sites)]
    outs = [torch.empty((8, n), dtype=torch.float64, device=dev), torch.empty(n, dtype=torch.float64, device=dev),
            torch.empty(n, dtype=torch.int32, device=dev), torch.empty((n, 28), dtype=torch.float64, device=dev),
            torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.uint8, device=dev),
            torch.empty(n, dtype=torch.uint8, device=dev)]
    kw = dict(fit_bstar=False, deep_space=deep_space)
    fit_observations_device(*args, *outs, **kw)   # warm-up
    torch.cuda.synchronize()
    ms = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fit_observations_device(*args, *outs, **kw)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    iters, status = outs[4].cpu().numpy(), outs[5].cpu().numpy()
    per_sat = np.diff(off).astype(np.int64)
    evals = float(((iters.astype(np.int64) + 1) * per_sat).sum() * 7)   # B* held: 6 variables + the nominal set
    sat = np.repeat(np.arange(n), per_sat)
    t0 = time.perf_counter()
    fit_observations(guess, sat, jd, fr, kd, val, sig, sta, sites, **kw)
    host_ms = (time.perf_counter() - t0) * 1e3
    pick = np.linspace(0, n - 1, min(cpu_sample, n)).astype(int)
    sub = [per[s] for s in pick]
    sj, sf, sk, sv, ss, st, so = O.concat(sub)
    threads = os.cpu_count() or 1
    O.restated_library()   # built before the clock starts
    t0 = time.perf_counter()
    O.restated_fit(guess[:, pick], sj, sf, sk, sv, ss, st, so, sites, fit_bstar=False, mixed=deep_space,
                   threads=threads)
    cpu_ms = (time.perf_counter() - t0) * 1e3 * n / len(pick)
    return {"workload": name, "sats": n, "obs": m, "residuals": int(np.isfinite(sig).sum()),
            "device_ms_best": round(min(ms), 2), "device_ms_spread": round(max(ms) - min(ms), 2),
            "host_ms_pageable": round(host_ms, 1), "iterations_hist": np.bincount(iters).tolist(),
            "status_hist": np.bincount(status, minlength=5).tolist(),
            "sgp4_evals_per_s": round(evals / (min(ms) * 1e-3), 0),
            "cpu_restatement_ms_scaled": round(cpu_ms, 0), "cpu_threads": threads, "cpu_sample": len(pick)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sats", type=int, default=13478)
    ap.add_argument("--cpu-sample", type=int, default=32)
    args = ap.parse_args()
    from astroz_b200 import synth
    from tests import fit_oracle as R
    from tests.fit_oracle import obs as O

    card = _card()
    el = synth.elements_from_tles(synth.near_earth_catalog(args.sats))
    jd, fr = synth.time_grid(1440)
    fr = np.arange(1440) * 2.0 / 1440.0 + fr[0]
    g = R.perturbed(el, seed=3)
    g[7] = el[7]
    ot1 = _run("OT1", el, g, _tracks(el, O.RADAR, O.RADAR_SITES, jd, fr), O.RADAR_SITES, args.cpu_sample, False)
    el3 = synth.elements_from_tles(synth.mixed_catalog(13478))
    el3 = el3[:, np.abs(el3[1] - 1.0027) < 0.001]
    g3 = R.perturbed(el3, seed=3)
    g3[3] = np.abs(g3[3])
    g3[7] = el3[7]
    sites = np.array([[30.0 * (-1) ** q, -180.0 + 60.0 * q, 2.0] for q in range(6)])
    t3 = np.concatenate([np.arange(0.0, 600.0, 5.0) + 1440.0 * k for k in range(3)]) / 1440.0
    jd3, fr3 = np.full(len(t3), np.floor(el3[0].min()) + 0.5), t3 + 0.3
    ot2 = _run("OT2", el3, g3, _tracks(el3, O.OPTICAL, sites, jd3, fr3), sites, args.cpu_sample, True)
    print(json.dumps({"tool": "fit_obs_timing", "card": card, "results": [ot1, ot2]}))


if __name__ == "__main__":
    main()
