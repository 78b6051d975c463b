"""Time K8, the element fit (astroz_b200/csrc/az_fit.cu), on four workloads and print one JSON line.

    python tools/fit_timing.py [--sats 13478] [--obs 1440] [--cpu-sample 64]

FT1: the config-2 catalogue, `--obs` observations per satellite at 1 min from the K1 grid (positions and velocities),
     from perturbed guesses (n + 1e-4 rev/day, e + 1e-4, 0.05 deg on each angle, B* x 2).
FT2: TEME states at epoch from K6, propagated one day at 1 min by K7 (TwoBody + J2, DP87), fitted from the elements the
     states came from.
FT3: the 1,536 deep-space sets of config 3 (GEO, Molniya, GPS-like), 1,440 observations at 1 min from the K2 grid, from
     the same perturbed guesses with B* held (deep_space=True: fit_deep_kernel).
FT4: the same sets over a 7-day arc at 10 min starting 2 days before their epochs, so both directions of the resonance
     lattice are used.
Reported per workload: device ms (one launch, CUDA events, after a warm-up; best of 3 and the spread), host-call ms with
pinned and with pageable buffers, the iteration histogram, SGP4 evaluations per second (trial sets x observations:
(1 + variables) x observations per pass; for FT3 and FT4 SDP4 evaluations, 7 per observation and pass), and the
threaded CPU restatement (tests/fit_oracle, its deep-space part for FT3 and FT4) on a sample of satellites scaled to the
whole batch, on the same host.  Card name, power limit and maximum SM clock are read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def _run(name, el, guess, sat, jd, fr, pos, vel, cpu_sample, deep_space=False):
    import torch

    from astroz_b200 import _lib
    from astroz_b200.fit import fit_elements, fit_elements_device
    from tests import fit_oracle as R
    from tests.fit_oracle import deep as D

    n, m = el.shape[1], len(sat)
    dev = torch.device("cuda", 0)
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a)).to(dev, dt)  # noqa: E731
    offsets = np.searchsorted(sat, np.arange(n + 1)).astype(np.int32)
    args = [t(guess), t(offsets, torch.int32), t(jd), t(fr), t(pos), t(vel)]
    outs = [torch.empty((8, n), dtype=torch.float64, device=dev), torch.empty((n, 2), dtype=torch.float64, device=dev),
            torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.uint8, device=dev)]
    kw = dict(fit_bstar=False, deep_space=True) if deep_space else {}
    fit_elements_device(*args, *outs, **kw)   # warm-up
    torch.cuda.synchronize()
    ms = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fit_elements_device(*args, *outs, **kw)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    iters = outs[2].cpu().numpy()
    status = outs[3].cpu().numpy()
    passes = iters.astype(np.int64) + 1
    per_sat = np.diff(offsets).astype(np.int64)
    evals = float((passes * per_sat).sum() * (7 if deep_space else 8))   # held B*: 6 variables + the nominal set
    host = {}
    for kind in ("pinned", "pageable"):
        if kind == "pinned":
            bufs = []
            for a in (jd, fr, pos, vel):
                p = _lib.pinned_empty(a.shape)
                p[...] = a
                bufs.append(p)
            j2, f2, p2, v2 = bufs
        else:
            j2, f2, p2, v2 = (np.array(a) for a in (jd, fr, pos, vel))
        best = []
        for _ in range(2):
            t0 = time.perf_counter()
            fit_elements(guess, sat, j2, f2, p2, v2, **kw)
            best.append((time.perf_counter() - t0) * 1e3)
        host[kind] = round(min(best), 1)
    pick = np.linspace(0, n - 1, min(cpu_sample, n)).astype(int)
    rows = np.concatenate([np.arange(offsets[s], offsets[s + 1]) for s in pick])
    off = np.concatenate([[0], np.cumsum(per_sat[pick])]).astype(np.uint32)
    threads = os.cpu_count() or 1
    t0 = time.perf_counter()
    restated = D.fit_mixed if deep_space else R.fit
    restated(guess[:, pick], off, jd[rows], fr[rows], pos[rows], vel[rows], threads=threads,
             **({"fit_bstar": False} if deep_space else {}))
    cpu_ms = (time.perf_counter() - t0) * 1e3 * n / len(pick)
    return {"workload": name, "sats": n, "obs": m, "device_ms_best": round(min(ms), 2),
            "device_ms_spread": round(max(ms) - min(ms), 2), "host_ms": host,
            "iterations_hist": np.bincount(iters).tolist(), "status_hist": np.bincount(status, minlength=5).tolist(),
            "sgp4_evals_per_s": round(evals / (min(ms) * 1e-3), 0), "cpu_restatement_ms_scaled": round(cpu_ms, 0),
            "cpu_threads": threads, "cpu_sample": len(pick)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sats", type=int, default=13478)
    ap.add_argument("--obs", type=int, default=1440)
    ap.add_argument("--cpu-sample", type=int, default=64)
    args = ap.parse_args()
    from astroz_b200 import synth
    from astroz_b200.constellation import Constellation, Layout
    from tests import fit_oracle as R
    from tests.test_gpu_fit import k7_case

    card = _card()
    el = synth.elements_from_tles(synth.near_earth_catalog(args.sats))
    c = Constellation.from_elements(*el)
    jd, fr = synth.time_grid(args.obs)
    pos, vel = c.propagate(jd, fr, layout=Layout.satelliteMajor)
    c.deinit()
    sat = np.repeat(np.arange(args.sats), args.obs)
    ft1 = _run("FT1", el, R.perturbed(el, seed=3), sat, np.tile(jd, args.sats), np.tile(fr, args.sats),
               np.array(pos).reshape(-1, 3), np.array(vel).reshape(-1, 3), args.cpu_sample)
    el2, sat2, jd2, fr2, pos2, vel2 = k7_case(args.sats)
    ft2 = _run("FT2", el2, el2, sat2, jd2, fr2, pos2, vel2, args.cpu_sample)
    el3 = synth.elements_from_tles(synth.mixed_catalog(13478))
    el3 = el3[:, 1440.0 / el3[1] > 225.0]
    g3 = R.perturbed(el3, seed=3)
    g3[7] = el3[7]
    n3 = el3.shape[1]
    c = Constellation.from_elements(*el3)
    ft = []
    for name, (jd3, fr3) in (("FT3", synth.time_grid(1440)),
                             ("FT4", (np.full(1008, el3[0].min() - 2.0), np.arange(1008) * 10.0 / 1440.0))):
        p3, v3 = c.propagate(jd3, fr3, layout=Layout.satelliteMajor)
        ft.append(_run(name, el3, g3, np.repeat(np.arange(n3), len(jd3)), np.tile(jd3, n3), np.tile(fr3, n3),
                       np.array(p3).reshape(-1, 3), np.array(v3).reshape(-1, 3), args.cpu_sample, deep_space=True))
    c.deinit()
    print(json.dumps({"tool": "fit_timing", "card": card, "results": [ft1, ft2, *ft]}))


if __name__ == "__main__":
    main()
