"""K12 track correlation timing (astroz_cuda_correlate[_device]).

    python tools/correlate_timing.py [--reps 3] [--quick]

Workloads (covariances are synthetic PSD matrices at a radar refit's scale, B* free on near-earth rows and held on
deep-space rows; tracks are noisy radar or optical observations of catalogue rows from six stations, formed from
propagate_pairs states by the numpy statement of the kinds -- geometric, so visibility is not modelled):
  CR1  the config-2 catalogue (13,478 near-earth rows) with covariance against 1,000 and 10,000 radar tracks of 10
       observations (10^4 and 10^5 observations);
  CR2  the same catalogue and tracks with no covariance (P = 0: one propagation per observation per pair);
  CR3  config 3's GEO rows against 1,000 optical tracks of 12 observations over two hours;
  CR4  one radar track against the config-2 catalogue;
  CR5  config 3 (11,942 near-earth and 1,536 deep-space rows) against 1,000 radar tracks of near-earth rows: a mixed
       catalogue, where both scoring kernels run over every row chunk.
Prints one JSON record per workload: device ms (CUDA events, best of --reps, and the spread), pairs / s and SGP4 / SDP4
evaluations / s counted from the definition ((1 + nvar) x L per pair, nvar 0 without covariance), host-call ms with
pageable and pinned buffers, the C restatement (tests/fit_oracle/correlate.c: each row's sets built once, the stacked
form per pair) on every host thread over a sample of --cpu-sample tracks against every row, scaled to the workload's
tracks, and the card, power limit and maximum SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception:   # noqa: BLE001
        return ["unknown", "unknown", "unknown"]


def _tracks(el, rows, kind, L, step_s, seed):
    from tests.fit_oracle.correlate import device_tracks

    return device_tracks(el, rows, kind, L, step_s, seed)


def _device_ms(el, P, model, trk, reps):
    import torch

    from astroz_b200.correlate import correlate_device, correlate_scratch_bytes

    ids, jd, fr, kind, value, sigma, station = trk
    dev = torch.device("cuda", 0)
    g = lambda a, dt: None if a is None else torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa
    n, t, best = el.shape[1], int(ids.max()) + 1, 4
    offsets = np.searchsorted(ids, np.arange(t + 1)).astype(np.int32)
    args = [g(el, torch.float64), g(P, torch.float64), g(model, torch.uint8), g(offsets, torch.int32),
            g(jd, torch.float64), g(fr, torch.float64), g(kind, torch.uint8), g(value, torch.float64),
            g(sigma, torch.float64), g(station.astype(np.int32), torch.int32),
            g(np.array([[42.6, -71.5, 0.12], [9.4, 167.5, 0.01], [-31.0, 136.0, 0.15], [69.3, 16.0, 0.05],
                        [36.0, 139.0, 0.2], [-22.0, -47.0, 0.7]]), torch.float64),
            torch.zeros(correlate_scratch_bytes(n, t, best), dtype=torch.uint8, device=dev)]
    out = [torch.zeros((t, best), dtype=torch.int32, device=dev), torch.zeros((t, best), dtype=torch.float64,
                                                                               device=dev)]
    out += [torch.zeros(t, dtype=torch.int32, device=dev) for _ in range(3)]
    out += [torch.zeros(t, dtype=torch.uint8, device=dev), torch.zeros(n, dtype=torch.uint8, device=dev)]
    correlate_device(*args, *out)
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        correlate_device(*args, *out)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return times, out[5].cpu().numpy()


def _host_ms(el, P, model, trk, pinned):
    import torch

    from astroz_b200.correlate import correlate

    ids, jd, fr, kind, value, sigma, station = trk
    if pinned:
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()  # noqa: E731
        el, jd, fr, value, sigma = pin(el), pin(jd), pin(fr), pin(value), pin(sigma)
        P = None if P is None else pin(P)
    t0 = time.perf_counter()
    correlate(el, ids, jd, fr, kind, value, sigma, station, _stations(), covariance=P, model=model)
    return (time.perf_counter() - t0) * 1e3


def _cpu_s(el, P, model, trk, sample):
    """seconds of the C restatement over all the workload's pairs, on every host thread, scaled from `sample` tracks"""
    from tests.fit_oracle import correlate as cr

    ids, jd, fr, kind, value, sigma, station = trk
    t = int(ids.max()) + 1
    k = min(sample, t)
    e = int(np.searchsorted(ids, k))
    tr = cr.Tracks([(jd[:e], fr[:e], kind[:e], value[:e], sigma[:e], station[:e])], _stations())
    tr.offsets = np.searchsorted(ids[:e], np.arange(k + 1)).astype(np.uint32)
    tr.t = k
    t0 = time.perf_counter()
    cr.restated_sweep(el, P, model, tr)
    return (time.perf_counter() - t0) * t / k


def _stations():
    from tests.fit_oracle import obs as O

    return O.RADAR_SITES


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="CR1 / CR2 at 1,000 tracks only")
    ap.add_argument("--cpu-sample", type=int, default=8, help="tracks of the C restatement's sample")
    args = ap.parse_args()
    from astroz_b200 import synth
    from tests.fit_oracle import conjunction_cases as cc
    from tests.fit_oracle import obs as O

    name, power, clock = _card()
    el2 = synth.elements_from_tles(synth.near_earth_catalog(13478, 13478))
    n2 = el2.shape[1]
    P2 = cc.P_words(n2, scale=0.3, seed=12)
    el3 = synth.elements_from_tles(synth.mixed_catalog())
    geo = np.flatnonzero((el3[1] > 0.9) & (el3[1] < 1.1))
    elg = np.ascontiguousarray(el3[:, geo])
    Pg = cc.P_words(len(geo), scale=0.3, seed=13, deep=np.ones(len(geo), bool))
    mg = np.ones(len(geo), np.uint8)
    rng = np.random.default_rng(1)
    work = []
    for t in ((1000,) if args.quick else (1000, 10000)):
        trk = _tracks(el2, rng.integers(0, n2, t), O.RADAR, 10, 10.0, seed=t)
        work.append((f"CR1 {t} tracks", el2, P2, None, trk, 7))
        work.append((f"CR2 {t} tracks", el2, None, None, trk, 0))
    work.append(("CR3 GEO optical 1000 tracks", elg, Pg, mg,
                 _tracks(elg, rng.integers(0, len(geo), 1000), O.OPTICAL, 12, 600.0, seed=3), 6))
    work.append(("CR4 one track", el2, P2, None, _tracks(el2, np.array([17]), O.RADAR, 10, 10.0, seed=4), 7))
    deep3 = (1440.0 / el3[1]) > 225.0
    P3 = cc.P_words(el3.shape[1], scale=0.3, seed=14, deep=deep3)
    near3 = np.flatnonzero(~deep3)
    work.append(("CR5 config 3 mixed, 1000 tracks", el3, P3, deep3.astype(np.uint8),
                 _tracks(el3, rng.choice(near3, 1000), O.RADAR, 10, 10.0, seed=5), 7))
    for label, el, P, model, trk, _ in work:
        times, status = _device_ms(el, P, model, trk, args.reps)
        n, t, m = el.shape[1], int(trk[0].max()) + 1, len(trk[0])
        pairs = n * t
        if P is None:
            evals = m * n
        else:   # 1 + nvar per row: 8 with B* free, 7 with its row of P zero
            bstar = [q for q, (j, k) in enumerate(zip(*np.triu_indices(7))) if j == 6 or k == 6]
            evals = m * int(np.sum(np.where(np.any(P[:, bstar] != 0, axis=1), 8, 7)))
        best = min(times)
        rec = dict(workload=label, rows=n, tracks=t, observations=m, device_ms=best,
                   device_ms_spread=max(times) - best, pairs_per_s=pairs / (best * 1e-3),
                   evals_per_s=evals / (best * 1e-3), host_ms_pageable=_host_ms(el, P, model, trk, False),
                   host_ms_pinned=_host_ms(el, P, model, trk, True),
                   cpu_restatement_s=_cpu_s(el, P, model, trk, args.cpu_sample), cpu_threads=os.cpu_count(),
                   status_counts={int(k): int(v) for k, v in zip(*np.unique(status, return_counts=True))},
                   card=name, power_limit=power, max_sm_clock=clock)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
