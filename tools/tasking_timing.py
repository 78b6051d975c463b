"""K18 sensor tasking timing (astroz_cuda_tasking[_device]).

    python tools/tasking_timing.py [--reps 3] [--cpu-rows 64]

Workloads (covariances are synthetic PSD matrices at a radar refit's scale, as tools/correlate_timing.py builds them;
B* free on near-earth rows and held on deep-space rows; the Sun from tasking.sun_direction):
  TK1  the config-2 catalogue (13,478 near-earth rows) x 6 radars x 1,440 one-minute slots;
  TK2  config 3's 1,536 deep-space rows x 3 optical sites x 3 nights (three 12-hour windows) at 2 minutes;
  TK3  config 3 (11,942 near-earth and 1,536 deep-space rows) x 6 radars + 3 optical sites x 1 day at 2 minutes.
Prints one JSON record per workload: device ms (CUDA events around the device call, best of --reps, and the spread),
(row, slot) cells / s, SGP4 / SDP4 evaluations / s counted from the definition (one nominal per (row, slot) plus nvar
per (row, slot) visible to any sensor; the visible share is taken from the host build on --cpu-rows random rows), the
visible fraction of (row, sensor, slot) cells, host-call ms with pageable and pinned buffers, the share of the device
call not covered by the tasking kernels (torch.profiler, a run of its own: launch gaps between slots), the host build
(tests/host_emul/emul_tasking.cu) on 8 threads over --cpu-rows rows scaled to the workload's rows, and the card, power
limit and maximum SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from correlate_timing import _card  # noqa: E402


def _scene(el, P, model, radar, optical, jd, fr):
    from astroz_b200.tasking import sun_direction
    from tests.fit_oracle import tasking as TK

    kind, station, sigma, limits, stations = TK.sensors(radar, optical)
    return TK.Scene(np.ascontiguousarray(el), model, P, kind, station, sigma, limits, stations, jd, fr,
                    np.ascontiguousarray(sun_direction(jd, fr)))


def _device(sc, reps, profile=False):
    import torch

    from astroz_b200.tasking import plan_device, plan_scratch_bytes

    d = torch.device("cuda", 0)
    g = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=d)  # noqa: E731
    n, S, T = sc.n, sc.S, sc.T
    args = [g(sc.el), g(sc.P), g(sc.model, torch.uint8), g(sc.kind, torch.uint8),
            g(sc.station.astype(np.int32), torch.int32), g(sc.sigma), g(sc.limits), g(sc.stations), g(sc.jd),
            g(sc.fr), g(sc.sun), torch.zeros(plan_scratch_bytes(n, S), dtype=torch.uint8, device=d)]
    z = lambda shape, dt=torch.float64: torch.zeros(shape, dtype=dt, device=d)  # noqa: E731
    out = [z((S, T), torch.int32), z((S, T)), z((S, T, 4)), z((S, T, 4)), z((S, T), torch.int32), z((n, 28)),
           z(n, torch.int32), z(n, torch.int32), z(n, torch.int32), z(n, torch.uint8)]
    plan_device(*args, *out)
    torch.cuda.synchronize()
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof

        with prof(activities=[ProfilerActivity.CUDA]) as p:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            plan_device(*args, *out)
            b.record()
            torch.cuda.synchronize()
        kern = sum(e.device_time_total for e in p.key_averages() if e.key.startswith("az::task_")) * 1e-3
        return 1.0 - kern / a.elapsed_time(b)
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        plan_device(*args, *out)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return times, out[7].cpu().numpy(), out[0].cpu().numpy()


def _host_ms(sc, pinned):
    import torch

    from astroz_b200.tasking import Sensor, plan

    arr = [sc.el, sc.jd, sc.fr, sc.sun, sc.P, sc.model]
    if pinned:
        arr = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy() for a in arr]
    el, jd, fr, sun, P, md = arr
    sens = [Sensor(int(sc.kind[k]), *sc.stations[k], sigma=tuple(sc.sigma[k]), el_min=np.rad2deg(sc.limits[k, 0]),
                   range_max=sc.limits[k, 1], sun_el_max=np.rad2deg(sc.limits[k, 2]),
                   exclusion=np.rad2deg(sc.limits[k, 3])) for k in range(sc.S)]
    t0 = time.perf_counter()
    plan(el, sens, jd, fr, sun=sun, covariance=P, model=md)
    return (time.perf_counter() - t0) * 1e3


def _cpu(sc, rows, threads=8):
    """(seconds of the host build on `threads` threads scaled to every row, share of (row, slot) visible to any
    sensor) from `rows` random rows"""
    from tests.fit_oracle import tasking as TK

    L = TK.emul_library()
    pick = np.sort(np.random.default_rng(0).choice(sc.n, min(rows, sc.n), replace=False))
    parts = [p for p in np.array_split(pick, threads) if len(p)]
    sub = lambda p: TK.Scene(np.ascontiguousarray(sc.el[:, p]), sc.model[p], sc.P[p], sc.kind, sc.station,  # noqa
                             sc.sigma, sc.limits, sc.stations, sc.jd, sc.fr, sc.sun)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(len(parts)) as ex:
        list(ex.map(lambda p: TK.emul(L, sub(p)), parts))
    sec = (time.perf_counter() - t0) * sc.n / len(pick)
    s1 = sub(pick[:16])
    anyvis = np.mean([np.mean(TK.emul_slot(L, s1, t, s1.P)[2] != 0) for t in range(0, sc.T, max(1, sc.T // 48))])
    return sec, anyvis


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-rows", type=int, default=64)
    args = ap.parse_args()
    from astroz_b200 import synth
    from tests.fit_oracle import conjunction_cases as cc
    from tests.fit_oracle import obs as O
    from tests.fit_oracle import tasking as TK

    name, power, clock = _card()
    el2 = synth.elements_from_tles(synth.near_earth_catalog(13478, 13478))
    P2 = cc.P_words(el2.shape[1], scale=0.3, seed=12)
    el3 = synth.elements_from_tles(synth.mixed_catalog())
    deep3 = (1440.0 / el3[1]) > 225.0
    P3 = cc.P_words(el3.shape[1], scale=0.3, seed=14, deep=deep3)
    t0 = float(el2[0].max())
    day = lambda T, step: (np.full(T, np.floor(t0 - 0.5) + 0.5), (t0 - (np.floor(t0 - 0.5) + 0.5)) +  # noqa: E731
                           np.arange(T) * step / 1440.0)
    jd1, fr1 = day(1440, 1.0)
    nights = np.concatenate([np.arange(360) * 2.0 / 1440.0 + q for q in range(3)])
    jd2, fr2 = np.full(1080, np.floor(t0 - 0.5) + 0.5), (t0 - (np.floor(t0 - 0.5) + 0.5)) + nights
    jd3, fr3 = day(720, 2.0)
    dp = np.flatnonzero(deep3)
    work = [("TK1 config 2 x 6 radars x 1440 slots",
             _scene(el2, P2, np.zeros(el2.shape[1], np.uint8), O.RADAR_SITES, np.zeros((0, 3)), jd1, fr1)),
            ("TK2 1536 deep-space rows x 3 optical x 3 nights",
             _scene(el3[:, dp], P3[dp], np.ones(len(dp), np.uint8), np.zeros((0, 3)), TK.OPTICAL_SITES, jd2, fr2)),
            ("TK3 config 3 x 9 sensors x 1 day",
             _scene(el3, P3, deep3.astype(np.uint8), O.RADAR_SITES, TK.OPTICAL_SITES, jd3, fr3))]
    for label, sc in work:
        times, n_visible, task_row = _device(sc, args.reps)
        gap = _device(sc, 1, profile=True)
        cpu_s, anyvis = _cpu(sc, args.cpu_rows)
        best = min(times)
        cells = sc.n * sc.T
        nvar = np.where(sc.model == 1, 6, 7)
        evals = cells + anyvis * sc.T * float(nvar.sum())
        rec = dict(workload=label, rows=sc.n, sensors=sc.S, slots=sc.T, device_ms=best,
                   device_ms_spread=max(times) - best, cells_per_s=cells / (best * 1e-3),
                   evals_per_s=evals / (best * 1e-3), visible_fraction=float(n_visible.sum()) / (cells * sc.S),
                   any_visible_fraction_sampled=float(anyvis), tasks=int(np.sum(task_row >= 0)),
                   host_ms_pageable=_host_ms(sc, False), host_ms_pinned=_host_ms(sc, True),
                   launch_gap_share=gap, host_build_8_threads_s=cpu_s, card=name, power_limit=power,
                   max_sm_clock=clock)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
