"""K13 initial-orbit timing (astroz_cuda_initial_orbits[_device]).

    python tools/iod_timing.py [--tracks 100000] [--reps 3] [--cpu-sample 2000] [--cpu-threads N]

Workload: --tracks mixed tracks of a synthetic mixed catalogue (tests/fit_oracle/iod.py's mixed_tracks, the device
tests' mix: 65 % radar tracks of near-earth rows, 10 observations at 30 s, every 20th cut to its first and last
observations, a Lambert pair 270 s apart; 25 % optical tracks of deep-space rows, 12 at 300 s; 10 % TEME-state
tracks, 3 at 60 s), noisy, from propagate_pairs states.  Prints one JSON record: the device call's time (CUDA events around
astroz_cuda_initial_orbits_device, best of --reps and the spread), split into the IOD kernel and the conversion (the
K8 fits and the finishing kernel) by torch.profiler kernel times; the host call (pageable buffers); the host build of
the same source (tests/host_emul/emul_iod.cu) on --cpu-threads host threads (default: every usable CPU) over
--cpu-sample tracks, scaled to the workload;
statuses and winning methods; and the card, power limit and maximum SM clock read in the same run.
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
    except (OSError, IndexError, subprocess.TimeoutExpired):
        return None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-sample", type=int, default=2000)
    ap.add_argument("--cpu-threads", type=int, default=len(os.sched_getaffinity(0)))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from astroz_b200.iod import initial_orbits, initial_orbits_device, initial_orbits_scratch_bytes
    from tests.fit_oracle import correlate as cr
    from tests.fit_oracle import iod as I

    tr = I.mixed_tracks(args.tracks, 31)
    t = tr.t
    d = torch.device("cuda", 0)
    cu = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a)).to(dt).to(d)  # noqa: E731
    ins = (cu(tr.offsets.astype(np.int32), torch.int32), cu(tr.jd, torch.float64), cu(tr.fr, torch.float64),
           cu(tr.kind, torch.uint8), cu(tr.value, torch.float64), cu(tr.sigma, torch.float64),
           cu(tr.station.astype(np.int32), torch.int32), cu(tr.stations, torch.float64), None)
    out = dict(elements=torch.zeros((8, t), dtype=torch.float64, device=d),
               state=torch.zeros((t, 6), dtype=torch.float64, device=d),
               wrms=torch.zeros(t, dtype=torch.float64, device=d), method=torch.zeros(t, dtype=torch.uint8, device=d),
               candidates=torch.zeros(t, dtype=torch.int32, device=d),
               conv=torch.zeros((t, 2), dtype=torch.float64, device=d),
               deep_space=torch.zeros(t, dtype=torch.uint8, device=d), status=torch.zeros(t, dtype=torch.uint8, device=d))
    scratch = torch.zeros(initial_orbits_scratch_bytes(t), dtype=torch.uint8, device=d)
    run = lambda: initial_orbits_device(*ins, scratch, **out)  # noqa: E731
    run()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            key = "iod_kernel" if "iod_kernel" in e.name else "conversion"
            kern[key] = kern.get(key, 0.0) + e.device_time / 1000.0
    t0 = time.perf_counter()
    res = initial_orbits(tr.track_ids(), tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station, tr.stations)
    host_ms = (time.perf_counter() - t0) * 1e3
    from concurrent.futures import ThreadPoolExecutor

    L = I.emul_library()
    picks = np.random.default_rng(0).choice(t, min(args.cpu_sample, t), replace=False)
    threads = args.cpu_threads
    parts = [p for p in np.array_split(picks, threads) if len(p)]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(len(parts)) as ex:
        list(ex.map(lambda p: I.emul(L, cr.subset(tr, p)), parts))
    cpu_s = (time.perf_counter() - t0) * t / len(picks)
    print(json.dumps({
        "workload": "IOD mixed tracks", "tracks": t, "observations": int(len(tr.jd)),
        "device_ms_best": min(times), "device_ms_spread": max(times) - min(times),
        "iod_kernel_ms": kern.get("iod_kernel"), "conversion_ms": kern.get("conversion"),
        "host_call_ms_pageable": host_ms, "cpu_host_build_s_scaled": cpu_s, "cpu_threads": threads,
        "cpu_sample": len(picks), "reps": args.reps,
        "statuses": np.bincount(res.status, minlength=5).tolist(),
        "methods": {int(k): int(v) for k, v in zip(*np.unique(res.method, return_counts=True))},
        "card": _card()}))


if __name__ == "__main__":
    main()
