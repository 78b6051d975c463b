"""K17 track-linking timing (astroz_cuda_link_tracks[_device]).

    python tools/link_timing.py [--objects 300] [--max-gap 1.5] [--reps 3] [--cpu-sample 400] [--cpu-threads N]

Workload: 2 x --objects optical tracks of GEO rows of a synthetic catalogue (tests/fit_oracle/link.py's geo_tracks: 12
observations at 300 s, one track on each of two consecutive days, 1" noise, from propagate_pairs states), every pair of
tracks whose anchors are at most --max-gap days apart, max_revs = 1.  Prints one JSON record: the device call's time
(CUDA events around astroz_cuda_link_tracks_device, best of --reps and the spread), split into the link kernel and the
conversion (the K8 fits and the finishing kernel) by torch.profiler kernel times; pairs/s; Lambert problems/s (32 x 32
ranges x 2 directions per optical pair, each solving 2 max_revs + 1 slots) and admissible states scored/s; the host call
(pageable buffers); the host build of the same source (tests/host_emul/emul_link.cu) on --cpu-threads host threads
(default: every usable CPU) over --cpu-sample pairs, scaled to the workload; statuses; how many true pairs (one object's
two tracks) end at a two-body wrms below 3, a measure of whether the range grid seeds their refinement well enough; and
the card, power limit and maximum SM clock read in the same run.
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
    ap.add_argument("--objects", type=int, default=300)
    ap.add_argument("--max-gap", type=float, default=1.5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-sample", type=int, default=400)
    ap.add_argument("--cpu-threads", type=int, default=len(os.sched_getaffinity(0)))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from astroz_b200.iod import (LINK_R_MAX, LINK_R_MIN, anchor_times, candidate_pairs, link_tracks, link_tracks_device,
                                 link_tracks_scratch_bytes)
    from tests.fit_oracle import link as K

    tr, owner = K.geo_tracks(args.objects, 41)
    pairs = candidate_pairs(anchor_times(tr.track_ids(), tr.jd, tr.fr, tr.kind, tr.sigma), args.max_gap)
    p = len(pairs)
    d = torch.device("cuda", 0)
    cu = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a)).to(dt).to(d)  # noqa: E731
    ins = (cu(tr.offsets.astype(np.int32), torch.int32), cu(tr.jd, torch.float64), cu(tr.fr, torch.float64),
           cu(tr.kind, torch.uint8), cu(tr.value, torch.float64), cu(tr.sigma, torch.float64),
           cu(tr.station.astype(np.int32), torch.int32), cu(tr.stations, torch.float64),
           cu(pairs.astype(np.int32), torch.int32), None)
    f64 = lambda *s: torch.zeros(s, dtype=torch.float64, device=d)  # noqa: E731
    u8 = lambda: torch.zeros(p, dtype=torch.uint8, device=d)  # noqa: E731
    i32 = lambda: torch.zeros(p, dtype=torch.int32, device=d)  # noqa: E731
    out = dict(elements=f64(8, p), state=f64(p, 6), rho=f64(p, 2), revs=u8(), flags=u8(), wrms=f64(p), used=i32(),
               hypotheses=i32(), conv=f64(p, 2), deep_space=u8(), status=u8())
    scratch = torch.zeros(link_tracks_scratch_bytes(p), dtype=torch.uint8, device=d)
    run = lambda: link_tracks_device(*ins, scratch, **out)  # noqa: E731
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
            key = "link_kernel" if "link_kernel" in e.name else "conversion"
            kern[key] = kern.get(key, 0.0) + e.device_time / 1000.0
    t0 = time.perf_counter()
    res = link_tracks(tr.track_ids(), tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station, tr.stations, pairs,
                      r_min=LINK_R_MIN, r_max=LINK_R_MAX)
    host_ms = (time.perf_counter() - t0) * 1e3
    from concurrent.futures import ThreadPoolExecutor

    L = K.emul_library()
    picks = np.random.default_rng(0).choice(p, min(args.cpu_sample, p), replace=False)
    parts = [q for q in np.array_split(picks, args.cpu_threads) if len(q)]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(len(parts)) as ex:
        list(ex.map(lambda q: K.emul(L, tr, pairs[q], LINK_R_MIN, LINK_R_MAX), parts))
    cpu_s = (time.perf_counter() - t0) * p / len(picks)
    best = min(times) / 1e3
    problems = 32 * 32 * 2 * p
    true = owner[pairs[:, 0]] == owner[pairs[:, 1]]
    ok = res.status == 0
    print(json.dumps({
        "workload": "GEO optical track pairs", "tracks": tr.t, "pairs": p, "max_gap_days": args.max_gap,
        "max_revs": 1, "device_ms_best": min(times), "device_ms_spread": max(times) - min(times),
        "link_kernel_ms": kern.get("link_kernel"), "conversion_ms": kern.get("conversion"),
        "pairs_per_s": p / best, "lambert_problems_per_s": problems / best, "lambert_slots_per_s": 3 * problems / best,
        "admissible_states_per_s": float(res.hypotheses.sum()) / best,
        "hypotheses_per_pair_mean": float(res.hypotheses.mean()),
        "host_call_ms_pageable": host_ms, "cpu_host_build_s_scaled": cpu_s, "cpu_threads": args.cpu_threads,
        "cpu_sample": len(picks), "reps": args.reps, "statuses": np.bincount(res.status, minlength=6).tolist(),
        "true_pairs": int(true.sum()), "true_pairs_ok": int((true & ok).sum()),
        "true_pairs_wrms_below_3": int((true & ok & (res.wrms < 3.0)).sum()),
        "other_pairs_wrms_below_3": int((~true & ok & (res.wrms < 3.0)).sum()),
        "card": _card()}))


if __name__ == "__main__":
    main()
