"""K16 manoeuvre-trial timing (astroz_cuda_conjunction_maneuver[_device]) and the avoidance planner.

    python tools/avoidance_timing.py [--reps 3] [--workloads AV1,AV2] [--host-subset 256]

AV1: tools/conjunction_mc_timing.py's 1,000 LEO crossings (MC1, +-1 min) x 8 leads x 2 signs x 32 tangential
magnitudes (geometric, 1 m/s down by halves), 512,000 trials; AV2: its 100 GEO crossings (MC2, +-30 min), same trial
shape.  Per workload: device ms of the _device call (CUDA events, best of --reps and the spread), trials per second,
each stage's kernel time from torch.profiler in a run of its own (the two covariance passes, the conversion fit, K11
and the avoid_* kernels), the host call's ms from pageable and from pinned buffers, and the host build
(tests/host_emul/emul_avoid.cu) on 8 threads, each running a share of --host-subset trials, scaled to the workload.
Then the planner on AV1 (rounds 20, pc_max 1e-6).  Prints one JSON record per line, with the card, power limit and
maximum SM clock read in the same run.
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

from conjunction_is_timing import _event_ms  # noqa: E402
from conjunction_mc_timing import _workloads  # noqa: E402
from conjunction_timing import _card, _covariances  # noqa: E402

LEADS = 8
LADDER = 32


def _trials(el, pr, jd, fr, w):
    """(candidate, burn_jd, burn_fr, dv (t, 3)): every candidate x 8 leads (0.5 .. 4 orbits before the window) x 2 signs
    x 32 tangential magnitudes"""
    m = len(pr)
    period = 1.0 / el[1, pr]
    c, l, s, k = (a.reshape(-1) for a in np.meshgrid(np.arange(m), np.arange(LEADS), np.arange(2), np.arange(LADDER),
                                                       indexing="ij"))
    mags = 1e-3 * 2.0 ** (np.arange(LADDER) - (LADDER - 1))
    dv = np.zeros((len(c), 3))
    dv[:, 1] = np.where(s == 0, -1.0, 1.0) * mags[k]
    return c, jd[c], fr[c] - w / 1440.0 - 0.5 * (l + 1) * period[c], dv


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default="AV1,AV2")
    ap.add_argument("--host-subset", type=int, default=256)
    args = ap.parse_args()
    import torch

    from astroz_b200.collision import avoidance, maneuver_trials, maneuver_trials_device, maneuver_trials_scratch_bytes
    from tests.fit_oracle import avoid as av

    card = _card()
    dev = torch.device("cuda:0")
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
    L = av.emul_library()
    wl = {"AV1": _workloads()[0], "AV2": _workloads()[1]}
    for name in args.workloads.split(","):
        _, el, pr, se, jd, fr, w, deep, _ = wl[name]
        n, m = el.shape[1], len(pr)
        model = np.full(n, deep, np.uint8)
        P = _covariances(n, model.astype(bool))
        ca, bj, bf, dv = _trials(el, pr, jd, fr, w)
        T = len(ca)
        ins = [t(el), t(P), t(model, torch.uint8), t(pr, torch.int32), t(se, torch.int32), t(jd), t(fr),
               t(np.full(m, w)), t(np.full(m, 0.02)), t(ca, torch.int32), t(bj), t(bf), t(dv), None]
        outs = [torch.zeros((T, 13), dtype=torch.float64, device=dev), None, None, None,
                torch.zeros(T, dtype=torch.uint8, device=dev)]
        scratch = torch.empty(maneuver_trials_scratch_bytes(T), dtype=torch.uint8, device=dev)
        run = lambda: maneuver_trials_device(*ins, *outs, scratch)  # noqa: E731
        ms = _event_ms(run, args.reps)
        st = np.bincount(outs[4].cpu().numpy(), minlength=9).tolist()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            key = e.key.split("(")[0]
            if key.startswith(("az::", "void az::")):
                kern[key.replace("void ", "")] = round(getattr(e, "device_time_total",
                                                               getattr(e, "cuda_time_total", 0)) / 1e3, 3)
        host_ms = {}
        for label, pin in (("pageable", False), ("pinned", True)):
            arr = [el, P, bj, bf, dv]
            if pin:
                arr = [torch.as_tensor(np.ascontiguousarray(a)).pin_memory().numpy() for a in arr]
            call = lambda: maneuver_trials(arr[0], pr, se, jd, fr, window_min=w, hbr_km=0.02, candidate=ca,  # noqa: E731
                                           burn_jd=arr[2], burn_fr=arr[3], dv_rtn=arr[4], covariance=arr[1],
                                           model=model)
            call()
            best = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                call()
                best.append((time.perf_counter() - t0) * 1e3)
            host_ms[label] = round(min(best), 2)
        sub = np.random.default_rng(1).choice(T, min(args.host_subset, T), replace=False)
        parts = np.array_split(sub, 8)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(8) as ex:
            list(ex.map(lambda s: av.emul(L, el, P, model, pr, se, jd, fr, w, 0.02, ca[s], bj[s], bf[s], dv[s]),
                        parts))
        host8 = (time.perf_counter() - t0) * T / len(sub)
        print(json.dumps({"workload": name, "trials": T, "device_ms_best": round(min(ms), 2),
                          "device_ms_spread": round(max(ms) - min(ms), 2),
                          "trials_per_s": f"{T / (min(ms) * 1e-3):.3e}", "kernel_ms": kern, "host_call_ms": host_ms,
                          "host_build_8_threads_s_scaled": round(host8, 1), "statuses": st,
                          "card": card[0], "power_limit": card[1], "max_sm_clock": card[2]}), flush=True)
    # the planner on AV1
    _, el, pr, se, jd, fr, w, deep, _ = wl["AV1"]
    n = el.shape[1]
    P = _covariances(n, np.zeros(n, bool))
    t0 = time.perf_counter()
    r = avoidance(el, pr, se, jd, fr, window_min=w, hbr_km=0.02, lead_min=w + 0.5 * (np.arange(LEADS) + 1) * 95.0,
                  pc_max=1e-6, dv_max_kms=1e-3, ladder=LADDER, rounds=20, covariance=P, model=np.zeros(n, np.uint8))
    s = time.perf_counter() - t0
    print(json.dumps({"workload": "planner AV1, 20 rounds", "s": round(s, 2),
                      "found": int(np.isfinite(r.dv_kms).sum()), "cells": int(r.dv_kms.size),
                      "nominal_above_target": int((r.pc_nominal > 1e-6).sum()),
                      "card": card[0], "power_limit": card[1]}), flush=True)


if __name__ == "__main__":
    main()
