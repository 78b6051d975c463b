"""K19 reentry prediction timing (astroz_cuda_reentry[_device]).

    python tools/reentry_timing.py [--reps 3] [--budget-s 300] [--cpu-threads 16] [--workloads RE1,RE2]

Workloads:
  RE1  1,000 synthetic near-earth rows with perigees of 150-300 km (apogee up to 200 km higher, B* 5e-5 .. 5e-4, a
       diagonal covariance at a fitted row's scale with a 10 % B* spread) x 1,000 samples, density_sigma 0.2, 60 days;
  RE2  the nominals of the config-2 catalogue (13,478 near-earth rows, astroz_b200.synth) over 30 days: every
       trajectory runs to the horizon, the horizon-bound case.
Prints one JSON record per workload: device ms (CUDA events around the device call after one warm-up call, best of
--reps, and the spread), trajectories / s, DP87 attempts (sums over every trajectory, from the words the call returns),
warp divergence (max over mean attempts per work item: 32 consecutive samples of a row, or 32 consecutive nominals),
the fp64 rate from the FLOP count fixed below, the host build (tests/host_emul/emul_reentry.cu) on --cpu-threads
threads over a subset scaled to the workload's trajectories, and the card, power limit and maximum SM clock read in the
same run.  When a first timing of one tenth of RE1's rows says a call would exceed --budget-s, RE1 is timed on that
tenth and the record says so.

FLOP count, fixed before measuring (fp64 add, mul, div, sqrt each 1; exp 20; the 27 band compares not counted):
  force evaluation: two-body + J2 22, co-rotating drag 16, geodetic height 40, density 24: 102;
  DP87 attempt: 13 evaluations, the stage sums 2 x 6 per non-zero a_ij (59), the 8th / 7th-order sums 2 x 6 per
  non-zero weight (9 + 8), the error norm 6 x 6: 13 x 102 + 708 + 204 + 36 = 2,274.
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

FLOP_PER_ATTEMPT = 13 * 102 + 2 * 6 * 59 + 2 * 6 * 17 + 36


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def _re1(rows=1000, seed=21):
    from tests.test_gpu_reentry import scene

    rng = np.random.default_rng(seed)
    el, P, md = scene(n_leo=rows, n_gto=0, seed=seed)
    hp = rng.uniform(150, 300, rows)   # perigees of 150-300 km in place of the scene's
    from tests.test_reentry_cpu import leo
    for i in range(rows):
        e = el[:, i]
        el[:, i] = leo(hp[i], hp[i] + rng.uniform(0, 200), incl=e[3], node=e[4], argp=e[5], ma=e[6], bstar=e[7])
    return dict(el=el, P=P, md=md, samples=1000, horizon=60.0, sigma=0.2)


def _re2():
    from astroz_b200 import synth

    el = synth.elements_from_tles(synth.near_earth_catalog(13478))
    n = el.shape[1]
    return dict(el=el, P=np.zeros((n, 28)), md=np.zeros(n, np.uint8), samples=0, horizon=30.0, sigma=0.0)


def _device(w, reps):
    import torch

    from astroz_b200.reentry import predict_device, predict_scratch_bytes

    d = torch.device("cuda", 0)
    g = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=d)  # noqa: E731
    el, P, md, S = w["el"], w["P"], w["md"], w["samples"]
    m = el.shape[1]
    rec, nst, st = torch.zeros((m, 8), dtype=torch.float64, device=d), torch.zeros(m, dtype=torch.uint8, device=d), \
        torch.zeros(m, dtype=torch.uint8, device=d)
    counts = torch.zeros((m, 3), dtype=torch.int64, device=d)
    so = torch.zeros((m, S, 4), dtype=torch.float64, device=d) if S else None
    args = [g(el), g(P), g(md, torch.uint8), g(np.arange(m), torch.int32), None, g(np.full(m, S), torch.int64), None,
            g(np.full(m, 7), torch.int64), rec, None, nst, counts, so, st,
            torch.zeros(predict_scratch_bytes(m), dtype=torch.uint8, device=d)]
    kw = dict(interface_km=80.0, horizon_days=w["horizon"], density_sigma=w["sigma"])
    predict_device(*args, **kw)   # warm-up: module load, scan tuning
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        predict_device(*args, **kw)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return ms, rec.cpu().numpy(), counts.cpu().numpy(), None if so is None else so.cpu().numpy(), st.cpu().numpy()


def _divergence(rec, so):
    """max over mean attempts per work item, and the attempts per item"""
    items = []
    if so is not None:
        att = so[:, :, 3]
        for row in att:
            for q in range(0, len(row), 32):
                items.append(row[q:q + 32])
    nom = rec[:, 6] + rec[:, 7]
    for q in range(0, len(nom), 32):
        items.append(nom[q:q + 32])
    ratio = np.array([it.max() / it.mean() for it in items if it.mean() > 0])
    return float(ratio.mean()), float(np.percentile(ratio, 99))


def _host(w, rows, threads):
    from tests.fit_oracle import reentry as ro

    L = ro.emul_library()
    el, P, md = w["el"][:, :rows], w["P"][:rows], w["md"][:rows]
    S = min(w["samples"], 32)
    t0 = time.perf_counter()
    ro.emul(L, el, P, md, np.arange(rows), samples=S, horizon_days=w["horizon"], sigma=w["sigma"], seed=7,
            threads=threads)
    dt = time.perf_counter() - t0
    per = dt / (rows * (1 + S))
    return per * w["el"].shape[1] * (1 + w["samples"]), rows, S


def run(name, w, reps, budget, threads):
    out = dict(workload=name, card=_card())
    m = w["el"].shape[1]
    if name == "RE1":
        tenth = dict(w, el=w["el"][:, : m // 10], P=w["P"][: m // 10], md=w["md"][: m // 10])
        ms, *_ = _device(tenth, 1)
        est = min(ms) * 10 / 1e3
        out["estimate_full_s"] = est
        if est > budget:
            w, m = tenth, m // 10
            out["scaled"] = f"timed on {m} rows (one tenth): a full call was estimated at {est:.0f} s"
    ms, rec, counts, so, st = _device(w, reps)
    traj = m * (1 + w["samples"])
    att = float((rec[:, 6] + rec[:, 7]).sum() + (0 if so is None else so[:, :, 3].sum()))
    best = min(ms)
    div_mean, div_p99 = _divergence(rec, so)
    host_s, hrows, hs = _host(w, 16 if name == "RE1" else 64, threads)
    out.update(rows=m, samples=w["samples"], horizon_days=w["horizon"], device_ms=best,
               spread=(max(ms) - best) / best, trajectories_per_s=traj / (best / 1e3), attempts=att,
               attempts_per_trajectory=att / traj, divergence_mean=div_mean, divergence_p99=div_p99,
               fp64_tflops=att * FLOP_PER_ATTEMPT / (best / 1e3) / 1e12,
               counts=[int(x) for x in counts.sum(0)], nominal_reentered=int((rec[:, 0] < np.inf).sum()),
               host_build_s=host_s, host_build_subset=f"{hrows} rows x {hs} samples, {threads} threads, scaled",
               status_ok=int((st == 0).sum()))
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--budget-s", type=float, default=300.0)
    ap.add_argument("--cpu-threads", type=int, default=16)
    ap.add_argument("--workloads", default="RE1,RE2")
    a = ap.parse_args()
    for name in a.workloads.split(","):
        run(name, _re1() if name == "RE1" else _re2(), a.reps, a.budget_s, a.cpu_threads)


if __name__ == "__main__":
    main()
