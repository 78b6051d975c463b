#!/usr/bin/env python
"""K7 timing (DESIGN.md section 3 "K7 numerical"): one JSON line.

    python tools/numerical_timing.py [--n 100000] [--reps 3] [--cpu-states 200]

N1: n LEO states (synth.monte_carlo_catalog turned into TEME states at epoch with propagate_pairs), J2 + drag with the
ballistic coefficient dispersed per state, one day at dt 60 s, DP87 at the default tolerances.  N2: N1 with RK4 at
dt 10 s.  N3: the config-2 catalogue's TEME states at the headline epoch, J2 only, one day at 60 s, DP87.
Per workload: device time from CUDA events after a warm-up call, state-samples/s, accepted / rejected steps, divergence
(per warp of 32 consecutive states, max attempts / mean attempts, averaged over warps), fp64 FLOP/s from the per-stage
count fixed in DESIGN.md against astroz_cuda_fp64_pipe_peak, and the threaded C restatement's time on a subset.
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

MU, R_EQ, J2 = 398600.5, 6378.137, 0.00108262998905
# fp64 operations per stage (DESIGN.md section 3 "K7 numerical"): a derivative costs 15 (two-body: 5 mul/add for r^2,
# sqrt, 3 for r^3 and the division, 3 products), J2 adds 22, drag adds 24 (its exp counted as 10); a DP87 stage adds
# 2 x 6 per tableau weight, an RK4 stage 2 x 6
DERIV = {0: 15, 1: 37, 2: 39, 3: 61}
DP87_WEIGHTS = 78 + 8 + 7   # non-zero a, b8, b7
RK4_COMBINE = 4 * 12 + 30


def teme_states(tles, jd, fr):
    import astroz_b200

    c = astroz_b200.Constellation(tles)
    n = len(tles)
    pos, vel, _ = c.propagate_pairs(np.arange(n, dtype=np.uint32), np.full(n, jd), np.full(n, fr))
    return np.concatenate([pos, vel], axis=1)


def run(y, forces, integrator, dt, drag, reps, peak):
    import torch

    from astroz_b200 import numerical
    from tests import numerical_oracle as N

    dev = torch.device("cuda", 0)
    n = len(y)
    samples = len(numerical.numerical_times(0.0, 86400.0, dt))
    ds = torch.from_numpy(np.ascontiguousarray(y)).to(dev)
    out = torch.empty((n, samples, 6), dtype=torch.float64, device=dev)
    st = torch.empty(n, dtype=torch.uint8, device=dev)
    steps = torch.empty((n, 2), dtype=torch.int64, device=dev)
    kw = dict(j2=J2 if forces & 1 else None, r_eq=R_EQ, integrator=integrator)
    if forces & 2:
        kw.update(drag_cd=torch.full((n,), 2.2, dtype=torch.float64, device=dev),
                  drag_area=torch.from_numpy(drag).to(dev), drag_mass=torch.full((n,), 500.0, dtype=torch.float64,
                                                                                    device=dev))
    numerical.propagate_numerical_batch_device(ds, 0.0, 86400.0, dt, MU, out, st, steps, **kw)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        e0.record()
        numerical.propagate_numerical_batch_device(ds, 0.0, 86400.0, dt, MU, out, st, steps, **kw)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    cnt = steps.cpu().numpy()
    status = np.bincount(st.cpu().numpy(), minlength=4).tolist()
    att = cnt.sum(axis=1).astype(np.float64)
    w = att[: n // 32 * 32].reshape(-1, 32)
    divergence = float(np.mean(w.max(axis=1) / np.maximum(w.mean(axis=1), 1)))
    stages = 13 if integrator == "dp87" else 4
    per_attempt = stages * DERIV[forces] + (DP87_WEIGHTS * 12 + 40 if integrator == "dp87" else RK4_COMBINE)
    flops = float(att.sum()) * per_attempt
    best = min(ms)
    res = {"n": n, "samples": samples, "device_ms": round(best, 3), "device_ms_all": [round(x, 3) for x in ms],
           "state_samples_per_s": round(n * samples / best * 1e3, 1), "accepted": int(cnt[:, 0].sum()),
           "rejected": int(cnt[:, 1].sum()), "status_counts": status, "divergence_max_over_mean": round(divergence, 3),
           "fp64_tflops": round(flops / best * 1e-9, 3), "fp64_share_of_pipe_peak": round(flops / best * 1e-9 / peak, 4)}
    sub = min(n, ARGS.cpu_states)
    threads = len(os.sched_getaffinity(0))
    t0 = time.perf_counter()
    dk = dict(drag_cd=2.2, drag_area=drag[:sub], drag_mass=500.0) if forces & 2 else {}
    N.propagate(y[:sub], 0.0, 86400.0, dt, MU, j2=J2 if forces & 1 else None, r_eq=R_EQ, integrator=integrator,
                threads=threads, **dk)
    cpu = time.perf_counter() - t0
    res["cpu_restatement"] = {"states": sub, "threads": threads, "s": round(cpu, 3),
                              "s_scaled_to_n": round(cpu * n / sub, 2)}
    return res


def main():
    import astroz_b200
    from astroz_b200 import synth

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    peak = astroz_b200.fp64_pipe_peak_tflops()
    rng = np.random.default_rng(0)
    jd0 = synth.BENCH_JD0
    mc = synth.monte_carlo_catalog(ARGS.n)
    y1 = teme_states(mc, jd0, 0.0)
    area = rng.uniform(1.0, 20.0, len(y1))
    out = {"card_power_limit_max_sm_clock": card, "fp64_pipe_peak_tflops": round(peak, 2), "reps": ARGS.reps}
    out["N1"] = run(y1, 3, "dp87", 60.0, area, ARGS.reps, peak)
    out["N2"] = run(y1, 3, "rk4", 10.0, area, ARGS.reps, peak)
    y3 = teme_states(synth.near_earth_catalog(synth.HEADLINE_SATS, seed=13478), jd0, 0.0)   # bench.py's config2
    out["N3"] = run(y3, 1, "dp87", 60.0, np.ones(len(y3)), ARGS.reps, peak)
    print(json.dumps(out))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-states", type=int, default=200)
    ARGS = ap.parse_args()
    main()
