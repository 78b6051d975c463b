#!/usr/bin/env python
"""K7 maneuver timing (DESIGN.md section 3 "K7 maneuvers"): one JSON line.

    python tools/maneuver_timing.py [--n1 20000] [--n2 10000] [--reps 3] [--sample 256]

M1: n1 LEO states (a Monte-Carlo catalogue's TEME states at one epoch), each with three prograde burns at dispersed
times and magnitudes, the Spacecraft force set (TwoBody + J2 + Drag: cd 2.2, 0.05 m^2, 300 kg, cut-off 1000 km), RK4 at
10 s over one day.  M2: n2 LEO states, one phasing maneuver each at 1 h, the angle swept over [-0.1, 0.1] rad (wider
phasing orbits of these LEO states dip into the dense atmosphere or the Earth), DP87 over one day at 60 s.  M3: M1's
states with empty schedules, alternated with the model-list kernel on the same states: the price of the maneuver loop
itself, and the bytes compared.  C: the threaded scalar restatement on --sample states of M1
and M2, scaled to the full batch.
Device times are CUDA events around the device call after a warm-up call, best of --reps; divergence is the warp's
largest step count over its mean, averaged over warps.  The card name, power limit and max SM clock are read in the same
run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MU, R_EQ, J2 = 398600.5, 6378.137, 0.00108262998905


def spacecraft():
    from astroz_b200 import numerical as P

    return [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.Drag(R_EQ, 1.225, 7.249, 2.2, 0.05, 300.0, 1000.0)]


def device_ms(fn, reps):
    import torch

    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def divergence(steps):
    s = steps.sum(axis=1).astype(np.float64)
    s = s[: len(s) // 32 * 32].reshape(-1, 32)
    return round(float(np.mean(s.max(axis=1) / np.maximum(s.mean(axis=1), 1))), 3)


def run(y, duration, h, models, sched, integrator, reps):
    """The C device call on tensors and schedules uploaded once (the timed window holds the kernel alone); rows sized
    by the wrapper's estimate"""
    import ctypes as C

    import torch

    from astroz_b200 import numerical as P
    from astroz_b200._lib import check, lib

    dev = torch.device("cuda", 0)
    n = len(y)
    off, imp = P.pack_schedules(sched, n)
    S = P._estimate_samples(y, 0.0, duration, h, off, imp, MU)
    ds = torch.from_numpy(np.ascontiguousarray(y)).to(dev)
    d_off = torch.from_numpy(off.view(np.int32)).to(dev)
    d_imp = torch.from_numpy(imp.view(np.uint8)).to(dev)
    times = torch.empty((n, S), dtype=torch.float64, device=dev)
    out = torch.empty((n, S, 6), dtype=torch.float64, device=dev)
    cnt = torch.empty(n, dtype=torch.int64, device=dev)
    st = torch.empty(n, dtype=torch.uint8, device=dev)
    steps = torch.empty((n, 2), dtype=torch.int64, device=dev)
    descs, keep = P._descriptors(models, n, 0, P._host_array)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    call = lambda: check(lib().astroz_cuda_propagate_maneuvers_device(  # noqa: E731
        p(ds), n, 0.0, duration, h, MU, p(d_off), p(d_imp), len(imp), C.cast(descs, C.c_void_p), len(descs),
        P._integrator(integrator), 1e-9, 1e-12, S, 0, p(times), p(out), p(cnt), p(st), p(steps), None))
    ms = device_ms(call, reps)
    c, s, k = cnt.cpu().numpy(), st.cpu().numpy(), steps.cpu().numpy()
    best = min(ms)
    res = {"n": n, "row_samples": S, "samples": int(c.sum()), "device_ms": round(best, 3),
           "device_ms_all": [round(x, 3) for x in ms], "state_samples_per_s": round(float(c.sum()) / best * 1e3, 1),
           "accepted": int(k[:, 0].sum()), "rejected": int(k[:, 1].sum()), "warp_max_over_mean_steps": divergence(k),
           "status_counts": np.bincount(s, minlength=6).tolist()}
    del times, out, keep
    torch.cuda.empty_cache()
    return res


def price_loop(y, reps):
    """M3: empty schedules against the model-list kernel, alternated, bytes compared"""
    import torch

    from astroz_b200 import numerical as P

    dev = torch.device("cuda", 0)
    n = len(y)
    K = len(P.numerical_times(0.0, 86400.0, 10.0))
    ds = torch.from_numpy(np.ascontiguousarray(y)).to(dev)
    a = [torch.empty((n, K, 6), dtype=torch.float64, device=dev), torch.empty(n, dtype=torch.uint8, device=dev),
         torch.empty((n, 2), dtype=torch.int64, device=dev)]
    b = [torch.empty((n, K), dtype=torch.float64, device=dev), torch.empty((n, K, 6), dtype=torch.float64, device=dev),
         torch.empty(n, dtype=torch.int64, device=dev), torch.empty(n, dtype=torch.uint8, device=dev),
         torch.empty((n, 2), dtype=torch.int64, device=dev)]
    models = spacecraft()
    import ctypes as C

    from astroz_b200._lib import check, lib

    d_off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    descs, keep = P._descriptors(models, n, 0, P._host_array)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    lst = lambda: check(lib().astroz_cuda_propagate_numerical_models_device(  # noqa: E731
        p(ds), n, 0.0, 86400.0, 10.0, C.cast(descs, C.c_void_p), len(descs), 0, 1e-9, 1e-12, 0, *[p(t) for t in a],
        None))
    man = lambda: check(lib().astroz_cuda_propagate_maneuvers_device(  # noqa: E731
        p(ds), n, 0.0, 86400.0, 10.0, MU, p(d_off), None, 0, C.cast(descs, C.c_void_p), len(descs), 0, 1e-9, 1e-12, K,
        0, *[p(t) for t in b], None))
    ms = {"models": [], "maneuvers": []}
    for _ in range(reps):
        ms["models"] += device_ms(lst, 1)
        ms["maneuvers"] += device_ms(man, 1)
    same = bool(torch.equal(a[0].view(torch.int64), b[1].view(torch.int64)) and torch.equal(a[1], b[3]) and
                torch.equal(a[2], b[4]))
    res = {"n": n, "samples": K, "models_ms": round(min(ms["models"]), 3), "maneuvers_ms": round(min(ms["maneuvers"]), 3),
           "models_ms_all": [round(x, 3) for x in ms["models"]],
           "maneuvers_ms_all": [round(x, 3) for x in ms["maneuvers"]], "bytes_identical": same}
    res["maneuvers_over_models"] = round(res["maneuvers_ms"] / res["models_ms"], 3)
    del a, b, keep
    torch.cuda.empty_cache()
    return res


def restatement(y, duration, h, models, sched, integrator, n_full, threads):
    from tests.numerical_oracle import maneuvers as R

    t = time.perf_counter()
    R.propagate(y, 0.0, duration, h, models, sched, integrator=integrator, k7_forms=True, threads=threads)
    s = time.perf_counter() - t
    return {"sample": len(y), "threads": threads, "seconds": round(s, 3),
            "scaled_to_batch_s": round(s * n_full / len(y), 2)}


def main():
    from astroz_b200 import numerical as P, synth
    from tools.numerical_timing import teme_states

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    rng = np.random.default_rng(0)
    out = {"card_power_limit_max_sm_clock": card, "reps": ARGS.reps}
    y1 = teme_states(synth.monte_carlo_catalog(ARGS.n1), synth.BENCH_JD0, 0.0)
    s1 = [[P.Prograde(t, dv) for t, dv in zip(np.sort(rng.uniform(0, 86400, 3)), rng.uniform(-0.01, 0.01, 3))]
          for _ in range(len(y1))]
    out["M1"] = run(y1, 86400.0, 10.0, spacecraft(), s1, "rk4", ARGS.reps)
    y2 = teme_states(synth.monte_carlo_catalog(ARGS.n2, seed=777), synth.BENCH_JD0, 0.0)
    s2 = [[P.Phase(3600.0, a, 1.0)] for a in np.linspace(-0.1, 0.1, len(y2))]
    out["M2"] = run(y2, 86400.0, 60.0, spacecraft(), s2, "dp87", ARGS.reps)
    out["M3"] = price_loop(y1, ARGS.reps)
    threads = os.cpu_count() or 1
    k = ARGS.sample
    out["C"] = {"M1": restatement(y1[:k], 86400.0, 10.0, spacecraft(), s1[:k], "rk4", len(y1), threads),
                "M2": restatement(y2[:k], 86400.0, 60.0, spacecraft(), s2[:k], "dp87", len(y2), threads)}
    print(json.dumps(out))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--n1", type=int, default=20000)
    ap.add_argument("--n2", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=256)
    ARGS = ap.parse_args()
    main()
