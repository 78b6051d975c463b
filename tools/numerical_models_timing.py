#!/usr/bin/env python
"""K7 model-list timing (DESIGN.md section 3 "K7 model lists"): one JSON line.

    python tools/numerical_models_timing.py [--n 100000] [--reps 3]

F1: n dispersed GEO states, TwoBody + J2 + SRP + Sun + Moon, the Sun and Moon as per-interval tables from seeded circular
orbits (test data, not an ephemeris), DP87, 7 days at 300 s.  F2: n LEO states, TwoBody + J2 + J3 + J4 + ImprovedDrag with
per-state cd, area and mass, DP87, one day at 60 s.  F3: tools/numerical_timing.py's N1 (J2 + drag, DP87) and N3 (J2,
DP87) through the list path and through the fixed kernels, alternated, with the bytes compared.
Device times are CUDA events around the device call after a warm-up call, best of --reps; the card name, power limit and
max SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MU, R_EQ, J2, J3, J4 = 398600.5, 6378.137, 0.00108262998905, -0.00000253215306, -0.00000161098761
SUN_MU, MOON_MU, AU = 1.32712e11, 4902.80, 1.495978707e8
# fp64 operations per model evaluation, counted from az_numerical.cuh's model_accel (exp counted as 10, sqrt and division
# as 1) plus 3 for the Composite sum; a derivative is the sum over the list.  A DP87 attempt adds 2 x 6 per tableau
# weight and 40 for the error norm, as in tools/numerical_timing.py.
MODEL_FLOP = {"TwoBody": 15, "J2": 25, "J3": 34, "J4": 36, "Drag": 31, "ImprovedDrag": 43,
              "SolarRadiationPressure": 47, "ThirdBody": 34}
DP87_WEIGHTS = 78 + 8 + 7


def device_call(fn, reps):
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


def summary(ms, n, samples, steps, st, models):
    cnt = steps.cpu().numpy()
    att = float(cnt.sum())
    per_attempt = 13 * sum(MODEL_FLOP[type(m).__name__] + 3 for m in models) + DP87_WEIGHTS * 12 + 40
    best = min(ms)
    return {"n": n, "samples": samples, "device_ms": round(best, 3), "device_ms_all": [round(x, 3) for x in ms],
            "state_samples_per_s": round(n * samples / best * 1e3, 1), "accepted": int(cnt[:, 0].sum()),
            "rejected": int(cnt[:, 1].sum()),
            "status_counts": np.bincount(st.cpu().numpy(), minlength=4).tolist(),
            "fp64_tflops": round(att * per_attempt / best * 1e-9, 3)}


def tables(K, dt):
    t = np.arange(K) * dt
    rng = np.random.default_rng(42)
    ps, pm = rng.uniform(0, 2 * math.pi, 2)
    ws, wm = 2 * math.pi / (365.25 * 86400), 2 * math.pi / (27.32 * 86400)
    sun = AU * np.stack([np.cos(ws * t + ps), 0.917 * np.sin(ws * t + ps), 0.398 * np.sin(ws * t + ps)], axis=1)
    moon = 384400.0 * np.stack([np.cos(wm * t + pm), 0.91 * np.sin(wm * t + pm), 0.41 * np.sin(wm * t + pm)], axis=1)
    return sun, moon


def run_models(y, duration, dt, make_models, reps):
    import torch

    from astroz_b200 import numerical as P

    dev = torch.device("cuda", 0)
    n = len(y)
    samples = len(P.numerical_times(0.0, duration, dt))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    models = make_models(samples - 1, T)
    ds = T(y)
    out = torch.empty((n, samples, 6), dtype=torch.float64, device=dev)
    st = torch.empty(n, dtype=torch.uint8, device=dev)
    steps = torch.empty((n, 2), dtype=torch.int64, device=dev)
    ms = device_call(lambda: P.propagate_models_batch_device(ds, 0.0, duration, dt, models, out, st, steps), reps)
    res = summary(ms, n, samples, steps, st, models)
    del out
    torch.cuda.empty_cache()
    return res


def geo_states(n, rng):
    a = 42164.0 * (1 + 1e-4 * rng.standard_normal(n))
    lon = rng.uniform(0, 2 * math.pi, n)
    inc = np.radians(rng.uniform(0, 0.1, n))
    v = np.sqrt(MU / a)
    return np.stack([a * np.cos(lon), a * np.sin(lon) * np.cos(inc), a * np.sin(lon) * np.sin(inc),
                     -v * np.sin(lon), v * np.cos(lon) * np.cos(inc), v * np.cos(lon) * np.sin(inc)], axis=1)


def compare_paths(y, forces, area, reps):
    """One workload through the list path and the fixed kernel, alternated; returns both summaries and byte equality"""
    import torch

    from astroz_b200 import numerical as P

    dev = torch.device("cuda", 0)
    n = len(y)
    samples = len(P.numerical_times(0.0, 86400.0, 60.0))
    ds = torch.from_numpy(np.ascontiguousarray(y)).to(dev)
    outs = [torch.empty((n, samples, 6), dtype=torch.float64, device=dev) for _ in range(2)]
    sts = [torch.empty(n, dtype=torch.uint8, device=dev) for _ in range(2)]
    stp = [torch.empty((n, 2), dtype=torch.int64, device=dev) for _ in range(2)]
    kw = dict(j2=J2, r_eq=R_EQ)
    models = [P.TwoBody(MU), P.J2(MU, J2, R_EQ)]
    if forces & 2:
        dd = [torch.full((n,), 2.2, dtype=torch.float64, device=dev), torch.from_numpy(area).to(dev),
              torch.full((n,), 500.0, dtype=torch.float64, device=dev)]
        kw.update(drag_cd=dd[0], drag_area=dd[1], drag_mass=dd[2])
        models.append(P.Drag(R_EQ, 1.225, 7.249, dd[0], dd[1], dd[2], 1500.0))
    fixed = lambda: P.propagate_numerical_batch_device(ds, 0.0, 86400.0, 60.0, MU, outs[0], sts[0], stp[0], **kw)  # noqa
    lst = lambda: P.propagate_models_batch_device(ds, 0.0, 86400.0, 60.0, models, outs[1], sts[1], stp[1])  # noqa
    ms = {"fixed": [], "list": []}
    for _ in range(reps):
        ms["fixed"] += device_call(fixed, 1)
        ms["list"] += device_call(lst, 1)
    identical = bool(torch.equal(outs[0].view(torch.int64), outs[1].view(torch.int64)) and torch.equal(sts[0], sts[1])
                     and torch.equal(stp[0], stp[1]))
    res = {"n": n, "samples": samples, "fixed_ms": round(min(ms["fixed"]), 3), "list_ms": round(min(ms["list"]), 3),
           "fixed_ms_all": [round(x, 3) for x in ms["fixed"]], "list_ms_all": [round(x, 3) for x in ms["list"]],
           "bytes_identical": identical}
    res["list_over_fixed"] = round(res["list_ms"] / res["fixed_ms"], 3)
    del outs
    torch.cuda.empty_cache()
    return res


def main():
    import torch

    from astroz_b200 import numerical as P, synth
    from tools.numerical_timing import teme_states

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    rng = np.random.default_rng(0)
    out = {"card_power_limit_max_sm_clock": card, "reps": ARGS.reps}
    n = ARGS.n
    y1 = geo_states(n, rng)
    cr, area1 = rng.uniform(1.2, 1.8, n), rng.uniform(5.0, 40.0, n)

    def f1(K, T):
        sun, moon = tables(K, 300.0)
        return [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.SolarRadiationPressure(T(cr), T(area1), 1500.0, R_EQ, T(sun)),
                P.ThirdBody(SUN_MU, T(sun)), P.ThirdBody(MOON_MU, T(moon))]
    out["F1"] = run_models(y1, 7 * 86400.0, 300.0, f1, ARGS.reps)
    jd0 = synth.BENCH_JD0
    y2 = teme_states(synth.monte_carlo_catalog(n), jd0, 0.0)
    cd, area2, mass = rng.uniform(2.0, 2.4, len(y2)), rng.uniform(1.0, 20.0, len(y2)), rng.uniform(100, 1000, len(y2))

    def f2(K, T):
        return [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.J3(MU, J3, R_EQ), P.J4(MU, J4, R_EQ),
                P.ImprovedDrag(R_EQ, T(cd), T(area2), T(mass), 1500.0, 150.0)]
    out["F2"] = run_models(y2, 86400.0, 60.0, f2, ARGS.reps)
    out["F3"] = {"N1": compare_paths(y2, 3, rng.uniform(1.0, 20.0, len(y2)), ARGS.reps),
                 "N3": compare_paths(teme_states(synth.near_earth_catalog(synth.HEADLINE_SATS, seed=13478), jd0, 0.0),
                                     1, None, ARGS.reps)}
    torch.cuda.synchronize()
    print(json.dumps(out))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=3)
    ARGS = ap.parse_args()
    main()
