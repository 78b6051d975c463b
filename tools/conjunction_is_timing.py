"""K15 importance-sampled collision probability timing (astroz_cuda_conjunction_is[_device]) against K14.

    python tools/conjunction_is_timing.py [--reps 3] [--workloads MC1,MC2] [--tails 1e-5,1e-7,1e-9]

MC1 and MC2 are tools/conjunction_mc_timing.py's workloads (1,000 LEO crossings at +-1 min and 100 GEO crossings at
+-30 min, 10^5 samples each).  For each, K14 and K15 (linear shifts) run alternated in one process: device ms (CUDA
events, best of --reps, and the spread) and samples per second of both, and the proposal pass alone (K11's launch and
is_proposal_kernel, read from torch.profiler) for 100,000 LEO candidates.  For one LEO crossing at each K11 Pc of
--tails (sigma 200 m, R 20 m): the IS relative error at 10^6 samples, the samples and time IS needs for 10 % and what
plain draws need for the same (N = 99 (1 - Pc) / Pc at K14's measured rate).  Prints one JSON record per line, with the
card, power limit and maximum SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from conjunction_mc_timing import _workloads  # noqa: E402
from conjunction_timing import _card, _covariances  # noqa: E402


def _event_ms(fn, reps):
    import torch

    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return times


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", default="MC1,MC2")
    ap.add_argument("--tails", default="1e-5,1e-7,1e-9")
    args = ap.parse_args()
    import torch

    from astroz_b200.collision import (conjunctions, importance_sampling, importance_sampling_device,
                                       importance_sampling_scratch_bytes, monte_carlo_device,
                                       monte_carlo_scratch_bytes)
    from tests.fit_oracle import conjunction_is as ci

    card = _card()
    dev = torch.device("cuda:0")
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
    rates = {}
    for name, el, pr, se, jd, fr, w, deep, samples in _workloads():
        if name not in args.workloads.split(","):
            continue
        n, m = el.shape[1], len(pr)
        model = np.full(n, deep, np.uint8)
        P = _covariances(n, model.astype(bool))
        ins = [t(el), t(P), t(model, torch.uint8), t(pr, torch.int32), t(se, torch.int32), t(jd), t(fr),
               t(np.full(m, w)), t(np.full(m, 0.02)), t(np.full(m, samples), torch.int64), None,
               t(np.arange(m) + 1, torch.int64)]
        c3 = torch.zeros((m, 3), dtype=torch.int64, device=dev)
        c12 = torch.zeros((m, 12), dtype=torch.int64, device=dev)
        st = torch.zeros(m, dtype=torch.uint8, device=dev)
        kind = torch.zeros(m, dtype=torch.uint8, device=dev)
        s14 = torch.empty(monte_carlo_scratch_bytes(m), dtype=torch.uint8, device=dev)
        s15 = torch.empty(importance_sampling_scratch_bytes(m), dtype=torch.uint8, device=dev)
        mc_ms, is_ms = [], []
        for _ in range(args.reps):   # alternated
            mc_ms += _event_ms(lambda: monte_carlo_device(*ins, c3, None, st, s14), 1)
            is_ms += _event_ms(lambda: importance_sampling_device(*ins, None, c12, None, kind, None, st, s15), 1)
        total = float(m) * samples
        rates[name] = total / (min(mc_ms) * 1e-3)
        print(json.dumps({"workload": name, "candidates": m, "samples_each": samples,
                          "k14_ms_best": round(min(mc_ms), 3), "k14_ms_spread": round(max(mc_ms) - min(mc_ms), 3),
                          "is_ms_best": round(min(is_ms), 3), "is_ms_spread": round(max(is_ms) - min(is_ms), 3),
                          "k14_samples_per_s": f"{total / (min(mc_ms) * 1e-3):.3e}",
                          "is_samples_per_s": f"{total / (min(is_ms) * 1e-3):.3e}",
                          "is_over_k14": round(min(is_ms) / min(mc_ms), 4),
                          "kinds": np.bincount(kind.cpu().numpy(), minlength=3).tolist(),
                          "card": card[0], "power_limit": card[1], "max_sm_clock": card[2]}), flush=True)
    # the proposal pass for 100,000 LEO candidates: one sample each, kernels timed by the profiler
    name, el, pr, se, jd, fr, w, deep, _ = _workloads()[0]
    rng = np.random.default_rng(3)
    from tests.fit_oracle.conjunction_cases import crossings
    n0 = el.shape[1] - len(pr)   # the catalogue rows before the engineered copies
    rows = rng.integers(0, n0, 100000)
    cp, jd, fr = crossings(el[:, :n0], rows, rng.uniform(0.5, 120.0, len(rows)))
    el2 = np.concatenate([el[:, :n0], cp], axis=1)
    m = len(rows)
    P = _covariances(el2.shape[1], np.zeros(el2.shape[1], bool))
    ins = [t(el2), t(P), None, t(rows, torch.int32), t(n0 + np.arange(m), torch.int32), t(jd), t(fr),
           t(np.full(m, 1.0)), t(np.full(m, 0.02)), t(np.ones(m), torch.int64), None, None]
    c12 = torch.zeros((m, 12), dtype=torch.int64, device=dev)
    st = torch.zeros(m, dtype=torch.uint8, device=dev)
    kind = torch.zeros(m, dtype=torch.uint8, device=dev)
    s15 = torch.empty(importance_sampling_scratch_bytes(m), dtype=torch.uint8, device=dev)
    run = lambda: importance_sampling_device(*ins, None, c12, None, kind, None, st, s15)  # noqa: E731
    whole = _event_ms(run, args.reps)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    k = {}
    for e in prof.key_averages():
        if e.key.startswith(("az::conjunction", "az::is_", "az::mc_", "conjunction", "is_")) or "cub" in e.key:
            k[e.key.split("(")[0]] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e3, 3)
    print(json.dumps({"workload": "proposal pass, 100,000 LEO candidates x 1 sample", "call_ms_best": round(min(whole), 3),
                      "kernel_ms": k, "kinds": np.bincount(kind.cpu().numpy(), minlength=3).tolist(),
                      "card": card[0], "power_limit": card[1]}), flush=True)
    # the tails
    rate = rates.get("MC1")
    for target in [float(x) for x in args.tails.split(",") if x]:
        assess = lambda e, p, r: conjunctions(e, [0], [1], np.floor(e[0, 0] - 0.5) + 0.5,  # noqa: E731
                                              e[0, 0] - (np.floor(e[0, 0] - 0.5) + 0.5), window_min=1.0, hbr_km=r,
                                              covariance=p, model=np.zeros(2, np.uint8)).record[0]
        e, p, r = ci.leo_at_pc(assess, target)
        pc11 = assess(e, p, r)[12]
        jd0 = np.floor(e[0, 0] - 0.5) + 0.5
        call = lambda: importance_sampling(e, [0], [1], jd0, e[0, 0] - jd0, window_min=1.0, hbr_km=r,  # noqa: E731
                                           samples=10 ** 6, seed=7, covariance=p, model=np.zeros(2, np.uint8))
        res = call()
        ms = min(_event_ms(call, args.reps))
        rel = float(res.std_error[0] / res.pc[0])
        n10 = 10 ** 6 * (rel / 0.1) ** 2
        plain = 99.0 * (1 - res.pc[0]) / res.pc[0]
        print(json.dumps({"workload": f"one LEO candidate, K11 Pc {pc11:.2e}", "is_pc": f"{res.pc[0]:.4e}",
                          "is_rel_error_1e6": round(rel, 5), "is_samples_for_10pct": f"{n10:.3e}",
                          "is_ms_1e6": round(ms, 2), "is_ms_for_10pct": round(ms * n10 / 1e6, 3),
                          "plain_samples_for_10pct": f"{plain:.3e}",
                          "plain_s_for_10pct_at_k14_rate": None if rate is None else round(plain / rate, 1),
                          "card": card[0], "power_limit": card[1]}), flush=True)


if __name__ == "__main__":
    main()
