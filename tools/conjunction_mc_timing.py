"""K14 Monte Carlo collision probability timing (astroz_cuda_conjunction_mc[_device]).

    python tools/conjunction_mc_timing.py [--reps 3] [--restated-samples 2000] [--workloads MC1,MC2,MC3]

Workloads (covariances synthetic PSD matrices at a radar fit's scale, B* free on near-earth rows and held on deep-space
rows, as tools/conjunction_timing.py makes them):
  MC1  1,000 engineered LEO crossings among the config-2 rows, +-1 min, 10^5 samples each;
  MC2  100 engineered GEO-GEO crossings among config 3's GEO rows, +-30 min, 10^5 samples each (two SDP4 set builds
       and 32 lattices per 8 samples);
  MC3  one LEO crossing, +-1 min, 10^8 samples.
Prints one JSON record per workload: device ms (CUDA events, best of --reps, and the spread), samples per second,
host-call ms with pageable and pinned buffers, the C restatement (each sample's drawn pair through
tests/fit_oracle/conjunction.c on every CPU thread) scaled from --restated-samples samples, the counts, and the card,
power limit and maximum SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from conjunction_timing import _card, _covariances  # noqa: E402


def _workloads():
    from astroz_b200 import synth
    from tests.fit_oracle.conjunction_cases import crossings

    ne = synth.elements_from_tles(synth.near_earth_catalog())
    mix = synth.elements_from_tles(synth.mixed_catalog())
    geo = mix[:, np.abs(mix[1] - 1.0027) < 0.01]
    rng = np.random.default_rng(7)
    n, g = ne.shape[1], geo.shape[1]
    rows = rng.integers(0, n, 1000)
    cp, jd, fr = crossings(ne, rows, rng.uniform(0.5, 120.0, len(rows)))
    out = [("MC1", np.concatenate([ne, cp], axis=1), rows, n + np.arange(len(rows)), jd, fr, 1.0, 0, 10 ** 5)]
    rows = rng.integers(0, g, 100)
    cp, jd, fr = crossings(geo, rows, rng.uniform(0.02, 1.0, len(rows)))
    out.append(("MC2", np.concatenate([geo, cp], axis=1), rows, g + np.arange(len(rows)), jd, fr, 30.0, 1, 10 ** 5))
    rows = rows[:1] * 0
    cp, jd, fr = crossings(ne, rows, np.array([40.0]))
    out.append(("MC3", np.concatenate([ne, cp], axis=1), rows, n + np.arange(1), jd, fr, 1.0, 0, 10 ** 8))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--restated-samples", type=int, default=2000)
    ap.add_argument("--workloads", default="MC1,MC2,MC3")
    args = ap.parse_args()
    import torch

    from astroz_b200.collision import monte_carlo, monte_carlo_device, monte_carlo_scratch_bytes
    from tests.fit_oracle import conjunction_mc as mc

    card = _card()
    dev = torch.device("cuda:0")
    for name, el, pr, se, jd, fr, w, deep, samples in _workloads():
        if name not in args.workloads.split(","):
            continue
        n, m = el.shape[1], len(pr)
        model = np.full(n, deep, np.uint8)
        P = _covariances(n, model.astype(bool))
        hbr = 0.02
        t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
        args_dev = [t(el), t(P), t(model, torch.uint8), t(pr, torch.int32), t(se, torch.int32), t(jd), t(fr),
                    t(np.full(m, w)), t(np.full(m, hbr)), t(np.full(m, samples), torch.int64), None,
                    t(np.arange(m) + 1, torch.int64)]
        counts = torch.zeros((m, 3), dtype=torch.int64, device=dev)
        stat = torch.zeros(m, dtype=torch.uint8, device=dev)
        scratch = torch.empty(monte_carlo_scratch_bytes(m), dtype=torch.uint8, device=dev)
        monte_carlo_device(*args_dev, counts, None, stat, scratch)   # warm-up: module load
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            monte_carlo_device(*args_dev, counts, None, stat, scratch)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        c = counts.cpu().numpy()
        total = float(m) * samples
        record = {"workload": name, "candidates": m, "samples_each": samples,
                  "device_ms_best": round(min(times), 3), "device_ms_spread": round(max(times) - min(times), 3),
                  "samples_per_s": f"{total / (min(times) * 1e-3):.3e}",
                  "hits": int(c[:, 0].sum()), "edge": int(c[:, 1].sum()), "failed": int(c[:, 2].sum()),
                  "status_counts": {int(k): int(v) for k, v in zip(*np.unique(stat.cpu().numpy(),
                                                                               return_counts=True))},
                  "card": card[0], "power_limit": card[1], "max_sm_clock": card[2]}
        host = {}
        for kind in ("pageable", "pinned"):
            conv = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()) if kind == "pinned" \
                else (lambda a: np.ascontiguousarray(a))
            h = [conv(x) for x in (el, P, jd, fr, np.full(m, w), np.full(m, hbr))]
            best = float("inf")
            for _ in range(args.reps):
                s = time.perf_counter()
                res = monte_carlo(h[0], pr, se, h[2], h[3], window_min=h[4], hbr_km=h[5], samples=samples,
                                  seed=np.arange(m) + 1, covariance=h[1], model=model)
                best = min(best, (time.perf_counter() - s) * 1e3)
            host[kind] = round(best, 2)
            assert (res.hits == c[:, 0].astype(np.uint64)).all()
        k = args.restated_samples
        s = time.perf_counter()
        mc.restated(el, P, model, int(pr[0]), int(se[0]), jd[0], fr[0], w, k, 0, 1)
        ref_ms = (time.perf_counter() - s) * 1e3 * total / k
        record.update({"host_call_ms": host, "c_restatement_ms_scaled": round(ref_ms, 1),
                       "c_restatement_threads": os.cpu_count()})
        print(json.dumps(record), flush=True)


if __name__ == "__main__":
    main()
