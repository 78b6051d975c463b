"""K11 conjunction assessment timing (astroz_cuda_conjunction[_device]).

    python tools/conjunction_timing.py [--reps 3] [--device-only]

Workloads (covariances are synthetic PSD matrices at a radar fit's scale, B* free on near-earth rows and held on
deep-space rows, so each object's Sigma runs 8 or 7 propagations):
  PC1  100,000 engineered LEO crossings among the config-2 rows (13,478 near-earth): a row against a copy of itself
       with its inclination changed by 0.5 .. 120 deg, guessed at the row's node crossing, +-1 min.  Nearly every
       candidate holds a minimum in its window and runs the whole search;
  PC2  one primary against every other config-2 row: 13,477 candidates, +-1 min (a screen's one-against-all list);
  PC3  10,000 engineered GEO-GEO crossings among config 3's GEO rows (inclination changed by 0.02 .. 1 deg), +-30 min;
  PC1r 100,000 random config-2 pairs at a common guess time, +-1 min: almost all end WINDOW_EDGE after one round.
Engineered partners are appended to the catalogue as extra rows with their row's covariance.  Prints one JSON record
per workload: device ms (CUDA events, best of --reps, and the spread), SGP4 / SDP4 evaluations per second counted from
the definition (32 samples x 2 rows per search round, rounds from the window and the 1e-9 min tolerance, plus 1 + nvar
per row for Sigma), host-call ms with pageable and pinned buffers, the threaded C restatement
(tests/fit_oracle/conjunction.c) scaled from a subset, candidates by status, and the card, power limit and maximum SM
clock.  --device-only times the device call alone, for comparing measurement builds of the library
(ASTROZ_B200_LIB; AZ_TAG names the build in the record).
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


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception:   # noqa: BLE001
        return ["unknown", "unknown", "unknown"]


def _covariances(n, deep, seed=3):
    rng = np.random.default_rng(seed)
    iu = np.triu_indices(7)
    A = rng.standard_normal((n, 7, 7))
    Cm = A @ A.transpose(0, 2, 1) / 7.0 + 0.3 * np.eye(7)
    s = np.sqrt(np.einsum("nii->ni", Cm))
    d = np.tile(np.array([1e-7, 1e-6, 1e-6, 1e-5, 1e-5, 1e-5, 1e-5]), (n, 1))
    d[deep, 6] = 0.0
    Cm = Cm / (s[:, :, None] * s[:, None, :]) * d[:, :, None] * d[:, None, :]
    return np.ascontiguousarray(Cm[:, iu[0], iu[1]])


def _workloads():
    from astroz_b200 import synth
    from tests.fit_oracle.conjunction_cases import crossings

    ne = synth.elements_from_tles(synth.near_earth_catalog())
    mix = synth.elements_from_tles(synth.mixed_catalog())
    geo = mix[:, np.abs(mix[1] - 1.0027) < 0.01]
    rng = np.random.default_rng(7)
    out = []
    n = ne.shape[1]
    rows = rng.integers(0, n, 100000)
    cp, jd, fr = crossings(ne, rows, rng.uniform(0.5, 120.0, len(rows)))
    out.append(("PC1", np.concatenate([ne, cp], axis=1), rows, n + np.arange(len(rows)), jd, fr, 1.0, 0))
    t0 = float(np.max(ne[0])) + 0.5
    jd0 = np.full(n - 1, np.floor(t0 - 0.5) + 0.5)
    out.append(("PC2", ne, np.zeros(n - 1, np.int64), np.arange(1, n), jd0, t0 - jd0, 1.0, 0))
    g = geo.shape[1]
    rows = rng.integers(0, g, 10000)
    cp, jd, fr = crossings(geo, rows, rng.uniform(0.02, 1.0, len(rows)))
    out.append(("PC3", np.concatenate([geo, cp], axis=1), rows, g + np.arange(len(rows)), jd, fr, 30.0, 1))
    pr = rng.integers(0, n, 100000)
    se = (pr + rng.integers(1, n, 100000)) % n
    jd0 = np.full(len(pr), np.floor(t0 - 0.5) + 0.5)
    out.append(("PC1r", ne, pr, se, jd0, t0 - jd0, 1.0, 0))
    return out


def _evaluations(status, w, nvar):
    first = 2.0 * w / 31.0
    rounds = 1 + max(1, math.ceil(math.log(first / 1e-9) / math.log(31.0)))
    search = np.where(status == 3, 1, rounds) * 64
    return float(np.sum(np.where(status <= 3, search + 2 * (1 + nvar), 0)))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--restated", type=int, default=2000, help="candidates of the C restatement's subset")
    ap.add_argument("--device-only", action="store_true")
    args = ap.parse_args()
    import torch

    from astroz_b200.collision import conjunctions, conjunctions_device
    from tests.fit_oracle import conjunction as cj

    card = _card()
    dev = torch.device("cuda:0")
    for name, el, pr, se, jd, fr, w, deep in _workloads():
        n, m = el.shape[1], len(pr)
        model = np.full(n, deep, np.uint8)
        P = _covariances(n, model.astype(bool))
        t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
        args_dev = [t(el), t(P), t(model, torch.uint8), t(pr, torch.int32), t(se, torch.int32), t(jd), t(fr),
                    t(np.full(m, w)), t(np.full(m, 0.02))]
        rec = torch.zeros((m, 13), dtype=torch.float64, device=dev)
        sig = torch.zeros((m, 2, 21), dtype=torch.float64, device=dev)
        stat = torch.zeros(m, dtype=torch.uint8, device=dev)
        conjunctions_device(*args_dev, rec, None, sig, stat)   # warm-up: module load
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            conjunctions_device(*args_dev, rec, None, sig, stat)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        status = stat.cpu().numpy()
        nvar = np.where(model.astype(bool), 6, 7)
        evals = _evaluations(status, w, (nvar[pr] + nvar[se]) / 2.0)
        record = {"workload": name, "build": os.environ.get("AZ_TAG", "default"), "candidates": m,
                  "device_ms_best": round(min(times), 3), "device_ms_spread": round(max(times) - min(times), 3),
                  "evaluations_per_s": f"{evals / (min(times) * 1e-3):.3e}",
                  "status_counts": {int(c): int(v) for c, v in zip(*np.unique(status, return_counts=True))},
                  "card": card[0], "power_limit": card[1], "max_sm_clock": card[2]}
        if args.device_only:
            print(json.dumps(record))
            continue
        host = {}
        for kind in ("pageable", "pinned"):
            conv = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()) if kind == "pinned" \
                else (lambda a: np.ascontiguousarray(a))
            h = [conv(x) for x in (el, P, jd, fr, np.full(m, w), np.full(m, 0.02))]
            best = float("inf")
            for _ in range(args.reps):
                s = time.perf_counter()
                conjunctions(h[0], pr, se, h[2], h[3], window_min=h[4], hbr_km=h[5], covariance=h[1], model=model)
                best = min(best, (time.perf_counter() - s) * 1e3)
            host[kind] = round(best, 2)
        k = min(args.restated, m)
        s = time.perf_counter()
        cj.restated(el, P, model, pr[:k], se[:k], jd[:k], fr[:k], np.full(k, w))
        ref_ms = (time.perf_counter() - s) * 1e3 * m / k
        record.update({"host_call_ms": host, "c_restatement_ms_scaled": round(ref_ms, 1),
                       "c_restatement_threads": os.cpu_count()})
        print(json.dumps(record))


if __name__ == "__main__":
    main()
