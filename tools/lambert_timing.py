"""K9 timing on the GPU: batched Lambert solves and porkchop grids.  Prints one JSON line.

    python tools/lambert_timing.py

Workloads:
  L1  10^7 random LEO-GEO problems, max_revs = 0;
  L2  10^6 LEO problems with tof up to 1 day, max_revs = 15;
  P1  Constellation.porkchop: the ISS row against 2,000 config-2 targets, 144 departures x 144 arrivals over 1 day,
      max_revs = 15;
  P2  Constellation.porkchop: one GEO chaser against config 3's 1,024 GEO objects, 96 x 96 over 7 days, max_revs = 7.
L1 / L2 time lambert_batch_device with CUDA events after a warm-up, best of 3.  Their rate counts the slots attempted
(status OK or NOT_CONVERGED: a Householder iteration ran), and their warp imbalance is the mean over warps (32
consecutive problems) of the largest per-problem iteration total over the mean one.  P1 / P2 time the whole host call
(propagation, grid, download into pageable numpy arrays), best of 3, and report cells/s.  The threaded C statement of the
solver (tests/lambert_oracle) runs a subset of L1 / L2 on every host core, scaled up to the full count.  The card's name,
power limit and maximum SM clock are read in the same call.
"""
from __future__ import annotations

import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MU = 398600.5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", "0"], capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"gpu": q[0], "power_limit_w": float(q[1]), "max_sm_clock_mhz": float(q[2])}


def problems(rng, n, r_lo, r_hi, tof_hi):
    u1, w = rng.normal(size=(n, 3)), rng.normal(size=(n, 3))
    u1 /= np.linalg.norm(u1, axis=1)[:, None]
    w -= np.einsum("ij,ij->i", w, u1)[:, None] * u1
    w /= np.linalg.norm(w, axis=1)[:, None]
    ang = rng.uniform(0.01, 2 * np.pi - 0.01, n)
    u2 = np.cos(ang)[:, None] * u1 + np.sin(ang)[:, None] * w
    rad = lambda: np.exp(rng.uniform(math.log(r_lo), math.log(r_hi), n))[:, None]  # noqa: E731
    r1, r2 = u1 * rad(), u2 * rad()
    tof = np.exp(rng.uniform(math.log(300.0), math.log(tof_hi), n))
    normal = np.cross(r1, r2) * rng.choice([-1.0, 1.0], n)[:, None]
    return r1, r2, tof, normal / np.linalg.norm(normal, axis=1)[:, None]


def lambert_workload(name, n, max_revs, r_lo, r_hi, tof_hi, cpu_subset):
    import torch

    from astroz_b200.lambert import NOT_CONVERGED, OK, lambert_batch_device
    from tests import lambert_oracle as L

    r1, r2, tof, normal = problems(np.random.default_rng(hash(name) & 0xFFFF), n, r_lo, r_hi, tof_hi)
    S = 2 * max_revs + 1
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (r1, r2, tof, normal)]
    v1 = torch.empty((n, S, 3), dtype=torch.float64, device="cuda")
    v2 = torch.empty_like(v1)
    st = torch.empty((n, S), dtype=torch.uint8, device="cuda")
    it = torch.empty_like(st)
    call = lambda: lambert_batch_device(dev[0], dev[1], dev[2], v1, v2, st, MU, iterations=it,  # noqa: E731
                                        normal=dev[3], max_revs=max_revs)
    call()
    torch.cuda.synchronize()
    ms = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    status, iters = st.cpu().numpy(), it.cpu().numpy().astype(np.float64)
    attempted = int(np.sum((status == OK) | (status == NOT_CONVERGED)))
    per = iters.sum(axis=1)[: n // 32 * 32].reshape(-1, 32)
    imbalance = float(np.mean(per.max(axis=1) / np.maximum(per.mean(axis=1), 1e-30)))
    best = min(ms) / 1e3
    t0 = time.perf_counter()
    threads = os.cpu_count() or 1
    cs = L.solve(r1[:cpu_subset], r2[:cpu_subset], tof[:cpu_subset], MU, max_revs=max_revs, normal=normal[:cpu_subset],
                 threads=threads)
    cpu_s = (time.perf_counter() - t0) * n / cpu_subset
    return {"problems": n, "max_revs": max_revs, "slots_attempted": attempted, "kernel_ms": round(min(ms), 3),
            "solves_per_s": attempted / best, "ok_slots": int(np.sum(status == OK)),
            "not_converged_slots": int(np.sum(status == NOT_CONVERGED)), "warp_max_over_mean_iterations": imbalance,
            "cpu_threads": threads, "cpu_subset": cpu_subset, "cpu_scaled_s": cpu_s,
            "cpu_slot_status_equal_on_subset": bool(np.array_equal(cs[2], status[:cpu_subset]))}


def porkchop_workload(c, chaser, target, n_dep, n_arr, days, max_revs):
    jd0 = 2460437.5
    dep_jd, dep_fr = np.full(n_dep, jd0), np.arange(n_dep) * (days / n_dep)
    arr_jd, arr_fr = np.full(n_arr, jd0), 0.02 + np.arange(n_arr) * (days / n_arr)
    c.porkchop(chaser[:2], target[:2], dep_jd, dep_fr, arr_jd, arr_fr, max_revs=max_revs)
    secs = []
    for _ in range(3):
        t0 = time.perf_counter()
        dv, slot, st = c.porkchop(chaser, target, dep_jd, dep_fr, arr_jd, arr_fr, max_revs=max_revs)
        secs.append(time.perf_counter() - t0)
    cells = st.size
    return {"pairs": len(chaser), "departures": n_dep, "arrivals": n_arr, "days": days, "max_revs": max_revs,
            "cells": cells, "call_s": round(min(secs), 4), "cells_per_s": cells / min(secs),
            "ok_cells": int(np.sum(st == 0)), "status_counts": np.bincount(st.ravel(), minlength=5).tolist(),
            "median_total_dv_km_s": float(np.median(dv.sum(-1)[st == 0]))}


def main():
    from astroz_b200 import Constellation, device_count, synth
    from tests.golden.tles import ISS

    if device_count() < 1:
        raise SystemExit("lambert_timing needs a CUDA device")
    out = card()
    out["L1"] = lambert_workload("L1", 10_000_000, 0, 6600.0, 42164.0, 2 * 86400.0, 100_000)
    out["L2"] = lambert_workload("L2", 1_000_000, 15, 6600.0, 8000.0, 86400.0, 20_000)
    leo = [ISS] + synth.near_earth_catalog(2000)
    c = Constellation(leo, device=0)
    out["P1"] = porkchop_workload(c, np.zeros(2000, dtype=np.uint32), np.arange(1, 2001, dtype=np.uint32), 144, 144,
                                  1.0, 15)
    mixed = synth.mixed_catalog(2048)
    c3 = Constellation(mixed, device=0)
    geo = np.flatnonzero(np.asarray(c3.classes) == 2).astype(np.uint32)   # irez 1: the GEO objects
    out["P2"] = porkchop_workload(c3, np.full(len(geo), geo[0], dtype=np.uint32), geo, 96, 96, 7.0, 7)
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
