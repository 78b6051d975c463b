"""K10 state covariance timing (astroz_cuda_propagate_covariance[_device]).

    python tools/covariance_timing.py [--reps 3] [--device-only]

Workloads (covariances are synthetic PSD matrices at a radar fit's scale, B* free, so every query runs 8 propagations):
  CV1  the config-2 catalogue (13,478 near-earth rows) x 1,440 one-minute times from each epoch: 19.4 M queries;
  CV2  one query per config-2 row at a common time: 13,478 queries, bound by building the sets;
  CV3  config 3's 1,536 deep-space rows x 7 days at 10 min: 1.55 M queries.
Prints one JSON record per workload: device ms (CUDA events, best of --reps, and the spread), SGP4 / SDP4 evaluations
per second, the queries per work item (cov_chunk), host-call ms with pageable and pinned buffers, the threaded C
restatement scaled from a subset, and the card, power limit and maximum SM clock.  --device-only times the device
calls alone, for comparing measurement builds of the library (ASTROZ_B200_LIB; AZ_TAG names the build in the record).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception:   # noqa: BLE001
        return ["unknown", "unknown", "unknown"]


def _covariances(n, seed=3):
    rng = np.random.default_rng(seed)
    d = np.array([1e-7, 1e-6, 1e-6, 1e-5, 1e-5, 1e-5, 1e-5])
    iu = np.triu_indices(7)
    A = rng.standard_normal((n, 7, 7))
    Cm = A @ A.transpose(0, 2, 1) / 7.0 + 0.3 * np.eye(7)
    s = np.sqrt(np.einsum("nii->ni", Cm))
    Cm = Cm / (s[:, :, None] * s[:, None, :]) * np.outer(d, d)
    return np.ascontiguousarray(Cm[:, iu[0], iu[1]])


def _workloads():
    from astroz_b200 import synth

    ne = synth.elements_from_tles(synth.near_earth_catalog())
    mix = synth.elements_from_tles(synth.mixed_catalog())
    ds = mix[:, 1440.0 / mix[1] > 225.0]
    out = []
    n = ne.shape[1]
    jd0 = np.floor(ne[0] - 0.5) + 0.5
    sat = np.repeat(np.arange(n), 1440)
    out.append(("CV1", ne, np.zeros(n, np.uint8), sat, jd0[sat], (ne[0] - jd0)[sat] + np.tile(np.arange(1440) / 1440.0, n)))
    t0 = float(np.max(ne[0])) + 0.5
    out.append(("CV2", ne, np.zeros(n, np.uint8), np.arange(n), np.full(n, np.floor(t0) + 0.5), np.full(n, t0 % 1.0)))
    n = ds.shape[1]
    jd0 = np.floor(ds[0] - 0.5) + 0.5
    steps = 7 * 144
    sat = np.repeat(np.arange(n), steps)
    out.append(("CV3", ds, np.ones(n, np.uint8), sat, jd0[sat], (ds[0] - jd0)[sat] + np.tile(np.arange(steps) / 144.0, n)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--device-only", action="store_true")
    args = ap.parse_args()
    import torch

    from astroz_b200 import _lib as L
    from astroz_b200.covariance import propagate_covariance_device
    from tests.fit_oracle import covariance as K

    name, power, clock = _card()
    dev = torch.device("cuda:0")
    for tag, el, model, sat, jd, fr in _workloads():
        n, m = el.shape[1], len(sat)
        cov = _covariances(n)
        off = np.searchsorted(sat, np.arange(n + 1)).astype(np.uint32)
        d = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (el, cov, model, off.astype(np.int32), jd, fr)]
        sg = torch.empty(m, 21, dtype=torch.float64, device=dev)
        st = torch.empty(m, 6, dtype=torch.float64, device=dev)
        stt = torch.empty(m, dtype=torch.uint8, device=dev)
        times = []
        for _ in range(args.reps + 1):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            propagate_covariance_device(d[0], d[1], d[2], d[3], d[4], d[5], st, sg, None, stt)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        times = times[1:]
        ok = int((stt == 0).sum())
        evals = 8 * m
        rec = {"workload": tag, "build": os.environ.get("AZ_TAG", "default"), "rows": n, "queries": m, "ok": ok,
               "chunk": K.emul_library().emul_cov_chunk(m) if not os.environ.get("AZ_TAG") else None,
               "device_ms_best": round(min(times), 3), "device_ms_spread": round(max(times) - min(times), 3),
               "evals_per_s": f"{evals / (min(times) * 1e-3):.3e}"}
        if args.device_only:
            print(json.dumps(rec), flush=True)
            continue
        host = {}
        p = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731
        for pinned in (False, True):
            ins = [torch.from_numpy(np.ascontiguousarray(x)) for x in (el, cov, model, off, jd, fr)]
            outs = [torch.empty(m, 6, dtype=torch.float64), torch.empty(m, 21, dtype=torch.float64),
                    torch.empty(m, dtype=torch.uint8)]
            if pinned:
                ins, outs = [x.pin_memory() for x in ins], [x.pin_memory() for x in outs]
            t0 = time.perf_counter()
            rc = L.lib().astroz_cuda_propagate_covariance(p(ins[0]), n, 1, p(ins[1]), p(ins[2]), p(ins[3]), p(ins[4]),
                                                           p(ins[5]), m, 0, 0, p(outs[0]), p(outs[1]), None, p(outs[2]))
            host["pinned" if pinned else "pageable"] = round((time.perf_counter() - t0) * 1e3, 2)
            assert rc == 0
            assert outs[1].numpy().tobytes() == sg.cpu().numpy().tobytes()
        # the threaded C restatement on a subset of rows, scaled to the workload
        k = min(n, 40 if tag != "CV2" else 2000)
        sub = sat < k
        t0 = time.perf_counter()
        K.restated(el[:, :k], cov[:k], model[:k], off[:k + 1], jd[sub], fr[sub], 0)
        cpu_s = (time.perf_counter() - t0) * m / max(int(sub.sum()), 1)
        rec.update({"host_call_ms": host, "cpu_restatement_s_scaled": round(cpu_s, 2), "cpu_threads": os.cpu_count(),
                    "card": name, "power_limit": power, "max_sm_clock": clock})
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
