"""K6 (satellite, time) pairs on one GPU: device time of the _device call (sort included), host-call time with pinned
and with pageable buffers, for four workloads; the grid on the same catalogue x 1,440 epochs and the per-satellite
astroz_cuda_sgp4_array loop (the only earlier way to serve W1) in the same process.  Prints one JSON line.

  W1  config-2 catalogue (synth.near_earth_catalog()), 19,408,320 queries: satellites and times over the headline day
      drawn uniformly (seeded) -- the headline grid's cell count
  W2  the W1 queries grouped by satellite
  W3  config-3 mixed catalogue (synth.mixed_catalog()), 19,408,320 shuffled queries
  W4  100,000 W1-style queries (latency)

    python tools/pairs_timing.py [--reps 5] [--loop-sats 1000]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unknown"
    return name, q


def queries(n_sats, nq, seed):
    from astroz_b200 import synth

    rng = np.random.default_rng(seed)
    sat = rng.integers(0, n_sats, nq).astype(np.uint32)
    jd = np.full(nq, synth.BENCH_JD0)
    fr = rng.uniform(0.0, 1.0, nq)
    return sat, jd, fr


def device_ms(c, sat, jd, fr, reps):
    """CUDA events around the _device call on a dedicated torch stream (key, sort, split and K6 kernels)."""
    import torch

    dev = torch.device("cuda", 0)
    n = len(sat)
    ds = torch.from_numpy(sat.view(np.int32)).to(dev)
    dj, df = torch.from_numpy(jd).to(dev), torch.from_numpy(fr).to(dev)
    pos = torch.empty((n, 3), dtype=torch.float64, device=dev)
    vel = torch.empty_like(pos)
    st = torch.empty((n,), dtype=torch.uint8, device=dev)
    s = torch.cuda.Stream()   # a stream of its own: raw handle 0 would mean the library's stream, outside the events
    torch.cuda.synchronize()
    for _ in range(2):
        c.propagate_pairs_device(ds, dj, df, pos, vel, st, stream=s.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(reps):
        c.propagate_pairs_device(ds, dj, df, pos, vel, st, stream=s.cuda_stream)
    e1.record(s)
    torch.cuda.synchronize()
    out = (pos.cpu().numpy(), vel.cpu().numpy(), st.cpu().numpy())
    del ds, dj, df, pos, vel, st
    torch.cuda.empty_cache()
    return e0.elapsed_time(e1) / reps, out


def host_ms(c, sat, jd, fr, reps, pinned):
    from astroz_b200 import _lib

    n = len(sat)
    if pinned:
        bufs = [_lib.pinned_empty((n,), np.uint32), _lib.pinned_empty((n,)), _lib.pinned_empty((n,))]
        bufs[0][:], bufs[1][:], bufs[2][:] = sat, jd, fr
        out = [_lib.pinned_empty((n, 3)), _lib.pinned_empty((n, 3)), _lib.pinned_empty((n,), np.uint8)]
    else:
        bufs = [sat.copy(), jd.copy(), fr.copy()]
        out = [np.empty((n, 3)), np.empty((n, 3)), np.empty(n, dtype=np.uint8)]

    def call():
        rc = _lib.lib().astroz_cuda_constellation_propagate_pairs(
            c._h, C.c_void_p(bufs[0].ctypes.data), _lib.dptr(bufs[1]), _lib.dptr(bufs[2]), n, 0, _lib.dptr(out[0]),
            _lib.dptr(out[1]), C.c_void_p(out[2].ctypes.data))
        _lib.check(rc)

    call()
    t0 = time.perf_counter()
    for _ in range(reps):
        call()
    ms = (time.perf_counter() - t0) / reps * 1e3
    return ms, out


def grid_ms(c, n_sats, reps):
    import torch

    from astroz_b200 import synth

    jd, fr = synth.time_grid(1440)
    dev = torch.device("cuda", 0)
    pos = torch.empty((n_sats, 1440, 3), dtype=torch.float64, device=dev)
    vel = torch.empty_like(pos)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    for _ in range(2):
        c.propagate_device(jd, fr, pos, vel, stream=s.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(reps):
        c.propagate_device(jd, fr, pos, vel, stream=s.cuda_stream)
    e1.record(s)
    torch.cuda.synchronize()
    del pos, vel
    torch.cuda.empty_cache()
    return e0.elapsed_time(e1) / reps


def sgp4_array_loop_ms(tles, sat, jd, fr, n_loop, seed):
    """One astroz_cuda_sgp4_array call per satellite over that satellite's W1 times, pinned buffers, for n_loop
    satellites drawn at random; returns (measured ms for those, queries they cover)."""
    from astroz_b200 import _lib

    L = _lib.lib()
    rng = np.random.default_rng(seed)
    pick = rng.choice(len(tles), n_loop, replace=False)
    order = np.argsort(sat, kind="stable")
    bounds = np.searchsorted(sat[order], np.arange(len(tles) + 1))
    handles, work = [], []
    for s in pick:
        q = order[bounds[s]:bounds[s + 1]]
        m = len(q)
        pj, pf, res = _lib.pinned_empty((m,)), _lib.pinned_empty((m,)), _lib.pinned_empty((m, 6))
        pj[:], pf[:] = jd[q], fr[q]
        h = C.c_void_p()
        _lib.check(L.astroz_cuda_sgp4_init(tles[s][0].encode(), tles[s][1].encode(), 1, 0, C.byref(h)))
        ep = C.c_double()
        _lib.check(L.astroz_cuda_sgp4_epoch(h, C.byref(ep)))
        handles.append(h)
        work.append((h, pj, pf, ep.value, res, m))
    for h, pj, pf, ep, res, m in work:   # opens each handle's device resources
        _lib.check(L.astroz_cuda_sgp4_array(h, _lib.dptr(pj), _lib.dptr(pf), ep, _lib.dptr(res), m))
    t0 = time.perf_counter()
    for h, pj, pf, ep, res, m in work:
        _lib.check(L.astroz_cuda_sgp4_array(h, _lib.dptr(pj), _lib.dptr(pf), ep, _lib.dptr(res), m))
    ms = (time.perf_counter() - t0) * 1e3
    covered = sum(w[5] for w in work)
    for h in handles:
        L.astroz_cuda_sgp4_free(h)
    return ms, covered


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop-sats", type=int, default=1000)
    args = ap.parse_args()
    import astroz_b200
    from astroz_b200 import _lib, synth

    _lib.require_device()
    name, power = card()
    n_q = 19_408_320
    res = {"card": name, "power_limit_and_max_sm_clock": power, "queries_w1_w2_w3": n_q, "reps": args.reps}

    near = synth.near_earth_catalog()
    c1 = astroz_b200.Constellation(near)
    sat, jd, fr = queries(len(near), n_q, 1)
    grp = np.argsort(sat, kind="stable")
    w4 = queries(len(near), 100_000, 4)
    for wl, (s, j, f) in (("W1", (sat, jd, fr)), ("W2", (sat[grp], jd[grp], fr[grp])), ("W4", w4)):
        dms, dout = device_ms(c1, s, j, f, args.reps)
        pms, pout = host_ms(c1, s, j, f, args.reps, True)
        gms, gout = host_ms(c1, s, j, f, args.reps, False)
        same = all(np.array_equal(a, b) for a, b in zip(dout, pout)) and \
            all(np.array_equal(a, b) for a, b in zip(pout, gout))
        res[wl] = {"n": len(s), "device_ms": round(dms, 4), "device_Gprops_s": round(len(s) / dms / 1e6, 3),
                   "host_pinned_ms": round(pms, 3), "host_pageable_ms": round(gms, 3), "host_device_identical": same}
        if wl == "W1":
            w1_pos = dout[0]
        if wl == "W2":
            res[wl]["equals_W1_per_query"] = bool(np.array_equal(dout[0], w1_pos[grp]))
        del dout, pout, gout
    gms = grid_ms(c1, len(near), args.reps)
    res["grid_near_earth_x1440"] = {"cells": len(near) * 1440, "device_ms": round(gms, 4),
                                    "Gprops_s": round(len(near) * 1440 / gms / 1e6, 3)}
    loop_ms, covered = sgp4_array_loop_ms(near, sat, jd, fr, args.loop_sats, 7)
    est = loop_ms * n_q / covered
    res["sgp4_array_loop_W1"] = {"satellites_timed": args.loop_sats, "queries_timed": int(covered),
                                 "ms_timed": round(loop_ms, 2), "ms_scaled_to_W1": round(est, 1),
                                 "pairs_host_pinned_speedup": round(est / res["W1"]["host_pinned_ms"], 1)}
    del c1

    mixed = synth.mixed_catalog()
    c3 = astroz_b200.Constellation(mixed)
    s3, j3, f3 = queries(len(mixed), n_q, 3)
    dms, dout = device_ms(c3, s3, j3, f3, args.reps)
    pms, pout = host_ms(c3, s3, j3, f3, args.reps, True)
    gms_, gout = host_ms(c3, s3, j3, f3, args.reps, False)
    same = all(np.array_equal(a, b) for a, b in zip(dout, pout)) and all(np.array_equal(a, b) for a, b in zip(pout, gout))
    res["W3"] = {"n": n_q, "deep_space_share": round(float(np.mean(c3.classes[s3] > 0)), 4),
                 "device_ms": round(dms, 4), "device_Gprops_s": round(n_q / dms / 1e6, 3),
                 "host_pinned_ms": round(pms, 3), "host_pageable_ms": round(gms_, 3), "host_device_identical": same}
    del dout, pout, gout
    g3 = grid_ms(c3, len(mixed), args.reps)
    res["grid_mixed_x1440"] = {"cells": len(mixed) * 1440, "device_ms": round(g3, 4),
                               "Gprops_s": round(len(mixed) * 1440 / g3 / 1e6, 3)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
