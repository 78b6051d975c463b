#!/usr/bin/env python
"""Host-buffer calls that run the two-slot chunk pipeline (astroz_b200/csrc/az_hostcopy.cu, ChunkPipeline), each with
pinned and with pageable buffers: host clock around calls that end in a synchronise, best of --reps after a warm-up
call, and a SHA-256 of the result bytes.  Prints one JSON line with the card's name, power limit and
maximum SM clock.

  pairs W1 / W4  tools/pairs_timing.py's W1 (19,408,320 queries over the config-2 catalogue) and W4 (100,000 queries),
                 TEME with velocities and status
  sgp4_array     the ISS over 31,536,000 epochs at one second ("1 year (second)"), through astroz_cuda_sgp4_array
  numerical N1   tools/numerical_timing.py's N1 (100,000 LEO states, J2 + drag, one day at 60 s, DP87) through
                 astroz_cuda_propagate_numerical

    python tools/host_pipeline_timing.py [--reps 3]
    python tools/host_pipeline_timing.py --compare OTHER.so [--rounds 5]

--compare alternates processes on OTHER.so (through ASTROZ_B200_LIB) and on this tree's library, --rounds each, and
reports per call the best time of each library, the spread of its runs (slowest minus fastest) and whether every run of
both gave the same bytes.
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

MU, R_EQ, J2 = 398600.5, 6378.137, 0.00108262998905


def card() -> str:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return q.stdout.strip() or "unknown"


def checksum(arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(memoryview(np.ascontiguousarray(a)).cast("B"))
    return h.hexdigest()[:32]


def like(a: np.ndarray, pinned: bool) -> np.ndarray:
    from astroz_b200 import _lib

    if not pinned:
        return a.copy()
    p = _lib.pinned_empty(a.shape, a.dtype)
    p[...] = a
    return p


def empty(shape, dtype, pinned: bool) -> np.ndarray:
    from astroz_b200 import _lib

    return _lib.pinned_empty(shape, dtype) if pinned else np.empty(shape, dtype)


def best_ms(call, reps: int) -> float:
    call()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()   # every timed call returns after its own synchronise
        ms.append((time.perf_counter() - t0) * 1e3)
    return min(ms)


def ptr(a):
    return C.c_void_p(a.ctypes.data)


def pairs_case(c, queries, pinned, reps):
    from astroz_b200 import _lib

    sat, jd, fr = (like(x, pinned) for x in queries)
    n = len(sat)
    out = [empty((n, 3), np.float64, pinned), empty((n, 3), np.float64, pinned), empty((n,), np.uint8, pinned)]
    L = _lib.lib()
    ms = best_ms(lambda: _lib.check(L.astroz_cuda_constellation_propagate_pairs(
        c._h, ptr(sat), _lib.dptr(jd), _lib.dptr(fr), n, 0, _lib.dptr(out[0]), _lib.dptr(out[1]), ptr(out[2]))), reps)
    return ms, checksum(out)


def sgp4_array_case(s, jd0, fr0, pinned, reps):
    from astroz_b200 import _lib

    jd, fr = like(jd0, pinned), like(fr0, pinned)
    out = empty((len(jd), 6), np.float64, pinned)
    L = _lib.lib()
    ep = s.jdsatepoch + s.jdsatepochF
    ms = best_ms(lambda: _lib.check(L.astroz_cuda_sgp4_array(s._h, _lib.dptr(jd), _lib.dptr(fr), ep, _lib.dptr(out),
                                                             len(jd))), reps)
    return ms, checksum([out])


def numerical_case(y0, area0, samples, pinned, reps):
    from astroz_b200 import _lib

    n = len(y0)
    y, area = like(y0, pinned), like(area0, pinned)
    cd, mass = like(np.full(n, 2.2), pinned), like(np.full(n, 500.0), pinned)
    out = empty((n, samples, 6), np.float64, pinned)
    status, steps = empty((n,), np.uint8, pinned), empty((n, 2), np.uint64, pinned)
    L = _lib.lib()
    j2, req = C.c_double(J2), C.c_double(R_EQ)
    ms = best_ms(lambda: _lib.check(L.astroz_cuda_propagate_numerical(
        ptr(y), n, 0.0, 86400.0, 60.0, MU, 3, C.byref(j2), C.byref(req), ptr(cd), ptr(area), ptr(mass), 1, 1e-9, 1e-12,
        0, ptr(out), ptr(status), ptr(steps))), reps)
    return ms, checksum([out, status, steps])


def measure(reps: int) -> dict:
    import astroz_b200
    from astroz_b200 import _lib, numerical, synth
    from astroz_b200.api import WGS72, Satrec
    from numerical_timing import teme_states
    from pairs_timing import queries
    from tests.golden import tles as G

    _lib.require_device()
    res = {"card_power_limit_max_sm_clock": card(), "lib": os.path.relpath(_lib.LIB_PATH, ROOT), "reps": reps}

    def both(name, case, *args):
        for pinned in (True, False):
            ms, digest = case(*args, pinned, reps)
            res[f"{name}_{'pinned' if pinned else 'pageable'}"] = {"ms": round(ms, 3), "checksum": digest}

    near = synth.near_earth_catalog()
    c = astroz_b200.Constellation(near)
    both("pairs_W1", pairs_case, c, queries(len(near), 19_408_320, 1))
    both("pairs_W4", pairs_case, c, queries(len(near), 100_000, 4))
    del c
    s = Satrec.twoline2rv(*G.ISS, WGS72)
    n = 31_536_000
    both("sgp4_array_31.5M", sgp4_array_case, s, np.full(n, s.jdsatepoch), s.jdsatepochF + np.arange(n) / 86400.0)
    del s
    rng = np.random.default_rng(0)
    y1 = teme_states(synth.monte_carlo_catalog(100_000), synth.BENCH_JD0, 0.0)
    area = rng.uniform(1.0, 20.0, len(y1))
    both("numerical_N1", numerical_case, y1, area, len(numerical.numerical_times(0.0, 86400.0, 60.0)))
    return res


def compare(other: str, rounds: int, reps: int) -> dict:
    runs = {"other": [], "this": []}
    for r in range(rounds):
        for label in (("other", "this") if r % 2 == 0 else ("this", "other")):
            env = dict(os.environ)
            env.pop("ASTROZ_B200_LIB", None)
            if label == "other":
                env["ASTROZ_B200_LIB"] = os.path.abspath(other)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--reps", str(reps)], env=env,
                               capture_output=True, text=True, check=True)
            runs[label].append(json.loads(p.stdout.strip().splitlines()[-1]))
    first = runs["this"][0]
    res = {"card_power_limit_max_sm_clock": first["card_power_limit_max_sm_clock"], "other": other, "rounds": rounds,
           "reps": reps, "calls": {}}
    for key in (k for k in first if isinstance(first[k], dict)):
        row = {}
        for label in ("other", "this"):
            ms = [run[key]["ms"] for run in runs[label]]
            row[label] = {"best_ms": min(ms), "spread_ms": round(max(ms) - min(ms), 3)}
        row["same_bytes"] = len({run[key]["checksum"] for lab in runs for run in runs[lab]}) == 1
        res["calls"][key] = row
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--compare", metavar="OTHER.so")
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(compare(a.compare, a.rounds, a.reps) if a.compare else measure(a.reps)), flush=True)


if __name__ == "__main__":
    main()
