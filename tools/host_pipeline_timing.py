#!/usr/bin/env python
"""Host orchestration of the C ABI (astroz_b200/csrc/az_capi.cu, az_hostcopy.cu): the calls that run the two-slot chunk
pipeline (ChunkPipeline), the calls that place grid results in the caller's host block, and the single-pass calls
around them.  Host-buffer calls run with pinned and with pageable buffers.  Host clock around calls that end in a
synchronise, best of --reps after a warm-up call, and a SHA-256 of the result bytes.  Prints one JSON line with the
card's name, power limit and maximum SM clock.

  pairs W1 / W4  tools/pairs_timing.py's W1 (19,408,320 queries over the config-2 catalogue) and W4 (100,000 queries),
                 TEME with velocities and status
  sgp4_array     the ISS over 31,536,000 epochs at one second ("1 year (second)"), through astroz_cuda_sgp4_array
  numerical N1   tools/numerical_timing.py's N1 (100,000 LEO states, J2 + drag, one day at 60 s, DP87) through
                 astroz_cuda_propagate_numerical
  propagate      the config-2 mixed catalogue (13,478 satellites, 1,024 GEO, 256 Molniya, 256 GPS) over 1,440 epochs,
                 TEME with velocities, satellite- and time-major; also on a three-shard handle of one GPU
                 (ASTROZ_DEVICE_LIST=0,0,0)
  sgp4_into      astroz_cuda_sgp4_propagate_into, the 13,478 near-earth satellites over 1,440 epochs with a seeded
                 9-in-10 mask and per-satellite epoch offsets into a block 512 rows wider than the catalogue
  sdp4_into      astroz_cuda_sdp4_propagate_into, the mixed catalogue's deep-space members over 1,440 epochs at row 32 of
                 a block 64 rows wider, both layouts
  batch          astroz_cuda_sgp4_propagate_batch, the ISS (near) and a GEO satellite (deep) at 1, 63, 64 and 10,000
                 seeded epochs within a week of the element epoch
  screen         astroz_cuda_sgp4_screen (target 0, 10 km) and astroz_cuda_sgp4_screen_all (10 km) over the near-earth
                 catalogue and 1,440 epochs
  device         astroz_cuda_constellation_propagate_device_f32 (near-earth catalogue) and
                 astroz_cuda_sdp4_propagate_into_device (the mixed catalogue's deep-space members), 1,440 epochs

The whole-batch calls (one device block per call, no chunk pipeline), each at a workload of its family's timing tool:
  fit_elements FT1     tools/fit_timing.py's FT1: the config-2 catalogue, 1,440 K1-grid states each, perturbed guesses
  fit_observations OT1 tools/fit_obs_timing.py's OT1: the config-2 catalogue from radar tracks of six stations, B* held
  observe OT1          astroz_cuda_observe of OT1's observations, from propagate_pairs states at their times
  covariance CV2       tools/covariance_timing.py's CV2: one query per config-2 row at a common time, TEME
  conjunction PC1      tools/conjunction_timing.py's PC1: 100,000 engineered LEO crossings
  correlate CR1        tools/correlate_timing.py's CR1 at 1,000 radar tracks of 10 observations
  initial_orbits       tools/iod_timing.py's 100,000-track mix (tests/fit_oracle/iod.py mixed_tracks)
  lambert L1           tools/lambert_timing.py's L1 problem set (10^7 LEO-GEO problems, max_revs = 0), seed 1

    python tools/host_pipeline_timing.py [--reps 3] [--calls all|chunked|whole_batch]
    python tools/host_pipeline_timing.py --compare OTHER.so [--rounds 5] [--calls ...]

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


def propagate_case(c, jd, fr, layout, pinned, reps):
    shape = c._shape(len(jd), layout)
    pos, vel = empty(shape, np.float64, pinned), empty(shape, np.float64, pinned)
    ms = best_ms(lambda: c.propagate(jd, fr, pos, vel, 0, layout), reps)
    return ms, checksum([pos, vel])


def sgp4_into_case(c, times, off, mask, rows, time_major, pinned, reps):
    # masked and surplus rows keep what the block held before the call: a fill that is part of the checksum
    shape = (len(times), rows, 3) if time_major else (rows, len(times), 3)
    pos, vel = like(np.full(shape, 0.5), pinned), like(np.full(shape, -0.5), pinned)
    ms = best_ms(lambda: c.propagate_into(times, pos, vel, epoch_offsets=off, satellite_mask=mask,
                                          time_major=time_major, output_stride=rows), reps)
    return ms, checksum([pos, vel])


def sdp4_into_case(c, jd, fr, rows, offset, time_major, pinned, reps):
    shape = (len(jd), rows, 3) if time_major else (rows, len(jd), 3)
    pos, vel = like(np.full(shape, 0.5), pinned), like(np.full(shape, -0.5), pinned)
    ms = best_ms(lambda: c.propagate_sdp4_into(jd, fr, pos, vel, time_major=time_major, output_stride=rows,
                                               sat_offset=offset), reps)
    return ms, checksum([pos, vel])


def batch_case(s, times, reps):
    from astroz_b200 import _lib

    out = np.zeros((len(times), 6))
    L = _lib.lib()
    ms = best_ms(lambda: _lib.check(L.astroz_cuda_sgp4_propagate_batch(s._h, _lib.dptr(times), _lib.dptr(out),
                                                                       len(times))), reps)
    return ms, checksum([out])


def screen_case(c, times, off, reps):
    out = [None]

    def call():
        out[0] = c.screen_conjunction(times, 0, 10.0, epoch_offsets=off)

    return best_ms(call, reps), checksum(out[0])


def screen_all_case(c, times, off, reps):
    from astroz_b200 import _lib

    ns, cap = c.numSgp4, 2_000_000
    pairs, tidx, cnt = np.empty((cap, 2), np.uint32), np.empty(cap, np.uint32), C.c_uint64()
    L = _lib.lib()
    u32p = C.POINTER(C.c_uint32)
    ms = best_ms(lambda: _lib.check(L.astroz_cuda_sgp4_screen_all(
        c._h, _lib.dptr(times), len(times), _lib.dptr(off[:ns]), 10.0, pairs.ctypes.data_as(u32p),
        tidx.ctypes.data_as(u32p), cap, C.byref(cnt))), reps)
    # hits are appended in whatever order the threads find them: the hit set is compared in the API's sorted order
    from astroz_b200.constellation import _sorted_hits

    k = min(cnt.value, cap)
    return ms, checksum([np.array([cnt.value], np.uint64), *_sorted_hits(pairs[:k], tidx[:k])])


def device_f32_case(c, jd, fr, reps):
    import torch

    pos = torch.zeros((c.numSatellites, len(jd), 3), dtype=torch.float64, device="cuda:0")
    vel = torch.zeros_like(pos)

    def call():
        c.propagate_device_f32(jd, fr, pos, vel)
        torch.cuda.synchronize()

    return best_ms(call, reps), checksum([pos.cpu().numpy(), vel.cpu().numpy()])


def sdp4_device_case(c, jd, fr, reps):
    import torch

    from astroz_b200 import _lib

    nd = c.numSdp4
    block = torch.zeros((2, nd, len(jd), 3), dtype=torch.float64, device="cuda:0")
    L = _lib.lib()

    def call():
        _lib.check(L.astroz_cuda_sdp4_propagate_into_device(
            c._h, _lib.dptr(jd), _lib.dptr(fr), len(jd), C.c_void_p(block[0].data_ptr()),
            C.c_void_p(block[1].data_ptr()), 0, 0, nd, 0, None))
        c.synchronize()

    return best_ms(call, reps), checksum([block.cpu().numpy()])


class Out:
    """An output argument of a whole-batch call: zero-filled, pinned or pageable like the inputs."""

    def __init__(self, shape, dtype=np.float64):
        self.shape, self.dtype = shape, dtype


def whole_batch_case(name, args, pinned, reps):
    from astroz_b200 import _lib

    held = [like(np.zeros(a.shape, a.dtype), pinned) if isinstance(a, Out)
            else like(np.ascontiguousarray(a), pinned) if isinstance(a, np.ndarray) else a for a in args]
    outs = [h for a, h in zip(args, held) if isinstance(a, Out)]
    fn = getattr(_lib.lib(), f"astroz_cuda_{name}")
    values = [ptr(h) if isinstance(h, np.ndarray) else h for h in held]
    ms = best_ms(lambda: _lib.check(fn(*values)), reps)
    return ms, checksum(outs)


def whole_batch_workloads():
    """(record name, C function without its astroz_cuda_ prefix, arguments) of every whole-batch call"""
    import conjunction_timing
    import correlate_timing
    import covariance_timing
    import fit_obs_timing
    import lambert_timing

    from astroz_b200 import synth
    from astroz_b200.constellation import Constellation, Layout
    from tests import fit_oracle as R
    from tests.fit_oracle import conjunction_cases as cc
    from tests.fit_oracle import iod as I
    from tests.fit_oracle import obs as O

    u8, u32 = np.uint8, np.uint32
    el = synth.elements_from_tles(synth.near_earth_catalog(13478))
    n = el.shape[1]
    c = Constellation.from_elements(*el)
    jd, fr = synth.time_grid(1440)
    pos, vel = c.propagate(jd, fr, layout=Layout.satelliteMajor)
    m = n * 1440
    yield "fit_elements_FT1", "fit_elements", [
        R.perturbed(el, seed=3), n, 1, np.arange(n + 1, dtype=u32) * 1440, np.tile(jd, n), np.tile(fr, n),
        np.array(pos).reshape(-1, 3), np.array(vel).reshape(-1, 3), m, 1.0, 1e-3, 1, 25, 0, Out((8, n)), Out((n, 2)),
        Out(n, u32), Out(n, u8)]
    del pos, vel

    g = R.perturbed(el, seed=3)
    g[7] = el[7]
    fr2 = np.arange(1440) * 2.0 / 1440.0 + fr[0]
    ojd, ofr, kind, value, sigma, station, off = O.concat(
        fit_obs_timing._tracks(el, O.RADAR, O.RADAR_SITES, jd, fr2))
    off, station, sites = off.astype(u32), station.astype(u32), np.ascontiguousarray(O.RADAR_SITES, np.float64)
    m, k = len(ojd), len(sites)
    yield "fit_observations_OT1", "fit_observations", [
        g, n, 1, off, ojd, ofr, value, sigma, station, kind, m, sites, k, 0, 25, 0, Out((8, n)), Out(n), Out(n, u32),
        Out((n, 28)), Out(n, u32), Out(n, u8), Out(n, u8)]
    p, v, _ = c.propagate_pairs(np.repeat(np.arange(n), np.diff(off)), ojd, ofr)
    states = np.concatenate([np.asarray(p), np.asarray(v)], axis=1)
    yield "observe_OT1", "observe", [states, ojd, ofr, kind, station, m, sites, k, 0, Out((m, 6))]
    c.deinit()
    del states, value, sigma

    _, el_c, model, sat, qjd, qfr = next(w for w in covariance_timing._workloads() if w[0] == "CV2")
    m = len(sat)
    yield "covariance_CV2", "propagate_covariance", [
        el_c, n, 1, covariance_timing._covariances(n), model, np.searchsorted(sat, np.arange(n + 1)).astype(u32), qjd,
        qfr, m, 0, 0, Out((m, 6)), Out((m, 21)), None, Out(m, u8)]

    _, el_p, pr, se, cjd, cfr, w, deep = next(x for x in conjunction_timing._workloads() if x[0] == "PC1")
    np_, m = el_p.shape[1], len(pr)
    model = np.full(np_, deep, u8)
    yield "conjunction_PC1", "conjunction", [
        el_p, np_, 1, conjunction_timing._covariances(np_, model.astype(bool)), model, pr.astype(u32),
        se.astype(u32), cjd, cfr, np.full(m, w), np.full(m, 0.02), m, 0, 0, Out((m, 13)), Out((m, 2, 6)),
        Out((m, 2, 21)), Out(m, u8)]

    el2 = synth.elements_from_tles(synth.near_earth_catalog(13478, 13478))
    n2 = el2.shape[1]
    ids, tjd, tfr, kind, value, sigma, station = correlate_timing._tracks(
        el2, np.random.default_rng(1).integers(0, n2, 1000), O.RADAR, 10, 10.0, seed=1000)
    t, m, best = 1000, len(ids), 4
    yield "correlate_CR1", "correlate", [
        el2, n2, 1, cc.P_words(n2, scale=0.3, seed=12), None, np.searchsorted(ids, np.arange(t + 1)).astype(u32), t,
        tjd, tfr, kind, value, sigma, station.astype(u32), m, sites, k, 0.999, best, 0, Out((t, best), u32),
        Out((t, best)), Out(t, u32), Out(t, u32), Out(t, u32), Out(t, u8), Out(n2, u8)]

    tr = I.mixed_tracks(100_000, 31)
    t = tr.t
    yield "initial_orbits_100k", "initial_orbits", [
        tr.offsets, t, tr.jd, tr.fr, tr.kind, tr.value, tr.sigma, tr.station, len(tr.jd), tr.stations,
        len(tr.stations), None, 1, 0, Out((8, t)), Out((t, 6)), Out(t), Out(t, u8), Out(t, u32), Out((t, 2)),
        Out(t, u8), Out(t, u8)]

    n = 10_000_000
    r1, r2, tof, normal = lambert_timing.problems(np.random.default_rng(1), n, 6600.0, 42164.0, 2 * 86400.0)
    yield "lambert_L1", "lambert", [r1, r2, tof, normal, n, lambert_timing.MU, 0, 0, Out((n, 3)), Out((n, 3)),
                                    Out(n, u8), Out(n, u8)]


def measure(reps: int, calls: str = "all") -> dict:
    import astroz_b200
    from astroz_b200 import _lib, numerical, synth
    from astroz_b200.api import WGS72, Satrec
    from numerical_timing import teme_states
    from pairs_timing import queries
    from tests.golden import tles as G

    _lib.require_device()
    res = {"card_power_limit_max_sm_clock": card(), "lib": os.path.relpath(_lib.LIB_PATH, ROOT), "reps": reps}

    def record(name, ms, digest):
        res[name] = {"ms": round(ms, 3), "checksum": digest}
        print(f"{name}: {ms:.3f} ms", file=sys.stderr, flush=True)   # progress of a long run

    def both(name, case, *args):
        for pinned in (True, False):
            record(f"{name}_{'pinned' if pinned else 'pageable'}", *case(*args, pinned, reps))

    def one(name, case, *args):
        record(name, *case(*args, reps))

    if calls in ("all", "whole_batch"):
        for name, fn, args in whole_batch_workloads():
            both(name, whole_batch_case, fn, args)
    if calls == "whole_batch":
        return res

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

    jd, fr = synth.time_grid(1440)
    mixed = synth.mixed_catalog()
    c = astroz_b200.Constellation(mixed)
    for layout, tag in ((0, "sat"), (1, "time")):
        both(f"propagate_mixed_{tag}", propagate_case, c, jd, fr, layout)
    for time_major, tag in ((False, "sat"), (True, "time")):
        both(f"sdp4_into_wide_{tag}", sdp4_into_case, c, jd, fr, c.numSdp4 + 64, 32, time_major)
    one("sdp4_into_device", sdp4_device_case, c, jd, fr)
    del c
    os.environ["ASTROZ_DEVICE_LIST"] = "0,0,0"   # read when a device = -1 handle is made
    c = astroz_b200.Constellation(mixed, device=-1)
    del os.environ["ASTROZ_DEVICE_LIST"]
    for layout, tag in ((0, "sat"), (1, "time")):
        both(f"propagate_mixed_3shards_{tag}", propagate_case, c, jd, fr, layout)
    del c

    c = astroz_b200.Constellation(near)
    ns = c.numSgp4
    rng = np.random.default_rng(3)
    times = np.arange(1440, dtype=np.float64)
    off = rng.uniform(-1440.0, 0.0, ns)
    mask = (rng.uniform(size=ns) < 0.9).astype(np.uint8)
    for time_major, tag in ((False, "sat"), (True, "time")):
        both(f"sgp4_into_masked_wide_{tag}", sgp4_into_case, c, times, off, mask, ns + 512, time_major)
    one("sgp4_screen", screen_case, c, times, off)
    one("screen_all", screen_all_case, c, times, off)
    one("propagate_device_f32", device_f32_case, c, jd, fr)
    del c

    for tag, tle in (("near", G.ISS), ("deep", G.GEO28626)):
        s = Satrec.twoline2rv(*tle, WGS72)
        for n in (1, 63, 64, 10_000):
            one(f"batch_{tag}_{n}", batch_case, s, np.sort(np.random.default_rng(n).uniform(-1440.0, 10080.0, n)))
        del s
    return res


def compare(other: str, rounds: int, reps: int, calls: str) -> dict:
    runs = {"other": [], "this": []}
    for r in range(rounds):
        for label in (("other", "this") if r % 2 == 0 else ("this", "other")):
            env = dict(os.environ)
            env.pop("ASTROZ_B200_LIB", None)
            if label == "other":
                env["ASTROZ_B200_LIB"] = os.path.abspath(other)
            print(f"round {r}: {label}", file=sys.stderr, flush=True)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--reps", str(reps), "--calls", calls], env=env,
                               stdout=subprocess.PIPE, text=True, check=True)
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
    ap.add_argument("--calls", choices=("all", "chunked", "whole_batch"), default="all",
                    help="chunked: the calls above the whole-batch ones; whole_batch: those alone")
    a = ap.parse_args()
    print(json.dumps(compare(a.compare, a.rounds, a.reps, a.calls) if a.compare else measure(a.reps, a.calls)),
          flush=True)


if __name__ == "__main__":
    main()
