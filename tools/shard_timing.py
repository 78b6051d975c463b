#!/usr/bin/env python
"""Compute-only strong scaling of the headline grid, measured on ONE GPU: the 1/N satellite shard a rank of an N-GPU
run propagates (N = 1, 2, 4, 8), timed back to back on the launching stream, for the automatic epochs-per-CTA choice
and for fixed stripes (ASTROZ_K1_STRIPE).  efficiency = t(1) / (N * t(1/N)).
    python tools/shard_timing.py > shard_timing.jsonl
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from astroz_b200 import Constellation, synth  # noqa: E402
from astroz_b200.parallel import shard_bounds  # noqa: E402

tles = synth.near_earth_catalog()
jd, fr = synth.time_grid()
dev = torch.device("cuda", 0)
stream = torch.cuda.Stream(dev)
torch.cuda.set_stream(stream)
nt = len(jd)
for stripe in os.environ.get("AZ_STRIPES", "0,384,192,96").split(","):
    os.environ["ASTROZ_K1_STRIPE"] = stripe
    base = None
    for world in (1, 2, 4, 8):
        b, e = shard_bounds(len(tles), world)[0]
        c = Constellation(tles[b:e])
        n = e - b
        block = torch.empty((2, n, nt, 3), dtype=torch.float64, device=dev)
        step = lambda: c.propagate_device(jd, fr, block[0], block[1], stream=stream.cuda_stream)  # noqa: E731
        for _ in range(20):
            step()
        torch.cuda.synchronize()
        K = 400
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(K):
            step()
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / K
        kms = []
        c.set_timing(True)
        for _ in range(5):
            step()
            c.synchronize()
            kms.append(c.last_kernel_ms()[0])
        base = base or ms
        print(json.dumps({"stripe": "auto" if stripe == "0" else int(stripe), "n_gpus_emulated": world, "sats": n,
                          "ms_per_step": ms, "kernel_ms": min(kms), "Gprops": n * nt / ms / 1e6,
                          "compute_only_efficiency": base / (world * ms)}), flush=True)
        del c, block
