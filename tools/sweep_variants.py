#!/usr/bin/env python
"""On-device sweep of the K1 tuning variants (ASTROZ_SGP4_VARIANT) on the headline grid.
    python tools/sweep_variants.py [n_variants] > sweep.jsonl
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from astroz_b200 import Constellation, synth  # noqa: E402

nv = int(sys.argv[1]) if len(sys.argv) > 1 else 10
tles = synth.near_earth_catalog()
jd, fr = synth.time_grid()
dev = torch.device("cuda", 0)
n, nt = len(tles), len(jd)
block = torch.empty((2, n, nt, 3), dtype=torch.float64, device=dev)
stream = torch.cuda.Stream(dev)
torch.cuda.set_stream(stream)
ref = None
res = []
for v in [-1] + list(range(nv)):
    os.environ["ASTROZ_SGP4_VARIANT"] = str(v)
    c = Constellation(tles)
    for _ in range(5):
        c.propagate_device(jd, fr, block[0], block[1], stream=stream.cuda_stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    K = 20
    for _ in range(K):
        c.propagate_device(jd, fr, block[0], block[1], stream=stream.cuda_stream)
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    chk = block[:, ::97, ::13].clone()
    if ref is None:
        ref = chk
    same = bool(torch.equal(chk, ref))
    maxdiff = float((chk - ref).abs().max())
    res.append({"variant": v, "ms": ms, "Gprops": n * nt / ms / 1e6, "bitwise_same_as_default": same, "maxdiff": maxdiff})
    print(json.dumps(res[-1]), flush=True)
    del c
