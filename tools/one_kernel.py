#!/usr/bin/env python
"""Run one output specialisation of the near-earth grid a few times (an ncu target):
    ncu --set full -k regex:sgp4_grid_kernel --launch-skip 3 -c 1 -o prof python tools/one_kernel.py <layout> <mode> <vel> [n_sats]
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from astroz_b200 import Constellation, synth  # noqa: E402

layout, mode, vel = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
n = int(sys.argv[4]) if len(sys.argv) > 4 else synth.HEADLINE_SATS
tles = synth.near_earth_catalog(n)
jd, fr = synth.time_grid()
dev = torch.device("cuda", 0)
c = Constellation(tles)
nt = len(jd)
pos = torch.empty((n * nt * 3,), dtype=torch.float64, device=dev)
velb = torch.empty_like(pos) if vel else None
for _ in range(6):
    c.propagate_device(jd, fr, pos, velb, None, mode, layout)
c.synchronize()
