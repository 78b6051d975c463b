"""BASELINE config 5: 10,000 perturbed-TLE draws of one object x 1,440 epochs -- fp64 vs fp32 arithmetic.
Prints max / RMS of |dr| and |dv| (fp32 variants against the fp64 kernel) and the fp64 kernel's parity with
the CPU oracle on a sample of draws.   python tools/mc_fp32_study.py > mc_fp32.json"""
import json, os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from astroz_b200 import Constellation, synth
from oracle import oracle as orc   # checker only

tles = synth.monte_carlo_catalog(10000)
jd, fr = synth.time_grid(1440, jd0=2460437.5)
c = Constellation(tles)
c.set_timing(True)
dev = torch.device("cuda", 0); n, nt = len(tles), len(jd)
p64 = torch.empty((n, nt, 3), dtype=torch.float64, device=dev); v64 = torch.empty_like(p64)
for _ in range(3):
    c.propagate_device(jd, fr, p64, v64); c.synchronize()
k64 = c.last_kernel_ms()[0]
res = {"workload": "config5: 10,000 Gaussian draws of the ISS TLE x 1,440 epochs (seed 12345)", "cells": n * nt,
       "fp64_kernel_ms": k64}
rows = np.arange(0, n, 250)
po, vo, err, _ = orc.constellation_propagate([tles[i] for i in rows], jd, fr)
ridx = torch.as_tensor(rows, device=dev)
res["fp64_vs_oracle"] = {"max_dr_km": float(np.abs(p64[ridx].cpu().numpy() - po).max()),
                         "max_dv_kms": float(np.abs(v64[ridx].cpu().numpy() - vo).max()), "draws_checked": len(rows)}
for name, phase in (("fp32_all", False), ("fp32_with_fp64_phase", True)):
    p32 = torch.empty_like(p64); v32 = torch.empty_like(p64)
    c.propagate_device_f32(jd, fr, p32, v32, phase64=phase); c.synchronize()
    ms = c.last_kernel_ms()[0]
    dr = torch.linalg.norm(p32 - p64, dim=2); dv = torch.linalg.norm(v32 - v64, dim=2)
    res[name] = {"kernel_ms": ms, "max_dr_km": float(dr.max()), "rms_dr_km": float(dr.pow(2).mean().sqrt()),
                 "max_dv_kms": float(dv.max()), "rms_dv_kms": float(dv.pow(2).mean().sqrt()),
                 "dr_at_epoch_rms_km": float(dr[:, 0].pow(2).mean().sqrt()), "dr_at_24h_rms_km": float(dr[:, -1].pow(2).mean().sqrt())}
print(json.dumps(res, indent=1))
