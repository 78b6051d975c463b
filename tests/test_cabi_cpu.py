"""CPU-side checks of the drop-in boundary: the C-ABI library loads here (no GPU), exports exactly what
include/astroz_b200.h declares, and refuses loudly to propagate without a device (no CPU fallback)."""
import os
import re
import subprocess

import numpy as np
import pytest

from tests.golden import tles as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from astroz_b200 import build

    return build.build()


def test_header_and_exports_match(built):
    header = open(os.path.join(ROOT, "include", "astroz_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(astroz_cuda_[a-z0-9_]+)\s*\(", header)))
    out = subprocess.run(["nm", "-D", "--defined-only", built], capture_output=True, text=True, check=True).stdout
    exported = sorted({ln.split()[-1] for ln in out.splitlines() if "astroz_cuda_" in ln})
    assert declared == exported
    from astroz_b200 import _lib

    assert sorted(_lib.EXPORTS) == declared
    L = _lib.lib()
    for name in declared:
        assert hasattr(L, name)
    assert L.astroz_cuda_version() == 0x000100


def test_library_is_sm90a_with_tma(built):
    """The shipped kernels are sm_90a SASS and the element tile is staged by a TMA bulk copy (UBLKCP)."""
    sass = subprocess.run(["cuobjdump", "-sass", built], capture_output=True, text=True).stdout
    if not sass:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in sass and "sm_100" not in sass
    assert "UBLKCP" in sass and "DFMA" in sass and "MUFU.RCP64H" in sass


def test_no_cpu_fallback(built):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the loud-failure path is exercised on the CPU box")
    import astroz_b200
    from astroz_b200 import AstrozCudaError

    assert astroz_b200.device_count() == 0
    with pytest.raises(AstrozCudaError) as ei:
        astroz_b200.Constellation([G.ISS])
    assert ei.value.code == -201 and "no CPU" in str(ei.value)
    from astroz_b200.api import Satrec

    with pytest.raises(AstrozCudaError):
        Satrec.twoline2rv(*G.ISS)
    with pytest.raises(AstrozCudaError):
        astroz_b200.fp64_peak_tflops()


def test_product_does_not_touch_the_oracle():
    """Nothing under astroz_b200/ (or include/) may import, link or mention the oracle."""
    bad = []
    for base in ("astroz_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h")):
                    txt = open(os.path.join(dirpath, f), errors="replace").read()
                    if re.search(r"\boracle\b|azo_|astroz_oracle", txt):
                        bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_jday_and_days2mdhms():
    # src/Datetime.zig:307-324
    from astroz_b200.api import days2mdhms, jday

    jd, fr = jday(2019, 1, 5, 4, 28, 31.5)
    assert jd == 2458488.5 and abs(fr - 0.18647569444444444) < 1e-9
    mon, day, hr, minute, sec = days2mdhms(2019, 5.186475694444444)
    assert (mon, day, hr, minute) == (1, 5, 4, 28) and abs(sec - 31.5) < 0.01


def test_synthetic_catalog_is_valid(oracle):
    from astroz_b200 import synth

    tles = synth.near_earth_catalog(600)
    assert all(len(a) == 69 and len(b) == 69 for a, b in tles)
    jd, fr = synth.time_grid(4)
    _, _, err, klass = oracle.constellation_propagate(tles, jd, fr)
    assert not klass.any() and not err.any()
    isimp = sum(oracle.Sgp4(*t).el["isimp"] for t in tles)
    assert 0 < isimp < 60       # the low-perigee shell exercises the simplified drag branch
    mixed = synth.mixed_catalog(400, n_geo=40, n_molniya=20, n_gps=20)
    _, _, _, k2 = oracle.constellation_propagate(mixed, jd, fr)
    assert np.bincount(k2, minlength=4).tolist() == [320, 20, 40, 20]


def test_zig_bindings_cover_every_export():
    """zig/src/c_api/cuda.zig (the reference-side binding a maintainer copies to src/c_api/cuda.zig) is generated from
    the header and committed: it must be up to date and declare every exported symbol with the header's arity; the
    device branch of Constellation.zig (zig/src/Constellation.device.zig) may only call symbols that exist."""
    import sys

    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_zig_bindings.py"), "--check"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    header = open(os.path.join(ROOT, "include", "astroz_b200.h")).read()
    declared = set(re.findall(r"\b(astroz_cuda_[a-z0-9_]+)\s*\(", header))
    zig = open(os.path.join(ROOT, "zig", "src", "c_api", "cuda.zig")).read()
    bound = dict(re.findall(r"pub extern fn (astroz_cuda_[a-z0-9_]+)\(([^)]*)\)", zig))
    assert set(bound) == declared, sorted(declared ^ set(bound))
    stripped = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    for name, zargs in bound.items():
        cargs = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", stripped, flags=re.S).group(1).strip()
        n_c = 0 if cargs in ("", "void") else cargs.count(",") + 1
        n_z = len(re.findall(r"(?:^|, )\w+: ", zargs))
        assert n_c == n_z, (name, n_c, n_z)
    branch = open(os.path.join(ROOT, "zig", "src", "Constellation.device.zig")).read()
    used = set(re.findall(r"cuda\.(astroz_cuda_[a-z0-9_]+)\(", branch))
    assert used and used <= declared, sorted(used - declared)
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert "zig/src/c_api/cuda.zig" in doc and "zig/src/Constellation.device.zig" in doc
