"""The per-query cores of the (satellite, time) pairs path (astroz_b200/csrc/az_pairs.cuh) run on the CPU by the
test-only harness tests/host_emul/emul_pairs.cu: gathered column access into the near-earth tiles, the tsince
expression, GMST and the output epilogues, checked against the scalar oracle.  The device run is in
tests/test_gpu_pairs.py."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.golden import tles as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "host_emul")
NODES = 6   # lattice checkpoints per direction: 3,600 minutes, so most queries of a +-7 day spread step on past it


@pytest.fixture(scope="module")
def emul_pairs():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = os.path.join(EMUL_DIR, "libemul_pairs.so")
    src = os.path.join(EMUL_DIR, "emul_pairs.cu")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC", "-shared", "-I" + csrc, "-o", so, src], check=True, capture_output=True)
    L = C.CDLL(so)
    dp = C.POINTER(C.c_double)

    def run(tles, sat, jd, fr, mode):
        n, nq = len(tles), len(sat)
        a1 = (C.c_char_p * n)(*[t[0].encode() for t in tles])
        a2 = (C.c_char_p * n)(*[t[1].encode() for t in tles])
        sat = np.ascontiguousarray(sat, dtype=np.uint32)
        pos, vel, ts, ep = np.zeros((nq, 3)), np.zeros((nq, 3)), np.zeros(nq), np.zeros(nq)
        st = np.zeros(nq, dtype=np.uint8)
        ref = np.zeros(1)
        rc = L.emul_pairs(a1, a2, n, 1, sat.ctypes.data_as(C.c_void_p), jd.ctypes.data_as(dp), fr.ctypes.data_as(dp),
                          nq, mode, NODES, pos.ctypes.data_as(dp), vel.ctypes.data_as(dp),
                          st.ctypes.data_as(C.c_void_p), ts.ctypes.data_as(dp), ref.ctypes.data_as(dp),
                          ep.ctypes.data_as(dp))
        assert rc == 0
        return pos, vel, st, ts, float(ref[0]), ep

    return run


def _queries(n_sats, nq, seed):
    from astroz_b200 import synth

    rng = np.random.default_rng(seed)
    sat = rng.integers(0, n_sats, nq)
    t = synth.BENCH_JD0 + rng.uniform(-7.0, 7.0, nq)
    jd = np.floor(t - 0.5) + 0.5      # midnight-based jd, the rest in fr, like python-sgp4's jday
    return sat, jd, t - jd


def test_pairs_cores_match_scalar_oracle_all_modes(emul_pairs, oracle):
    from astroz_b200 import synth

    tles = synth.mixed_catalog(300, n_geo=60, n_molniya=40, n_gps=40) + [G.ISS, G.GEO28626, G.HEO09880, G.GPS20413]
    sat, jd, fr = _queries(len(tles), 1500, 7)
    p0, v0, st, ts, ref, ep = emul_pairs(tles, sat, jd, fr, 0)
    # every class takes part, near-earth and deep-space alike
    _, _, _, klass = oracle.constellation_propagate(tles, jd[:1], fr[:1])
    assert set(klass[sat]) == {0, 1, 2, 3}
    deep = klass[sat] > 0

    # tsince equals the host grid expression bit for bit: tbase[t] + toff[s] near earth, (jd + fr - epoch) * 1440 deep
    jf = jd + fr
    grid_near = (jf - ref) * 1440.0 + (ref - ep) * 1440.0
    grid_deep = (jf - ep) * 1440.0
    assert np.array_equal(ts[~deep], grid_near[~deep])
    assert np.array_equal(ts[deep], grid_deep[deep])

    # TEME against the scalar propagators
    models = {}
    for i, s in enumerate(sat):
        if s not in models:
            models[s] = (oracle.Sdp4 if klass[s] else oracle.Sgp4)(*tles[s])
        m = models[s]
        if klass[s]:
            rc, r, v = m.propagate(ts[i])
            if rc != 0:
                assert st[i] != 0 and not p0[i].any()
                continue
        else:
            r, v = m.propagate(ts[i])
        assert np.max(np.abs(p0[i] - r)) < 1e-6, (i, s, klass[s])
        assert np.max(np.abs(v0[i] - v)) < 1e-9, (i, s, klass[s])
    ok = st == 0
    assert ok.mean() > 0.99

    # ECEF: the pure GMST rotation of the query's own epoch
    p1, v1, st1, *_ = emul_pairs(tles, sat, jd, fr, 1)
    assert np.array_equal(st1, st)
    g = np.array([oracle.julian_to_gmst(x) for x in jf])
    cg, sg = np.cos(g), np.sin(g)
    rot = lambda a: np.stack([a[:, 0] * cg + a[:, 1] * sg, -a[:, 0] * sg + a[:, 1] * cg, a[:, 2]], axis=1)
    assert np.max(np.abs(p1[ok] - rot(p0)[ok])) < 1e-9
    assert np.max(np.abs(v1[ok] - rot(v0)[ok])) < 1e-12

    # geodetic: the reference's ECEF -> (lat, lon, alt) of that ECEF position
    p2, _, st2, *_ = emul_pairs(tles, sat, jd, fr, 2)
    assert np.array_equal(st2, st)
    lla = np.array([oracle.ecef_to_geodetic(e) for e in p1[ok]])
    assert np.max(np.abs(p2[ok][:, :2] - lla[:, :2])) < 1e-12
    assert np.max(np.abs(p2[ok][:, 2] - lla[:, 2])) < 1e-7


def test_pairs_cores_are_order_independent(emul_pairs):
    """A query's bits depend on (sat, jd, fr) alone: a shuffled, duplicated list gives each query the same result."""
    from astroz_b200 import synth

    tles = synth.mixed_catalog(120, n_geo=20, n_molniya=20, n_gps=10)
    sat, jd, fr = _queries(len(tles), 400, 11)
    p, v, st, *_ = emul_pairs(tles, sat, jd, fr, 1)
    perm = np.random.default_rng(3).permutation(np.concatenate([np.arange(400), np.arange(0, 400, 3)]))
    pp, vp, sp, *_ = emul_pairs(tles, sat[perm], jd[perm], fr[perm], 1)
    assert np.array_equal(pp, p[perm]) and np.array_equal(vp, v[perm]) and np.array_equal(sp, st[perm])
