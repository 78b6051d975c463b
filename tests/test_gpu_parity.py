"""Parity of the CUDA path against the CPU oracle and the reference's golden vectors.

Every test here calls the product through its C-ABI (ctypes wrappers in astroz_b200) on a real GPU.
Tolerances (fp64): the north star asks for the reference's Vallado tolerance (< 10 m, < 1e-6 km/s as
tested in src/Sgp4Batch.zig:264-269, "< 1 um/s" as worded in README.md:47).  We hold the CUDA path to
1e-6 km (1 mm) and 1e-9 km/s (1 um/s) against the scalar oracle -- tighter than either.
"""
import ctypes as C
import math

import numpy as np
import pytest

from tests.golden import tles as G

pytestmark = pytest.mark.gpu

POS_TOL = 1e-6   # km
VEL_TOL = 1e-9   # km/s


@pytest.fixture(scope="module")
def az():
    import astroz_b200

    astroz_b200.lib()
    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return astroz_b200


@pytest.fixture(scope="module")
def synth():
    from astroz_b200 import synth as s

    return s


def _maxerr(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))))


# ---------------------------------------------------------------------------------------------- goldens
def test_vallado_vectors_on_gpu(az):
    # src/Sgp4Batch.zig:235-296 -- WGS72, 0.01 km / 1e-6 km/s in the reference
    from astroz_b200.api import Satrec, WGS72

    for tle, t, pos, vel in G.VALLADO:
        sat = Satrec.twoline2rv(*tle, WGS72)
        assert sat.error == 0 and not sat.is_deep_space
        e, r, v = sat.sgp4_array(np.array([sat.jdsatepoch]), np.array([sat.jdsatepochF + t / 1440.0]))
        # jd/fr round trip quantises tsince to one ulp of the Julian date (~40 us)
        assert _maxerr(r[0], pos) < 1e-3, (tle[0], t, r[0] - np.array(pos))
        assert _maxerr(v[0], vel) < 1e-6
        out = np.zeros(6)
        from astroz_b200 import _lib

        _lib.check(_lib.lib().astroz_cuda_sgp4_propagate_batch(sat._h, _lib.dptr(np.array([t])), _lib.dptr(out), 1))
        assert _maxerr(out[:3], pos) < 2e-8 and _maxerr(out[3:], vel) < 1e-9  # exact tsince: print precision


def test_python_sgp4_table_on_gpu(az):
    # src/validation_tests.zig:331-374 (0.1 km / 1e-4 km/s with WGS84; the table itself is WGS72)
    from astroz_b200 import _lib
    from astroz_b200.api import Satrec, WGS72, WGS84

    times = np.array([row[0] for row in G.SGP4_REFERENCE_TABLE])
    pos = np.array([row[1] for row in G.SGP4_REFERENCE_TABLE])
    vel = np.array([row[2] for row in G.SGP4_REFERENCE_TABLE])
    for wc, ptol, vtol in ((WGS84, 0.1, 1e-4), (WGS72, 5e-8, 5e-10)):
        sat = Satrec.twoline2rv(*G.ISS_VALIDATION, wc)
        out = np.zeros((len(times), 6))
        _lib.check(_lib.lib().astroz_cuda_sgp4_propagate_batch(sat._h, _lib.dptr(times), _lib.dptr(out), len(times)))
        assert _maxerr(out[:, :3], pos) < ptol
        assert _maxerr(out[:, 3:], vel) < vtol


def test_iss_python_sgp4_epoch_state(az):
    # src/Sgp4.zig:906-948, WGS84: 1e-3 km / 1e-5 km/s
    from astroz_b200.api import Satrec, WGS84

    sat = Satrec.twoline2rv(*G.ISS, WGS84)
    e, r, v = sat.sgp4(sat.jdsatepoch, sat.jdsatepochF)
    assert e == 0
    assert np.linalg.norm(np.array(r) - np.array([-5887.061832, 3151.888264, -1263.887271])) < 1e-3
    assert np.linalg.norm(np.array(v) - np.array([-3.250642, -3.745001, 5.837125])) < 1e-5


def test_sdp4_vectors_on_gpu(az):
    # src/Sdp4.zig:1481-1559 -- GPS (irez 0), GEO (irez 1), HEO (irez 2); 0.01 km / 1e-5 km/s in the reference
    from astroz_b200 import _lib
    from astroz_b200.api import Satrec, WGS72

    for tle, t, pos, vel in G.SDP4_VECTORS:
        sat = Satrec.twoline2rv(*tle, WGS72)
        assert sat.error == 0 and sat.is_deep_space
        out = np.zeros(6)
        _lib.check(_lib.lib().astroz_cuda_sgp4_propagate_batch(sat._h, _lib.dptr(np.array([t])), _lib.dptr(out), 1))
        assert _maxerr(out[:3], pos) < 1e-6, (tle[0], t, out[:3] - np.array(pos))
        if vel is not None:
            assert _maxerr(out[3:], vel) < 1e-8


def test_classification_and_counts(az):
    # src/Constellation.zig:766-781
    c = az.Constellation([G.ISS, G.GEO28626, G.SAT55909, G.GPS20413, G.SAT55910])
    assert (c.numSatellites, c.numSgp4, c.numSdp4) == (5, 3, 2)
    assert list(c.classes) == [0, 2, 0, 1, 0]
    c2 = az.Constellation([G.ISS, G.SAT55909, G.SAT55910])
    assert (c2.numSgp4, c2.numSdp4) == (3, 0)
    c3 = az.Constellation([G.GEO28626, G.GPS20413, G.HEO09880])
    assert (c3.numSgp4, c3.numSdp4) == (0, 3) and list(c3.classes) == [2, 1, 3]


# ---------------------------------------------------------------------------------------------- config 1
def test_config1_iss_1440_epochs(az, oracle):
    """BASELINE config 1: ISS x 1,440 epochs, WGS72, jd = jdsatepoch, fr = jdsatepochF + i/1440
    (benchmarks/python_astroz_bench.py:69-71)."""
    from astroz_b200.api import Satrec, WGS72

    sat = Satrec.twoline2rv(*G.ISS, WGS72)
    jd = np.full(1440, sat.jdsatepoch)
    fr = sat.jdsatepochF + np.arange(1440) / 1440.0
    e, r, v = sat.sgp4_array(jd, fr)
    ref = oracle.Sgp4(*G.ISS, grav=oracle.WGS72)
    ts = ((jd + fr) - (sat.jdsatepoch + sat.jdsatepochF)) * 1440.0
    ro = np.array([ref.propagate(t)[0] for t in ts])
    vo = np.array([ref.propagate(t)[1] for t in ts])
    assert not e.any()
    assert _maxerr(r, ro) < POS_TOL and _maxerr(v, vo) < VEL_TOL
    # scalar entry point agrees with the batch one
    e1, r1, v1 = sat.sgp4(jd[7], fr[7])
    assert e1 == 0 and _maxerr(r1, r[7]) < 1e-9 and _maxerr(v1, v[7]) < 1e-12


# ---------------------------------------------------------------------------------------------- grids
@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_near_earth_grid_vs_oracle(az, oracle, synth, layout, mode):
    tles = synth.near_earth_catalog(1003)           # not a multiple of the 8-satellite tile
    jd, fr = synth.time_grid(1440)
    jd, fr = jd[::11][:131].copy(), fr[::11][:131].copy()   # 131 epochs: ragged vs the 32-lane warps
    c = az.Constellation(tles)
    assert c.numSgp4 == 1003
    p, v = c.propagate(jd, fr, outputMode=mode, layout=layout)
    po, vo, err, _ = oracle.constellation_propagate(tles, jd, fr, mode=mode, layout=layout)
    assert not err.any()
    if mode == 2:   # (lat rad, lon rad, alt km): src/Constellation.zig:497
        assert _maxerr(p[..., :2], po[..., :2]) < 1e-10
        assert _maxerr(p[..., 2], po[..., 2]) < POS_TOL
    else:
        assert _maxerr(p, po) < POS_TOL
    assert _maxerr(v, vo) < VEL_TOL


def test_mixed_grid_vs_oracle_with_status(az, oracle, synth):
    import torch

    tles = synth.mixed_catalog(1200, n_geo=160, n_molniya=80, n_gps=80)
    jd, fr = synth.time_grid(1440)
    jd, fr = jd[::7].copy(), fr[::7].copy()
    c = az.Constellation(tles)
    po, vo, err, klass = oracle.constellation_propagate(tles, jd, fr)
    assert list(c.classes) == list(klass)
    assert c.numSdp4 == 320 and set(klass) == {0, 1, 2, 3}
    nt = len(jd)
    dev = torch.device("cuda", 0)
    pos = torch.empty((len(tles), nt, 3), dtype=torch.float64, device=dev)
    vel = torch.empty_like(pos)
    st = torch.full((len(tles), nt), 255, dtype=torch.uint8, device=dev)
    c.propagate_device(jd, fr, pos, vel, st)
    c.synchronize()
    assert _maxerr(pos.cpu().numpy(), po) < POS_TOL
    assert _maxerr(vel.cpu().numpy(), vo) < VEL_TOL
    st = st.cpu().numpy()
    deep = klass > 0
    assert np.array_equal(st[deep], err[deep])
    # host-buffer API == device API, bit for bit
    ph, vh = c.propagate(jd, fr, layout=0)
    assert np.array_equal(ph, pos.cpu().numpy()) and np.array_equal(vh, vel.cpu().numpy())
    # layouts agree to the reference's own layout-equivalence tolerance (src/Constellation.zig:869: 1e-10); not bit for
    # bit, because the two layouts group epochs differently per thread and the choice between equally valid small-angle
    # series / Newton exits is made per group (cells differ by ~1e-12 km)
    ptm, vtm = c.propagate(jd, fr, layout=1)
    assert _maxerr(ptm.transpose(1, 0, 2), ph) < 1e-10 and _maxerr(vtm.transpose(1, 0, 2), vh) < 1e-13


def test_week_long_and_backwards_in_time(az, oracle, synth):
    """Config-4 horizon (10,080 epochs) on a subset, plus epochs *before* the element epochs: exercises the
    negative direction of the SDP4 resonance lattice.  Unpinned by any reference vector (SURVEY.md 8c):
    the scalar oracle is the only authority here."""
    tles = synth.mixed_catalog(96, n_geo=16, n_molniya=16, n_gps=8) + [G.GEO28626, G.HEO09880, G.GPS20413]
    jd, fr = synth.time_grid(10080)
    for shift in (0.0, -30.0):
        c = az.Constellation(tles)
        p, v = c.propagate(jd + shift, fr, layout=0)
        po, vo, err, _ = oracle.constellation_propagate(tles, jd + shift, fr)
        assert not err.any()
        assert _maxerr(p, po) < POS_TOL, shift
        assert _maxerr(v, vo) < VEL_TOL, shift


def test_deep_space_failures_are_zero_filled_per_satellite(az, oracle, synth):
    """A decaying Molniya-type object: cells the scalar path rejects (src/Sdp4.zig:913-967) come back
    zero-filled with their code; neighbours in the same 8-batch are untouched (the reference zero-fills
    the whole batch, src/Constellation.zig:468-471 -- documented supersede)."""
    import torch

    bad = synth.tle_lines(42000, 24, 120.0, 63.4, 0.0, 0.755, 0.0, 10.0, 2.006, 1e-3)
    tles = [G.GPS20413, bad, G.GEO28626, G.HEO09880]
    jd = np.full(40, 2460430.5)
    fr = np.linspace(0.0, 2000.0, 40)          # ~5.5 years
    c = az.Constellation(tles)
    dev = torch.device("cuda", 0)
    pos = torch.empty((4, 40, 3), dtype=torch.float64, device=dev)
    vel = torch.empty_like(pos)
    st = torch.zeros((4, 40), dtype=torch.uint8, device=dev)
    c.propagate_device(jd, fr, pos, vel, st)
    c.synchronize()
    po, vo, err, _ = oracle.constellation_propagate(tles, jd, fr)
    st = st.cpu().numpy()
    assert err[1].any() and set(np.unique(err[1])) >= {1, 2}, "fixture should exercise decayed and invalid-ecc"
    assert np.array_equal(st, err)
    p = pos.cpu().numpy()
    assert np.all(p[1][err[1] != 0] == 0.0)
    ok = err == 0
    assert _maxerr(p[ok], po[ok]) < 1e-5      # years of propagation: angles ~1e5 rad
    assert np.all(p[0] != 0.0) and np.all(p[2] != 0.0)


def test_satrec_array_time_model(az, oracle, synth):
    """SatrecArray.sgp4: reference = jd[0]+fr[0], offsets and times as bindings/python/astroz/api.py:300-302."""
    from astroz_b200.api import Satrec, SatrecArray, WGS72

    tles = synth.near_earth_catalog(257)
    sats = [Satrec.twoline2rv(l1, l2, WGS72) for l1, l2 in tles[:40]]
    assert all(s.error == 0 for s in sats)
    arr = SatrecArray([Satrec.twoline2rv(l1, l2, WGS72) for l1, l2 in tles])
    jd, fr = synth.time_grid(97)
    e, r, v = arr.sgp4(jd, fr)
    ro, vo = oracle.satrec_array_sgp4(tles, jd, fr)
    assert e.shape == (257, 97) and e.dtype == np.uint8 and not e.any()
    assert r.shape == (257, 97, 3) and _maxerr(r, ro) < POS_TOL and _maxerr(v, vo) < VEL_TOL
    e2, r2, v2 = arr.sgp4(jd, fr, velocities=False)
    assert np.array_equal(r2, r) and not v2.any()
    # scalar jd/fr are accepted like python-sgp4
    e3, r3, v3 = arr.sgp4(jd[0], fr[5])
    assert r3.shape == (257, 1, 3)


def test_stateless_propagate_into(az, oracle, synth):
    # Constellation.propagateConstellation via SatrecArray.propagate_into (satrec.zig:896-988): time-major
    tles = synth.near_earth_catalog(75)
    c = az.Constellation(tles)
    ep = c.epochs
    ref = 2460437.75
    times = np.arange(0.0, 300.0, 2.5)
    off = (ref - ep) * 1440.0
    p, v = c.propagate_into(times, epoch_offsets=off)
    assert p.shape == (len(times), 75, 3)
    for i in (0, 13, 74):
        s = oracle.Sgp4(*tles[i])
        ro = np.array([s.propagate(t + off[i])[0] for t in times])
        assert _maxerr(p[:, i], ro) < POS_TOL


# ---------------------------------------------------------------------------------------------- edges
def test_edge_shapes_and_errors(az, oracle):
    from astroz_b200 import AstrozCudaError

    c = az.Constellation([G.ISS])
    epoch = c.epochs[0]
    p, v = c.propagate(np.array([math.floor(epoch)]), np.array([epoch - math.floor(epoch)]))
    r, vv = oracle.Sgp4(*G.ISS).propagate(0.0)
    assert p.shape == (1, 1, 3) and _maxerr(p[0, 0], r) < POS_TOL and _maxerr(v[0, 0], vv) < VEL_TOL
    # empty time axis is a no-op
    p0, v0 = c.propagate(np.array([]), np.array([]))
    assert p0.shape == (0, 1, 3)
    # 7 satellites (one partial tile), 33 epochs (one full warp + 1)
    tles7 = [G.ISS, G.SAT55909, G.SAT55910, G.SAT06251, G.SAT00005, G.ISS_VALIDATION, G.ISS]
    c7 = az.Constellation(tles7)
    jd = np.full(33, 2460500.5)
    fr = np.arange(33) / 97.0
    p7, v7 = c7.propagate(jd, fr, layout=0)
    po, vo, _, _ = oracle.constellation_propagate(tles7, jd, fr)
    good = np.isfinite(po).all(axis=(1, 2))
    assert good.sum() >= 5
    assert _maxerr(p7[good], po[good]) < 1e-5 and np.array_equal(np.isfinite(p7), np.isfinite(po))
    assert np.array_equal(p7[0], p7[6])   # duplicate satellites give identical rows (Sgp4Batch.zig:226-231)
    # errors: unparsable TLE, invalid eccentricity at init, short buffer, bad mode
    with pytest.raises(AstrozCudaError) as ei:
        az.Constellation([("1 25544U", "2 25544")])
    assert ei.value.code == -1
    with pytest.raises(AstrozCudaError) as ei:
        c.propagate(jd, fr, resultsPos=np.zeros(5))
    assert ei.value.code == -12          # src/Constellation.zig:255-257
    with pytest.raises(AstrozCudaError) as ei:
        c.propagate(jd, fr, outputMode=7)
    assert ei.value.code == -20
    decayed = ("1 00001U 24001A   24100.00000000  .00000000  00000+0  10000-3 0  9990",
               "2 00001  51.6000 100.0000 0900000  10.0000  20.0000 16.40000000    10")
    with pytest.raises(AstrozCudaError) as ei:   # perigee below the surface: Sgp4.zig:117-118
        az.Constellation([G.ISS, decayed])
    assert ei.value.code == -12


# ---------------------------------------------------------------------------------------------- full size
def test_headline_grid_properties(az, oracle, synth):
    """BASELINE config 2 at full size (13,478 x 1,440 = 19.4 M cells) through size-independent properties:
    layout equivalence, velocity-off equivalence, determinism, physical sanity, and an oracle spot check of
    complete rows."""
    import torch

    tles = synth.near_earth_catalog()
    jd, fr = synth.time_grid()
    c = az.Constellation(tles)
    assert c.numSatellites == synth.HEADLINE_SATS and c.numSdp4 == 0
    n, nt = c.numSatellites, len(jd)
    dev = torch.device("cuda", 0)
    pos = torch.empty((n, nt, 3), dtype=torch.float64, device=dev)
    vel = torch.empty_like(pos)
    c.propagate_device(jd, fr, pos, vel)
    c.synchronize()
    pos2 = torch.empty_like(pos)
    c.propagate_device(jd, fr, pos2, None)
    c.synchronize()
    assert torch.equal(pos, pos2)                                  # velocities off: same positions, bitwise
    ptm = torch.empty((nt, n, 3), dtype=torch.float64, device=dev)
    vtm = torch.empty_like(ptm)
    c.propagate_device(jd, fr, ptm, vtm, layout=1)
    c.synchronize()
    # layout equivalence at the reference's own tolerance (src/Constellation.zig:869); see test_mixed_grid_vs_oracle
    assert float((ptm.transpose(0, 1) - pos).abs().max()) < 1e-10
    assert float((vtm.transpose(0, 1) - vel).abs().max()) < 1e-13
    rmag = torch.linalg.norm(pos, dim=2)
    vmag = torch.linalg.norm(vel, dim=2)
    assert torch.isfinite(pos).all() and torch.isfinite(vel).all()
    assert float(rmag.min()) > 6378.0 + 60.0 and float(rmag.max()) < 6378.0 + 12000.0   # low-perigee shell decays to ~95 km
    assert float(vmag.min()) > 3.0 and float(vmag.max()) < 9.5
    rows = np.random.default_rng(7).choice(n, 160, replace=False)
    sub = [tles[i] for i in rows]
    ph = pos[torch.as_tensor(rows, device=dev)].cpu().numpy()
    vh = vel[torch.as_tensor(rows, device=dev)].cpu().numpy()
    ref0 = c.referenceEpochJd
    for k, i in enumerate(rows[:160]):
        s = oracle.Sgp4(*tles[i])
        ts = (jd + fr - ref0) * 1440.0 + (ref0 - s.epochJd) * 1440.0     # Constellation.zig:153,268,425
        ro = np.array([s.propagate(t) for t in ts[::9]])
        assert _maxerr(ph[k, ::9], ro[:, 0]) < POS_TOL and _maxerr(vh[k, ::9], ro[:, 1]) < VEL_TOL
    # end-to-end host API on pinned buffers gives the same block
    p_host, v_host = c.propagate(jd, fr, layout=0)
    assert np.array_equal(p_host[rows], ph) and np.array_equal(v_host[rows], vh)


# ---------------------------------------------------------------------------------------------- BASELINE grids, every cell
def _report(name, **kw):
    """Per-config maxima, printed (pytest -s / -rP) and appended to $ASTROZ_PARITY_LOG when that is set."""
    import json
    import os

    line = json.dumps({"config": name, **kw})
    print("parity_full:", line)
    out = os.environ.get("ASTROZ_PARITY_LOG")
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def _device_vs_oracle(dev_block, ref, chunk_rows=2048):
    """max |device - oracle| over the whole block, streamed through the host in row chunks (the blocks are up to
    466 MB each; nothing is sampled)."""
    worst = 0.0
    for r0 in range(0, ref.shape[0], chunk_rows):
        got = dev_block[r0:r0 + chunk_rows].cpu().numpy()
        worst = max(worst, float(np.max(np.abs(got - ref[r0:r0 + chunk_rows]))))
    return worst


def _full_grid_both_layouts(az, oracle, tles, jd, fr, name):
    """Whole-constellation check in the manner of the reference's own (src/Constellation.zig:784-873), at BASELINE
    size: EVERY cell of the grid against the scalar oracle, satellite-major and time-major, status bytes included."""
    import torch

    c = az.Constellation(tles)
    n, nt = c.numSatellites, len(jd)
    po, vo, err, klass = oracle.constellation_propagate(tles, jd, fr, threads=0)
    assert list(c.classes) == list(klass)
    dev = torch.device("cuda", 0)
    pos = torch.empty((n, nt, 3), dtype=torch.float64, device=dev)
    vel = torch.empty_like(pos)
    status = torch.full((n, nt), 255, dtype=torch.uint8, device=dev)
    c.propagate_device(jd, fr, pos, vel, status)
    c.synchronize()
    dr, dv = _device_vs_oracle(pos, po), _device_vs_oracle(vel, vo)
    st = status.cpu().numpy()
    deep = np.asarray(klass) != 0
    # deep-space cells carry the oracle's codes; near-earth cells flag mrt < 1 (the scalar path's decay check,
    # src/Sgp4.zig:588-590, which the oracle's near-earth entry reports through its zero-fill only for SDP4)
    assert np.array_equal(st[deep], err[deep])
    assert dr < POS_TOL and dv < VEL_TOL, (name, dr, dv)
    del pos, vel
    ptm = torch.empty((nt, n, 3), dtype=torch.float64, device=dev)
    vtm = torch.empty_like(ptm)
    c.propagate_device(jd, fr, ptm, vtm, layout=1)
    c.synchronize()
    dr_t = _device_vs_oracle(ptm.transpose(0, 1), po)
    dv_t = _device_vs_oracle(vtm.transpose(0, 1), vo)
    assert dr_t < POS_TOL and dv_t < VEL_TOL, (name, dr_t, dv_t)
    _report(name, cells=n * nt, n_sgp4=c.numSgp4, n_sdp4=c.numSdp4, max_dr_km=dr, max_dv_kms=dv,
            max_dr_km_time_major=dr_t, max_dv_kms_time_major=dv_t, failed_cells=int((err != 0).sum()))
    return c


def test_config2_full_grid_every_cell(az, oracle, synth):
    """BASELINE config 2: 13,478 near-earth satellites (seed 13478) x 1,440 epochs = 19,408,320 cells, all compared."""
    tles = synth.near_earth_catalog(synth.HEADLINE_SATS, seed=13478)
    jd, fr = synth.time_grid(1440)
    c = _full_grid_both_layouts(az, oracle, tles, jd, fr, "config2")
    assert c.numSdp4 == 0 and c.numSatellites == 13478


def test_config3_full_grid_every_cell(az, oracle, synth):
    """BASELINE config 3: the 13,478-slot catalog with 1,024 GEO + 256 Molniya + 256 GPS-like deep-space members
    (seed 28626) x 1,440 epochs, all cells, all four classes, status bytes."""
    tles = synth.mixed_catalog(synth.HEADLINE_SATS, seed=28626, n_geo=1024, n_molniya=256, n_gps=256)
    jd, fr = synth.time_grid(1440)
    c = _full_grid_both_layouts(az, oracle, tles, jd, fr, "config3")
    assert c.numSdp4 == 1536 and set(np.asarray(c.classes).tolist()) == {0, 1, 2, 3}


def test_config4_week_grid_strided_epochs(az, oracle, synth):
    """BASELINE config 4 on one GPU: the whole 13,478 x 10,080 grid (135.9 M cells, 6.5 GB in HBM) is propagated;
    every 16th epoch out to the end of the week (630 epochs x all satellites = 8.5 M cells) is compared with the
    oracle.  Horizons beyond one day are pinned by no reference vector (DESIGN section 5): the scalar restatement is
    the authority here."""
    import torch

    tles = synth.near_earth_catalog(synth.HEADLINE_SATS, seed=13478)
    jd, fr = synth.time_grid(10080)
    c = az.Constellation(tles)
    n, nt = c.numSatellites, len(jd)
    dev = torch.device("cuda", 0)
    pos = torch.empty((n, nt, 3), dtype=torch.float64, device=dev)
    vel = torch.empty_like(pos)
    c.propagate_device(jd, fr, pos, vel)
    c.synchronize()
    po, vo, err, _ = oracle.constellation_propagate(tles, jd[::16].copy(), fr[::16].copy(), threads=0)
    dr = _device_vs_oracle(pos[:, ::16], po)
    dv = _device_vs_oracle(vel[:, ::16], vo)
    assert torch.isfinite(pos).all() and torch.isfinite(vel).all()
    assert dr < POS_TOL and dv < VEL_TOL, (dr, dv)
    _report("config4", cells=n * nt, compared_cells=int(po.shape[0] * po.shape[1]), max_dr_km=dr, max_dv_kms=dv)


def test_config5_all_draws_every_cell(az, oracle, synth):
    """BASELINE config 5: all 10,000 Monte-Carlo draws x 1,440 epochs in fp64, every cell against the oracle."""
    import torch

    tles = synth.monte_carlo_catalog(10000)
    jd, fr = synth.time_grid(1440, jd0=2460437.5)
    c = az.Constellation(tles)
    assert c.numSgp4 == 10000
    n, nt = c.numSatellites, len(jd)
    dev = torch.device("cuda", 0)
    pos = torch.empty((n, nt, 3), dtype=torch.float64, device=dev)
    vel = torch.empty_like(pos)
    c.propagate_device(jd, fr, pos, vel)
    c.synchronize()
    po, vo, err, _ = oracle.constellation_propagate(tles, jd, fr, threads=0)
    dr, dv = _device_vs_oracle(pos, po), _device_vs_oracle(vel, vo)
    assert dr < POS_TOL and dv < VEL_TOL, (dr, dv)
    _report("config5", cells=n * nt, max_dr_km=dr, max_dv_kms=dv)


# ---------------------------------------------------------------------------------------------- next rows (SURVEY 8f)
def test_fused_single_target_screen(az, oracle, synth):
    """Constellation.screenConstellation (src/Constellation.zig:683-756) fused on the device: minimum distance
    and its first time index per satellite against one target; 12 bytes per satellite come back."""
    tles = synth.near_earth_catalog(700)
    # make a few near-neighbours of the target so some minima fall below the threshold
    base = tles[5]
    for k in range(6):
        l2 = base[1]
        ma = (float(l2[43:51]) + 0.02 * (k + 1)) % 360.0
        l2 = l2[:43] + f"{ma:8.4f}" + l2[51:68]
        l2 = l2 + str(synth._checksum(l2))
        tles[100 + k] = (base[0], l2)
    c = az.Constellation(tles)
    times = np.arange(0.0, 1440.0, 1.0)
    ref = 2460437.5
    off = (ref - c.epochs) * 1440.0
    for target, thr in ((5, 50.0), (311, 500.0)):
        d, ti = c.screen_conjunction(times, target, thr, epoch_offsets=off, reference_jd=ref)
        do, tio = oracle.screen_constellation(tles, times, off, target, thr, ref)
        assert d.shape == (700,) and ti.dtype == np.uint32
        assert np.max(np.abs(d - do)) < 1e-6
        assert d[target] == thr and ti[target] == 0
        hit = do < thr
        assert hit.sum() >= 3
        same = ti == tio
        # an index may differ only where two epochs tie to rounding
        assert same[~hit].all() and (same[hit].mean() > 0.95)


def test_single_satellite_long_time_axis(az, oracle):
    """Satrec.sgp4_array over a long axis (the reference's other published benchmark family,
    benchmarks/zig_sgp4_bench.zig:46-52): 1 satellite x 200k epochs runs on the dedicated time-parallel kernel
    and must agree with the grid kernel and the oracle."""
    from astroz_b200.api import Satrec, WGS72

    sat = Satrec.twoline2rv(*G.ISS, WGS72)
    n = 200_003
    jd = np.full(n, sat.jdsatepoch)
    fr = sat.jdsatepochF + np.arange(n) * (1.0 / 86400.0)
    e, r, v = sat.sgp4_array(jd, fr)
    ts = ((jd + fr) - (sat.jdsatepoch + sat.jdsatepochF)) * 1440.0
    ref = oracle.Sgp4(*G.ISS, grav=oracle.WGS72)
    idx = np.r_[0:40, n - 40:n, np.arange(0, n, 4999)]
    ro = np.array([ref.propagate(ts[i]) for i in idx])
    assert _maxerr(r[idx], ro[:, 0]) < POS_TOL and _maxerr(v[idx], ro[:, 1]) < VEL_TOL
    assert np.isfinite(r).all() and np.isfinite(v).all()
    # same satellite through the grid kernel (2 copies -> K1) gives the same numbers
    c = az.Constellation([G.ISS, G.ISS])
    p2, v2 = c.propagate(jd[:3000], fr[:3000], layout=0)
    assert _maxerr(p2[0], r[:3000]) < 1e-6 and np.array_equal(p2[0], p2[1])


def test_single_satellite_chunked_pipeline(az, oracle):
    """An axis long enough for the chunked upload / propagate / download pipeline of astroz_cuda_sgp4_array (three
    chunks of 1.5 M epochs): chunk seams, the pageable-input staging and the pinned result must all line up."""
    from astroz_b200.api import Satrec, WGS72

    sat = Satrec.twoline2rv(*G.ISS, WGS72)
    n = 4_500_007
    jd = np.full(n, sat.jdsatepoch)
    fr = sat.jdsatepochF + np.arange(n) * (1.0 / 86400.0)
    e, r, v = sat.sgp4_array(jd, fr)
    assert r.shape == (n, 3) and np.isfinite(r).all() and np.isfinite(v).all()
    ts = ((jd + fr) - (sat.jdsatepoch + sat.jdsatepochF)) * 1440.0
    ref = oracle.Sgp4(*G.ISS, grav=oracle.WGS72)
    seams = [1_500_032, 3_000_064]
    idx = np.r_[0:8, n - 8:n, np.arange(0, n, 150_001)]
    for sm in seams:
        idx = np.r_[idx, sm - 4:sm + 4]
    ro = np.array([ref.propagate(ts[i]) for i in idx])
    assert _maxerr(r[idx], ro[:, 0]) < POS_TOL and _maxerr(v[idx], ro[:, 1]) < VEL_TOL
    # a window across the first seam, propagated on its own (one chunk), agrees to rounding
    a, b = seams[0] - 10_000, seams[0] + 10_000
    _, r2, v2 = sat.sgp4_array(jd[a:b], fr[a:b])
    assert _maxerr(r2, r[a:b]) < 1e-9 and _maxerr(v2, v[a:b]) < 1e-12


def test_config5_monte_carlo_draws_and_fp32_study(az, oracle, synth):
    """BASELINE config 5: perturbed draws of one object.  fp64 kernel vs oracle at the usual tolerance; the fp32
    study kernels must stay within the (much looser) envelope single precision allows."""
    import torch

    tles = synth.monte_carlo_catalog(400)
    jd, fr = synth.time_grid(1440, jd0=2460437.5)
    jd, fr = jd[::16].copy(), fr[::16].copy()
    c = az.Constellation(tles)
    assert c.numSgp4 == 400
    p, v = c.propagate(jd, fr, layout=0)
    po, vo, err, _ = oracle.constellation_propagate(tles, jd, fr)
    assert _maxerr(p, po) < POS_TOL and _maxerr(v, vo) < VEL_TOL
    spread = np.linalg.norm(p - p.mean(axis=0), axis=2).max()
    assert 1.0 < spread < 500.0          # the draws really differ (0.01 deg ~ 1 km) but stay one object
    dev = torch.device("cuda", 0)
    p64 = torch.as_tensor(p, device=dev)
    for phase, tol in ((True, 0.05), (False, 5.0)):
        p32 = torch.empty_like(p64)
        v32 = torch.empty_like(p64)
        c.propagate_device_f32(jd, fr, p32, v32, phase64=phase)
        c.synchronize()
        assert float((p32 - p64).abs().max()) < tol


def test_constellation_from_numeric_elements(az, oracle, synth):
    """OMM-style ingest: numeric mean elements instead of TLE text (src/Tle.zig:134-215) give the same
    constellation as the text route when fed the values the text encodes."""
    tles = synth.mixed_catalog(120, n_geo=10, n_molniya=6, n_gps=4)
    t = [oracle.parse_tle(*x) for x in tles]
    cols = {k: np.array([r[k] for r in t]) for k in ("epochJd", "nRevDay", "ecc", "inclDeg", "raanDeg", "argpDeg", "maDeg", "bstar")}
    a = az.Constellation(tles)
    b = az.Constellation.from_elements(cols["epochJd"], cols["nRevDay"], cols["ecc"], cols["inclDeg"], cols["raanDeg"],
                                       cols["argpDeg"], cols["maDeg"], cols["bstar"])
    assert list(a.classes) == list(b.classes) and np.array_equal(a.epochs, b.epochs)
    jd, fr = synth.time_grid(50)
    pa, va = a.propagate(jd, fr, layout=0)
    pb, vb = b.propagate(jd, fr, layout=0)
    assert np.array_equal(pa, pb) and np.array_equal(va, vb)
    with pytest.raises(az.AstrozCudaError) as ei:
        az.Constellation.from_elements([2460400.5], [15.5], [1.2], [51.0], [0.0], [0.0], [0.0], [1e-4])
    assert ei.value.code == -11   # eccentricity outside [0, 1): src/Sgp4.zig:111-113


def test_constellation_from_text_blob(az):
    """Tle.MultiIterator semantics (src/Tle.zig:103-132): 3-line sets with name lines, blank lines, CRLF, a
    dangling line 1 and a short line are all tolerated; pairs are (1..., 2...) lines of >= 69 columns."""
    text = ("ISS (ZARYA)\r\n" + G.ISS[0] + "\r\n" + G.ISS[1] + "\r\n\r\n"
            "GEO SAT\n  " + G.GEO28626[0] + "  \n" + G.GEO28626[1] + "\n"
            + G.SAT55909[0] + "\n"            # line 1 without its line 2: dropped when the next line 1 arrives
            + G.SAT55910[0] + "\n" + G.SAT55910[1] + "\n"
            "1 short line\n")
    c = az.Constellation.from_text(text)
    assert (c.numSatellites, c.numSgp4, c.numSdp4) == (3, 2, 1)
    ref = az.Constellation([G.ISS, G.GEO28626, G.SAT55910])
    assert np.array_equal(c.epochs, ref.epochs) and list(c.classes) == list(ref.classes)


def test_all_vs_all_coarse_screen(az, oracle, synth):
    """coarseScreen (bindings/python/src/conjunction.zig:11-149) on the device: same SET of (s, other, t) hits as
    the CPU cell list, both on an externally supplied block (either layout, with a mask and NaN rows) and
    through the fused propagate -> screen entry point."""
    import torch

    tles = synth.near_earth_catalog(900)
    base = tles[7]
    for k in range(10):       # a cluster of near-neighbours so there are hits at a 30 km threshold
        l2 = base[1]
        ma = (float(l2[43:51]) + 0.05 * (k + 1)) % 360.0
        l2 = l2[:43] + f"{ma:8.4f}" + l2[51:68]
        tles[200 + 3 * k] = (base[0], l2 + str(synth._checksum(l2)))
    c = az.Constellation(tles)
    times = np.arange(0.0, 360.0, 1.5)
    ref = 2460437.5
    off = (ref - c.epochs) * 1440.0
    p_tm, _ = c.propagate_into(times, epoch_offsets=off, want_velocities=False, time_major=True)
    p_sm = np.ascontiguousarray(p_tm.transpose(1, 0, 2))
    thr = 30.0
    want_pairs, want_t = oracle.coarse_screen(p_sm, thr)
    assert len(want_t) > 50
    got_pairs, got_t = c.screen_all(times, thr, epoch_offsets=off)
    assert np.array_equal(got_pairs, want_pairs) and np.array_equal(got_t, want_t)
    # external block, satellite-major, with a masked satellite and a NaN row
    dev = torch.device("cuda", 0)
    blk = p_sm.copy()
    blk[203] = np.nan
    mask = np.ones(900, dtype=np.uint8)
    mask[206] = 0
    w_pairs, w_t = oracle.coarse_screen(blk, thr, valid_mask=mask)
    g_pairs, g_t = c.coarse_screen_device(torch.as_tensor(blk, device=dev), thr, layout=0,
                                          valid_mask=torch.as_tensor(mask, device=dev))
    assert np.array_equal(g_pairs, w_pairs) and np.array_equal(g_t, w_t)
    assert not np.isin(203, g_pairs) and not np.isin(206, g_pairs)
    g2_pairs, g2_t = c.coarse_screen_device(torch.as_tensor(np.ascontiguousarray(blk.transpose(1, 0, 2)), device=dev),
                                            thr, layout=1, valid_mask=torch.as_tensor(mask, device=dev))
    assert np.array_equal(g2_pairs, w_pairs) and np.array_equal(g2_t, w_t)


def test_odd_offsets_and_strides_take_the_unaligned_paths(az, synth):
    """Output rows placed at an odd offset inside a larger block, odd epoch counts, odd row counts: the 128-bit
    store paths must fall back to 8-byte stores (no misaligned access) and give the same numbers."""
    import torch

    tles = synth.near_earth_catalog(41)
    c = az.Constellation(tles)
    dev = torch.device("cuda", 0)
    for nt in (97, 64):
        jd, fr = synth.time_grid(nt)
        sm_p, sm_v = c.propagate(jd, fr, layout=0)
        for layout in (0, 1):
            # the reference block in the SAME layout (same launch shape: bit for bit), rows at offset 0
            ref_p, ref_v = c.propagate(jd, fr, layout=layout)
            if layout == 1:
                ref_p, ref_v = ref_p.transpose(1, 0, 2), ref_v.transpose(1, 0, 2)
                # across layouts a cell may take a different series (the choice is per thread over its epochs): the
                # reference's own layout-equivalence bound (src/Constellation.zig:869)
                assert _maxerr(ref_p, sm_p) < 1e-10 and _maxerr(ref_v, sm_v) < 1e-13
            rows = 41 + 7
            shape = (rows, nt, 3) if layout == 0 else (nt, rows, 3)
            pos = torch.full(shape, -1.0, dtype=torch.float64, device=dev)
            vel = torch.full(shape, -1.0, dtype=torch.float64, device=dev)
            c.propagate_device(jd, fr, pos, vel, None, 0, layout, out_num_sats=rows, out_sat_offset=3)
            c.synchronize()
            p = pos.cpu().numpy() if layout == 0 else pos.cpu().numpy().transpose(1, 0, 2)
            v = vel.cpu().numpy() if layout == 0 else vel.cpu().numpy().transpose(1, 0, 2)
            assert np.array_equal(p[3:44], ref_p) and np.array_equal(v[3:44], ref_v)
            assert np.all(p[:3] == -1.0) and np.all(p[44:] == -1.0)     # neighbours untouched


def test_propagate_into_mask_and_output_stride(az, oracle, synth):
    """satellite_mask and output_stride of Sgp4Constellation.propagate_into (bindings/python/src/sgp4.zig:171-268,
    src/Constellation.zig:436-446,530-533): masked rows are left untouched, the block may be wider than the
    constellation."""
    tles = synth.near_earth_catalog(37)
    c = az.Constellation(tles)
    times = np.arange(0.0, 130.0, 2.0)
    off = (2460437.5 - c.epochs) * 1440.0
    full_p, full_v = c.propagate_into(times, epoch_offsets=off, time_major=False)
    mask = np.ones(37, dtype=np.uint8)
    mask[[0, 5, 8, 9, 36]] = 0
    for tm in (False, True):
        rows = 45
        shape = (rows, len(times), 3) if not tm else (len(times), rows, 3)
        p = np.full(shape, 7.0)
        v = np.full(shape, 7.0)
        c.propagate_into(times, p, v, epoch_offsets=off, satellite_mask=mask, time_major=tm, output_stride=rows)
        ps = p if not tm else p.transpose(1, 0, 2)
        vs = v if not tm else v.transpose(1, 0, 2)
        on = np.flatnonzero(mask)
        if tm:   # across layouts: the reference's layout-equivalence tolerance (src/Constellation.zig:869)
            assert _maxerr(ps[on], full_p[on]) < 1e-10 and _maxerr(vs[on], full_v[on]) < 1e-13
        else:
            assert np.array_equal(ps[on], full_p[on]) and np.array_equal(vs[on], full_v[on])
        assert np.all(ps[np.flatnonzero(mask == 0)] == 7.0) and np.all(ps[37:] == 7.0)
    with pytest.raises(ValueError):
        c.propagate_into(times, satellite_mask=np.ones(5, dtype=np.uint8))
    # caller buffers are validated before the raw pointers reach the C side (satrec.zig:927-941, sgp4.zig:144)
    good = np.zeros((37, len(times), 3))
    for bad in (good.astype(np.float32), np.zeros((37, len(times), 6))[:, :, ::2], np.zeros((36, len(times), 3))):
        with pytest.raises(ValueError):
            c.propagate_into(times, bad, None, epoch_offsets=off, time_major=False, want_velocities=False)
        with pytest.raises(ValueError):
            c.propagate_into(times, good, bad, epoch_offsets=off, time_major=False)
    with pytest.raises(ValueError):
        c.propagate_into(times, epoch_offsets=off[:20])
    # buffers the wrapper allocates itself: masked rows come back as zeros, not uninitialised pinned memory
    pm, vm = c.propagate_into(times, epoch_offsets=off, satellite_mask=mask, time_major=False)
    assert np.all(pm[mask == 0] == 0.0) and np.all(vm[mask == 0] == 0.0) and np.array_equal(pm[mask == 1], full_p[mask == 1])
    # a one-satellite constellation takes the time-parallel kernel only when no mask is given: a masked-out row stays
    one = az.Constellation(tles[:1])
    keep = np.full((1, 200, 3), 7.0)
    one.propagate_into(np.arange(200.0), keep, None, epoch_offsets=np.zeros(1), satellite_mask=np.zeros(1, dtype=np.uint8),
                       time_major=False, want_velocities=False)
    assert np.all(keep == 7.0)


def test_device_side_element_init_matches_host_init(az, oracle, synth):
    """K5 (SURVEY 8f-3): element columns resident in HBM -> classification + Sgp4/Sdp4.initElements + table build on the
    device (src/Constellation.zig:101-200, src/Sgp4.zig:108-417, src/Sdp4.zig:174-657).  Must reproduce the host
    ingest: same classes, row maps and reference epoch, and the same trajectories to the device libm's last ulps."""
    import torch
    for n in (1, 7, 1000, 2051):
        tles = synth.mixed_catalog(n, n_geo=max(1, n // 12), n_molniya=max(1, n // 40), n_gps=max(1, n // 40)) \
            if n >= 7 else synth.near_earth_catalog(n)
        el = synth.elements_from_tles(tles)
        host = az.Constellation.from_elements(*el)
        dev = az.Constellation.from_device_elements(torch.from_numpy(el).cuda())
        assert (dev.numSatellites, dev.numSgp4, dev.numSdp4) == (host.numSatellites, host.numSgp4, host.numSdp4)
        assert np.array_equal(dev.classes, host.classes) and np.array_equal(dev.epochs, host.epochs)
        assert dev.referenceEpochJd == host.referenceEpochJd
        if n >= 1000:
            assert host.numSdp4 > 0 and len(set(host.classes.tolist())) == 4
        jd = np.full(61, 2460437.5)
        fr = np.linspace(0.0, 3.0, 61)
        for layout in (az.Layout.satelliteMajor, az.Layout.timeMajor):
            ph, vh = host.propagate(jd, fr, layout=layout)
            pd, vd = dev.propagate(jd, fr, layout=layout)
            assert np.max(np.abs(pd - ph)) < 1e-8 and np.max(np.abs(vd - vh)) < 1e-11
            # and directly against the oracle (which parses the TLE text the element columns came from)
            po, vo, _, klass = oracle.constellation_propagate(tles, jd, fr, layout=int(layout), threads=0)
            assert list(dev.classes) == list(klass)
            assert _maxerr(pd, po) < POS_TOL and _maxerr(vd, vo) < VEL_TOL


def test_device_side_element_init_large_and_errors(az, oracle, synth):
    import torch
    # more than 1024 blocks of 256 element sets: the block-offset scan carries between its passes
    n = 300_001
    base = synth.elements_from_tles(synth.mixed_catalog(4096, n_geo=300, n_molniya=100, n_gps=100))
    idx = np.random.default_rng(5).integers(0, base.shape[1], n)
    el = np.ascontiguousarray(base[:, idx])
    host = az.Constellation.from_elements(*el)
    dev = az.Constellation.from_device_elements(torch.from_numpy(el).cuda())
    assert (dev.numSgp4, dev.numSdp4) == (host.numSgp4, host.numSdp4)
    assert np.array_equal(dev.classes, host.classes)
    jd = np.full(3, 2460437.5)
    fr = np.array([0.0, 0.4, 0.9])
    ph, vh = host.propagate(jd, fr)
    pd, vd = dev.propagate(jd, fr)
    assert np.max(np.abs(pd - ph)) < 1e-8 and np.max(np.abs(vd - vh)) < 1e-11
    # the 4,096 distinct element sets the draw came from, device-initialised, against the oracle directly
    base_tles = synth.mixed_catalog(4096, n_geo=300, n_molniya=100, n_gps=100)
    devb = az.Constellation.from_device_elements(torch.from_numpy(np.ascontiguousarray(base)).cuda())
    pb, vb = devb.propagate(jd, fr, layout=0)
    po, vo, _, klass = oracle.constellation_propagate(base_tles, jd, fr, threads=0)
    assert list(devb.classes) == list(klass)
    assert _maxerr(pb, po) < POS_TOL and _maxerr(vb, vo) < VEL_TOL
    # the first failing element set in catalog order decides the error (src/Constellation.zig:115-126)
    bad = el[:, :5000].copy()
    bad[2, 4100] = 1.5      # eccentricity >= 1  -> InvalidEccentricity
    bad[1, 3000] = 17.9     # perigee below the surface -> SatelliteDecayed
    with pytest.raises(az.AstrozCudaError) as eh:
        az.Constellation.from_elements(*bad)
    with pytest.raises(az.AstrozCudaError) as ed:
        az.Constellation.from_device_elements(torch.from_numpy(bad).cuda())
    assert ed.value.code == eh.value.code
    assert b"element set 3000 " in az.lib().astroz_cuda_last_error()
    empty = az.Constellation.from_device_elements(torch.empty((8, 0), dtype=torch.float64, device="cuda"))
    assert empty.numSatellites == 0


def test_python_sgp4_attribute_surface(az, oracle):
    """Attributes / methods of the native Satrec and SatrecArray the reference exposes beyond sgp4():
    bindings/python/src/satrec.zig:385-494 (getters), :256-343 (sgp4_array_into), :807 (epochs), :896-988
    (propagate_into)."""
    import math
    from astroz_b200.api import Satrec, SatrecArray, WGS72
    from tests.golden import tles as T
    l1, l2 = T.ISS
    s = Satrec.twoline2rv(l1, l2, WGS72)
    assert s.satnum == 25544 and s.epochyr == 24 and abs(s.epochdays - 127.82853009) < 1e-12
    assert abs(s.ecco - 0.0003580) < 1e-15 and abs(s.inclo - math.radians(51.6393)) < 1e-15
    assert abs(s.nodeo - math.radians(160.4574)) < 1e-15 and abs(s.argpo - math.radians(140.6673)) < 1e-15
    assert abs(s.mo - math.radians(205.7250)) < 1e-15 and abs(s.bstar - 0.27310e-3) < 1e-18
    assert abs(s.no_kozai - 15.50957674 * 2 * math.pi / 1440.0) < 1e-15
    assert abs(s.ndot - 0.00015698 * 2 * math.pi / 1440.0 ** 2) < 1e-20
    n_unkozai = s.no_unkozai
    assert abs(s.a - (0.0743669161331734132 / n_unkozai) ** (2.0 / 3.0)) < 1e-14  # a = (xke / no)^(2/3), src/Sgp4.zig:228
    assert 1.06 < s.a < 1.07 and abs(n_unkozai / s.no_kozai - 1.0) < 2e-3
    assert abs(s.alta - (s.a * (1 + s.ecco) - 1)) < 1e-15 and abs(s.altp - (s.a * (1 - s.ecco) - 1)) < 1e-15
    assert not s.is_deep_space
    jd = np.full(70, s.jdsatepoch)
    fr = s.jdsatepochF + np.arange(70) / 1440.0
    e, r, v = s.sgp4_array(jd, fr)
    r2, v2 = np.zeros((70, 3)), np.zeros((70, 3))
    s.sgp4_array_into(jd, fr, r2, v2)
    assert np.array_equal(r, r2) and np.array_equal(v, v2)
    sats = [Satrec.twoline2rv(a, b, WGS72) for a, b in (T.ISS, T.SAT55909, T.GEO28626, T.SAT55910)]
    arr = SatrecArray(sats)
    assert arr.num_satellites == 4 and len(arr.epochs) == 4
    assert abs(arr.epochs[0] - (s.jdsatepoch + s.jdsatepochF)) < 1e-9
    times = np.arange(0.0, 90.0, 1.5)
    p = np.zeros((len(times), 3, 3))
    vv = np.zeros((len(times), 3, 3))
    arr.propagate_into(times, p, vv)      # near-earth members only, minutes since each satellite's own epoch
    for k, (a, b) in enumerate((T.ISS, T.SAT55909, T.SAT55910)):
        oo = oracle.Sgp4(a, b, oracle.WGS72)
        for j in (0, 17, 59):
            ro, vo = oo.propagate(times[j])
            assert np.max(np.abs(p[j, k] - ro)) < 1e-6 and np.max(np.abs(vv[j, k] - vo)) < 1e-9
    with pytest.raises(ValueError):
        arr.propagate_into(times, np.zeros((3, 3, 3)))


def test_high_level_frontend_propagate_and_screen(az, oracle):
    """astroz.propagate / astroz.screen / astroz.Constellation mirrors (bindings/python/astroz/__init__.py:305-660)
    and the native sdp4_batch_propagate_into (bindings/python/src/satrec.zig:505-644)."""
    from datetime import datetime, timezone
    from astroz_b200 import frontend
    from astroz_b200.api import Satrec, sdp4_batch_propagate_into, WGS72
    from tests.golden import tles as T
    order_in = [T.GEO28626, T.ISS, T.HEO09880, T.SAT55909, T.SAT55910, T.GPS20413]
    text = "\n".join("NAME\n" + a + "\n" + b for a, b in order_in)
    c = frontend.Constellation(text)
    near = [T.ISS, T.SAT55909, T.SAT55910]
    deep = [T.GEO28626, T.HEO09880, T.GPS20413]
    assert c.num_satellites == 6 and (c._n_sgp4, c._n_sdp4) == (3, 3)
    start = datetime(2024, 7, 6, 3, 0, 0, tzinfo=timezone.utc)
    start_jd = 2440587.5 + start.timestamp() / 86400.0
    times = np.arange(0.0, 200.0, 7.0)
    pos, vel = frontend.propagate(c, times, start_time=start, output="teme", velocities=True)
    assert pos.shape == (len(times), 6, 3) and vel.shape == pos.shape
    for k, (a, b) in enumerate(near):      # rows [0, n_sgp4): tsince = times + (start - epoch) * 1440
        o = oracle.Sgp4(a, b, oracle.WGS72)
        off = (start_jd - c.epochs[k]) * 1440.0
        for j in (0, 11, len(times) - 1):
            r, v = o.propagate(times[j] + off)
            assert np.max(np.abs(pos[j, k] - r)) < 1e-6 and np.max(np.abs(vel[j, k] - v)) < 1e-9
    for k, (a, b) in enumerate(deep):      # rows after them: the deep-space members, filled (unlike the reference)
        o = oracle.Sdp4(a, b, oracle.WGS72)
        for j in (0, 11, len(times) - 1):
            _, r, v = o.propagate(((start_jd + times[j] / 1440.0) - c.epochs[3 + k]) * 1440.0)
            assert np.max(np.abs(pos[j, 3 + k] - r)) < 2e-5 and np.max(np.abs(vel[j, 3 + k] - v)) < 2e-9
    # default output is ECEF = Rz(GMST) * TEME (src/Constellation.zig:930-964)
    ecef = frontend.propagate(c, times, start_time=start)
    for j in (0, 5, len(times) - 1):
        g = oracle.julian_to_gmst(start_jd + times[j] / 1440.0)
        cg, sg = np.cos(g), np.sin(g)
        x, y = pos[j, :, 0], pos[j, :, 1]
        assert np.max(np.abs(ecef[j, :, 0] - (cg * x + sg * y))) < 1e-6
        assert np.max(np.abs(ecef[j, :, 1] - (-sg * x + cg * y))) < 1e-6
        assert np.max(np.abs(ecef[j, :, 2] - pos[j, :, 2])) < 1e-9
    # single-target and all-vs-all screens of a pure near-earth catalogue
    cn = frontend.Constellation("\n".join(a + "\n" + b for a, b in near))
    dist, tidx = frontend.screen(cn, times, threshold=5000.0, target=0, start_time=start)
    pn = frontend.propagate(cn, times, start_time=start, output="teme")
    d = np.linalg.norm(pn - pn[:, :1], axis=2)
    assert np.allclose(dist[1:], d.min(axis=0)[1:], atol=1e-6) and np.array_equal(tidx[1:], d.argmin(axis=0)[1:])
    pairs, tt = frontend.screen(cn, times, threshold=8000.0, start_time=start)
    want = {(t, i, j) for t in range(len(times)) for i in range(3) for j in range(i + 1, 3)
            if np.linalg.norm(pn[t, i] - pn[t, j]) < 8000.0}
    assert {(int(t), int(min(p)), int(max(p))) for p, t in zip(pairs, tt)} == want
    # the mixed catalogue goes through propagate + the cell-list screen
    pairs_m, tt_m = frontend.screen(c, times, threshold=9000.0, start_time=start)
    want_m = {(t, i, j) for t in range(len(times)) for i in range(6) for j in range(i + 1, 6)
              if np.linalg.norm(pos[t, i] - pos[t, j]) < 9000.0}
    assert {(int(t), int(min(p)), int(max(p))) for p, t in zip(pairs_m, tt_m)} == want_m
    # sdp4_batch_propagate_into: time-major, strided, offset rows; other rows untouched
    sats = [Satrec.twoline2rv(a, b, WGS72) for a, b in deep]
    jd = np.full(len(times), np.floor(start_jd) + 0.5)
    fr = (start_jd - jd[0]) + times / 1440.0
    p2 = np.full((len(times), 7, 3), -1.0)
    v2 = np.full((len(times), 7, 3), -1.0)
    sdp4_batch_propagate_into(sats, jd, fr, p2, v2, output_stride=7, sat_offset=2)
    assert np.all(p2[:, :2] == -1.0) and np.all(p2[:, 5:] == -1.0) and np.all(v2[:, :2] == -1.0)
    for k, (a, b) in enumerate(deep):
        o = oracle.Sdp4(a, b, oracle.WGS72)
        for j in (0, 9, len(times) - 1):
            _, r, v = o.propagate(((jd[j] + fr[j]) - c.epochs[3 + k]) * 1440.0)
            assert np.max(np.abs(p2[j, 2 + k] - r)) < 2e-5 and np.max(np.abs(v2[j, 2 + k] - v)) < 2e-9
    with pytest.raises(ValueError):
        sdp4_batch_propagate_into([Satrec.twoline2rv(*T.ISS, WGS72)], jd, fr, p2, v2)


def test_many_satrec_objects_are_cheap_until_propagated(az, oracle, synth):
    """python-sgp4 style: one Satrec per element set, then a SatrecArray over them (benchmarks/python_astroz_bench.py
    does this for the whole catalogue).  Satrec handles parse and classify on the host and open their device resources
    lazily, so building thousands of them costs milliseconds, not streams and allocations."""
    import time
    from astroz_b200.api import Satrec, SatrecArray, WGS72
    tles = synth.near_earth_catalog(3000)
    t0 = time.perf_counter()
    sats = [Satrec.twoline2rv(a, b, WGS72) for a, b in tles]
    dt = time.perf_counter() - t0
    assert dt < 3.0, f"3000 Satrec objects took {dt:.2f} s"
    assert all(s.error == 0 and not s.is_deep_space for s in sats) and sats[17].satnum == 10017
    jd, fr = synth.time_grid(90)
    e, r, v = SatrecArray(sats).sgp4(jd, fr)
    assert r.shape == (3000, 90, 3) and not e.any()
    for k in (0, 1234, 2999):     # a lazily opened handle gives the same numbers as the batch
        e1, r1, v1 = sats[k].sgp4(jd[5], fr[5])
        assert e1 == 0 and _maxerr(np.array(r1), r[k, 5]) < 1e-9 and _maxerr(np.array(v1), v[k, 5]) < 1e-12


# ---------------------------------------------------------------------------------------------- multi-device handle
def _device_block(ptr, shape):
    """Copy a raw device block (a pointer the library owns) to the host."""
    from cuda import cudart

    out = np.empty(shape)
    (err,) = cudart.cudaMemcpy(out.ctypes.data, ptr, out.nbytes, cudart.cudaMemcpyKind.cudaMemcpyDeviceToHost)
    assert int(err) == 0, err
    return out


def test_multi_device_handle_shards_are_bit_identical(az, oracle, synth, monkeypatch):
    """device = -1: ONE handle whose propagate call fans out over the devices (src/Constellation.zig:327-385 fans out
    over threads).  On a one-GPU box ASTROZ_DEVICE_LIST repeats the ordinal, so the sharding, the per-shard row
    offsets and strided copies, and the shared reference epoch are exercised all the same: every result must equal
    the single-device handle's bit for bit."""
    tles = synth.mixed_catalog(1003, n_geo=90, n_molniya=40, n_gps=30)
    jd, fr = synth.time_grid(1440)
    jd, fr = jd[::7].copy(), fr[::7].copy()
    single = az.Constellation(tles, device=0)
    monkeypatch.setenv("ASTROZ_DEVICE_LIST", "0,0,0")
    multi = az.Constellation(tles, device=-1)
    monkeypatch.delenv("ASTROZ_DEVICE_LIST")
    ids, rows = multi.devices
    assert ids == [0, 0, 0] and rows[0] == 0 and rows[-1] == 1003 and all(r % 8 == 0 for r in rows[:-1])
    assert all(250 < rows[k + 1] - rows[k] < 420 for k in range(3))   # equal-cost ranges (deep-space rows weigh 2.4)
    assert (multi.numSatellites, multi.numSgp4, multi.numSdp4) == (single.numSatellites, single.numSgp4, single.numSdp4)
    assert np.array_equal(multi.classes, single.classes) and np.array_equal(multi.epochs, single.epochs)
    assert multi.referenceEpochJd == single.referenceEpochJd
    for layout in (az.Layout.satelliteMajor, az.Layout.timeMajor):
        for mode in (az.OutputMode.teme, az.OutputMode.ecef, az.OutputMode.geodetic):
            for velocities in (True, False):
                ps, vs = single.propagate(jd, fr, outputMode=mode, layout=layout, velocities=velocities)
                pm, vm = multi.propagate(jd, fr, outputMode=mode, layout=layout, velocities=velocities)
                assert np.array_equal(ps, pm), (layout, mode, velocities)
                assert (vs is None and vm is None) or np.array_equal(vs, vm)
    # caller-owned pageable buffers take the same route
    pp, vp = np.zeros((1003, len(jd), 3)), np.zeros((1003, len(jd), 3))
    multi.propagate(jd, fr, pp, vp, layout=az.Layout.satelliteMajor)
    ps, vs = single.propagate(jd, fr, layout=az.Layout.satelliteMajor)
    assert np.array_equal(pp, ps) and np.array_equal(vp, vs)
    po, vo, _, _ = oracle.constellation_propagate(tles, jd, fr, threads=0)
    assert _maxerr(pp, po) < POS_TOL and _maxerr(vp, vo) < VEL_TOL
    # the stateless near-earth path, with a mask and a wider block
    ns = single.numSgp4
    times = np.arange(0.0, 300.0, 3.0)
    off = (2460437.5 - single.epochs[np.asarray(single.classes) == 0]) * 1440.0
    mask = np.ones(ns, dtype=np.uint8)
    mask[::5] = 0
    for tm in (False, True):
        shape = (ns + 9, len(times), 3) if not tm else (len(times), ns + 9, 3)
        a_p, a_v, b_p, b_v = (np.full(shape, 3.0) for _ in range(4))
        single.propagate_into(times, a_p, a_v, epoch_offsets=off, satellite_mask=mask, time_major=tm, output_stride=ns + 9)
        multi.propagate_into(times, b_p, b_v, epoch_offsets=off, satellite_mask=mask, time_major=tm, output_stride=ns + 9)
        assert np.array_equal(a_p, b_p) and np.array_equal(a_v, b_v)
    # a shared reference epoch can be moved, and every shard follows
    multi.referenceEpochJd = single.referenceEpochJd + 0.25
    single.referenceEpochJd = single.referenceEpochJd + 0.25
    assert np.array_equal(multi.propagate(jd, fr, layout=0)[0], single.propagate(jd, fr, layout=0)[0])
    # device-pointer entry points need one device
    import torch

    t = torch.empty((1003, len(jd), 3), dtype=torch.float64, device="cuda")
    with pytest.raises(az.AstrozCudaError) as ei:
        multi.propagate_device(jd, fr, t)
    assert ei.value.code == -20
    # the all-gather behind one handle: every device of the handle ends with the whole block
    single.referenceEpochJd = single.referenceEpochJd - 0.25
    multi.referenceEpochJd = multi.referenceEpochJd - 0.25
    ids, ppos, pvel = multi.propagate_replicated(jd, fr)
    ps, vs = single.propagate(jd, fr, layout=0)
    for k in range(len(ids)):
        assert np.array_equal(_device_block(ppos[k], ps.shape), ps)
        assert np.array_equal(_device_block(pvel[k], vs.shape), vs)
    ids1, p1, v1 = single.propagate_replicated(jd, fr, velocities=False)
    assert ids1 == [0] and v1 == [0] and np.array_equal(_device_block(p1[0], ps.shape), ps)


def test_multi_device_handle_device_count_knob(az, synth, monkeypatch):
    """ASTROZ_DEVICES caps the GPUs of a device = -1 handle the way ASTROZ_THREADS caps the reference's threads
    (src/Constellation.zig:61-74); with one device left the handle is an ordinary single-device one."""
    import torch

    tles = synth.near_earth_catalog(512)
    monkeypatch.setenv("ASTROZ_DEVICES", "1")
    c = az.Constellation(tles, device=-1)
    assert c.devices == ([0], [0, 512])
    monkeypatch.delenv("ASTROZ_DEVICES")
    c2 = az.Constellation(tles, device=-1)
    ids, rows = c2.devices
    assert len(ids) == min(torch.cuda.device_count(), 8) and rows[-1] == 512
    jd, fr = synth.time_grid(64)
    assert np.array_equal(c.propagate(jd, fr)[0], c2.propagate(jd, fr)[0])
    with pytest.raises(az.AstrozCudaError):
        az.Constellation(tles, device=-2)


def test_caller_owned_pageable_and_registered_buffers(az, synth):
    """The reference writes into whatever slices the caller passes (src/Constellation.zig:245-258; numpy buffers from
    Python, bindings/python/src/satrec.zig:917-942).  Pageable destinations are served through the handle's pinned
    ring + host copy pool, page-locked ones by direct DMA: all three routes must give the same bytes, for blocks that
    span several ring pieces, both layouts, and the strided (wider block) form."""
    tles = synth.near_earth_catalog(2100)
    jd, fr = synth.time_grid(1440)
    c = az.Constellation(tles)
    n, nt = 2100, 1440                                  # 72.6 MB per array: three 32 MB ring pieces
    for layout in (az.Layout.satelliteMajor, az.Layout.timeMajor):
        ref_p, ref_v = c.propagate(jd, fr, layout=layout)                     # pinned (the wrapper's own allocation)
        shape = ref_p.shape
        pg_p, pg_v = np.full(shape, -1.0), np.full(shape, -1.0)              # pageable
        c.propagate(jd, fr, pg_p, pg_v, layout=layout)
        assert np.array_equal(pg_p, ref_p) and np.array_equal(pg_v, ref_v)
        rg_p = np.full(shape, -2.0)                                           # page-locked in place by the caller
        az.host_register(rg_p)
        try:
            c.propagate(jd, fr, rg_p, None, layout=layout, velocities=False)
        finally:
            az.host_unregister(rg_p)
        assert np.array_equal(rg_p, ref_p)
    # a result block placed by the library for the handle (NUMA-bound, page-locked; freed with the array)
    for layout in (az.Layout.satelliteMajor, az.Layout.timeMajor):
        blk = c.host_block(nt, layout)
        assert blk.shape == ((n, nt, 3) if layout == 0 else (nt, n, 3)) and blk.dtype == np.float64
        c.propagate(jd, fr, blk, None, layout=layout, velocities=False)
        assert np.array_equal(blk, c.propagate(jd, fr, layout=layout, velocities=False)[0])
        del blk
    # stateless path into a wider pageable block: rows beyond the constellation and the pitch gaps stay untouched
    times = np.arange(0.0, 1440.0, 1.0)
    off = (2460437.5 - c.epochs) * 1440.0
    want_p, want_v = c.propagate_into(times, epoch_offsets=off, time_major=True)
    wide_p, wide_v = np.full((nt, n + 7, 3), 5.0), np.full((nt, n + 7, 3), 5.0)
    c.propagate_into(times, wide_p, wide_v, epoch_offsets=off, time_major=True, output_stride=n + 7)
    assert np.array_equal(wide_p[:, :n], want_p) and np.array_equal(wide_v[:, :n], want_v)
    assert np.all(wide_p[:, n:] == 5.0) and np.all(wide_v[:, n:] == 5.0)
