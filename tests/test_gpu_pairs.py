"""Arbitrary (satellite, time) pairs on the device (K6, astroz_b200/csrc/az_pairs.cu): against the grid path, the
scalar oracle, and itself under reordering, chunking and every kind of host buffer."""
import ctypes as C

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


@pytest.fixture(scope="module")
def mixed(az, synth):
    tles = synth.mixed_catalog(1200, n_geo=160, n_molniya=80, n_gps=80)
    return tles, az.Constellation(tles)


def _maxerr(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b)))) if np.size(a) else 0.0


def _host_call(c, sat, jd, fr, mode, pos, vel=None, status=None):
    """The C entry point on caller-owned buffers (pageable, registered or pinned)."""
    from astroz_b200._lib import dptr, lib

    sat = np.ascontiguousarray(sat, dtype=np.uint32)
    return lib().astroz_cuda_constellation_propagate_pairs(
        c._h, C.c_void_p(sat.ctypes.data), dptr(jd), dptr(fr), len(sat), int(mode), dptr(pos),
        dptr(vel) if vel is not None else None, C.c_void_p(status.ctypes.data) if status is not None else None)


def _device_call(c, sat, jd, fr, mode=0, velocities=True):
    import torch

    dev = torch.device("cuda", 0)
    n = len(sat)
    ds = torch.from_numpy(np.ascontiguousarray(sat, dtype=np.uint32).view(np.int32)).to(dev)
    dj = torch.from_numpy(np.ascontiguousarray(jd)).to(dev)
    df = torch.from_numpy(np.ascontiguousarray(fr)).to(dev)
    pos = torch.full((n, 3), 7.0, dtype=torch.float64, device=dev)
    vel = torch.full((n, 3), 7.0, dtype=torch.float64, device=dev) if velocities else None
    st = torch.full((n,), 255, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    c.propagate_pairs_device(ds, dj, df, pos, vel, st, outputMode=mode)
    c.synchronize()
    return pos.cpu().numpy(), (vel.cpu().numpy() if vel is not None else None), st.cpu().numpy()


def _off_grid(synth, n_sats, nq, seed, days=7.0):
    rng = np.random.default_rng(seed)
    sat = rng.integers(0, n_sats, nq).astype(np.uint32)
    t = synth.BENCH_JD0 + rng.uniform(-days, days, nq)
    jd = np.floor(t - 0.5) + 0.5
    return sat, jd, t - jd


def _scalar_check(oracle, tles, klass, ref, sat, jd, fr, pos, vel, st, sample):
    """TEME results of `sample` queries against the scalar propagators at the grid's tsince (ref: the handle's reference
    epoch)."""
    models = {}
    for i in sample:
        s = int(sat[i])
        if s not in models:
            models[s] = (oracle.Sdp4 if klass[s] else oracle.Sgp4)(*tles[s])
        m = models[s]
        jf = jd[i] + fr[i]
        if klass[s]:
            rc, r, v = m.propagate((jf - m.epochJd) * 1440.0)
            if rc != 0:
                assert st[i] != 0 and not pos[i].any()
                continue
        else:
            r, v = m.propagate((jf - ref) * 1440.0 + (ref - m.epochJd) * 1440.0)
        assert st[i] in (0, 1)
        assert _maxerr(pos[i], r) < POS_TOL, (i, s, klass[s])
        assert _maxerr(vel[i], v) < VEL_TOL, (i, s, klass[s])


# ------------------------------------------------------------------------------------------------ vs grid / oracle
def test_pairs_match_grid_and_oracle(az, oracle, synth, mixed):
    import torch

    tles, c = mixed
    jd, fr = synth.time_grid(1440)
    jd, fr = jd[::7].copy(), fr[::7].copy()
    n, nt = len(tles), len(jd)
    rng = np.random.default_rng(20)
    s = rng.integers(0, n, 200_000).astype(np.uint32)   # drawn from grid cells: shuffled, with duplicates
    t = rng.integers(0, nt, 200_000)
    po, vo, err, klass = oracle.constellation_propagate(tles, jd, fr)
    dev = torch.device("cuda", 0)
    gp = torch.empty((n, nt, 3), dtype=torch.float64, device=dev)
    gv = torch.empty_like(gp)
    gs = torch.full((n, nt), 255, dtype=torch.uint8, device=dev)
    for mode in (az.OutputMode.teme, az.OutputMode.ecef, az.OutputMode.geodetic):
        c.propagate_device(jd, fr, gp, gv, gs, outputMode=mode)
        c.synchronize()
        P, V, S = gp.cpu().numpy()[s, t], gv.cpu().numpy()[s, t], gs.cpu().numpy()[s, t]
        pos, vel, st = c.propagate_pairs(s, jd[t], fr[t], outputMode=mode)
        assert np.array_equal(st, S), mode
        if mode == az.OutputMode.geodetic:
            assert _maxerr(pos[:, :2], P[:, :2]) < 2e-14
            assert _maxerr(pos[:, 2], P[:, 2]) < 1e-10
        else:
            assert _maxerr(pos, P) < 1e-10, mode
        assert _maxerr(vel, V) < 1e-13, mode
        if mode == az.OutputMode.teme:
            assert _maxerr(pos, po[s, t]) < POS_TOL and _maxerr(vel, vo[s, t]) < VEL_TOL
            deep = klass[s] > 0
            assert np.array_equal(st[deep], err[s, t][deep])


def test_pairs_off_grid_times_and_lattice_growth(az, oracle, synth):
    """Each query at its own epoch, +-7 days around the element epochs (before them too).  A fresh handle first sees a
    short reach, then a week's: the second call grows the resonance lattice."""
    tles = synth.mixed_catalog(400, n_geo=60, n_molniya=40, n_gps=30) + [G.GEO28626, G.HEO09880, G.GPS20413, G.ISS]
    c = az.Constellation(tles)
    klass = c.classes
    for days, seed in ((0.3, 1), (7.0, 2)):
        sat, jd, fr = _off_grid(synth, len(tles), 20_000, seed, days)
        pos, vel, st = c.propagate_pairs(sat, jd, fr)
        sample = np.random.default_rng(seed).choice(len(sat), 2500, replace=False)
        _scalar_check(oracle, tles, klass, c.referenceEpochJd, sat, jd, fr, pos, vel, st, sample)
        dp, dv, dst = _device_call(c, sat, jd, fr)
        assert np.array_equal(dp, pos) and np.array_equal(dv, vel) and np.array_equal(dst, st)


def test_pairs_failures_are_zero_filled_per_query(az, oracle, synth):
    bad = synth.tle_lines(42000, 24, 120.0, 63.4, 0.0, 0.755, 0.0, 10.0, 2.006, 1e-3)
    tles = [G.GPS20413, bad, G.GEO28626, G.HEO09880]
    jd = np.full(40, 2460430.5)
    fr = np.linspace(0.0, 2000.0, 40)
    po, vo, err, _ = oracle.constellation_propagate(tles, jd, fr)
    assert err[1].any() and set(np.unique(err[1])) >= {1, 2}
    s, t = np.meshgrid(np.arange(4), np.arange(40), indexing="ij")
    perm = np.random.default_rng(4).permutation(160)
    s, t = s.ravel()[perm].astype(np.uint32), t.ravel()[perm]
    c = az.Constellation(tles)
    pos, vel, st = c.propagate_pairs(s, jd[t], fr[t])
    assert np.array_equal(st, err[s, t])
    assert np.all(pos[st != 0] == 0.0) and np.all(vel[st != 0] == 0.0)
    ok = st == 0
    assert _maxerr(pos[ok], po[s, t][ok]) < 1e-5
    assert np.all(pos[(s == 0) | (s == 2)] != 0.0)   # the GPS and GEO objects never fail over these years
    gp, gv = c.propagate(jd, fr, layout=az.Layout.satelliteMajor)
    assert _maxerr(pos[s != 1], gp[s, t][s != 1]) < 1e-10


# ------------------------------------------------------------------------------------------------ order, buffers
def test_pairs_order_independence_and_buffers(az, synth, mixed):
    from astroz_b200 import _lib

    tles, c = mixed
    sat, jd, fr = _off_grid(synth, len(tles), 30_000, 9)
    base = c.propagate_pairs(sat, jd, fr, outputMode=az.OutputMode.ecef)
    n = len(sat)
    orders = {
        "shuffled": np.random.default_rng(5).permutation(n),
        "grouped": np.argsort(sat, kind="stable"),
        "reversed": np.arange(n)[::-1].copy(),
        "duplicated": np.concatenate([np.arange(n), np.arange(0, n, 2), np.arange(0, n, 3)]),
    }
    for name, o in orders.items():
        p, v, st = c.propagate_pairs(sat[o], jd[o], fr[o], outputMode=az.OutputMode.ecef)
        assert np.array_equal(p, base[0][o]) and np.array_equal(v, base[1][o]) and np.array_equal(st, base[2][o]), name
    dp, dv, dst = _device_call(c, sat, jd, fr, mode=az.OutputMode.ecef)
    assert np.array_equal(dp, base[0]) and np.array_equal(dv, base[1]) and np.array_equal(dst, base[2])
    # pageable, registered and pinned destinations (and pinned queries) are byte-identical
    pg = [np.full((n, 3), 9.0), np.full((n, 3), 9.0), np.full(n, 200, dtype=np.uint8)]
    assert _host_call(c, sat, jd, fr, 1, *pg) == 0
    reg = [np.full((n, 3), 9.0), np.full((n, 3), 9.0), np.full(n, 200, dtype=np.uint8)]
    for a in reg:
        _lib.host_register(a)
    try:
        assert _host_call(c, sat, jd, fr, 1, *reg) == 0
    finally:
        for a in reg:
            _lib.host_unregister(a)
    pin = [_lib.pinned_empty((n, 3)), _lib.pinned_empty((n, 3)), _lib.pinned_empty((n,), np.uint8)]
    psat, pjd, pfr = _lib.pinned_empty((n,), np.uint32), _lib.pinned_empty((n,)), _lib.pinned_empty((n,))
    psat[:], pjd[:], pfr[:] = sat, jd, fr
    assert _host_call(c, psat, pjd, pfr, 1, *pin) == 0
    for bufs in (pg, reg, pin):
        for a, b in zip(bufs, base):
            assert a.tobytes() == b.tobytes()


def test_pairs_host_chunks_match_device_call(az, synth, monkeypatch):
    """Four host chunks (two device slots, each reused) against one device call, bit for bit, for pageable and pinned
    buffers: the pageable path takes queries and results through the pinned ring."""
    from astroz_b200 import _lib

    tles = synth.mixed_catalog(500, n_geo=50, n_molniya=30, n_gps=20)
    monkeypatch.setenv("ASTROZ_PAIRS_CHUNK", "4096")
    c = az.Constellation(tles)
    monkeypatch.delenv("ASTROZ_PAIRS_CHUNK")
    sat, jd, fr = _off_grid(synth, len(tles), 3 * 4096 + 1234, 13)
    n = len(sat)
    dp, dv, dst = _device_call(c, sat, jd, fr, mode=az.OutputMode.geodetic)
    pg = [np.zeros((n, 3)), np.zeros((n, 3)), np.zeros(n, dtype=np.uint8)]
    assert _host_call(c, sat, jd, fr, 2, *pg) == 0
    assert np.array_equal(pg[0], dp) and np.array_equal(pg[1], dv) and np.array_equal(pg[2], dst)
    p, v, st = c.propagate_pairs(sat, jd, fr, outputMode=az.OutputMode.geodetic)
    assert np.array_equal(p, dp) and np.array_equal(v, dv) and np.array_equal(st, dst)
    # positions only, no status: the same bytes where they are written
    p2 = np.zeros((n, 3))
    assert _host_call(c, sat, jd, fr, 2, p2) == 0
    assert np.array_equal(p2, dp)


# ------------------------------------------------------------------------------------------------ edges
def test_pairs_edge_cases(az, synth, mixed, monkeypatch):
    import torch

    from astroz_b200 import AstrozCudaError

    tles, c = mixed
    p, v, st = c.propagate_pairs(np.zeros(0, dtype=np.uint32), np.zeros(0), np.zeros(0))
    assert p.shape == (0, 3) and v.shape == (0, 3) and st.shape == (0,)
    sat, jd, fr = _off_grid(synth, len(tles), 64, 21)
    full = c.propagate_pairs(sat, jd, fr)
    one = c.propagate_pairs(sat[5:6], jd[5:6], fr[5:6])
    assert all(np.array_equal(a, b[5:6]) for a, b in zip(one, full))
    p, v, st = c.propagate_pairs(sat, jd, fr, velocities=False)
    assert v is None and np.array_equal(p, full[0]) and np.array_equal(st, full[2])
    pp = np.zeros((64, 3))
    assert _host_call(c, sat, jd, fr, 0, pp) == 0 and np.array_equal(pp, full[0])
    with pytest.raises(ValueError):
        c.propagate_pairs(sat, jd[:-1], fr)
    # out-of-range rows: the host call refuses and writes nothing ...
    bad = sat.copy()
    bad[[3, 40]] = [len(tles), 0xFFFFFFFF]
    bufs = [np.full((64, 3), 9.0), np.full((64, 3), 9.0), np.full(64, 200, dtype=np.uint8)]
    assert _host_call(c, bad, jd, fr, 0, *bufs) == -20
    assert np.all(bufs[0] == 9.0) and np.all(bufs[1] == 9.0) and np.all(bufs[2] == 200)
    with pytest.raises(AstrozCudaError) as ei:
        c.propagate_pairs(bad.astype(np.int64), jd, fr)
    assert ei.value.code == -20
    # ... the device call gives those queries zeros and ASTROZ_CELL_BAD_SATELLITE, the others their results
    dp, dv, dst = _device_call(c, bad, jd, fr)
    badq = np.isin(np.arange(64), [3, 40])
    assert np.all(dst[badq] == 3) and np.all(dp[badq] == 0.0) and np.all(dv[badq] == 0.0)
    assert np.array_equal(dp[~badq], full[0][~badq]) and np.array_equal(dst[~badq], full[2][~badq])
    # device call without velocity / status
    dev = torch.device("cuda", 0)
    pos = torch.zeros((64, 3), dtype=torch.float64, device=dev)
    c.propagate_pairs_device(torch.from_numpy(sat.view(np.int32)).to(dev), torch.from_numpy(jd).to(dev),
                             torch.from_numpy(fr).to(dev), pos)
    c.synchronize()
    assert np.array_equal(pos.cpu().numpy(), full[0])
    # a multi-device handle refuses both entry points
    many = synth.mixed_catalog(1003, n_geo=90, n_molniya=40, n_gps=30)
    monkeypatch.setenv("ASTROZ_DEVICE_LIST", "0,0,0")
    multi = az.Constellation(many, device=-1)
    monkeypatch.delenv("ASTROZ_DEVICE_LIST")
    assert len(multi.devices[0]) == 3
    with pytest.raises(AstrozCudaError) as ei:
        multi.propagate_pairs(sat, jd, fr)
    assert ei.value.code == -20
    with pytest.raises(AstrozCudaError) as ei:
        multi.propagate_pairs_device(torch.from_numpy(sat.view(np.int32)).to(dev), torch.from_numpy(jd).to(dev),
                                     torch.from_numpy(fr).to(dev), pos)
    assert ei.value.code == -20
