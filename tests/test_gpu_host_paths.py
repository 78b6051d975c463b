"""Host orchestration of the C ABI (astroz_b200/csrc/az_capi.cu, az_hostcopy.cu): what last_kernel_ms reports after
each kind of call, the stateless deep-space entry points, and several entry points in sequence on one handle, which
share its pinned time-axis slots, its epoch-offset staging and its pinned ring."""
import ctypes as C

import numpy as np
import pytest

from tests.golden import tles as G

pytestmark = pytest.mark.gpu

NOT_INITIALIZED = -102


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
def mixed_tles(synth):
    return synth.mixed_catalog(1200, n_geo=160, n_molniya=80, n_gps=80)


def _empty(shape, fill=0.0):
    import torch

    return torch.full(shape, fill, dtype=torch.float64, device=torch.device("cuda", 0))


def _sdp4_into_device(c, jd, fr, pos, vel, mode, layout, rows, offset):
    from astroz_b200._lib import check, dptr, lib

    check(lib().astroz_cuda_sdp4_propagate_into_device(
        c._h, dptr(jd), dptr(fr), len(jd), C.c_void_p(pos.data_ptr()), C.c_void_p(vel.data_ptr()), int(mode),
        int(layout), int(rows), int(offset), None))
    c.synchronize()


def _sgp4_into_device(c, times, off, pos, vel):
    from astroz_b200._lib import check, dptr, lib

    check(lib().astroz_cuda_sgp4_propagate_into_device(
        c._h, dptr(times), len(times), dptr(off), C.c_void_p(pos.data_ptr()), C.c_void_p(vel.data_ptr()), 0, 0.0, 1,
        None, 0, None))
    c.synchronize()


def _batch(sat, times):
    from astroz_b200 import _lib

    out = np.zeros((len(times), 6))
    rc = _lib.lib().astroz_cuda_sgp4_propagate_batch(sat._h, _lib.dptr(times), _lib.dptr(out), len(times))
    assert rc == 0, rc
    return out


def _not_initialized(c):
    from astroz_b200._lib import AstrozCudaError

    with pytest.raises(AstrozCudaError) as e:
        c.last_kernel_ms()
    return e.value.code == NOT_INITIALIZED


def test_last_kernel_ms_reports_what_each_call_timed(az, synth, mixed_tles):
    """[0] = the near-earth kernel, [2] = the deep-space kernel, 0.0 where the call ran none; [1] = the call's span
    where one was timed, else [0] + [2].  After a host-buffer propagate all three hold the span."""
    near = az.Constellation(synth.near_earth_catalog(3000))
    mixed = az.Constellation(mixed_tles)
    jd, fr = synth.time_grid(512)
    times = np.arange(0.0, 512.0)
    n, m = near.numSatellites, mixed.numSatellites
    for c in (near, mixed):
        c.set_timing(True)

    near.propagate_device(jd, fr, _empty((n, 512, 3)), _empty((n, 512, 3)))
    k1, span, k2 = near.last_kernel_ms()
    assert k1 > 0 and k2 == 0.0 and span >= k1

    mixed.propagate_device(jd, fr, _empty((m, 512, 3)), _empty((m, 512, 3)))
    k1, span, k2 = mixed.last_kernel_ms()
    assert k1 > 0 and k2 > 0 and span > 0      # the two grids overlap: the span is timed on its own

    # a call that returns before any work leaves the record as it was
    mixed.propagate_device(jd[:0], fr[:0], _empty((m, 1, 3)))
    assert mixed.last_kernel_ms() == (k1, span, k2)

    nd = mixed.numSdp4
    _sdp4_into_device(mixed, jd, fr, _empty((nd, 512, 3)), _empty((nd, 512, 3)), 0, 0, nd, 0)
    k1, span, k2 = mixed.last_kernel_ms()
    assert k1 == 0.0 and k2 > 0 and span == k2

    off = np.zeros(near.numSgp4)
    _sgp4_into_device(near, times, off, _empty((512, n, 3)), _empty((512, n, 3)))
    k1, span, k2 = near.last_kernel_ms()
    assert k1 > 0 and k2 == 0.0 and span == k1

    near.screen_conjunction(times, 7, 50.0, epoch_offsets=off)
    k1, span, k2 = near.last_kernel_ms()
    assert k1 > 0 and k2 == 0.0 and span == k1

    near.propagate_device_f32(jd, fr, _empty((n, 512, 3)), _empty((n, 512, 3)))
    near.synchronize()
    k1, span, k2 = near.last_kernel_ms()
    assert k1 > 0 and k2 == 0.0 and span == k1

    for c in (near, mixed):   # host buffers: the grid runs in chunks with the copies, all three slots are the span
        c.propagate(jd, fr, layout=az.Layout.timeMajor)
        k1, span, k2 = c.last_kernel_ms()
        assert span > 0 and k1 == span and k2 == span

    sat = np.arange(m, dtype=np.uint32)
    mixed.propagate_pairs(sat, np.full(m, jd[0]), np.full(m, 0.25))
    assert _not_initialized(mixed)             # the pairs kernels are not timed

    near.set_timing(False)
    assert _not_initialized(near)
    near.propagate_device(jd, fr, _empty((n, 512, 3)))
    near.synchronize()
    assert _not_initialized(near)


def _deep_rows(c, grid, layout):
    rows = np.flatnonzero(c.classes != 0)
    return grid[rows] if layout == 0 else grid[:, rows]


@pytest.mark.parametrize("layout", [0, 1])
def test_sdp4_propagate_into_matches_the_grid(az, synth, mixed_tles, layout):
    """astroz_cuda_sdp4_propagate_into (host) and _into_device write deep-space satellite i to row sat_offset + i of
    a block with out_num_sats rows: bit for bit the deep-space rows of a grid call on the same handle, into a dense
    block or a wider one, pageable or pinned; rows outside the handle's range stay untouched."""
    from astroz_b200 import _lib

    c = az.Constellation(mixed_tles)
    nd = c.numSdp4
    jd, fr = synth.time_grid(300)
    nt = len(jd)
    tm = layout == 1
    for mode in (az.OutputMode.teme, az.OutputMode.ecef):
        gp, gv = c.propagate(jd, fr, outputMode=mode, layout=layout)
        want_p, want_v = _deep_rows(c, gp, layout), _deep_rows(c, gv, layout)
        for rows, offset in ((nd, 0), (nd + 9, 5)):
            shape = (rows, nt, 3) if layout == 0 else (nt, rows, 3)
            inside = (slice(offset, offset + nd),) if layout == 0 else (slice(None), slice(offset, offset + nd))
            outside = np.ones(shape, dtype=bool)
            outside[inside] = False
            pinned = _lib.pinned_empty(shape)
            pinned.fill(-3.0)
            for pos in (np.full(shape, -3.0), pinned):
                vel = np.full(shape, -4.0)
                c.propagate_sdp4_into(jd, fr, pos, vel, outputMode=mode, time_major=tm, output_stride=rows,
                                      sat_offset=offset)
                assert np.array_equal(pos[inside], want_p) and np.array_equal(vel[inside], want_v)
                assert np.all(pos[outside] == -3.0) and np.all(vel[outside] == -4.0)
            dp, dv = _empty(shape, -3.0), _empty(shape, -4.0)
            _sdp4_into_device(c, jd, fr, dp, dv, mode, layout, rows, offset)
            dp, dv = dp.cpu().numpy(), dv.cpu().numpy()
            assert np.array_equal(dp[inside], want_p) and np.array_equal(dv[inside], want_v)
            assert np.all(dp[outside] == -3.0) and np.all(dv[outside] == -4.0)


def test_constellation_entry_points_in_sequence(az, synth, mixed_tles):
    """One handle through host propagate, the stateless near-earth path, the single-target screen, the device grid,
    host propagate again on the same axis (the cached axis), and pairs: each result is bit for bit that of the same
    call on a fresh handle."""
    jd, fr = synth.time_grid(700)
    times = np.arange(0.0, 700.0)
    c = az.Constellation(mixed_tles)
    n, ns = c.numSatellites, c.numSgp4
    off = (2460437.5 - c.epochs[c.classes == 0]) * 1440.0
    rng = np.random.default_rng(5)
    q_sat = rng.integers(0, n, 50_000).astype(np.uint32)
    q_jd = np.full(len(q_sat), jd[0])
    q_fr = rng.uniform(0.0, 2.0, len(q_sat))

    def host(h):
        return h.propagate(jd, fr, np.full((n, 700, 3), 9.0), np.full((n, 700, 3), 9.0), layout=0)

    def into(h):
        return h.propagate_into(times, np.full((700, ns, 3), 9.0), np.full((700, ns, 3), 9.0), epoch_offsets=off)

    def screen(h):
        return h.screen_conjunction(times, 11, 200.0, epoch_offsets=off)

    def device(h):
        p, v = _empty((n, 700, 3)), _empty((n, 700, 3))
        h.propagate_device(jd, fr, p, v)
        h.synchronize()
        return p.cpu().numpy(), v.cpu().numpy()

    def pairs(h):
        return h.propagate_pairs(q_sat, q_jd, q_fr)

    steps = [host, into, screen, device, host, pairs]
    for step in steps:
        got, want = step(c), step(az.Constellation(mixed_tles))
        for g, w in zip(got, want):
            assert np.array_equal(g, w), step.__name__


def test_satrec_entry_points_in_sequence(az, mixed_tles):
    """One Satrec handle through a chunked sgp4_array, sgp4_propagate_batch below and above 64 epochs, and sgp4_array
    again; a deep-space Satrec through batch and sgp4_array.  Each result is bit for bit the same call's on a fresh
    handle."""
    from astroz_b200.api import Satrec, WGS72

    iss = Satrec.twoline2rv(*G.ISS, WGS72)
    n = 2_200_003                            # two chunks of the sgp4_array pipeline, pageable epochs
    jd = np.full(n, iss.jdsatepoch)
    fr = iss.jdsatepochF + np.arange(n) * (1.0 / 86400.0)
    short = np.linspace(-30.0, 900.0, 40)
    long = np.linspace(-1440.0, 4320.0, 3001)
    deep_tle = next(t for t in mixed_tles if Satrec.twoline2rv(*t, WGS72).is_deep_space)
    deep = Satrec.twoline2rv(*deep_tle, WGS72)

    def fresh_iss():
        return Satrec.twoline2rv(*G.ISS, WGS72)

    def array(s):
        return s.sgp4_array(jd, fr)[1:]

    calls = [(iss, fresh_iss, array), (iss, fresh_iss, lambda s: (_batch(s, short),)),
             (iss, fresh_iss, lambda s: (_batch(s, long),)), (iss, fresh_iss, array),
             (deep, lambda: Satrec.twoline2rv(*deep_tle, WGS72), lambda s: (_batch(s, long),)),
             (deep, lambda: Satrec.twoline2rv(*deep_tle, WGS72), lambda s: s.sgp4_array(jd[:5000], fr[:5000])[1:])]
    for k, (handle, fresh, call) in enumerate(calls):
        for g, w in zip(call(handle), call(fresh())):
            assert np.array_equal(g, w), k
