"""Every output specialisation of the grid kernels against the scalar oracle, at the launch shapes they run.

K1 (sgp4_grid_kernel), K1t (sgp4_times_kernel) and K2 (sdp4_grid_kernel) each have 12 specialisations: TEME / ECEF /
geodetic x satellite-major / time-major x velocities on / off.  Which K1 code runs also follows the launch shape: the
epochs per thread (launch_k1_shaped), the epochs per CTA (the stripe, launch_k1) and, time-major, the store path of each
satellite pair: `paired` 16-byte stores, `adjacent` 8-byte stores, or lone rows.  `k1_launch` and `tm_store_paths` restate
that choice, and every fixture asserts the shape it is meant to reach, so a fixture that drifts onto another path fails
instead of quietly testing that path.

Tolerances are the suite's: 1e-6 km and 1e-9 km/s against the oracle; geodetic latitude and longitude 1e-10 rad, altitude
1e-6 km.  Within one shape, positions with velocities off equal positions with velocities on, bit for bit.  Geodetic cells
within 1e-5 rad of a pole, where the oracle's p / cos(lat) - N loses digits, are compared with a 40-digit solution of the
oracle's ECEF position instead (test_geodetic_near_the_poles).  Each comparison prints one line and appends it to
$ASTROZ_PARITY_LOG when that is set.
"""
import json
import math
import os

import numpy as np
import pytest

from astroz_b200 import synth
from tests.golden import tles as G

pytestmark = pytest.mark.gpu

POS_TOL = 1e-6    # km
VEL_TOL = 1e-9    # km/s
ANG_TOL = 1e-10   # rad, geodetic latitude and longitude
POLE_BAND = 1e-5  # rad: geodetic cells this close to a pole are compared with the 40-digit solution
RE_KM = 6378.135  # WGS72 radiusearthkm: the near-earth status reference |r| / RE
SENTINEL = -7.25  # rows of the block outside the handle (or masked) keep this value
TILE = 8          # kTileSats
# the deep-space cells of the decaying Molniya fixture run ~5.5 years: angles of ~1e5 rad, so positions get
# test_gpu_parity's 1e-5 km there, and geodetic angles the 2e-9 rad that 1e-5 km makes at the Earth's surface
LONG_POS_TOL, LONG_VEL_TOL, LONG_ANG_TOL = 1e-5, VEL_TOL, 2e-9


# ---------------------------------------------------------------------------------------------- the launch shape
def k1_launch(layout, mode, n_times, n_sgp4, sms, masked=False, out_num_sats=None, stripe_override=0):
    """The near-earth launch, restated from az_kernels.cu: launch_sgp4_grid (590-613) picks K1t for one unmasked
    near-earth satellite over >= 64 epochs whose block is satellite-major or one row wide; launch_k1_shaped (533-551)
    picks the epochs per thread; launch_k1 (444-483) halves the stripe, in whole passes of 32 x epochs per thread,
    until the grid gives every resident CTA slot (3 per SM, k1_resident_slots 421-432) about eight CTAs, and
    ASTROZ_K1_STRIPE overrides it (rounded down to whole passes, at least one)."""
    rows = n_sgp4 if out_num_sats is None else out_num_sats
    if n_sgp4 == 1 and n_times >= 64 and not masked and (layout == 0 or rows == 1):
        return {"kernel": "K1t", "lanes": 2}                                  # kTimesLanes
    if layout == 1:
        lanes, k_stripe = 3, 384          # AZ_TIME_MAJOR_K1 / AZ_TM_ECEF_K1 (geodetic time-major too)
    elif mode == 2:
        lanes, k_stripe = 2, 256          # AZ_GEODETIC_K1 = AZ_COMPACT_K1
    else:
        runs1, runs2, runs3 = -(-n_times // 32), -(-n_times // 64) * 2, -(-n_times // 96) * 3
        if runs3 <= runs2 and runs3 <= runs1:
            lanes, k_stripe = 3, 384      # AZ_DEFAULT_K1
        elif runs2 <= runs1:
            lanes, k_stripe = 2, 256      # AZ_COMPACT_K1
        else:
            lanes, k_stripe = 1, 256
    k_pass = 32 * lanes
    tiles = -(-n_sgp4 // TILE)
    stripe = k_stripe
    while stripe > k_pass and tiles * -(-n_times // stripe) < 8 * 3 * sms:
        half = -(-(stripe // 2) // k_pass) * k_pass
        if half >= stripe:
            break
        stripe = half
    if stripe_override:
        stripe = max(k_pass, stripe_override // k_pass * k_pass)
    return {"kernel": "K1", "lanes": lanes, "pass": k_pass, "stripe": stripe, "ctas_per_tile": -(-n_times // stripe)}


def tm_store_paths(orig, out_num_sats, out_sat_offset=0, mask=None, base_aligned=True):
    """The time-major store path of every satellite pair of K1 (az_kernels.cu:209-229).  orig[i] is the output row of
    near-earth satellite i; a pair is two consecutive satellites of an 8-satellite tile.  Both active and in adjacent
    rows: `paired` when the block's rows are an even number of doubles apart and the pair's first record is 16-byte
    aligned, else `adjacent`; a satellite without its partner (masked, a deep-space row between, the odd last row of a
    tile) is `lone`."""
    even = (out_num_sats * 3) % 2 == 0
    n, paths = len(orig), set()
    for sat0 in range(0, n, TILE):
        n_real = min(TILE, n - sat0)
        for pr in range((n_real + 1) // 2):
            a = sat0 + 2 * pr
            n_pair = min(2, n_real - 2 * pr)
            row_a = int(orig[a])
            row_b = int(orig[a + 1]) if n_pair == 2 else row_a
            act_a = mask is None or mask[row_a] != 0
            act_b = n_pair == 2 and (mask is None or mask[row_b] != 0)
            if not (act_a or act_b):
                continue
            adjacent = act_a and act_b and row_b == row_a + 1
            paired = adjacent and even and base_aligned and (out_sat_offset + row_a) % 2 == 0
            paths.add("paired" if paired else "adjacent" if adjacent else "lone")
    return paths


# ---------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def az():
    import astroz_b200

    astroz_b200.lib()
    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return astroz_b200


@pytest.fixture(scope="module")
def sms(az):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _report(kernel, shape, mode, layout, velocities, cells, **maxima):
    """One line per compared run, printed (pytest -rP) and appended to $ASTROZ_PARITY_LOG when that is set."""
    line = json.dumps({"config": "output_stage", "kernel": kernel, "shape": shape, "mode": mode, "layout": layout,
                       "velocities": velocities, "cells": int(cells), **maxima})
    print("output_stage:", line)
    out = os.environ.get("ASTROZ_PARITY_LOG")
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def _oracle(oracle, tles, jd, fr, mode):
    """The oracle, satellite-major (time-major comparisons transpose the device block instead)."""
    return oracle.constellation_propagate(tles, jd, fr, mode=mode, layout=0, threads=0)


def _sat_major(block, layout, rows=slice(None)):
    """(satellites, epochs, 3) view of a device block in either layout, rows `rows` of it."""
    return block[rows] if layout == 0 else block.transpose(0, 1)[rows]


def _diff(got, po, vo, mode, vel=None, cells=None, tols=(POS_TOL, VEL_TOL, ANG_TOL)):
    """Maxima of |device - oracle| over the cells selected by the boolean (satellites, epochs) array `cells` (all when
    None), asserted against `tols`.  Geodetic: latitude, longitude (wrapped to +-pi) and altitude separately; cells within
    POLE_BAND of a pole are left to test_geodetic_near_the_poles for longitude and altitude."""
    import torch

    dev = got.device
    ref = torch.from_numpy(np.ascontiguousarray(po)).to(dev)
    sel = torch.ones(ref.shape[:2], dtype=torch.bool, device=dev) if cells is None else torch.from_numpy(cells).to(dev)
    ptol, vtol, atol = tols
    out = {}
    if mode == 2:
        d = (got - ref).abs()
        dlon = torch.remainder(got[..., 1] - ref[..., 1] + math.pi, 2 * math.pi) - math.pi
        off_pole = sel & (ref[..., 0].abs() < math.pi / 2 - POLE_BAND)
        out["lat_rad"] = float(d[..., 0][sel].max()) if sel.any() else 0.0
        out["lon_rad"] = float(dlon.abs()[off_pole].max()) if off_pole.any() else 0.0
        out["alt_km"] = float(d[..., 2][off_pole].max()) if off_pole.any() else 0.0
        ok = out["lat_rad"] < atol and out["lon_rad"] < atol and out["alt_km"] < ptol
    else:
        out["dr_km"] = float((got - ref).abs()[sel].max()) if sel.any() else 0.0
        ok = out["dr_km"] < ptol
    if vel is not None:
        out["dv_kms"] = float((vel - torch.from_numpy(np.ascontiguousarray(vo)).to(dev)).abs()[sel].max()) if sel.any() else 0.0
        ok = ok and out["dv_kms"] < vtol
    assert ok, out
    return out


def _device_grid(c, jd, fr, mode, layout, velocities=True, rows=None, offset=0, status=False):
    """propagate_device into fresh blocks filled with SENTINEL (status: 255) of `rows` rows, this handle at `offset`."""
    import torch

    n, nt = c.numSatellites, len(jd)
    rows = n if rows is None else rows
    shape = (rows, nt, 3) if layout == 0 else (nt, rows, 3)
    pos = torch.full(shape, SENTINEL, dtype=torch.float64, device="cuda")
    vel = torch.full_like(pos, SENTINEL) if velocities else None
    st = torch.full((n, nt), 255, dtype=torch.uint8, device="cuda") if status else None
    assert pos.data_ptr() % 16 == 0 and (vel is None or vel.data_ptr() % 16 == 0)
    # the fills run on torch's stream, the grid on the handle's own non-blocking stream: with the time axis already on the
    # device the grid can start before the fills end, so they are waited for
    torch.cuda.synchronize()
    c.propagate_device(jd, fr, pos, vel, st, mode, layout, out_num_sats=rows, out_sat_offset=offset)
    c.synchronize()
    return pos, vel, st


def _outside_untouched(block, layout, keep):
    """Rows of a device block outside `keep` (a boolean per row) still hold SENTINEL."""
    import torch

    other = torch.from_numpy(~keep).to(block.device)
    view = _sat_major(block, layout)
    return bool((view[other] == SENTINEL).all())


def _run_matrix(c, tles, jd, fr, oracle, kernel, shape, layouts, modes=(0, 1, 2), rows=None, offset=0, cells=None,
                expect=None, tols=(POS_TOL, VEL_TOL, ANG_TOL), ref=None):
    """Every (mode, layout, velocities) of this handle through propagate_device against the oracle; velocities off must
    give the velocities-on positions bit for bit.  `expect(mode, layout)` asserts the launch shape first."""
    import torch

    n = c.numSatellites
    rows_n = n if rows is None else rows
    keep = np.zeros(rows_n, dtype=bool)
    keep[offset:offset + n] = True
    for mode in modes:
        po, vo, err, _ = ref[mode] if ref is not None else _oracle(oracle, tles, jd, fr, mode)
        for layout in layouts:
            if expect is not None:
                expect(mode, layout)
            pos, vel, _ = _device_grid(c, jd, fr, mode, layout, True, rows, offset)
            cells_n = int(n * len(jd) if cells is None else cells.sum())
            sl = slice(offset, offset + n)
            m = _diff(_sat_major(pos, layout, sl), po, vo, mode, _sat_major(vel, layout, sl), cells, tols)
            _report(kernel, shape, mode, layout, True, cells_n, **m)
            pos2, vel2, _ = _device_grid(c, jd, fr, mode, layout, False, rows, offset)
            assert vel2 is None and torch.equal(pos, pos2), (kernel, shape, mode, layout)
            _report(kernel, shape, mode, layout, False, cells_n, bitwise_equal_to_velocities_on=True)
            if rows_n != n:
                assert _outside_untouched(pos, layout, keep) and _outside_untouched(vel, layout, keep)
            del pos, vel, pos2


# ---------------------------------------------------------------------------------------------- the shape model itself
def test_shape_model_reproduces_the_known_shapes(sms):
    """The restatement reproduces what the suite relies on elsewhere: 1003 x 131 satellite-major TEME runs one epoch
    per thread on a stripe of one pass, 1003 rows time-major never take the paired stores, one satellite takes K1t."""
    s = k1_launch(0, 0, 131, 1003, sms)
    assert s["lanes"] == 1 and s["stripe"] == s["pass"] == 32
    assert k1_launch(0, 0, 1440, 13478, 132)["stripe"] == 384     # the headline grid on 132 SMs: full stripes
    assert "paired" not in tm_store_paths(np.arange(1003), 1003)
    assert tm_store_paths(np.arange(1002), 1002) == {"paired"}
    assert k1_launch(0, 1, 64, 1, sms)["kernel"] == "K1t" and k1_launch(0, 1, 63, 1, sms)["kernel"] == "K1"
    assert k1_launch(1, 0, 300, 1, sms, out_num_sats=4)["kernel"] == "K1"
    assert k1_launch(0, 0, 300, 1, sms, masked=True)["kernel"] == "K1"
    assert k1_launch(1, 0, 1440, 13478, 132, stripe_override=1000)["stripe"] == 960


# ---------------------------------------------------------------------------------------------- K1, epochs per thread
@pytest.mark.parametrize("n_times,lanes", [(1440, 3), (97, 2), (131, 1)])
def test_k1_satellite_major_epochs_per_thread(az, oracle, sms, n_times, lanes):
    """203 near-earth satellites (a ragged last tile) satellite-major at three, two and one epochs per thread (TEME and
    ECEF; geodetic always runs two), each on a stripe of one pass."""
    tles = synth.near_earth_catalog(203)
    jd, fr = synth.time_grid(1440)
    step = 1440 // n_times if n_times < 1440 else 1
    jd, fr = jd[::step][:n_times].copy(), fr[::step][:n_times].copy()
    c = az.Constellation(tles)

    def expect(mode, layout):
        s = k1_launch(layout, mode, n_times, 203, sms)
        assert s["kernel"] == "K1" and s["lanes"] == (2 if mode == 2 else lanes) and s["stripe"] == s["pass"], s

    _run_matrix(c, tles, jd, fr, oracle, "K1", f"203x{n_times} lanes={lanes} one pass", (0,), expect=expect)


# ---------------------------------------------------------------------------------------------- K1, full stripes
@pytest.fixture
def stripe_env(az):
    """Sets ASTROZ_K1_STRIPE for the handles a test creates.  The override is a process-wide static that a later handle
    created without the variable does not clear, so teardown creates one with ASTROZ_K1_STRIPE=0 (automatic)."""
    def make(tles, stripe):
        os.environ["ASTROZ_K1_STRIPE"] = str(stripe)
        try:
            return az.Constellation(tles)
        finally:
            del os.environ["ASTROZ_K1_STRIPE"]

    yield make
    make([G.ISS], 0)


def _full_stripe_catalog(sms):
    """Enough near-earth satellites that 1440 epochs keep the full stripe in every mode: tiles * ceil(1440 / 384) must
    reach 8 CTAs per resident slot; one more tile of two satellites keeps the row count even (paired time-major stores)."""
    tiles = -(-8 * 3 * sms // -(-1440 // 384))
    return synth.near_earth_catalog(TILE * tiles + 2, seed=6400)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_k1_full_stripe_and_forced_stripes(az, oracle, sms, stripe_env, mode):
    """The full stripe without the override (several warp-runs per CTA, a ragged last stripe), both layouts, against the
    oracle -- run once per mode and transposed for time-major.  Then the stripe forced to one, two and three passes, 384,
    the automatic stripe itself and an odd request: every specialisation gives the automatic result bit for bit.  The
    override is process-wide and outlives the handle that set it, so it is reset first and all four automatic results
    are computed before any handle forces a stripe."""
    import torch

    stripe_env([G.ISS], 0)
    tles = _full_stripe_catalog(sms)
    n = len(tles)
    jd, fr = synth.time_grid(1440)
    c = az.Constellation(tles)
    assert c.numSgp4 == n and n % 2 == 0
    for layout in (0, 1):
        s = k1_launch(layout, mode, 1440, n, sms)
        assert s["stripe"] == (256 if (mode == 2 and layout == 0) else 384), s
        assert s["stripe"] >= 2 * s["pass"] and 1440 % s["stripe"] != 0, s
    assert tm_store_paths(np.arange(n), n) == {"paired"}
    ref = {mode: _oracle(oracle, tles, jd, fr, mode)}
    _run_matrix(c, tles, jd, fr, oracle, "K1", f"{n}x1440 full stripe", (0, 1), modes=(mode,), ref=ref)
    del ref
    specs = [(layout, velocities) for layout in (0, 1) for velocities in (True, False)]
    auto = {sv: _device_grid(c, jd, fr, mode, *sv) for sv in specs}
    for layout, velocities in specs:
        auto_p, auto_v, _ = auto[layout, velocities]
        s = k1_launch(layout, mode, 1440, n, sms)
        k_pass = s["pass"]
        forced = set()
        for req in dict.fromkeys((k_pass, 2 * k_pass, 3 * k_pass, 384, s["stripe"], 1000, 7)):
            stripe = k1_launch(layout, mode, 1440, n, sms, stripe_override=req)["stripe"]
            forced.add(stripe)
            f = stripe_env(tles, req)
            p, v, _ = _device_grid(f, jd, fr, mode, layout, velocities)
            assert torch.equal(p, auto_p) and (v is None or torch.equal(v, auto_v)), (mode, layout, velocities, req)
            del f, p, v
        assert {k_pass, 2 * k_pass, 3 * k_pass, s["stripe"]} <= forced
        _report("K1", f"{n}x1440 forced stripes {sorted(forced)}, automatic {s['stripe']}", mode, layout, velocities,
                n * 1440, bitwise_equal_to_automatic=True)
        del auto[layout, velocities], auto_p, auto_v


# ---------------------------------------------------------------------------------------------- K1, time-major stores
TM_CASES = {
    # name: (satellites, block rows, row offset, store paths the pairs take)
    "paired": (202, 202, 0, {"paired"}),
    "adjacent_odd_rows": (202, 203, 0, {"adjacent"}),
    "adjacent_odd_offset": (202, 204, 1, {"adjacent"}),
    "lone_odd_last_row": (203, 206, 0, {"paired", "lone"}),
}


@pytest.mark.parametrize("case", sorted(TM_CASES))
def test_k1_time_major_store_paths(az, oracle, sms, case):
    """Each store path of the time-major K1 epilogue in all three modes, into blocks wider than the handle whose other
    rows keep their sentinel."""
    n, rows, off, paths = TM_CASES[case]
    tles = synth.near_earth_catalog(n, seed=4242)
    jd, fr = synth.time_grid(1440)
    jd, fr = jd[::11][:131].copy(), fr[::11][:131].copy()
    c = az.Constellation(tles)
    assert tm_store_paths(np.arange(n), rows, off) == paths

    def expect(mode, layout):
        assert k1_launch(layout, mode, 131, n, sms, out_num_sats=rows)["kernel"] == "K1"

    _run_matrix(c, tles, jd, fr, oracle, "K1", f"{n}x131 time-major {case}", (1,), rows=rows, offset=off, expect=expect)


def test_k1_time_major_masked_partners(az, oracle, sms):
    """Lone rows from masked partners: propagate_into with a satellite mask, time-major, every mode, against the oracle;
    masked rows keep the caller's contents."""
    import torch

    n, nt = 96, 131
    tles = synth.near_earth_catalog(n, seed=977)
    jd, fr = synth.time_grid(1440)
    jd, fr = jd[::11][:nt].copy(), fr[::11][:nt].copy()
    c = az.Constellation(tles)
    ref_jd = c.referenceEpochJd
    times = ((jd + fr) - ref_jd) * 1440.0            # the grid's time axis, so ref_jd + times / 1440 is jd + fr again
    assert np.array_equal(ref_jd + times / 1440.0, jd + fr)
    off = (ref_jd - c.epochs) * 1440.0
    mask = np.ones(n, dtype=np.uint8)
    mask[::3] = 0
    paths = tm_store_paths(np.arange(n), n, mask=mask)
    assert paths == {"paired", "lone"}, paths
    assert k1_launch(1, 0, nt, n, sms, masked=True)["kernel"] == "K1"
    on = mask == 1
    for mode in (0, 1, 2):
        po, vo, _, _ = _oracle(oracle, tles, jd, fr, mode)
        p = np.full((nt, n, 3), SENTINEL)
        v = np.full((nt, n, 3), SENTINEL)
        c.propagate_into(times, p, v, epoch_offsets=off, satellite_mask=mask, outputMode=mode, reference_jd=ref_jd,
                         time_major=True)
        p2 = np.full((nt, n, 3), SENTINEL)
        c.propagate_into(times, p2, None, epoch_offsets=off, satellite_mask=mask, outputMode=mode, reference_jd=ref_jd,
                         time_major=True, want_velocities=False)
        assert np.array_equal(p, p2)
        ps, vs = p.transpose(1, 0, 2), v.transpose(1, 0, 2)
        assert np.all(ps[~on] == SENTINEL) and np.all(vs[~on] == SENTINEL)
        m = _diff(torch.from_numpy(np.ascontiguousarray(ps[on])), po[on], vo[on], mode, torch.from_numpy(np.ascontiguousarray(vs[on])))
        _report("K1", f"{n}x{nt} time-major masked partners", mode, 1, True, int(on.sum()) * nt, **m)


# ---------------------------------------------------------------------------------------------- K2 (and K1 beside it)
def test_k2_mixed_catalog_every_specialisation(az, oracle, sms):
    """A mixed catalog with all four classes, deep-space rows at odd and even positions and between near-earth rows,
    over 1100 epochs (two full 512-epoch K2 stripes and a ragged third): every mode, layout and velocities setting,
    near-earth and deep-space cells reported apart, status bytes equal to the oracle's codes."""
    tles = synth.mixed_catalog(300, seed=1100, n_geo=20, n_molniya=12, n_gps=12)
    jd, fr = synth.time_grid(1100)
    c = az.Constellation(tles)
    klass = np.asarray(c.classes)
    deep = klass > 0
    rows = np.flatnonzero(deep)
    assert set(klass.tolist()) == {0, 1, 2, 3}
    assert {0, 1} <= set((rows % 2).tolist())
    near_rows = np.flatnonzero(~deep)
    assert np.any(np.diff(near_rows) == 2)                   # a deep-space row between two near-earth rows
    assert "lone" in tm_store_paths(near_rows, len(tles)) and 1100 % 512 != 0
    nt = len(jd)

    def expect_k1(mode, layout):
        # 1100 epochs: one epoch per thread satellite-major (runs 35 < 36), two geodetic, three time-major; 32 tiles
        # are far from filling the GPU, so the stripe is one pass
        s = k1_launch(layout, mode, nt, len(near_rows), sms, out_num_sats=len(tles))
        assert s["kernel"] == "K1" and s["lanes"] == (3 if layout == 1 else 2 if mode == 2 else 1), s
        assert s["stripe"] == s["pass"], s

    for mode in (0, 1, 2):
        po, vo, err, kl = _oracle(oracle, tles, jd, fr, mode)
        assert list(kl) == list(klass) and not err.any()
        ref = {mode: (po, vo, err, kl)}
        for kernel, sel in (("K2", deep), ("K1", ~deep)):
            cells = np.repeat(sel[:, None], nt, axis=1)
            _run_matrix(c, tles, jd, fr, oracle, kernel, f"mixed 300x{nt}", (0, 1), modes=(mode,), cells=cells, ref=ref,
                        expect=expect_k1 if kernel == "K1" else None)
        for layout in (0, 1):
            _, _, st = _device_grid(c, jd, fr, mode, layout, False, status=True)
            assert np.array_equal(st.cpu().numpy()[deep], err[deep])


@pytest.mark.parametrize("layout", [0, 1])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_k2_failed_cells_are_zero_in_every_frame(az, oracle, mode, layout):
    """The decaying Molniya object of test_deep_space_failures_are_zero_filled_per_satellite in every mode and layout:
    failed cells are exactly (0, 0, 0) in position and velocity -- the oracle zero-fills before the frame conversion and
    the kernel skips it -- their status codes equal the oracle's, and the other cells match it."""
    import torch

    bad = synth.tle_lines(42000, 24, 120.0, 63.4, 0.0, 0.755, 0.0, 10.0, 2.006, 1e-3)
    tles = [G.GPS20413, bad, G.GEO28626, G.HEO09880]
    jd = np.full(40, 2460430.5)
    fr = np.linspace(0.0, 2000.0, 40)
    c = az.Constellation(tles)
    po, vo, err, _ = _oracle(oracle, tles, jd, fr, mode)
    assert err[1].any() and set(np.unique(err[1])) >= {1, 2}
    failed = err != 0
    for velocities in (True, False):
        pos, vel, st = _device_grid(c, jd, fr, mode, layout, velocities, status=True)
        assert np.array_equal(st.cpu().numpy(), err)
        p = _sat_major(pos, layout).cpu().numpy()
        assert np.all(p[failed] == 0.0)
        if velocities:
            v = _sat_major(vel, layout).cpu().numpy()
            assert np.all(v[failed] == 0.0)
            m = _diff(_sat_major(pos, layout), po, vo, mode, _sat_major(vel, layout), ~failed,
                      (LONG_POS_TOL, LONG_VEL_TOL, LONG_ANG_TOL))
            _report("K2", "4x40 failing Molniya, 5.5 years", mode, layout, True, int((~failed).sum()),
                    failed_cells=int(failed.sum()), **m)
            ref_p = pos
        else:
            assert torch.equal(pos, ref_p)


# ---------------------------------------------------------------------------------------------- K1t
@pytest.mark.parametrize("n_times", [64, 255, 256, 257, 5000])
def test_k1t_every_specialisation(az, oracle, sms, n_times):
    """The ISS alone over n_times epochs runs K1t: satellite-major and as a one-row time-major block, every mode."""
    jd, fr = synth.time_grid(n_times)
    c = az.Constellation([G.ISS])

    def expect(mode, layout):
        assert k1_launch(layout, mode, n_times, 1, sms)["kernel"] == "K1t"

    _run_matrix(c, [G.ISS], jd, fr, oracle, "K1t", f"ISS x{n_times}", (0, 1), expect=expect)


def test_k1t_single_near_earth_row_of_a_mixed_catalog(az, oracle, sms):
    """One near-earth row among deep-space rows: satellite-major it runs K1t, time-major (four rows) K1 with a lone row."""
    tles = [G.GEO28626, G.ISS, G.GPS20413, G.HEO09880]
    jd, fr = synth.time_grid(300)
    c = az.Constellation(tles)
    assert c.numSgp4 == 1 and list(c.classes) == [2, 0, 1, 3]
    assert tm_store_paths([1], 4) == {"lone"}
    near = np.zeros((4, 300), dtype=bool)
    near[1] = True
    for layout, kernel in ((0, "K1t"), (1, "K1")):
        def expect(mode, lay, kernel=kernel):
            assert k1_launch(lay, mode, 300, 1, sms, out_num_sats=4)["kernel"] == kernel

        _run_matrix(c, tles, jd, fr, oracle, kernel, "mixed 4x300, one near-earth row", (layout,), cells=near,
                    expect=expect)


# ---------------------------------------------------------------------------------------------- near-earth status
def _status_reference(po):
    """ASTROZ_CELL_DECAYED where the oracle's |r| / RE < 1 (SGP4's |r| is mrt * RE up to rounding); cells within 1e-12
    of 1, or not finite, are not compared."""
    ratio = np.linalg.norm(po, axis=-1) / RE_KM
    comparable = np.isfinite(ratio) & (np.abs(ratio - 1.0) > 1e-12)
    return (ratio < 1.0).astype(np.uint8), comparable, ratio


def test_near_earth_status_bytes(az, oracle, sms):
    """The heavy-drag sets of test_gpu_cold_paths over two weeks: the status byte is ASTROZ_CELL_DECAYED exactly where
    the oracle's radius is below one Earth radius -- K1 in both layouts, K1t on the decaying satellite alone, and
    propagate_pairs."""
    from tests.test_gpu_cold_paths import FIXTURES

    tles = FIXTURES["drag_angle"][0]
    n = len(tles)
    jd = np.full(4033, 2460437.5)
    fr = np.linspace(0.0, 14.0, 4033)
    po, _, _, klass = _oracle(oracle, tles, jd, fr, 0)
    assert not klass.any()
    want, comparable, ratio = _status_reference(po)
    assert (want[comparable] == 1).any() and (want[comparable] == 0).any()
    c = az.Constellation(tles)
    for layout in (0, 1):
        assert k1_launch(layout, 0, 4033, n, sms)["kernel"] == "K1"
        _, _, st = _device_grid(c, jd, fr, 0, layout, False, status=True)
        st = st.cpu().numpy()
        assert np.array_equal(st[comparable], want[comparable]), layout
        _report("K1", f"{n}x4033 heavy drag, status", 0, layout, False, int(comparable.sum()),
                decayed=int(want[comparable].sum()))
    sat = np.repeat(np.arange(n, dtype=np.int64), len(jd))
    _, _, pst = c.propagate_pairs(sat, np.tile(jd, n), np.tile(fr, n), velocities=False)
    assert np.array_equal(pst.reshape(n, -1)[comparable], want[comparable])
    _report("pairs", f"{n}x4033 heavy drag, status", 0, 0, False, int(comparable.sum()), decayed=int(want[comparable].sum()))
    # K1t: the satellite that decays, alone, on a one-minute axis; cells just above the surface are there too
    k = int(np.argmax((want * comparable).sum(axis=1)))
    jd1 = np.full(20161, 2460437.5)
    fr1 = np.linspace(0.0, 14.0, 20161)
    po1, _, _, _ = _oracle(oracle, [tles[k]], jd1, fr1, 0)
    want1, comp1, ratio1 = _status_reference(po1)
    assert (want1[comp1] == 1).any() and (comp1 & (ratio1 > 1.0) & (ratio1 < 1.001)).sum() >= 10
    one = az.Constellation([tles[k]])
    assert k1_launch(0, 0, len(jd1), 1, sms)["kernel"] == "K1t"
    _, _, st1 = _device_grid(one, jd1, fr1, 0, 0, False, status=True)
    assert np.array_equal(st1.cpu().numpy()[comp1], want1[comp1])
    _report("K1t", "1x20161 heavy drag, status", 0, 0, False, int(comp1.sum()), decayed=int(want1[comp1].sum()))


# ---------------------------------------------------------------------------------------------- geodetic near the poles
def _geodetic_40_digits(ecef):
    """(lat, lon, alt) of an ECEF position on WGS84, to 40 digits: the reference's fixed point lat = atan2(z + e2 N sin
    lat, p), iterated to convergence, and the altitude as p cos lat + z sin lat - a sqrt(1 - e2 sin^2 lat), which is
    p / cos lat - N without the cancellation."""
    import mpmath as mp

    with mp.workdps(40):
        a = mp.mpf(6378.137)
        f = 1 / mp.mpf("298.257223563")
        e2 = 2 * f - f * f
        x, y, z = (mp.mpf(float(u)) for u in ecef)
        p = mp.sqrt(x * x + y * y)
        lat = mp.atan2(z, p * (1 - e2))
        for _ in range(60):
            s = mp.sin(lat)
            lat = mp.atan2(z + e2 * (a / mp.sqrt(1 - e2 * s * s)) * s, p)
        s, co = mp.sin(lat), mp.cos(lat)
        alt = p * co + z * s - a * mp.sqrt(1 - e2 * s * s)
        return float(lat), float(mp.atan2(y, x)), float(alt), float(p)


def _polar_axis(oracle):
    """Epochs around the pole crossings of a 90-degree orbit: the crossing times come from the oracle (minimum of
    sqrt(x^2 + y^2), the same in TEME and ECEF), then offsets from 0 to 30 s either side."""
    from scipy.optimize import minimize_scalar

    tle = synth.tle_lines(45000, 24, 128.0, 90.0, 30.0, 1e-3, 0.0, 0.0, 15.2, 1e-5)
    s = oracle.Sgp4(*tle)
    period = 1440.0 / 15.2
    jd0 = 2460433.5
    times = []
    for k in range(6):
        guess = (k + 0.5) * period / 2.0            # argument of latitude 90 and 270 degrees
        res = minimize_scalar(lambda t: float(np.hypot(*s.propagate(t)[0][:2])),
                              bounds=(guess - 0.2 * period, guess + 0.2 * period), method="bounded",
                              options={"xatol": 1e-9})
        for dt in (0.0, 1e-4, -1e-4, 1e-3, -1e-3, 2e-3, -2e-3, 5e-3, -5e-3, 0.05, -0.05, 0.5, -0.5, 30.0, -30.0):
            times.append(res.x + dt / 60.0)
    times = np.sort(np.array(times))
    fr = (s.epochJd - jd0) + times / 1440.0
    return tle, np.full(len(times), jd0), fr


def test_geodetic_near_the_poles(az, oracle, sms):
    """A 90-degree orbit sampled within 1e-5 rad of both poles: cells in that band against the 40-digit solution of the
    oracle's ECEF position (latitude 1e-10 rad, altitude 1e-6 km, longitude as p * dlon < 1e-6 km: on the axis the
    longitude is only as good as the position), the others against the oracle's geodetic output; K1t, and K1 in both
    layouts."""
    tle, jd, fr = _polar_axis(oracle)
    nt = len(jd)
    assert nt >= 64
    po_ecef, _, _, _ = _oracle(oracle, [tle, tle], jd, fr, 1)
    po_geo, vo, _, _ = _oracle(oracle, [tle, tle], jd, fr, 2)
    e = po_ecef[0]
    polar_dist = np.arctan2(np.hypot(e[:, 0], e[:, 1]), np.abs(e[:, 2]))
    band = polar_dist < POLE_BAND
    assert band.sum() >= 40 and (polar_dist < 1e-7).any() and (e[band, 2] > 0).any() and (e[band, 2] < 0).any()
    exact = np.array([_geodetic_40_digits(e[t]) for t in range(nt)])
    for kernel, tles, layout in (("K1t", [tle], 0), ("K1", [tle, tle], 0), ("K1", [tle, tle], 1)):
        c = az.Constellation(tles)
        assert k1_launch(layout, 2, nt, len(tles), sms)["kernel"] == kernel
        pos, vel, _ = _device_grid(c, jd, fr, 2, layout, True)
        got = _sat_major(pos, layout).cpu().numpy()
        m = _diff(_sat_major(pos, layout), po_geo[:len(tles)], vo[:len(tles)], 2, _sat_major(vel, layout))
        g = got[:, band]
        dlat = float(np.max(np.abs(g[..., 0] - exact[band, 0])))
        dalt = float(np.max(np.abs(g[..., 2] - exact[band, 2])))
        dlon = np.remainder(g[..., 1] - exact[band, 1] + np.pi, 2 * np.pi) - np.pi
        darc = float(np.max(np.abs(dlon) * exact[band, 3]))
        assert dlat < ANG_TOL and dalt < POS_TOL and darc < POS_TOL, (kernel, layout, dlat, dalt, darc)
        _report(kernel, f"{len(tles)}x{nt} polar orbit", 2, layout, True, len(tles) * nt, polar_cells=int(band.sum()),
                polar_lat_rad=dlat, polar_alt_km=dalt, polar_lon_arc_km=darc, **m)


# ---------------------------------------------------------------------------------------------- status block and offset
@pytest.mark.parametrize("layout", [0, 1])
def test_status_block_stays_the_handles_own_with_a_row_offset(az, oracle, layout):
    """d_status is the handle's own n x n_times bytes, satellite-major, also when out_sat_offset places the positions in
    a larger block: the status block is the first n * n_times bytes of a tensor of 255s, out_num_sats = n + 7,
    out_sat_offset = 3; row i must land at i * n_times and every byte after the block must stay 255."""
    import torch

    from tests.test_gpu_cold_paths import FIXTURES

    bad = synth.tle_lines(42000, 24, 120.0, 63.4, 0.0, 0.755, 0.0, 10.0, 2.006, 1e-3)
    tles = [G.GPS20413, bad] + FIXTURES["drag_angle"][0][4:] + [G.GEO28626]
    n = len(tles)
    jd = np.full(80, 2460430.5)
    fr = np.linspace(0.0, 2000.0, 80)
    c = az.Constellation(tles)
    base_p, base_v, base_st = _device_grid(c, jd, fr, 0, layout, True, status=True)
    want = base_st.cpu().numpy()
    assert len({bytes(r) for r in want}) >= 3           # rows that differ, so a misplaced row shows
    _, _, err, klass = _oracle(oracle, tles, jd, fr, 0)
    assert np.array_equal(want[klass > 0], err[klass > 0])
    nt = len(jd)
    guard = torch.full(((n + 7) * nt,), 255, dtype=torch.uint8, device="cuda")
    rows = n + 7
    shape = (rows, nt, 3) if layout == 0 else (nt, rows, 3)
    pos = torch.full(shape, SENTINEL, dtype=torch.float64, device="cuda")
    vel = torch.full_like(pos, SENTINEL)
    torch.cuda.synchronize()   # the fills (torch's stream) end before the grid (the handle's stream) starts
    c.propagate_device(jd, fr, pos, vel, guard[:n * nt], 0, layout, out_num_sats=rows, out_sat_offset=3)
    c.synchronize()
    g = guard.cpu().numpy()
    assert np.array_equal(g[:n * nt].reshape(n, nt), want)
    assert np.all(g[n * nt:] == 255)
    keep = np.zeros(rows, dtype=bool)
    keep[3:3 + n] = True
    # the decayed near-earth row turns to NaN after some years: compare bits
    for got, ref in ((pos, base_p), (vel, base_v)):
        assert torch.equal(_sat_major(got, layout, slice(3, 3 + n)).contiguous().view(torch.int64),
                           _sat_major(ref, layout).contiguous().view(torch.int64))
    assert _outside_untouched(pos, layout, keep) and _outside_untouched(vel, layout, keep)
