"""Both conjunction screens on the device against exact references (the block fixtures and references are in
tests/test_screens_cpu.py):

* K4 (all-vs-all, coarse_screen_device / the C ABI): every crafted block -- threshold flips between the reference's
  rounded d^2 and a fused one, cell edges, hash collisions, epoch-batch seams, non-finite and masked rows, a tiny
  threshold -- in both layouts, with and without a mask, equals brute force and the oracle's cell list exactly.
* K3 (single target, screen_conjunction): at several axis lengths the reported epoch of every hit is one where the
  oracle's distance is within eps of its minimum and of the reported distance; copies of the target come back at
  exactly (0.0, 0).
"""
import ctypes as C

import numpy as np
import pytest

from tests import test_screens_cpu as S

pytestmark = pytest.mark.gpu

EPS = 2e-6   # km: twice the suite's position tolerance against the scalar oracle


@pytest.fixture(scope="module")
def az():
    import astroz_b200

    astroz_b200.lib()
    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return astroz_b200


@pytest.fixture(scope="module")
def handle(az):
    from astroz_b200 import synth

    return az.Constellation(synth.near_earth_catalog(8))


def _device_screen(c, pos_sm, thr, layout, mask):
    import torch

    dev = torch.device("cuda", c.device)
    blk = pos_sm if layout == 0 else pos_sm.transpose(1, 0, 2)
    return c.coarse_screen_device(torch.as_tensor(np.ascontiguousarray(blk), device=dev), thr, layout=layout,
                                  valid_mask=None if mask is None else torch.as_tensor(mask, device=dev))


def _same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---------------------------------------------------------------------------------------------- K4
def test_k4_decides_the_threshold_like_the_reference(handle, oracle):
    """Pairs within an ulp of thr^2 where fma(dz,dz, fma(dx,dx, dy*dy)) and the reference's (dx^2 + dy^2) + dz^2
    disagree: the device keeps exactly the reference's hits."""
    for pos, thr, planted in S.fma_flip_block():
        want = S.brute_force(pos, thr)
        assert _same(oracle.coarse_screen(pos, thr), want)
        got_set = {(int(a), int(b), int(t)) for (a, b), t in zip(*want)}
        assert all(((a, b, t) in got_set) == ref_hit for a, b, t, ref_hit in planted)
        for layout in (0, 1):
            got = _device_screen(handle, pos, thr, layout, None)
            assert _same(got, want), (thr, layout)


@pytest.mark.parametrize("layout", [0, 1])
def test_k4_block_fixtures_equal_brute_force(handle, oracle, layout):
    for name, pos, thr, mask in S.all_k4_cases():
        masks = [mask] if mask is not None else [None, np.ones(pos.shape[0], dtype=np.uint8)]
        for m in masks:
            want = S.brute_force(pos, thr, m)
            assert _same(oracle.coarse_screen(pos, thr, valid_mask=m), want), name
            got = _device_screen(handle, pos, thr, layout, m)
            assert _same(got, want), (name, layout, m is None)


def test_k4_block_size_does_not_depend_on_the_handle(handle):
    """A 20,000-row block through a handle of 8 satellites, then a 50-row block through the same handle (its
    scratch is reused)."""
    rng = np.random.default_rng(9)
    big = S._background(rng, 20_000, 2, 6800.0, 7200.0)
    for i in range(40):   # clusters so there are hits at a 5 km threshold
        big[500 * i + 1:500 * i + 4] = big[500 * i] + rng.normal(size=(3, 2, 3))
    want = S.brute_force(big, 5.0)
    assert len(want[1]) >= 80
    assert _same(_device_screen(handle, big, 5.0, 1, None), want)
    small = big[:50].copy()
    want = S.brute_force(small, 5.0)
    assert len(want[1]) > 0
    assert _same(_device_screen(handle, small, 5.0, 0, None), want)


def test_k4_max_results_overflow_through_the_c_abi(handle):
    """More hits than max_results: count is the true total, the stored prefix is a subset of the true set without
    duplicates, and the words after max_results in both device buffers are untouched."""
    import torch

    from astroz_b200._lib import check, lib

    pos = S.cell_edge_block(10.0)
    want = S.brute_force(pos, 10.0)
    n = len(want[1])
    truth = {(int(a), int(b), int(t)) for (a, b), t in zip(*want)}
    dev = torch.device("cuda", handle.device)
    blk = torch.as_tensor(pos, device=dev)
    sentinel = 0x5EED5EED
    for m in (n // 3, n - 1):
        pairs = torch.full((m + 16, 2), sentinel, dtype=torch.int64, device=dev).to(torch.int32)
        tidx = torch.full((m + 16,), sentinel, dtype=torch.int64, device=dev).to(torch.int32)
        cnt = C.c_uint64()
        torch.cuda.synchronize(dev)
        check(lib().astroz_cuda_constellation_coarse_screen_device(
            handle._h, C.c_void_p(blk.data_ptr()), pos.shape[0], pos.shape[1], 0, 10.0, None,
            C.c_void_p(pairs.data_ptr()), C.c_void_p(tidx.data_ptr()), m, C.byref(cnt)))
        p = pairs.cpu().numpy().view(np.uint32)
        t = tidx.cpu().numpy().view(np.uint32)
        assert cnt.value == n
        assert (p[m:] == sentinel).all() and (t[m:] == sentinel).all()
        stored = {(int(a), int(b), int(x)) for (a, b), x in zip(p[:m], t[:m])}
        assert len(stored) == m and stored <= truth


# ---------------------------------------------------------------------------------------------- K3
def _catalog_with_neighbours(n, target, seed):
    """n near-earth sets; rows after the target carry co-orbital copies of it shifted in mean anomaly by 0.02-0.1 deg
    (minima below the threshold) and by 1e-4 deg (distance nearly constant over the axis: near ties)."""
    from astroz_b200 import synth

    tles = synth.near_earth_catalog(n, seed=seed)
    base = tles[target]
    for k, shift in enumerate((0.02, 0.05, 0.1, 0.0001, 0.0002, -0.0001)):
        l2 = base[1]
        ma = (float(l2[43:51]) + shift) % 360.0
        l2 = l2[:43] + f"{ma:8.4f}" + l2[51:68]
        tles[(target + 3 + 5 * k) % n] = (base[0], l2 + str(synth._checksum(l2)))
    return tles


def _oracle_tracks(oracle, tles, times, off):
    out = np.zeros((len(tles), len(times), 3))
    for s, t in enumerate(tles):
        m = oracle.Sgp4(*t)
        for k, x in enumerate(times):
            out[s, k] = m.propagate(x + off[s])[0]
    return out


@pytest.mark.parametrize("target", [2, 58])
def test_k3_reported_epochs_meet_the_oracle_minimum(az, oracle, target):
    """61 satellites (the last tile holds 5), the target in tile 0 or in the last tile, axes of 1, 31, 63, 64, 65 and
    1441 epochs.  A hit's epoch t satisfies d_o(t) <= min d_o + eps and |d - d_o(t)| <= eps; a satellite whose oracle
    minimum is above thr + eps returns exactly (thr, 0)."""
    tles = _catalog_with_neighbours(61, target, 501)
    c = az.Constellation(tles)
    assert c.numSgp4 == 61
    off = S.screen_offsets(tles)
    thr = 40.0
    full = S.screen_times(1441)
    tracks = _oracle_tracks(oracle, tles, full, off)
    n_hits = 0
    for nt in (1, 31, 63, 64, 65, 1441):
        times = full[:nt]
        d, ti = c.screen_conjunction(times, target, thr, epoch_offsets=off, reference_jd=S.REF_JD)
        do = np.linalg.norm(tracks[:, :nt] - tracks[target, :nt][None], axis=2)
        dmin = do.min(axis=1)
        assert d[target] == thr and ti[target] == 0
        for s in range(61):
            if s == target:
                continue
            if d[s] < thr:
                n_hits += 1
                t = int(ti[s])
                assert t < nt and do[s, t] <= dmin[s] + EPS and abs(d[s] - do[s, t]) <= EPS, (nt, s)
            if dmin[s] > thr + EPS:
                assert d[s] == thr and ti[s] == 0, (nt, s)
            if dmin[s] < thr - EPS:
                assert d[s] < thr, (nt, s)
    assert n_hits >= 6 * 6


def test_k3_copies_of_the_target_meet_it_at_zero(az, oracle):
    """Copies of the target in its own tile, in another tile and in the last, partial tile return exactly 0.0 km at
    epoch 0.  The target's first cell differs between one cell per call and the screen's two-lane shape (host
    emulation), so this holds only because the track is computed in the screen's shape."""
    from astroz_b200 import synth

    times = S.screen_times(300)
    cands = S.divergence_candidates()
    so = S.load_emul_screen()
    tgt, gap = S.pick_divergent_target(so, cands, times)
    assert 0.0 < gap < 1e-9
    base = synth.near_earth_catalog(61, seed=77)
    target, copies = 2, [5, 30, 59]
    tles = S.with_duplicates(base, cands[tgt], [target] + copies)
    off = S.screen_offsets(tles)
    c = az.Constellation(tles)
    for nt in (1, 65, 300):
        d, ti = c.screen_conjunction(times[:nt], target, 25.0, epoch_offsets=off, reference_jd=S.REF_JD)
        assert (d[copies] == 0.0).all() and (ti[copies] == 0).all(), nt
        do, _ = oracle.screen_constellation(tles, times[:nt], off, target, 25.0, S.REF_JD)
        assert (do[copies] == 0.0).all()
        assert np.max(np.abs(d - do)) < 1e-6


def test_mixed_handle_screens_the_near_earth_rows(az, oracle):
    """On a handle with deep-space rows, screen_conjunction and screen_all screen the near-earth rows: `target` and the
    result index near-earth rows in catalogue order, and epoch_offsets[:numSgp4] are their offsets."""
    from astroz_b200 import synth

    tles = synth.mixed_catalog(48, n_geo=5, n_molniya=3, n_gps=3)
    c = az.Constellation(tles)
    near = c.classes == 0
    assert 0 < c.numSgp4 < c.numSatellites
    near_tles = [t for t, k in zip(tles, near) if k]
    off = (S.REF_JD - c.epochs[near]) * 1440.0
    times = S.screen_times(200)
    d, ti = c.screen_conjunction(times, 4, 5000.0, epoch_offsets=off, reference_jd=S.REF_JD)
    do, tio = oracle.screen_constellation(near_tles, times, off, 4, 5000.0, S.REF_JD)
    assert d.shape == (c.numSgp4,)
    assert np.max(np.abs(d - do)) < 1e-6
    hit = do < 5000.0 - EPS
    assert hit.sum() >= 2 and (d[hit] < 5000.0).all()
    p_tm, _ = c.propagate_into(times, epoch_offsets=off, want_velocities=False, time_major=True)
    assert p_tm.shape[1] == c.numSgp4
    want = S.brute_force(np.ascontiguousarray(p_tm.transpose(1, 0, 2)), 300.0)
    assert _same(c.screen_all(times, 300.0, epoch_offsets=off), want)
