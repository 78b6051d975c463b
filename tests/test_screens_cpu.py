"""The two conjunction screens without a GPU: the per-thread code of K4 (cell coordinates, the 13 forward offsets, the
collision filter, the distance predicate) and K3's lane shape, both from astroz_b200/csrc/az_screen.cuh, run on the CPU
by tests/host_emul/emul_screen.cu.  They are checked against plain references kept in this file:

* a brute-force all-pairs search per epoch that rounds each product and sums (dx^2 + dy^2) + dz^2, the reference's
  order (bindings/python/src/conjunction.zig:119-124), with a strict `< thr * thr`;
* the scalar oracle, cell by cell, for K3.

The block fixtures built here are shared with tests/test_gpu_screens.py, which runs them through the device kernels.
The fixtures that put a pair's squared distance within an ulp of thr^2, where a fused multiply-add decides differently,
only prove something on the device: the host compiler does not contract.

Tiny thresholds: when |coordinate| / threshold exceeds the int range, cell coordinates saturate (INT32_MIN / INT32_MAX),
like the device conversion.  Saturation is monotonic, so the hit set still equals brute force; no call is refused.
"""
import ctypes as C
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "host_emul")
REF_JD = 2460437.5


# ---------------------------------------------------------------------------------------------- references
def sorted_hits(pairs, tidx):
    """(pairs[n, 2], t[n]) as uint32, ordered by (t, s, other) like the package's screens."""
    pairs = np.asarray(pairs, dtype=np.uint32).reshape(-1, 2)
    tidx = np.asarray(tidx, dtype=np.uint32).reshape(-1)
    order = np.lexsort((pairs[:, 1], pairs[:, 0], tidx)) if len(tidx) else np.zeros(0, dtype=np.int64)
    return np.ascontiguousarray(pairs[order]), np.ascontiguousarray(tidx[order])


def brute_force(pos_sm, thr, valid_mask=None, chunk=256):
    """Every pair (s < o) of rows that take part (mask set, x finite) with (dx*dx + dy*dy) + dz*dz < thr*thr, each
    operation rounded (numpy does not contract)."""
    pos_sm = np.asarray(pos_sm, dtype=np.float64)
    ns, nt = pos_sm.shape[:2]
    thr2 = thr * thr
    rows = np.ones(ns, dtype=bool) if valid_mask is None else np.asarray(valid_mask) != 0
    pairs, ts = [], []
    for t in range(nt):
        p = pos_sm[:, t]
        idx = np.flatnonzero(rows & np.isfinite(p[:, 0]))
        q = p[idx]
        for a0 in range(0, len(idx), chunk):
            b = q[a0:a0 + chunk]
            with np.errstate(invalid="ignore", over="ignore"):
                dx = b[:, None, 0] - q[None, :, 0]
                dy = b[:, None, 1] - q[None, :, 1]
                dz = b[:, None, 2] - q[None, :, 2]
                d2 = (dx * dx + dy * dy) + dz * dz
            i, j = np.nonzero(d2 < thr2)
            i = i + a0
            keep = i < j
            if keep.any():
                pairs.append(np.stack([idx[i[keep]], idx[j[keep]]], axis=1))
                ts.append(np.full(int(keep.sum()), t))
    if not pairs:
        return sorted_hits(np.zeros((0, 2)), np.zeros(0))
    return sorted_hits(np.concatenate(pairs), np.concatenate(ts))


def _rn(x: Fraction) -> Fraction:
    return Fraction(float(x))  # int / int true division rounds correctly to nearest even


def ref_d2_exact(dx, dy, dz) -> Fraction:
    """The reference's d^2: each product rounded, (dx^2 + dy^2) + dz^2 rounded after each sum."""
    fx, fy, fz = Fraction(dx), Fraction(dy), Fraction(dz)
    return _rn(_rn(_rn(fx * fx) + _rn(fy * fy)) + _rn(fz * fz))


def fma_d2_exact(dx, dy, dz) -> Fraction:
    """d^2 as fma(dz, dz, fma(dx, dx, dy * dy)): what nvcc made of the plain expression in the K4 kernel."""
    fx, fy, fz = Fraction(dx), Fraction(dy), Fraction(dz)
    return _rn(fz * fz + _rn(fx * fx + _rn(fy * fy)))


def _ulp(x):
    return np.spacing(np.abs(x))


def _background(rng, ns, nt, r0=20000.0, r1=40000.0):
    """Rows spread over a thick shell, far apart at a few-km threshold."""
    v = rng.normal(size=(ns, nt, 3))
    v /= np.linalg.norm(v, axis=2, keepdims=True)
    return v * rng.uniform(r0, r1, size=(ns, nt, 1))


# ---------------------------------------------------------------------------------------------- K4 fixtures
def fma_flip_offsets(thr, per_kind, seed):
    """Offsets (dx, dy, dz), multiples of 2^-40 (the ulp of coordinates in [4096, 8192) km), whose squared length sits
    so close to thr^2 that the reference's rounded sum and the fused form decide `< thr^2` differently.  Returns
    (ref_hit_only, fma_hit_only): two lists of per_kind offsets."""
    rng = np.random.default_rng(seed)
    q = 2.0 ** -40
    thr2 = thr * thr
    kinds = ([], [])
    while min(len(kinds[0]), len(kinds[1])) < per_kind:
        m = 200_000
        dx = np.round(thr * rng.uniform(0.3, 0.6, m) / q) * q
        dy = np.round(thr * rng.uniform(0.3, 0.6, m) / q) * q
        dz0 = np.round(np.sqrt(thr2 - dx * dx - dy * dy) / q) * q
        for k in range(-3, 4):
            dz = dz0 + k * q
            near = np.abs(((dx * dx + dy * dy) + dz * dz) - thr2) <= 2 * _ulp(thr2)
            for i in np.flatnonzero(near):
                d = (float(dx[i]), float(dy[i]), float(dz[i]))
                r, f = ref_d2_exact(*d) < thr2, fma_d2_exact(*d) < thr2
                if r != f and len(kinds[0 if r else 1]) < per_kind:
                    kinds[0 if r else 1].append(d)
    return kinds


def fma_flip_block(seed=5):
    """Pairs whose decision flips between the two d^2 forms, at thresholds 1, 10, 30 and 7.3 km (7.3 is no power-of-two
    fraction), at varied epochs of a 40-epoch block.  Returns a list of (pos_sm, thr, [(row, row, t, ref_hit)])."""
    out = []
    for j, thr in enumerate((1.0, 10.0, 30.0, 7.3)):
        ref_only, fma_only = fma_flip_offsets(thr, 3, seed + j)
        rng = np.random.default_rng(100 + j)
        nt = 40
        fix = [(d, True) for d in ref_only] + [(d, False) for d in fma_only]
        pos = _background(rng, 2 * len(fix) + 4, nt)
        planted = []
        for i, (d, ref_hit) in enumerate(fix):
            t = (7 * i + 3 * j) % nt
            s = rng.uniform(4200.0, 8000.0, 3) * rng.choice([-1.0, 1.0], 3)
            o = s - np.array(d)
            for c in range(3):  # the planted offset is exactly the difference the kernel forms
                assert Fraction(s[c]) - Fraction(o[c]) == Fraction(d[c])
            pos[2 * i, t], pos[2 * i + 1, t] = s, o
            planted.append((2 * i, 2 * i + 1, t, ref_hit))
        out.append((pos, thr, planted))
    return out


def cell_edge_block(thr, seed=1):
    """Cell-boundary cases on a 4-epoch block: coordinates exactly at k*thr; x with x * (1/thr) rounding up onto an
    integer; pairs straddling 0 on each axis (negative coordinates, -0.0); pairs one cell apart along all 26 neighbour
    offsets (the 13 forward ones and their negations), each pair in its own region of space."""
    rng = np.random.default_rng(seed)
    inv = 1.0 / thr
    rows = []

    def pair(a, b):
        rows.append(np.asarray(a, dtype=np.float64))
        rows.append(np.asarray(b, dtype=np.float64))

    # exactly on cell edges: at distance thr (no hit, strict <), and just inside it
    for k in (3, 17, -5):
        base = np.array([k * thr, 2 * k * thr, -k * thr])
        pair(base, base + np.array([thr, 0.0, 0.0]))
        a = base + 500.0
        pair(a, [a[0], a[1], np.nextafter(a[2] + thr, -np.inf)])   # one ulp of the coordinate inside thr
        pair(base - 700.0, base - 700.0 + np.array([0.0, thr * 0.5, thr * 0.5]))
    # x off a multiple of thr whose product with 1/thr still rounds onto an integer: the cell follows the product
    found = 0
    for k in range(100, 100000):
        for x in (np.nextafter(k * thr, -np.inf), np.nextafter(k * thr, np.inf)):
            prod = x * inv
            if found < 4 and prod == np.floor(prod) and (Fraction(x) / Fraction(thr)).denominator != 1:
                y = 3000.0 + found * 10 * thr
                pair([x, y, 100.0], [x - 0.95 * thr, y, 100.0])
                pair([x, y + 2000.0, 100.0], [x + 0.95 * thr, y + 2000.0, 100.0])
                found += 1
        if found == 4:
            break
    assert found == 4
    # straddling 0 on each axis, with -0.0 and negative coordinates
    for ax in range(3):
        for a, b in ((-0.0, 0.3 * thr), (-0.2 * thr, 0.0), (-0.4 * thr, 0.4 * thr), (-0.0, -0.7 * thr),
                     (-1e-300, 1e-300)):
            p, o = np.full(3, 9000.0 + 40 * thr * ax), np.full(3, 9000.0 + 40 * thr * ax)
            p[ax], o[ax] = a, b
            p[(ax + 1) % 3] = o[(ax + 1) % 3] = -3000.0 - 7 * thr * len(rows)
            pair(p, o)
    # one cell apart along every neighbour offset: close to the shared face / edge / corner, 0.1 thr per axis
    offsets = [(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1) if (dx, dy, dz) != (0, 0, 0)]
    for i, off in enumerate(offsets):
        cell = np.array([200 + 5 * i, -150 - 3 * i, 60 + 7 * i], dtype=np.float64)
        frac = np.array([0.95 if c > 0 else 0.05 if c < 0 else 0.5 for c in off])
        a = (cell + frac) * thr
        b = a + np.array(off, dtype=np.float64) * 0.1 * thr
        assert tuple(np.floor(b * inv) - np.floor(a * inv)) == off
        pair(a, b)
    nt = 4
    pos = _background(rng, len(rows), nt, 60000.0, 90000.0)
    pos[:, 1] = np.array(rows)
    pos[:, 3] = np.array(rows)[::-1]  # the same pairs with their row order reversed
    return pos


def _hash16(cx, cy, cz):
    m = np.uint64(2654435761)
    mask = np.uint64(0xFFFFFFFF)
    h = cx.astype(np.int64).astype(np.uint64) & mask
    h = (h * m) & mask
    h ^= cy.astype(np.int64).astype(np.uint64) & mask
    h = (h * m) & mask
    h ^= cz.astype(np.int64).astype(np.uint64) & mask
    h = (h * m) & mask
    return h & np.uint64(0xFFFF)


# offsets of coarse_search's 14 cells in its order: own cell, then the 13 lexicographically forward neighbours
FORWARD = [(n // 9 - 1, (n // 3) % 3 - 1, n % 3 - 1) for n in range(13, 27)]


def near_collisions(n_groups, seed):
    """(cell, o1, o2): two distinct cells cell + o1 and cell + o2 of one satellite's searched set (FORWARD) that share a
    bucket.  A partner in one of them is met once through each, so without the collision filter it is counted twice."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n_groups:
        cells = rng.integers(-800, 800, size=(300_000, 3))
        h = [_hash16(cells[:, 0] + o[0], cells[:, 1] + o[1], cells[:, 2] + o[2]) for o in FORWARD]
        for a in range(len(FORWARD)):
            for b in range(a + 1, len(FORWARD)):
                for k in np.flatnonzero(h[a] == h[b]):
                    if len(out) < n_groups:
                        out.append((cells[k], np.array(FORWARD[a]), np.array(FORWARD[b])))
    return out


def far_collisions(n_groups, seed):
    """(c1, c2): cells at least 2 apart that share a bucket, anywhere in space."""
    rng = np.random.default_rng(seed)
    cells = rng.integers(-800, 800, size=(400_000, 3))
    h = _hash16(cells[:, 0], cells[:, 1], cells[:, 2])
    order = np.argsort(h, kind="stable")
    hs = h[order]
    out = []
    for i in np.flatnonzero(hs[1:] == hs[:-1]):
        c1, c2 = cells[order[i]], cells[order[i + 1]]
        if np.max(np.abs(c1 - c2)) >= 2 and len(out) < n_groups:
            out.append((c1, c2))
    return out


def hash_collision_block(thr=10.0, seed=2):
    """Cells that share a bucket (spatial_hash & 0xffff).

    Near groups: two cells of one satellite's searched set share a bucket, and the satellite's partner (0.1 thr away)
    sits in one of them; the collision filter is what keeps that pair from being counted twice.  Far groups: cells at
    least 2 apart share a bucket, each with a cross-cell and a same-cell pair, so chains mix members of distant cells.
    Returns (pos, near) with near = [(row, partner_row, cell, o1, o2)]."""
    inv = 1.0 / thr
    rows, near = [], []
    for g, (cell, o1, o2) in enumerate(near_collisions(10, seed)):
        o = o1 if g % 2 == 0 else o2                  # the partner's cell: either member of the colliding pair
        frac = np.where(o > 0, 0.95, np.where(o < 0, 0.05, 0.5))
        a = (cell + frac) * thr
        b = a + (o if o.any() else np.array([1, 0, 0])) * 0.1 * thr
        assert np.array_equal(np.floor(a * inv), cell) and np.array_equal(np.floor(b * inv), cell + o)
        near.append((len(rows), len(rows) + 1, cell, o1, o2))
        rows += [a, b]
    for c1, c2 in far_collisions(12, seed):
        for c in (c1, c2):
            a = (c + np.array([0.5, 0.5, 0.95])) * thr
            rows.append(a)
            rows.append(a + np.array([0.0, 0.0, 0.1 * thr]))      # in the cell above: a cross-cell hit
            rows.append(a + np.array([0.0, 0.0, -0.8 * thr]))     # same cell, 0.8 thr away: a same-cell hit
    pos = np.array(rows)[:, None, :].repeat(2, axis=1)
    pos[:, 1] = pos[::-1, 0]
    return pos, near


def epoch_batch_block(nt, seed=3):
    """A block of nt epochs with hits planted at t = 0, 127, 128, 255, 256 and the last epoch (those that exist)."""
    rng = np.random.default_rng(seed + nt)
    pos = _background(rng, 30, nt, 7000.0, 7400.0)
    hits_at = sorted({t for t in (0, 127, 128, 255, 256, nt - 1) if t < nt})
    for i, t in enumerate(hits_at):
        a = rng.uniform(-5000.0, 5000.0, 3)
        pos[2 * i, t], pos[2 * i + 1, t] = a, a + rng.normal(size=3) * 0.5
    return pos, hits_at


def non_finite_block(thr=10.0):
    """Rows with NaN in y or z (x finite), rows with +-inf, masked rows, and a masked row in the same cell as a real
    hit.  Returns (pos, mask)."""
    base = np.array([1234.5, -2345.25, 3456.75])
    rows = [base, base + 1.0,                                         # a real hit
            [base[0] + 0.5, np.nan, base[2]],                         # NaN y next to it
            [base[0] - 0.5, base[1], np.nan],                         # NaN z
            [base[0], np.inf, base[2]],                               # +inf y
            [np.inf, base[1], base[2]],                               # +inf x: not listed
            [-np.inf, -np.inf, -np.inf],
            [np.nan, base[1], base[2]],                               # NaN x: not listed
            base + 0.25,                                              # masked, same cell as the real hit
            base + [0.0, 0.0, 2.0],                                   # another real hit partner
            [base[0] + 0.1, -np.inf, base[2]]]
    pos = np.array(rows, dtype=np.float64)[:, None, :].repeat(3, axis=1)
    pos[:, 2] = pos[::-1, 0]
    mask = np.ones(len(rows), dtype=np.uint8)
    mask[8] = 0
    mask[4] = 0
    return pos, mask


def tiny_threshold_block():
    """thr = 1e-6 km at GEO radius: |coordinate| / thr ~ 4e10, beyond the int range of a cell coordinate."""
    thr = 1e-6
    rng = np.random.default_rng(4)
    rows = []
    for sgn in (1.0, -1.0):
        for k in range(6):
            a = np.array([sgn * 42164.0, sgn * (3000.0 + 100.0 * k), sgn * 0.0])
            a = a + rng.uniform(-1, 1, 3) * 1e-3
            rows.append(a)
            rows.append(a + np.array([0.4e-6, 0.0, 0.0]))        # hit
            rows.append(a + np.array([0.0, 1.5e-6, 0.0]))        # miss
            rows.append(a + np.array([0.3e-6, 0.3e-6, 0.3e-6]))  # hit (with the first), not with the second
    pos = np.array(rows)[:, None, :].repeat(2, axis=1)
    pos[:, 1] = pos[::-1, 0]
    return pos, thr


def all_k4_cases():
    """(name, pos_sm, thr, mask) for every K4 block fixture except the fma flips."""
    cases = []
    for thr in (10.0, 7.3):
        pos = cell_edge_block(thr)
        mask = np.ones(pos.shape[0], dtype=np.uint8)
        mask[5::7] = 0
        cases += [(f"cell_edges_{thr}", pos, thr, None), (f"cell_edges_masked_{thr}", pos, thr, mask)]
    pos, _ = hash_collision_block()
    cases.append(("hash_collisions", pos, 10.0, None))
    for nt in (1, 127, 128, 129, 257):
        pos, _ = epoch_batch_block(nt)
        cases.append((f"epochs_{nt}", pos, 2.0, None))
    pos, mask = non_finite_block()
    cases += [("non_finite", pos, 10.0, mask), ("non_finite_unmasked", pos, 10.0, None)]
    pos, thr = tiny_threshold_block()
    cases.append(("tiny_threshold", pos, thr, None))
    return cases


# ---------------------------------------------------------------------------------------------- host emulation
@pytest.fixture(scope="module")
def emul_screen():
    return load_emul_screen()


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    return nvcc


def _compile_emul(so, includes):
    src = os.path.join(EMUL_DIR, "emul_screen.cu")
    subprocess.run([_nvcc(), "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                    "-Xcompiler", "-fPIC", "-shared", *["-I" + d for d in includes], "-o", so, src], check=True,
                   capture_output=True)
    return _load(so)


def load_emul_screen():
    """Build (when stale) and load tests/host_emul/emul_screen.cu."""
    _nvcc()
    so = os.path.join(EMUL_DIR, "libemul_screen.so")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = [os.path.join(EMUL_DIR, "emul_screen.cu")]
    deps += [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".hpp"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        return _compile_emul(so, [csrc])
    return _load(so)


def _load(so):
    L = C.CDLL(so)
    L.emul_coarse_screen.restype = C.c_uint64
    L.emul_coarse_screen.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_double, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_uint64]
    return L


def emul_coarse(L, pos_sm, thr, layout=0, valid_mask=None, max_results=100_000):
    """K4 on the CPU; the block is passed in `layout` (0: satellite-major, 1: time-major)."""
    ns, nt = pos_sm.shape[:2]
    blk = np.ascontiguousarray(pos_sm if layout == 0 else pos_sm.transpose(1, 0, 2), dtype=np.float64)
    pairs = np.zeros((max_results, 2), dtype=np.uint32)
    tidx = np.zeros(max_results, dtype=np.uint32)
    m = None if valid_mask is None else np.ascontiguousarray(valid_mask, dtype=np.uint8)
    k = L.emul_coarse_screen(blk.ctypes.data, ns, nt, layout, float(thr), m.ctypes.data if m is not None else None,
                             pairs.ctypes.data, tidx.ctypes.data, max_results)
    assert k <= max_results
    return sorted_hits(pairs[:k], tidx[:k])


def _lines(tles):
    n = len(tles)
    return (C.c_char_p * n)(*[t[0].encode() for t in tles]), (C.c_char_p * n)(*[t[1].encode() for t in tles])


def emul_track(L, tles, times, offsets, sat, lanes):
    a1, a2 = _lines(tles)
    out = np.zeros((len(times), 3))
    dp = C.POINTER(C.c_double)
    rc = L.emul_screen_track(a1, a2, len(tles), 1, np.ascontiguousarray(times).ctypes.data_as(dp), len(times),
                             np.ascontiguousarray(offsets).ctypes.data_as(dp), sat, lanes, out.ctypes.data_as(dp))
    assert rc == 0
    return out


def emul_k3(L, tles, times, offsets, target, thr):
    a1, a2 = _lines(tles)
    n = len(tles)
    d, ti = np.zeros(n), np.zeros(n, dtype=np.uint32)
    dp = C.POINTER(C.c_double)
    rc = L.emul_screen_conjunction(a1, a2, n, 1, np.ascontiguousarray(times).ctypes.data_as(dp), len(times),
                                   np.ascontiguousarray(offsets).ctypes.data_as(dp), target, C.c_double(thr),
                                   d.ctypes.data_as(dp), ti.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return d, ti


# ---------------------------------------------------------------------------------------------- K3 fixtures
def divergence_candidates(n=160):
    """Near-earth sets to pick a K3 target from (pick_divergent_target)."""
    from astroz_b200 import synth

    return synth.near_earth_catalog(n)


def screen_times(nt):
    return np.arange(nt, dtype=np.float64) * 1.0


def screen_offsets(tles):
    from oracle import oracle as orc

    return np.array([(REF_JD - orc.parse_tle(*t)["epochJd"]) * 1440.0 for t in tles])


def pick_divergent_target(L, cands, times):
    """The first candidate whose first cell differs between sgp4_cell<1> and K3's lane shape (host emulation)."""
    off = screen_offsets(cands)
    for s in range(len(cands)):
        one = emul_track(L, cands, times, off, s, 1)
        two = emul_track(L, cands, times, off, s, 2)
        if not np.array_equal(one[0], two[0]):
            return s, float(np.max(np.abs(one - two)))
    raise AssertionError("no candidate target whose first cell differs between the two lane shapes")


def with_duplicates(base, target_tle, slots):
    """base with target_tle written into the given rows."""
    tles = list(base)
    for r in slots:
        tles[r] = target_tle
    return tles


# ---------------------------------------------------------------------------------------------- tests
def test_fma_flip_fixtures_straddle_the_threshold():
    """Each planted pair's exact evaluations disagree: the reference's rounded sum and the fused form fall on opposite
    sides of thr^2.  A fixture that stops straddling fails here instead of passing silently on the device."""
    n_ref, n_fma = 0, 0
    for pos, thr, planted in fma_flip_block():
        thr2 = Fraction(thr * thr)
        for a, b, t, ref_hit in planted:
            d = tuple(float(v) for v in pos[a, t] - pos[b, t])
            r, f = ref_d2_exact(*d) < thr2, fma_d2_exact(*d) < thr2
            assert r != f and r == ref_hit
            n_ref += r
            n_fma += f
    assert n_ref >= 8 and n_fma >= 8


def test_brute_force_reference_on_flip_fixtures():
    """The brute-force reference decides the flips the reference's way (and so does the host emulation, which is
    uncontracted; the device run in test_gpu_screens.py is the one that can tell the two forms apart)."""
    for pos, thr, planted in fma_flip_block():
        pairs, ts = brute_force(pos, thr)
        got = {(int(a), int(b), int(t)) for (a, b), t in zip(pairs, ts)}
        for a, b, t, ref_hit in planted:
            assert ((a, b, t) in got) == ref_hit


@pytest.mark.parametrize("layout", [0, 1])
def test_k4_search_matches_brute_force_and_oracle(emul_screen, oracle, layout):
    for name, pos, thr, mask in all_k4_cases():
        masks = [mask] if mask is not None else [None, np.ones(pos.shape[0], dtype=np.uint8)]
        for m in masks:
            want = brute_force(pos, thr, m)
            got = emul_coarse(emul_screen, pos, thr, layout, m)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (name, m is None)
            ora = oracle.coarse_screen(pos, thr, valid_mask=m)
            assert np.array_equal(ora[0], want[0]) and np.array_equal(ora[1], want[1]), (name, m is None)


def test_hash_collision_fixture_needs_the_collision_filter(emul_screen, tmp_path):
    """The near collision groups bite: the two colliding cells are distinct members of the satellite's searched set,
    and the same search built without the collision filter counts each of those pairs twice, while the shipped
    search equals brute force."""
    pos, near = hash_collision_block()
    thr = 10.0
    for row, partner, cell, o1, o2 in near:
        assert not np.array_equal(o1, o2) and tuple(o1) in FORWARD and tuple(o2) in FORWARD
        c1, c2 = cell + o1, cell + o2
        assert _hash16(*[np.array([v]) for v in c1])[0] == _hash16(*[np.array([v]) for v in c2])[0]
        assert np.array_equal(np.floor(pos[row, 0] / thr), cell)
    want = brute_force(pos, thr)
    got = emul_coarse(emul_screen, pos, thr)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])

    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    text = open(os.path.join(csrc, "az_screen.cuh")).read()
    keep = "                continue;  // hash collision"
    assert text.count(keep) == 1
    (tmp_path / "az_screen.cuh").write_text(text.replace(keep, "                (void)0;  // hash collision"))
    unfiltered = _compile_emul(str(tmp_path / "libemul_screen_unfiltered.so"), [str(tmp_path), csrc])
    bad = emul_coarse(unfiltered, pos, thr)
    counts = {}
    for (a, b), t in zip(*bad):
        counts[(int(a), int(b), int(t))] = counts.get((int(a), int(b), int(t)), 0) + 1
    for row, partner, *_ in near:
        assert counts[(row, partner, 0)] == 2


def test_k4_fixtures_reach_their_cases(emul_screen):
    """The fixtures contain what they claim: hits at the epoch-batch seams, the tiny threshold beyond the int range,
    straddle pairs across 0, masked and non-finite rows kept out, and cell-edge pairs at exactly thr kept out."""
    for nt in (1, 127, 128, 129, 257):
        pos, hits_at = epoch_batch_block(nt)
        _, ts = brute_force(pos, 2.0)
        assert set(hits_at) <= set(ts.tolist())
    pos, thr = tiny_threshold_block()
    assert np.max(np.abs(pos)) / thr > 2.0 ** 31
    pairs, _ = brute_force(pos, thr)
    assert len(pairs) >= 24
    pos, mask = non_finite_block()
    pairs, ts = brute_force(pos, 10.0, mask)
    rows = set(pairs[ts < 2].ravel().tolist())   # epoch 2 holds the rows in reverse order
    assert {0, 1, 9} <= rows and not rows & {2, 3, 4, 5, 6, 7, 8, 10}
    pos = cell_edge_block(10.0)
    pairs, ts = brute_force(pos, 10.0)
    assert len(pairs) > 60 and (pos[:, 1] < 0).any() and np.signbit(pos[:, 1]).sum() > (pos[:, 1] < 0).sum()
    # a pair exactly thr apart on an axis is not a hit (strict <); the one just inside it is
    assert not ((pairs[:, 0] == 0) & (pairs[:, 1] == 1) & (ts == 1)).any()
    assert ((pairs[:, 0] == 2) & (pairs[:, 1] == 3) & (ts == 1)).any()


def test_k4_emulation_counts_past_max_results(emul_screen):
    pos = cell_edge_block(10.0)
    want = brute_force(pos, 10.0)
    n = len(want[1])
    got_pairs, got_t = emul_coarse(emul_screen, pos, 10.0, 0, None, max_results=100_000)
    assert len(got_t) == n
    ns, nt = pos.shape[:2]
    blk = np.ascontiguousarray(pos)
    m = n // 3
    pairs = np.full((m + 4, 2), 0xDEADBEEF, dtype=np.uint32)
    tidx = np.full(m + 4, 0xDEADBEEF, dtype=np.uint32)
    k = emul_screen.emul_coarse_screen(blk.ctypes.data, ns, nt, 0, 10.0, None, pairs.ctypes.data, tidx.ctypes.data, m)
    assert k == n
    assert (pairs[m:] == 0xDEADBEEF).all() and (tidx[m:] == 0xDEADBEEF).all()
    stored = {(int(a), int(b), int(t)) for (a, b), t in zip(pairs[:m], tidx[:m])}
    assert len(stored) == m and stored <= {(int(a), int(b), int(t)) for (a, b), t in zip(*want)}


def test_k3_duplicates_of_the_target_meet_it_at_zero(emul_screen, oracle):
    """Copies of the target (in its tile, in another tile, in the last, partial tile) come back at exactly 0.0 km and
    epoch 0, because the track and the screen evaluate the same lane shape.  The target is chosen so that its first cell
    differs between one cell per call and that shape: with the track on one lane, a copy would not meet it at epoch 0."""
    from astroz_b200 import synth

    times = screen_times(300)
    cands = divergence_candidates()
    tgt, gap = pick_divergent_target(emul_screen, cands, times)
    assert 0.0 < gap < 1e-9
    base = synth.near_earth_catalog(61, seed=77)
    target, copies = 2, [5, 30, 59]            # target in tile 0; copies in tile 0, tile 3 and the last tile (56..60)
    tles = with_duplicates(base, cands[tgt], [target] + copies)
    off = screen_offsets(tles)
    d, ti = emul_k3(emul_screen, tles, times, off, target, 25.0)
    assert (d[copies] == 0.0).all() and (ti[copies] == 0).all()
    do, tio = oracle.screen_constellation(tles, times, off, target, 25.0, REF_JD)
    assert (do[copies] == 0.0).all() and (tio[copies] == 0).all()
    others = np.setdiff1d(np.arange(len(tles)), copies + [target])
    assert np.max(np.abs(d[others] - do[others])) < 1e-6
    assert d[target] == 25.0 and ti[target] == 0
