"""The fp64 math primitives of az_math.cuh / az_device.cuh, each against a 40-digit mpmath reference at the accuracy its
own comment states, over the operand ranges the propagation cores feed it and at the edges where such code goes wrong.

The primitives run through a test-only probe (tests/device_probe/probe.cu) built from the product headers, in two
builds: the host loop tests/host_emul runs (fp32 seeds, host table) on any machine, and a small kernel on the device
(the MUFU seeds rcp.approx / rsqrt.approx, the __constant__ table) under the gpu mark.  The host and device builds differ
exactly in the seeds and the table, so the last test asserts that they agree to the stated bounds: what host emulation
can vouch for, and what it cannot (the seeds themselves).
"""
import ctypes as C
import math
import os
import shutil
import struct
import subprocess
from fractions import Fraction

import numpy as np
import pytest

mpmath = pytest.importorskip("mpmath")
mp = mpmath.mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_DIR = os.path.join(ROOT, "tests", "device_probe")
CSRC = os.path.join(ROOT, "astroz_b200", "csrc")

# tests/device_probe/probe.cu, enum ProbeOp
(RCP_SEED, RCP_FAST, RCP, DIV_NR, RSQRT_SEED, RSQRT_NR, RSQRT_NR1, SQRT, SQRT_NR1, SINCOS_FULL, SINCOS_QUARTER,
 SINCOS_TINY, SINCOS_MICRO, ROTATE_SMALL, ATAN2_SEED, ANGLE_OF_UNIT, RESONANCE_NODE, ABS_GT, ABS_LT, GE_ONE, HALF_OF,
 EXPO, FLOOR_AT, CLAMP_ABS) = range(24)

# Relative accuracy of the reciprocal / rsqrt seeds: the host's fp32 seeds ~2^-23, the device's MUFU seeds 1e-6
# (rcp.approx.ftz.f64 2^-20.0, rsqrt.approx.ftz.f64 2^-20.1 at most, measured on an H100).  One Newton step squares the
# seed's error for the reciprocal and leaves 3/2 of its square for 1/sqrt, always from below (az_math.cuh).
SEED_BOUND = {0: 2.0 ** -23, 1: 1e-6}
RCP1_BOUND = {d: b * b + 2.0 ** -53 for d, b in SEED_BOUND.items()}
RSQRT1_BOUND = {d: 1.5 * b * b + 2.0 ** -53 for d, b in SEED_BOUND.items()}
BUILDS = [pytest.param(0, id="host"), pytest.param(1, id="device", marks=pytest.mark.gpu)]


@pytest.fixture(scope="module")
def probe():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = os.path.join(PROBE_DIR, "libprobe.so")
    src = os.path.join(PROBE_DIR, "probe.cu")
    deps = [src] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".hpp", ".inc"))]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        # the product's own flags (astroz_b200/build.py): nvcc's default contraction (-fmad=true), like the library
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared", "-I" + CSRC, "-o", so, src],
                       check=True, capture_output=True)
    L = C.CDLL(so)
    dp = C.POINTER(C.c_double)
    L.probe_eval.argtypes = [C.c_int, dp, dp, dp, C.c_int, dp, dp, C.c_int]
    L.probe_eval.restype = C.c_int
    L.probe_constants.argtypes = [dp, C.c_int]

    def run(op, x, y=None, z=None, device=0):
        x = np.ascontiguousarray(x, dtype=np.float64)
        y = np.zeros_like(x) if y is None else np.ascontiguousarray(np.broadcast_to(y, x.shape), dtype=np.float64)
        z = np.zeros_like(x) if z is None else np.ascontiguousarray(np.broadcast_to(z, x.shape), dtype=np.float64)
        a = np.zeros_like(x)
        b = np.zeros_like(x)
        rc = L.probe_eval(op, x.ctypes.data_as(dp), y.ctypes.data_as(dp), z.ctypes.data_as(dp), len(x),
                          a.ctypes.data_as(dp), b.ctypes.data_as(dp), device)
        assert rc == 0, f"probe_eval(op {op}, device {device}) returned {rc}"
        return a, b

    k = np.zeros(12)
    L.probe_constants(k.ctypes.data_as(dp), 12)
    run.hi = dict(zip(("tiny", "quarter", "clamp", "emfloor", "micro", "linear"), (int(v) for v in k[:6])))
    run.value = dict(zip(("tiny", "quarter", "clamp", "emfloor", "micro", "linear"), k[6:].tolist()))
    return run


@pytest.fixture(autouse=True)
def _forty_digits():
    with mpmath.workdps(40):
        yield


# ---------------------------------------------------------------------------------------------- helpers
def _from_bits(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def largest_selected(hi):
    """The largest double a `!abs_gt(x, hi)` selector lets through: the threshold's high word, all-ones low word."""
    return _from_bits((hi << 32) | 0xFFFFFFFF)


def pow2_and_all_ones(k0, k1):
    """Exact powers of two and all-ones mantissas (the largest double below the next power) for exponents k0..k1."""
    k = np.arange(k0, k1 + 1, dtype=np.float64)
    return np.concatenate([2.0 ** k, (2.0 - 2.0 ** -52) * 2.0 ** k])


def abs_err(got, ref):
    """|got - ref| in 40 digits, per element, as float."""
    return np.array([float(abs(mp.mpf(float(g)) - r)) for g, r in zip(got, ref)])


def rel_err(got, ref):
    return np.array([float(abs((mp.mpf(float(g)) - r) / r)) for g, r in zip(got, ref)])


def ulp_err(got, ref):
    """|got - ref| in units of the spacing of doubles at ref."""
    return np.array([float(abs(mp.mpf(float(g)) - r)) / np.spacing(abs(float(r))) for g, r in zip(got, ref)])


def _rng(seed):
    return np.random.default_rng(seed)


# operand ranges the cores feed the primitives (az_device.cuh)
def rcp_operands():
    r = _rng(1)
    e = r.uniform(0.0, 0.999, 1500)
    return np.concatenate([
        1.0 - e * e,                            # 1 - e^2 (kepler_posvel prologue)
        r.uniform(0.03, 2.0, 1500),             # 1 - e cos E (Newton loop, a / r)
        1.0 + r.uniform(0.0, 1.0, 500),         # 1 + betal
        r.uniform(0.2, 1.0, 300),               # sin of the perturbed inclination (SDP4 phs)
        np.geomspace(1.5e-12, 2.0, 300),        # 1 + cos i down to xlcof's guard (retrograde equatorial)
        pow2_and_all_ones(-40, 40),
        np.array([1.5e-12, 0.002, 0.03, 1.0, 2.0, 3.0, 0.1, 1.0 / 3.0]),
    ])


def rsqrt_operands():
    r = _rng(2)
    return np.concatenate([
        r.uniform(0.9, 12.0, 1500),             # am, Earth radii
        np.geomspace(1e-6, 1.0, 1500),          # omel2 = 1 - e_L^2
        r.uniform(0.04, 1.0, 300),              # alfdp^2 + betdp^2 (Lyddane)
        np.geomspace(1e6, 5e9, 500),            # p^2, x^2 + y^2 + z^2 in km^2 (geodetic epilogue)
        pow2_and_all_ones(-40, 40),
        np.array([1e-6, 0.9, 1.0, 2.0, 3.0, 4.0, 12.0, 0.5]),
    ])


# ---------------------------------------------------------------------------------------------- reciprocals
@pytest.mark.parametrize("device", BUILDS)
def test_reciprocals(probe, device):
    """rcp_fast to the seed's error squared (one Newton step; 2^-46 on the host, 1e-12 on the device), rcp <= 1 ulp,
    div_nr <= 1 ulp for the quotients the cores form."""
    x = rcp_operands()
    ref = [1 / mp.mpf(float(v)) for v in x]
    fast, _ = probe(RCP_FAST, x, device=device)
    assert rel_err(fast, ref).max() <= RCP1_BOUND[device]
    full, _ = probe(RCP, x, device=device)
    assert ulp_err(full, ref).max() <= 1.0
    a = _rng(3).uniform(-3.0, 3.0, len(x))
    q, _ = probe(DIV_NR, a, x, device=device)
    qref = [mp.mpf(float(u)) / mp.mpf(float(v)) for u, v in zip(a, x)]
    assert ulp_err(q, qref).max() <= 1.0


@pytest.mark.parametrize("device", BUILDS)
def test_reciprocal_square_roots(probe, device):
    """rsqrt_nr <= 1 ulp, rsqrt_nr1 3/2 the seed's error squared (1.5 * 2^-46 host, 1.5e-12 device), sqrt_ and the Heron-corrected sqrt_from_rsqrt(x, rsqrt_nr1(x)) <= 1 ulp."""
    x = rsqrt_operands()
    ref = [1 / mpmath.sqrt(mp.mpf(float(v))) for v in x]
    sref = [mpmath.sqrt(mp.mpf(float(v))) for v in x]
    y, _ = probe(RSQRT_NR, x, device=device)
    assert ulp_err(y, ref).max() <= 1.0
    y1, _ = probe(RSQRT_NR1, x, device=device)
    assert rel_err(y1, ref).max() <= RSQRT1_BOUND[device]
    s, _ = probe(SQRT, x, device=device)
    assert ulp_err(s, sref).max() <= 1.0
    s1, _ = probe(SQRT_NR1, x, device=device)
    assert ulp_err(s1, sref).max() <= 1.0


# ---------------------------------------------------------------------------------------------- sin / cos
def _sincos_ref(x):
    return [mpmath.sin(mp.mpf(float(v))) for v in x], [mpmath.cos(mp.mpf(float(v))) for v in x]


@pytest.mark.parametrize("device", BUILDS)
def test_sincos_full(probe, device):
    """< 2e-16 absolute: dense sweep, the 1024-point lattice's nodes and midpoints (the remainder at its largest), one
    bit either side of a midpoint, and arguments up to |x| = 1e6."""
    r = _rng(4)
    h = 2.0 * np.pi / 1024.0
    k = np.arange(-1100, 1100, 3)
    mid = (k + 0.5) * h
    x = np.concatenate([np.linspace(-20.0, 20.0, 1601), k * h, mid, np.nextafter(mid, np.inf),
                        np.nextafter(mid, -np.inf), r.uniform(-1e3, 1e3, 600), r.uniform(-1e5, 1e5, 600),
                        r.uniform(-1e6, 1e6, 600), np.array([1e6, -1e6, 999999.5, 0.0, -0.0, 5e-324, 1e-300])])
    s, c = probe(SINCOS_FULL, x, device=device)
    rs, rc = _sincos_ref(x)
    assert abs_err(s, rs).max() < 2e-16
    assert abs_err(c, rc).max() < 2e-16


def _series_args(xmax, seed):
    r = _rng(seed)
    edge = np.array([xmax, -xmax, np.nextafter(xmax, 0.0), xmax * 0.5, 0.0, -0.0, 1e-300, 5e-324])
    return np.concatenate([r.uniform(-xmax, xmax, 1500), np.geomspace(1e-12, xmax, 300), edge])


@pytest.mark.parametrize("device", BUILDS)
def test_sincos_series_at_their_selected_ranges(probe, device):
    """Each series up to the largest argument its high-word selector lets through (the threshold's high word with an
    all-ones low word: 2^-20 relative above the nominal limit), at the bound its comment states.  The sine bounds are
    the whole error; the cosines, near 1, carry the rounding of their last FMA on top of the series' error (half an
    ulp of 1, 1.1e-16), which the bound adds explicitly."""
    half_ulp_one = 2.0 ** -53
    # micro, |x| <= 2e-3: the 21-bit -1/6 moves sin by 4e-8 |x|^3 (the omitted x^5 / 120 only cancels part of it),
    # < 3e-16 in all; cos moved by x^4 1e-8 <= 2e-19
    x = _series_args(largest_selected(probe.hi["micro"]), 5)
    assert x.max() > 2e-3
    s, c = probe(SINCOS_MICRO, x, device=device)
    rs, rc = _sincos_ref(x)
    es = abs_err(s, rs)
    assert np.all(es <= 4e-8 * np.abs(x) ** 3 + 0.5 * np.spacing(np.abs(s))) and es.max() < 3e-16
    assert abs_err(c, rc).max() <= 2e-19 + half_ulp_one
    # tiny, |x| <= 0.05: < 1e-17 (sin), and the cosine's series error as small beneath its rounding
    x = _series_args(largest_selected(probe.hi["tiny"]), 6)
    assert x.max() > 0.05
    s, c = probe(SINCOS_TINY, x, device=device)
    rs, rc = _sincos_ref(x)
    assert abs_err(s, rs).max() < 1e-17
    assert abs_err(c, rc).max() < 1e-17 + half_ulp_one
    # quarter, |x| <= 0.78 as selected for the drag angle (and pi/4 as documented): the fitted kernels' 3.4e-17 /
    # 8.4e-17 plus rounding, inside sincos_full's 2e-16
    x = np.concatenate([_series_args(largest_selected(probe.hi["quarter"]), 7), [np.pi / 4, -np.pi / 4]])
    s, c = probe(SINCOS_QUARTER, x, device=device)
    rs, rc = _sincos_ref(x)
    assert abs_err(s, rs).max() < 2e-16
    assert abs_err(c, rc).max() < 2e-16


@pytest.mark.parametrize("device", BUILDS)
def test_rotate_small_both_branches(probe, device):
    """rotate_small_n<1>: the micro rotation for |d| up to its selector's limit, and the cold general branch (sincos_full)
    above it, which only this probe reaches.  Against the exact rotation of the given unit vector."""
    r = _rng(8)
    lim = largest_selected(probe.hi["micro"])
    d = np.concatenate([r.uniform(-lim, lim, 800), [lim, -lim, np.nextafter(lim, np.inf), -np.nextafter(lim, np.inf)],
                        r.uniform(-3.0, 3.0, 800), np.geomspace(2.1e-3, 10.0, 200)])
    a = r.uniform(-np.pi, np.pi, len(d))
    s0 = np.array([float(mpmath.sin(mp.mpf(float(v)))) for v in a])
    c0 = np.array([float(mpmath.cos(mp.mpf(float(v)))) for v in a])
    s, c = probe(ROTATE_SMALL, s0, c0, d, device=device)
    rs = [mp.mpf(float(p)) * mpmath.cos(mp.mpf(float(q))) + mp.mpf(float(w)) * mpmath.sin(mp.mpf(float(q)))
          for p, w, q in zip(s0, c0, d)]
    rc = [mp.mpf(float(w)) * mpmath.cos(mp.mpf(float(q))) - mp.mpf(float(p)) * mpmath.sin(mp.mpf(float(q)))
          for p, w, q in zip(s0, c0, d)]
    small = np.abs(d) <= lim
    # micro: the series' 3e-16 |d| plus the rotation's two roundings (ulp-sized); general: sincos_full's 2e-16 plus
    # the same roundings
    es, ec = abs_err(s, rs), abs_err(c, rc)
    assert np.all(es[small] <= 3e-16 * np.abs(d[small]) + 2.3e-16)
    assert np.all(ec[small] <= 3e-16 * np.abs(d[small]) + 2.3e-16)
    assert es[~small].max() < 4.3e-16 and ec[~small].max() < 4.3e-16


@pytest.mark.parametrize("device", BUILDS)
def test_angle_of_unit(probe, device):
    """atan2_seed within 2e-5 rad, and angle_of_unit (the seed snapped to the k / 128 lattice, the table, the three-term
    arcsine) equal to atan2 of the given pair to 3e-16, lattice points and midpoints included."""
    k = np.arange(-402, 403)
    ang = np.concatenate([k / 128.0, (k + 0.5) / 128.0, (k + 0.4999) / 128.0, np.linspace(-np.pi, np.pi, 3001),
                          [np.pi, -np.pi, np.nextafter(np.pi, 0.0)]])
    ang = ang[(ang >= -np.pi) & (ang <= np.pi)]
    s = np.array([float(mpmath.sin(mp.mpf(float(v)))) for v in ang])
    c = np.array([float(mpmath.cos(mp.mpf(float(v)))) for v in ang])
    ref = [mpmath.atan2(mp.mpf(float(p)), mp.mpf(float(q))) for p, q in zip(s, c)]
    seed, _ = probe(ATAN2_SEED, s, c, device=device)
    assert abs_err(seed, ref).max() < 2e-5
    got, _ = probe(ANGLE_OF_UNIT, s, c, device=device)
    assert abs_err(got, ref).max() < 3e-16


# ---------------------------------------------------------------------------------------------- resonance lattice
@pytest.mark.parametrize("device", BUILDS)
def test_resonance_node_exact(probe, device):
    """resonance_node(t) is the number of whole 720-minute steps the reference's `while |t - atime| >= 720` loop takes:
    floor(|t| / 720) in exact arithmetic, at every node k 720 and one ulp either side, k up to 30 000, both signs."""
    k = np.arange(0, 30001, dtype=np.float64)
    node = k * 720.0
    t = np.concatenate([node, np.nextafter(node, np.inf), np.nextafter(node, -np.inf)])
    t = np.concatenate([t, -t, _rng(9).uniform(-2.2e7, 2.2e7, 5000)])
    got, _ = probe(RESONANCE_NODE, t, device=device)
    want = np.array([int(abs(Fraction(float(v))) // 720) for v in t], dtype=np.float64)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(float(t[i]), got[i], want[i]) for i in bad[:5]]


# ---------------------------------------------------------------------------------------------- bit predicates
NAN_POS = _from_bits(0x7FF8000000000000)
NAN_NEG = _from_bits(0xFFF8000000000000)
SUB = 5e-324                       # smallest subnormal
SUB_MAX = _from_bits(0x000FFFFFFFFFFFFF)
INF = math.inf


@pytest.mark.parametrize("device", BUILDS)
def test_bit_predicates_special_values(probe, device):
    """The high-word predicates on +-0, subnormals, +-inf and both signs of NaN.  The expected values are what the bit
    tests compute, listed here so a change to any of them is seen: a NaN whose sign bit is clear compares as larger than
    any limit and as >= 1 (the device's canonical NaN, 0x7fffffff..., is such a NaN); a NaN with the sign bit set is
    "negative" to the signed tests (ge_one false, floor_at returns the floor)."""
    vals = np.array([0.0, -0.0, SUB, -SUB, SUB_MAX, INF, -INF, NAN_POS, NAN_NEG])
    hi = probe.hi["micro"]
    a, _ = probe(ABS_GT, vals, float(hi), device=device)
    assert a.tolist() == [0, 0, 0, 0, 0, 1, 1, 1, 1]
    a, _ = probe(ABS_LT, vals, float(hi), device=device)
    assert a.tolist() == [1, 1, 1, 1, 1, 0, 0, 0, 0]
    a, _ = probe(GE_ONE, vals, device=device)
    assert a.tolist() == [0, 0, 0, 0, 0, 1, 0, 1, 0]
    a, _ = probe(EXPO, vals, device=device)
    assert a.tolist() == [0, 0, 0, 0, 0, 2047, 2047, 2047, 2047]
    fl = probe.value["emfloor"]
    a, _ = probe(FLOOR_AT, vals, float(probe.hi["emfloor"]), fl, device=device)
    want = [fl, fl, fl, fl, fl, INF, fl, None, fl]
    assert [_bits(v) for i, v in enumerate(a) if i != 7] == [_bits(w) for i, w in enumerate(want) if i != 7]
    assert math.isnan(a[7])
    cl = probe.value["clamp"]
    a, _ = probe(CLAMP_ABS, vals, float(probe.hi["clamp"]), cl, device=device)
    assert [_bits(v) for v in a] == [_bits(w) for w in [0.0, -0.0, SUB, -SUB, SUB_MAX, cl, -cl, cl, -cl]]
    # half_of is x / 2 for a normal x away from underflow only; at the special values it is an exponent-field wrap
    a, _ = probe(HALF_OF, np.array([0.0, -0.0, INF, -INF, NAN_POS]), device=device)
    assert [_bits(v) for v in a] == [0xFFF0000000000000, 0x7FF0000000000000, 0x7FE0000000000000,
                                     0xFFE0000000000000, 0x7FE8000000000000]


@pytest.mark.parametrize("device", BUILDS)
def test_bit_predicates_at_their_thresholds(probe, device):
    """Each selector threshold: the largest double it lets through and the next one up, both signs; the nominal value
    it stands for lies within 2^-20 relative of the first, and every series keeps its bound there (tested above)."""
    for name, hi in probe.hi.items():
        top = largest_selected(hi)
        nxt = np.nextafter(top, np.inf)
        assert abs(top / probe.value[name] - 1.0) < 2.0 ** -20, name
        v = np.array([top, -top, nxt, -nxt, np.nextafter(_from_bits(hi << 32), -np.inf)])
        gt, _ = probe(ABS_GT, v, float(hi), device=device)
        assert gt.tolist() == [0, 0, 1, 1, 0], name
        lt, _ = probe(ABS_LT, v, float(hi), device=device)
        assert lt.tolist() == [0, 0, 0, 0, 1], name
    # ge_one: exactly 1.0 and the largest double below it, both signs
    v = np.array([1.0, np.nextafter(1.0, 0.0), -1.0, 2.0, 1e300])
    a, _ = probe(GE_ONE, v, device=device)
    assert a.tolist() == [1, 0, 0, 1, 1]
    # floor_at: the floor itself and its neighbours, negative values (sign bit set: compare low)
    fl, hfl = probe.value["emfloor"], probe.hi["emfloor"]
    v = np.array([fl, np.nextafter(fl, 0.0), largest_selected(hfl), np.nextafter(largest_selected(hfl), np.inf),
                  -0.5, 0.3, np.nextafter(_from_bits(hfl << 32), 0.0)])
    a, _ = probe(FLOOR_AT, v, float(hfl), fl, device=device)
    # (one ulp below the floor shares its high word and is kept: the 2^-20 slack of every high-word test)
    assert a.tolist() == [fl, v[1], largest_selected(hfl), v[3], fl, 0.3, fl]
    # clamp_abs: +-0.95 and above
    cl, hcl = probe.value["clamp"], probe.hi["clamp"]
    v = np.array([0.5, -0.5, largest_selected(hcl), -largest_selected(hcl), np.nextafter(largest_selected(hcl), 2.0),
                  -3.0, 12.0])
    a, _ = probe(CLAMP_ABS, v, float(hcl), cl, device=device)
    assert a.tolist() == [0.5, -0.5, largest_selected(hcl), -largest_selected(hcl), cl, -cl, cl]


@pytest.mark.parametrize("device", BUILDS)
def test_half_of_and_expo_on_mantissa_edges(probe, device):
    """half_of(x) == x / 2 exactly and expo(x) is the biased exponent for powers of two and all-ones mantissas over the
    whole normal range above the smallest normal's double (the operands are O(1) reciprocal square roots)."""
    x = pow2_and_all_ones(-1021, 1023)
    x = np.concatenate([x, -x, rsqrt_operands()])
    h, _ = probe(HALF_OF, x, device=device)
    assert np.array_equal(h, x / 2.0)
    e, _ = probe(EXPO, x, device=device)
    assert np.array_equal(e, np.frexp(x)[1] + 1022.0)


# ---------------------------------------------------------------------------------------------- seeds, host vs device
@pytest.mark.gpu
def test_host_and_device_builds_agree(probe):
    """The MUFU seeds (device) and the fp32 seeds (host) differ, and so do the one-Newton-step results built on them:
    host emulation cannot vouch for those to better than the device's bound.  Both seeds are asserted at their bounds;
    past the seeds the builds agree to the device's stated bound (the Newton steps never overshoot, so the two errors
    share a sign), to 1 ulp where two Newton steps are taken, and the table paths bit for bit."""
    x = np.concatenate([rcp_operands(), rsqrt_operands()])
    for op, ref in ((RCP_SEED, lambda v: 1 / mp.mpf(float(v))), (RSQRT_SEED, lambda v: 1 / mpmath.sqrt(mp.mpf(float(v))))):
        r = [ref(v) for v in x]
        for dev in (0, 1):
            y, _ = probe(op, x, device=dev)
            assert rel_err(y, r).max() < SEED_BOUND[dev], (op, dev)
    for op, bound in ((RCP_FAST, RCP1_BOUND[1]), (RSQRT_NR1, RSQRT1_BOUND[1])):
        yh, _ = probe(op, x)
        yd, _ = probe(op, x, device=1)
        assert np.max(np.abs(yh - yd) / np.abs(yh)) <= bound
    for op in (RCP, RSQRT_NR, SQRT, SQRT_NR1):
        yh, _ = probe(op, x)
        yd, _ = probe(op, x, device=1)
        assert np.all(np.abs(yh - yd) <= np.spacing(np.abs(yh)))
    # everything that involves no seed is the same arithmetic on the same constants: bit-identical
    r = _rng(10)
    ang = np.concatenate([r.uniform(-1e6, 1e6, 2000), r.uniform(-0.8, 0.8, 2000)])
    for op in (SINCOS_FULL, SINCOS_QUARTER, SINCOS_TINY, SINCOS_MICRO):
        sh, ch = probe(op, ang)
        sd, cd = probe(op, ang, device=1)
        assert np.array_equal(sh, sd) and np.array_equal(ch, cd), op
    # angle_of_unit: the fp32 seed divides differently (__fdividef), so near a lattice midpoint the builds may snap to
    # neighbouring nodes; each is within 3e-16 of atan2, so they agree to twice that
    s, c = np.sin(ang), np.cos(ang)
    ah, _ = probe(ANGLE_OF_UNIT, s, c)
    ad, _ = probe(ANGLE_OF_UNIT, s, c, device=1)
    assert np.max(np.abs(ah - ad)) < 6e-16
