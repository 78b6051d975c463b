"""The per-state cores of K7 (astroz_b200/csrc/az_numerical.cuh) run on the CPU by the test-only harness
tests/host_emul/emul_numerical.cu, against the scalar restatement (tests/numerical_oracle), plus the C ABI's argument
checks, which run before any device is touched.  The device run is in tests/test_gpu_numerical.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import numerical_oracle as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "host_emul")
MU, R_EQ, J2 = 398600.5, 6378.137, 0.00108262998905


@pytest.fixture(scope="module")
def emul():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = os.path.join(EMUL_DIR, "libemul_numerical.so")
    src = os.path.join(EMUL_DIR, "emul_numerical.cu")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("az_numerical.cuh", "az_math.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-I" + csrc, "-o", so, src], check=True,
                       capture_output=True)
    return C.CDLL(so)


def _steps(t0, duration, dt):
    t, out = t0, []
    while t < t0 + duration:
        out.append(min(dt, t0 + duration - t))
        t += out[-1]
    return np.array(out)


def run_emul(L, states, t0, duration, dt, *, j2=None, r_eq=None, drag=None, integrator="dp87", rtol=1e-9, atol=1e-12):
    states = np.ascontiguousarray(np.atleast_2d(states), dtype=np.float64)
    n = len(states)
    steps = _steps(t0, duration, dt)
    K = len(steps)
    forces = (1 if j2 is not None else 0) | (2 if drag is not None else 0)
    par = np.array([MU, j2 or 0.0, r_eq or 0.0, rtol, atol])
    d = [np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (n,))) for x in drag] if drag else [None] * 3
    out = np.zeros((n, K + 1, 6))
    st = np.zeros(n, dtype=np.uint8)
    cnt = np.zeros((n, 2), dtype=np.uint64)
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    assert L.emul_numerical(p(states), n, p(steps), K, C.c_double(dt), p(par), forces, *map(p, d),
                            0 if integrator == "rk4" else 1, p(out), p(st), p(cnt)) == 0
    return out, st, cnt


def fixtures():
    """LEO, SSO, a 150 km perigee, GEO, Molniya, a hyperbola, a state at the centre (stopped under DP87) and a circular
    orbit at 80 km, which under drag crawls down through the atmosphere on steps its stiff drag term keeps short (hundreds
    of accepted and some rejected steps per hour, where a LEO state takes one step per minute)."""
    def kep(a, e, inc, M):
        E = M
        for _ in range(60):
            E -= (E - e * math.sin(E) - M) / (1 - e * math.cos(E))
        p = a * (1 - e * e)
        c, s = (math.cos(E) - e) / (1 - e * math.cos(E)), math.sqrt(1 - e * e) * math.sin(E) / (1 - e * math.cos(E))
        r, h = p / (1 + e * c), math.sqrt(MU * p)
        x, y, vx, vy = r * c, r * s, -MU / h * s, MU / h * (e + c)
        return [x, y * math.cos(inc), y * math.sin(inc), vx, vy * math.cos(inc), vy * math.sin(inc)]
    return np.array([kep(6778, 0.001, 0.9, 0.1), kep(7078, 0.0012, 1.71, 2.0), kep(R_EQ + 900, 1 - (R_EQ + 150) /
                     (R_EQ + 900), 0.6, -0.4), kep(42164, 0.0002, 0.001, 1.0), kep(26600, 0.72, 1.1, 0.2),
                     [7000.0, 0, 0, 0, 12.0, 1.0], [0.0, 0, 0, 0, 0, 0], kep(R_EQ + 80, 0.0, 0.5, 0.0)])


def test_tableau_is_the_oracles_and_its_zero_pattern_holds(emul):
    c, a, b8, b7 = np.zeros(13), np.zeros((13, 12)), np.zeros(13), np.zeros(13)
    nz = np.zeros((13, 14), dtype=np.uint8)
    p = lambda x: C.c_void_p(x.ctypes.data)  # noqa: E731
    emul.emul_numerical_tableau(p(c), p(a), p(b8), p(b7), p(nz))
    oc, oa, ob8, ob7 = N.tableau()
    for mine, theirs in ((c, oc), (a, oa), (b8, ob8), (b7, ob7)):
        assert np.array_equal(mine.view(np.uint64), theirs.view(np.uint64))
    assert np.array_equal(nz[:, :12].astype(bool), a != 0)
    assert np.array_equal(nz[:, 12].astype(bool), b8 != 0) and np.array_equal(nz[:, 13].astype(bool), b7 != 0)


@pytest.mark.parametrize("forces", ["none", "j2", "drag", "j2drag"])
def test_rk4_cores_equal_the_oracle(emul, forces):
    """Same operations in the same order, no contraction: two-body and J2 are bit-identical; with drag only exp may
    differ (glibc on both sides here, so the host build is bit-identical too).  The state at the centre goes to NaN: its
    status is non-finite on both sides."""
    kw = {"j2": J2 if "j2" in forces else None, "r_eq": R_EQ if forces != "none" else None}
    y = fixtures()
    drag = (2.2, np.linspace(1, 20, len(y)), 200.0) if "drag" in forces else None
    out, st, cnt = run_emul(emul, y, 0.0, 7200.0, 30.0, drag=drag, integrator="rk4", **kw)
    dk = dict(drag_cd=drag[0], drag_area=drag[1], drag_mass=drag[2]) if drag else {}
    _, ref, rst, rcnt = N.propagate(y, 0.0, 7200.0, 30.0, MU, integrator="rk4", **kw, **dk)
    assert np.array_equal(st, rst) and np.array_equal(cnt, rcnt) and st[6] == 3
    assert np.array_equal(out, ref, equal_nan=True)


STIFF = 7   # fixtures() row of the stiff crawl


@pytest.mark.parametrize("forces", ["none", "j2", "drag", "j2drag"])
def test_dp87_cores_match_the_oracle(emul, forces):
    """K7's operations are the reference's except the step factor errNorm^(-1/8): three square roots in K7, pow in the
    reference (<= 1 ulp apart).  With the restatement forming that factor as K7 does, the host build of the cores is
    bit-identical to it, steps, status and states alike (host exp is glibc's on both sides).  Against the reference's pow
    the states agree to 1e-6 km / 1e-9 km/s relative to the orbit's scale, and the step counts are equal wherever no
    error norm falls within rounding of 1.0.  The stiff crawl under drag is the exception: its error norm hovers around
    1.0 for thousands of attempts, so some accept / reject decisions flip and the counts differ by a fraction of a
    percent (the bound is 1 %), while each flip is a decision on an errNorm of 1.0 to the last bits."""
    kw = {"j2": J2 if "j2" in forces else None, "r_eq": R_EQ if forces != "none" else None}
    y = fixtures()
    drag = (2.2, np.linspace(1, 20, len(y)), 200.0) if "drag" in forces else None
    out, st, cnt = run_emul(emul, y, 0.0, 21600.0, 60.0, drag=drag, **kw)
    dk = dict(drag_cd=drag[0], drag_area=drag[1], drag_mass=drag[2]) if drag else {}
    _, same, sst, scnt = N.propagate(y, 0.0, 21600.0, 60.0, MU, k7_step_factor=True, **kw, **dk)
    assert np.array_equal(st, sst) and np.array_equal(cnt, scnt) and np.array_equal(out, same)
    _, ref, rst, rcnt = N.propagate(y, 0.0, 21600.0, 60.0, MU, **kw, **dk)
    assert np.array_equal(st, rst) and st[6] == 1
    calm = np.arange(len(y)) != STIFF if drag else np.ones(len(y), dtype=bool)
    assert np.array_equal(cnt[calm], rcnt[calm])
    if drag:
        assert cnt[STIFF, 0] > 50 * cnt[0, 0] and cnt[STIFF, 1] > 0   # the stiff crawl really is one
        assert np.all(np.abs(cnt[STIFF].astype(float) - rcnt[STIFF]) <= 0.01 * rcnt[STIFF].sum())
    scale = np.maximum(1.0, np.abs(ref[..., :3]).max(axis=(1, 2)) / 7000.0)[:, None, None]
    assert np.max(np.abs(out[calm][..., :3] - ref[calm][..., :3]) / scale[calm]) < 1e-6
    assert np.max(np.abs(out[calm][..., 3:] - ref[calm][..., 3:]) / scale[calm]) < 1e-9


def test_substep_limit_matches_the_oracle(emul):
    """One interval of 1e6 s at rtol 1e-14 hits the 10,000-substep cap; the next interval continues from where the cap
    left the state, with the step size the capped interval ended on.  At rtol 1e-14 the error norm sits near 1.0 on
    most attempts, so against the reference's pow the counts flip by a fraction of a percent (and a capped sample then lies
    at a different time, so its position is not comparable); with K7's step factor the restatement is bit-identical."""
    y = np.array([[7000.0, 0, 0, 0, 7.5, 0], [6778.0, 0, 0, 0, 7.67, 0.1]])
    out, st, cnt = run_emul(emul, y, 0.0, 1.2e6, 1e6, rtol=1e-14, atol=1e-14)
    _, same, sst, scnt = N.propagate(y, 0.0, 1.2e6, 1e6, MU, rtol=1e-14, atol=1e-14, k7_step_factor=True)
    assert np.array_equal(st, sst) and (st == 2).all() and (cnt[:, 0] > 10000).all()
    assert np.array_equal(cnt, scnt) and np.array_equal(out, same)
    _, ref, rst, rcnt = N.propagate(y, 0.0, 1.2e6, 1e6, MU, rtol=1e-14, atol=1e-14)
    assert np.array_equal(st, rst)
    assert np.all(np.abs(cnt.astype(float) - rcnt) <= 0.01 * rcnt.sum(axis=1, keepdims=True))


def test_cores_are_batch_independent(emul):
    y = fixtures()
    out, st, cnt = run_emul(emul, y, 0.0, 7200.0, 60.0, j2=J2, r_eq=R_EQ)
    perm = np.array([3, 1, 1, 6, 0, 5, 2, 4, 3, 7])
    o2, s2, c2 = run_emul(emul, y[perm], 0.0, 7200.0, 60.0, j2=J2, r_eq=R_EQ)
    assert np.array_equal(o2, out[perm]) and np.array_equal(s2, st[perm]) and np.array_equal(c2, cnt[perm])


def test_cabi_refuses_bad_arguments_and_writes_nothing():
    """The argument checks run before any device is touched, so they hold on a CPU box too."""
    from astroz_b200._lib import lib

    L = lib()
    y = np.zeros((1, 6))
    out = np.full((1, 20, 6), 7.0)
    st = np.full(1, 9, dtype=np.uint8)
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    d = lambda x: C.pointer(C.c_double(x))  # noqa: E731
    dragv = np.ones(1)
    cases = [  # (t0, duration, dt, mu, forces, j2, r_eq, drag, integrator, rtol, atol, device)
        (0, 100, 0.0, MU, 0, None, None, None, 1, 1e-9, 1e-12, 0),
        (0, 100, -1.0, MU, 0, None, None, None, 1, 1e-9, 1e-12, 0),
        (0, math.inf, 10, MU, 0, None, None, None, 1, 1e-9, 1e-12, 0),
        (math.nan, 100, 10, MU, 0, None, None, None, 1, 1e-9, 1e-12, 0),
        (0, 100, 10, math.nan, 0, None, None, None, 1, 1e-9, 1e-12, 0),
        (0, 100, 10, MU, 1, d(J2), None, None, 1, 1e-9, 1e-12, 0),
        (0, 100, 10, MU, 1, None, d(R_EQ), None, 1, 1e-9, 1e-12, 0),
        (0, 100, 10, MU, 2, None, d(R_EQ), None, 1, 1e-9, 1e-12, 0),
        (0, 100, 10, MU, 2, None, None, dragv, 1, 1e-9, 1e-12, 0),
        (0, 100, 10, MU, 4, None, d(R_EQ), None, 1, 1e-9, 1e-12, 0),
        (0, 100, 10, MU, 0, None, None, None, 2, 1e-9, 1e-12, 0),
        (0, 100, 10, MU, 0, None, None, None, 1, math.inf, 1e-12, 0),
        (1e17, 1000, 1.0, MU, 0, None, None, None, 1, 1e-9, 1e-12, 0),   # t + step == t: the loop never ends
        (0, 1e12, 1e-3, MU, 0, None, None, None, 1, 1e-9, 1e-12, 0),  # 1e15 steps
        (0, 100, 10, MU, 0, None, None, None, 1, 1e-9, 1e-12, -1),
    ]
    for t0, dur, dt, mu, forces, j2, req, drag, integ, rtol, atol, dev in cases:
        dp = [p(drag)] * 3 if drag is not None else [None] * 3
        rc = L.astroz_cuda_propagate_numerical(p(y), 1, t0, dur, dt, mu, forces, j2, req, *dp, integ, rtol, atol, dev,
                                               p(out), p(st), None)
        assert rc == -20, (t0, dur, dt, forces, integ, dev)
        rc = L.astroz_cuda_propagate_numerical_device(p(y), 1, t0, dur, dt, mu, forces, j2, req, *dp, integ, rtol,
                                                      atol, dev, p(out), p(st), None, None)
        assert rc == -20
    assert (out == 7.0).all() and st[0] == 9
    # n = 0 with otherwise valid arguments on device -1 is still refused
    assert L.astroz_cuda_propagate_numerical(p(y), 0, 0.0, 100.0, 10.0, MU, 0, None, None, None, None, None, 1, 1e-9,
                                             1e-12, -1, p(out), p(st), None) == -20
    # an output of n x samples x 48 bytes that does not fit in size_t: refused before anything is read or written
    big = 0xFFFFFFFF
    for fn in (L.astroz_cuda_propagate_numerical, L.astroz_cuda_propagate_numerical_device):
        extra = [None] if fn is L.astroz_cuda_propagate_numerical_device else []
        assert fn(p(y), big, 0.0, 1e8, 1.0, MU, 0, None, None, None, None, None, 1, 1e-9, 1e-12, 0, p(out), p(st),
                  None, *extra) == -20
    assert (out == 7.0).all() and st[0] == 9
    cnt = C.c_uint64(5)
    times = np.full(3, 7.0)
    assert L.astroz_cuda_numerical_times(0.0, 100.0, 0.0, p(times), C.byref(cnt)) == -20
    assert L.astroz_cuda_numerical_times(1e17, 1000.0, 1.0, p(times), C.byref(cnt)) == -20
    assert cnt.value == 5 and (times == 7.0).all()


def test_frontend_positional_call_and_defaults_without_a_loop():
    """The reference parses everything after mu as positional-or-keyword, None meaning the default; with no step to take
    (duration <= 0) it returns ([t0], [state]) whatever dt is.  None of this needs the device."""
    import inspect

    from astroz_b200 import frontend

    params = inspect.signature(frontend.propagate_numerical).parameters
    assert all(p.kind is inspect.Parameter.POSITIONAL_OR_KEYWORD for p in params.values())
    assert list(params) == ["state", "t0", "duration", "dt", "mu", "j2", "r_eq", "drag_cd", "drag_area", "drag_mass",
                            "integrator", "rtol", "atol"]
    s = (7000.0, 0.0, 0.0, 0.0, 7.5, 0.0)
    assert frontend.propagate_numerical(s, 5.0, 0.0, 60.0, frontend.EARTH_MU, frontend.EARTH_J2,
                                        frontend.EARTH_R_EQ) == ([5.0], [s])
    assert frontend.propagate_numerical(s, 5.0, -3.0, 0.0, frontend.EARTH_MU, None, None, None, None, None, None, None,
                                        None) == ([5.0], [s])
    with pytest.raises(ValueError, match="dt must be positive"):
        frontend.propagate_numerical(s, 0.0, 10.0, 0.0, frontend.EARTH_MU)
    with pytest.raises(ValueError, match="r_eq is required"):
        frontend.propagate_numerical(s, 0.0, 10.0, 1.0, frontend.EARTH_MU, frontend.EARTH_J2)
