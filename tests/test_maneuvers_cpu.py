"""Impulsive maneuvers (astroz_b200.numerical.propagate_maneuvers_batch) on the CPU:
- numpy statements of the four burns and of the abnormal-orbit test against the scalar restatement
  (tests/numerical_oracle/maneuvers.c);
- hand-worked sample-time sequences of the loop at its edges, with RK4 and DP87;
- the K7 maneuver core (az_numerical.cuh) under host emulation, bit-identical to the restatement on the reference's
  Spacecraft test schedules, and to the K7 model-list core when the schedules are empty;
- the C ABI's argument errors.
The device run is in tests/test_gpu_maneuvers.py."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from astroz_b200 import numerical as P
from tests.numerical_oracle import maneuvers as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "host_emul")
MU, R_EQ, J2 = 398600.5, 6378.137, 0.00108262998905
TWO_BODY = [P.TwoBody(MU)]
# Spacecraft.createForceModels (src/Spacecraft.zig:124-147) for the Cube size at 300 kg: TwoBody + J2 + Drag with the
# earth's 1.225 kg/m^3 and 7.249 km (src/constants.zig:145-165), cd 2.2, 0.05 m^2, cut-off 1000 km
SPACECRAFT = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.Drag(R_EQ, 1.225, 7.249, 2.2, 0.05, 300.0, 1000.0)]


def leo(r=7000.0, incl=0.3):
    v = math.sqrt(MU / r)
    return np.array([r, 0.0, 0.0, 0.0, v * math.cos(incl), v * math.sin(incl)])


def state_from_elements(n_rev_day, e, i_deg, raan_deg, argp_deg, ma_deg):
    """TEME-like state of mean elements, a from n by Kepler's third law (the physical one; SURVEY Appendix C)"""
    n = n_rev_day * 2 * math.pi / 86400.0
    a = (MU / (n * n)) ** (1.0 / 3.0)
    M = math.radians(ma_deg)
    E = M
    for _ in range(30):
        E = E - (E - e * math.sin(E) - M) / (1 - e * math.cos(E))
    nu = 2 * math.atan2(math.sqrt(1 + e) * math.sin(E / 2), math.sqrt(1 - e) * math.cos(E / 2))
    p = a * (1 - e * e)
    r = p / (1 + e * math.cos(nu))
    rp = np.array([r * math.cos(nu), r * math.sin(nu), 0.0])
    vp = np.array([-math.sin(nu), e + math.cos(nu), 0.0]) * math.sqrt(MU / p)
    O, w, i = math.radians(raan_deg), math.radians(argp_deg), math.radians(i_deg)
    Rz = lambda t: np.array([[math.cos(t), -math.sin(t), 0], [math.sin(t), math.cos(t), 0], [0, 0, 1]])  # noqa: E731
    Rx = np.array([[1, 0, 0], [0, math.cos(i), -math.sin(i)], [0, math.sin(i), math.cos(i)]])
    Q = Rz(O) @ Rx @ Rz(w)
    return np.concatenate([Q @ rp, Q @ vp])


# 1 55909U 23035B   24187.51050877 ... / 2 55909  43.9978 311.8012 0011446 278.6226  81.3336 15.05761711 71371
Y55909 = state_from_elements(15.05761711, 0.0011446, 43.9978, 311.8012, 278.6226, 81.3336)
# its epoch in J2000 seconds: 2024 day 187.51050877, JD 2460497.01050877
T0_55909 = (2460311.5 + 187.51050877 - 2451545.0) * 86400.0


# ---- the burns and the energy test, stated in numpy ---------------------------------------------------------------
def np_burn(y, b, mu=MU):
    y = y.copy()
    vmag = np.sqrt(y[:, 3] ** 2 + y[:, 4] ** 2 + y[:, 5] ** 2)
    if b.kind == 0:
        dv = np.broadcast_to(np.array(b.p), (len(y), 3))
    elif b.kind in (1, 2):
        if b.kind == 1:
            mag = np.full(len(y), b.p[0])
        else:   # calculatePhaseChange with Zig's pow forms: x * (x * x) and exp((2/3 - 1) log x) * x
            r = np.sqrt(y[:, 0] ** 2 + y[:, 1] ** 2 + y[:, 2] ** 2)
            mag = np.zeros(len(y))
            for j, rr in enumerate(r):
                period = 2.0 * math.pi * math.sqrt(rr * (rr * rr) / mu)
                dT = b.p[0] * period / (2.0 * math.pi * b.p[1])
                x = (period + dT) * math.sqrt(mu) / (2.0 * math.pi)
                aT = math.exp((2.0 / 3.0 - 1.0) * math.log(x)) * x
                mag[j] = math.sqrt(mu * (2.0 / rr - 1.0 / aT)) - math.sqrt(mu / rr)
        dv = np.stack([y[:, 3] / vmag * mag, y[:, 4] / vmag * mag, y[:, 5] / vmag * mag], axis=1)
    else:
        di, dr = b.p[0], b.p[1]
        total = math.sqrt(di * di + dr * dr)
        if total < 1e-10:
            return y
        dvm = 2.0 * vmag * math.sin(total / 2.0)
        h = np.stack([y[:, 1] * y[:, 5] - y[:, 2] * y[:, 4], y[:, 2] * y[:, 3] - y[:, 0] * y[:, 5],
                      y[:, 0] * y[:, 4] - y[:, 1] * y[:, 3]], axis=1)
        hm = np.sqrt(h[:, 0] ** 2 + h[:, 1] ** 2 + h[:, 2] ** 2)
        dv = np.stack([h[:, 0] / hm * dvm * math.sin(di), h[:, 1] / hm * dvm * math.sin(di),
                       h[:, 2] / hm * dvm * math.cos(di)], axis=1)
    y[:, 3:] = y[:, 3:] + dv
    return y


def random_orbits(rng, m):
    r = rng.uniform(6700, 45000, m)
    u = rng.standard_normal((m, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    w = np.cross(u, rng.standard_normal((m, 3)))
    w /= np.linalg.norm(w, axis=1)[:, None]
    v = w * (np.sqrt(MU / r) * rng.uniform(0.9, 1.1, m))[:, None]
    return np.concatenate([u * r[:, None], v], axis=1)


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float64:
        a, b = a.view(np.uint64), b.view(np.uint64)
    return a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("burn", [P.Absolute(0.0, (0.01, -0.02, 0.003)), P.Prograde(0.0, 0.05), P.Prograde(0.0, -0.2),
                                  P.Phase(0.0, math.pi / 2), P.Phase(0.0, -0.3, 2.5), P.PlaneChange(0.0, 0.17, 0.08),
                                  P.PlaneChange(0.0, -0.05, 0.0), P.PlaneChange(0.0, 5e-11, 5e-11)],
                         ids=repr)
def test_numpy_statement_of_each_burn(burn):
    y = random_orbits(np.random.default_rng(3), 300)
    assert same(np_burn(y, burn), R.apply_burn(y, burn, k7_forms=True))


def test_restatement_burns_are_the_ones_the_loop_applies():
    """The sample after a burn at t0 is the burned state; the phasing burn's first half is followed by its coast."""
    y = random_orbits(np.random.default_rng(5), 40)
    for b in (P.Absolute(0.0, (0.0, 0.01, 0.02)), P.Prograde(-5.0, 0.1), P.PlaneChange(0.0, 0.2, -0.1)):
        t, traj, cnt, st, _ = R.propagate(y, 0.0, 10.0, 10.0, TWO_BODY, [b], k7_forms=True)
        assert same(traj[:, 1], np_burn(y, b)) and (st == 0).all() and (t[:, :2] == 0.0).all()
    t, traj, cnt, st, _ = R.propagate(y[:1], 0.0, 10.0, 10.0, TWO_BODY, [P.Phase(0.0, 0.5, 0.01)], k7_forms=True)
    b = np_burn(y[:1], P.Phase(0.0, 0.5, 0.01))
    # the coast's first sample is one RK4 step of h from the burned state
    first = R.propagate(b, 0.0, 10.0, 10.0, TWO_BODY, [], k7_forms=True)[1]
    assert same(traj[0, 1], first[0, 1]) and t[0, 1] == 10.0


def test_abnormal_orbit_stops_the_trajectory():
    y = np.stack([leo(), leo()])
    v_esc = math.sqrt(2 * MU / 7000.0)
    # a hyperbolic burn: energy > 0 after the first regular step
    sched = [[P.Prograde(0.0, v_esc - math.sqrt(MU / 7000.0) + 0.5)],
             [P.Prograde(0.0, v_esc - math.sqrt(MU / 7000.0) - 0.05)]]   # bound, apogee far beyond 100,000 km
    for integ in ("rk4", "dp87"):
        t, traj, cnt, st, _ = R.propagate(y, 0.0, 4 * 86400.0, 600.0, TWO_BODY, sched, integrator=integ, k7_forms=True)
        assert list(st) == [P.ABNORMAL, P.ABNORMAL]
        assert cnt[0] == 3 and t[0, 2] == 600.0                       # y0, the burn, one step
        last = traj[1, int(cnt[1]) - 1]
        r, v = np.linalg.norm(last[:3]), np.linalg.norm(last[3:])
        assert r > 100000 and 0.5 * v * v - MU / r < 0
        prev = traj[1, int(cnt[1]) - 2]
        assert np.linalg.norm(prev[:3]) <= 100000
        assert (traj[1, int(cnt[1]):] == 0).all() and (t[1, int(cnt[1]):] == 0).all()


# ---- sample times of the loop, worked by hand (t0 = 0, h = 10) ---------------------------------------------------
def times_of(sched, duration=50.0, integrator="rk4", h=10.0, y=None):
    y = leo() if y is None else y
    t, traj, cnt, st, steps = R.propagate(y, 0.0, duration, h, TWO_BODY, [sched], integrator=integrator,
                                          k7_forms=True)
    return list(t[0, :int(cnt[0])]), traj[0, :int(cnt[0])], int(st[0])


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_hand_worked_sample_times(integrator):
    cases = [
        ([P.Prograde(10.0, 0.01)], 50.0, [0, 10, 10, 20, 30, 40, 50]),                 # exactly at t + h
        ([P.Prograde(0.0, 0.01)], 50.0, [0, 0, 10, 20, 30, 40, 50]),                   # at t0
        ([P.Prograde(-5.0, 0.01)], 50.0, [0, 0, 10, 20, 30, 40, 50]),                  # before t0: fires at once
        ([P.Prograde(15.0, 0.01), P.Prograde(15.0, 0.01)], 50.0, [0, 10, 15, 15, 15, 25, 35, 45, 50]),  # two at once
        ([P.Prograde(30.0, 0.01), P.Prograde(12.0, 0.01)], 50.0, [0, 10, 20, 30, 30, 30, 40, 50]),      # unsorted
        ([P.Prograde(48.0, 0.01)], 45.0, [0, 10, 20, 30, 40, 48, 48, 45]),             # in (tf, tf + h]
        ([P.Prograde(56.0, 0.01)], 45.0, [0, 10, 20, 30, 40, 45]),                     # beyond tf + h: never fires
    ]
    for sched, duration, want in cases:
        got, _, st = times_of(sched, duration, integrator)
        assert got == [float(x) for x in want] and st == 0, (sched, got)


def test_two_burns_at_one_time_and_unsorted_lists_fire_in_list_order():
    _, a, _ = times_of([P.Prograde(15.0, 0.01), P.Absolute(15.0, (0.0, 0.0, 0.02))])
    _, b, _ = times_of([P.Absolute(15.0, (0.0, 0.0, 0.02)), P.Prograde(15.0, 0.01)])
    assert same(a[3], np_burn(a[2:3], P.Prograde(0, 0.01))[0]) and not same(a[4], b[4])


def test_plane_change_below_threshold_leaves_the_state():
    t, y, st = times_of([P.PlaneChange(20.0, 5e-11, 5e-11)])
    assert t == [0, 10, 20, 20, 30, 40, 50] and same(y[2], y[3])
    t, y, st = times_of([P.PlaneChange(20.0, 1e-10, 0.0)])
    assert not same(y[2], y[3])


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_phasing_coast_past_tf_ends_with_a_negative_step(integrator):
    r, h, orbits = 7000.0, 60.0, 0.05
    period = 2.0 * math.pi * math.sqrt(r * (r * r) / MU)
    t, traj, st = times_of([P.Phase(60.0, math.pi / 4, orbits)], 200.0, integrator, h=h)
    coast = [60.0 + h * k for k in range(1, 100) if 60.0 + h * (k - 1) < 60.0 + period * orbits]
    want = [0.0, 60.0] + coast + [coast[-1], 200.0]
    assert coast[-1] == 360.0 and t == want and st == 0
    if integrator == "dp87":
        # a step of -160 s makes no attempt (and leaves DP87's step size at -160 s): the state is kept
        assert same(traj[-1], traj[-2])
    else:   # RK4 steps back by -160 s
        assert not same(traj[-1], traj[-2])


# ---- host emulation of the K7 maneuver core ----------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = os.path.join(EMUL_DIR, "libemul_maneuvers.so")
    src = os.path.join(EMUL_DIR, "emul_maneuvers.cu")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("az_numerical.cuh", "az_math.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-I" + csrc, "-o", so, src], check=True,
                       capture_output=True)
    return C.CDLL(so)


def run_emul(L, states, t0, duration, h, models, schedules, cap, integrator="rk4", mu=MU, rtol=1e-9, atol=1e-12):
    from tests.numerical_oracle import models as M

    states = np.ascontiguousarray(np.atleast_2d(states), dtype=np.float64)
    n = len(states)
    off, imp = P.pack_schedules(schedules, n)
    descs, keep = M.descriptors(models, n, 1)
    times, out = np.zeros((n, cap)), np.zeros((n, cap, 6))
    cnt, st, steps = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint8), np.zeros((n, 2), dtype=np.uint64)
    p = lambda a: C.c_void_p(a.ctypes.data) if a.size else None  # noqa: E731
    d = C.c_double
    assert L.emul_maneuvers(p(states), n, d(t0), d(duration), d(h), d(mu), p(off), p(imp), C.cast(descs, C.c_void_p),
                            len(descs), d(rtol), d(atol), 0 if integrator == "rk4" else 1, C.c_uint32(cap), p(times),
                            p(out), p(cnt), p(st), p(steps)) == 0
    del keep
    return times, out, cnt, st, steps


# the reference's Spacecraft tests (src/Spacecraft.zig:388-392, 426-431, 477-485), their literal times against t0 = the
# TLE epoch in J2000 seconds: every impulse lies before t0 and fires at t0, in list order
SPACECRAFT_SCHEDULES = [
    [P.Prograde(2635014.50, 0.2), P.Prograde(2638026.50, 0.2), P.Prograde(2638103.50, 0.2)],
    [P.Phase(2500000.0, math.pi / 2.0, 1.0)],
    [P.PlaneChange(2500000.0, math.pi / 18.0, math.pi / 36.0)],
]


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_cores_equal_the_restatement_on_the_spacecraft_tests(emul, integrator):
    y = np.stack([Y55909] * 3)
    ref = R.propagate(y, T0_55909, 3 * 86400.0, 1.0, SPACECRAFT, SPACECRAFT_SCHEDULES, integrator=integrator,
                      k7_forms=True, threads=3)
    cap = ref[0].shape[1]
    got = run_emul(emul, y, T0_55909, 3 * 86400.0, 1.0, SPACECRAFT, SPACECRAFT_SCHEDULES, cap, integrator)
    for a, b in zip(ref, got):
        assert same(a, b)
    cnt = ref[2]
    assert (ref[3] == 0).all() and cnt[0] == 259201 + 3 and cnt[2] == 259201 + 1
    assert (ref[0][[0, 2], 1] == T0_55909).all()                          # the burns fire at t0
    # the phasing burn: its coast samples every second from t0 + 1 for one period, then the return burn's sample
    t1 = ref[0][1, :int(cnt[1])]
    rep = np.flatnonzero(np.diff(t1) == 0)
    assert t1[1] == T0_55909 + 1.0 and len(rep) == 1 and 5000 < rep[0] < 6500
    r = np.linalg.norm(ref[1][:, :, :3], axis=2)
    for i in range(3):
        assert (r[i, :int(cnt[i])] > R_EQ).all()                          # the reference tests' assertion


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_cores_equal_the_restatement_on_burn_sweeps(emul, integrator):
    rng = np.random.default_rng(11)
    y = random_orbits(rng, 12)
    sched = []
    for i in range(12):
        s = [P.Prograde(rng.uniform(-100, 9000), rng.uniform(-0.05, 0.05)),
             P.Absolute(rng.uniform(0, 9000), rng.uniform(-0.02, 0.02, 3)),
             P.PlaneChange(rng.uniform(0, 9000), rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2))]
        if i % 3 == 0:
            s.append(P.Phase(rng.uniform(0, 9000), rng.uniform(-1, 1), rng.uniform(0.3, 1.5)))
        sched.append(s)
    models = SPACECRAFT + [P.ThirdBody(4902.8, (300000.0, 200000.0, 10000.0))]
    ref = R.propagate(y, 100.0, 10800.0, 30.0, models, sched, integrator=integrator, k7_forms=True)
    got = run_emul(emul, y, 100.0, 10800.0, 30.0, models, sched, ref[0].shape[1], integrator)
    for a, b in zip(ref, got):
        assert same(a, b)
    # a short row: the first samples, the full count, TRUNCATED
    short = run_emul(emul, y, 100.0, 10800.0, 30.0, models, sched, 50, integrator)
    assert same(short[0], ref[0][:, :50]) and same(short[1], ref[1][:, :50]) and same(short[2], ref[2])
    assert (short[3] == P.TRUNCATED).all()


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_empty_schedules_equal_the_model_list_core(emul, integrator):
    from tests.test_numerical_models_cpu import run_emul as run_models

    models_lib = _models_emul()
    y = random_orbits(np.random.default_rng(2), 6)
    out, st, cnt = run_models(models_lib, y, 0.0, 7300.0, 60.0, SPACECRAFT, integrator)
    t, traj, n, s, steps = run_emul(emul, y, 0.0, 7300.0, 60.0, SPACECRAFT, [], out.shape[1], integrator)
    assert same(traj, out) and same(steps, cnt) and (n == out.shape[1]).all() and (s == st).all()
    assert same(t[0], P.numerical_times(0.0, 7300.0, 60.0))


def _models_emul():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    so = os.path.join(EMUL_DIR, "libemul_numerical_models.so")
    src = os.path.join(EMUL_DIR, "emul_numerical_models.cu")
    csrc = os.path.join(ROOT, "astroz_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("az_numerical.cuh", "az_math.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.run([nvcc, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "--expt-relaxed-constexpr",
                        "-Xcompiler", "-fPIC,-ffp-contract=off", "-shared", "-I" + csrc, "-o", so, src], check=True,
                       capture_output=True)
    return C.CDLL(so)


def test_wrapper_estimate_and_schedule_packing():
    off, imp = P.pack_schedules([P.Prograde(1.0, 0.1), P.Phase(2.0, 0.5, 2.0)], 3)
    assert list(off) == [0, 2, 4, 6] and list(imp["kind"]) == [1, 2] * 3 and imp["p"][1, 1] == 2.0
    off, imp = P.pack_schedules([[], [P.PlaneChange(0.0, 0.1, 0.2)], []], 3)
    assert list(off) == [0, 0, 1, 1] and imp.itemsize == 40   # sizeof(astroz_impulse_t)
    with pytest.raises(ValueError):
        P.pack_schedules([[], []], 3)
    with pytest.raises(ValueError):
        P.pack_schedules([P.Phase(0.0, 0.1, 0.0)], 1)
    with pytest.raises(ValueError):
        P.pack_schedules([P.Prograde(math.nan, 0.1)], 1)
    # the estimate covers the regular samples, 3 per burn and the coast at the initial radius
    y = np.stack([leo()] * 2)
    off, imp = P.pack_schedules([[P.Prograde(5.0, 0.01)], [P.Phase(5.0, 0.3, 2.0)]], 2)
    est = P._estimate_samples(y, 0.0, 600.0, 10.0, off, imp, MU)
    full = R.propagate(y, 0.0, 600.0, 10.0, TWO_BODY, [[P.Prograde(5.0, 0.01)], [P.Phase(5.0, 0.3, 2.0)]],
                       k7_forms=True)[2]
    assert est >= full.max()


# ---- C ABI argument errors ---------------------------------------------------------------------------------------
def test_cabi_refuses_bad_arguments_and_writes_nothing():
    from astroz_b200._lib import lib

    L = lib()
    y = np.zeros((2, 6))
    y[:, 0], y[:, 4] = 7000.0, 7.5
    times, out = np.full((2, 8), 7.0), np.full((2, 8, 6), 7.0)
    cnt, st = np.full(2, 3, dtype=np.uint64), np.full(2, 9, dtype=np.uint8)
    p = lambda a: C.c_void_p(a.ctypes.data) if a is not None and a.size else None  # noqa: E731
    two_body = (P._ForceModelC * 1)()
    two_body[0].kind, two_body[0].mu = 0, MU
    table = (P._ForceModelC * 1)()
    tab = np.zeros((4, 3))
    table[0].kind, table[0].flags, table[0].mu, table[0].pos_table = 7, 8, 4902.8, tab.ctypes.data
    nan_model = (P._ForceModelC * 1)()
    nan_model[0].kind, nan_model[0].mu = 0, math.nan

    def sched(*bs, off=None):
        imp = np.zeros(len(bs), dtype=P.IMPULSE_DTYPE)
        for k, b in enumerate(bs):
            imp[k] = b
        off = np.array([0, len(bs), len(bs)] if off is None else off, dtype=np.uint32)
        return off, imp

    ok = sched((10.0, 1, 0, (0.01, 0, 0)))
    base = dict(t0=0.0, dur=100.0, h=10.0, mu=MU, s=ok, models=two_body, integ=0, rtol=1e-9, atol=1e-12, cap=8, dev=0)
    common = [dict(h=0.0), dict(h=-1.0), dict(t0=math.nan), dict(dur=math.inf), dict(h=math.nan), dict(mu=math.nan),
              dict(rtol=math.nan), dict(atol=math.inf), dict(cap=0), dict(models=table), dict(models=nan_model),
              dict(integ=2), dict(dev=-1), dict(t0=1e17, dur=1000.0, h=1.0)]
    host_only = [dict(s=sched((10.0, 4, 0, (0, 0, 0)))), dict(s=sched((10.0, -1, 0, (0, 0, 0)))),
                 dict(s=sched((math.nan, 1, 0, (0.1, 0, 0)))), dict(s=sched((1.0, 0, 0, (0.1, math.inf, 0)))),
                 dict(s=sched((1.0, 1, 0, (0.1, 0, math.nan)))), dict(s=sched((1.0, 2, 0, (0.1, 0.0, 0)))),
                 dict(s=sched((1.0, 2, 0, (0.1, -1.0, 0)))), dict(s=sched((1.0, 1, 0, (0.1, 0, 0)), off=[0, 1, 0])),
                 dict(s=sched((1.0, 1, 0, (0.1, 0, 0)), off=[1, 0, 1])),
                 dict(s=sched((1.0, 1, 0, (0.1, 0, 0)), off=[0, 0, 0])),
                 dict(s=sched((1.0, 1, 0, (0.1, 0, 0)), off=[0, 1, 2]))]

    def call(fn, a, device):
        off, imp = a["s"]
        extra = [None] if device else []
        return fn(p(y), 2, a["t0"], a["dur"], a["h"], a["mu"], p(off), p(imp), len(imp),
                  C.cast(a["models"], C.c_void_p), 1, a["integ"], a["rtol"], a["atol"], a["cap"], a["dev"], p(times),
                  p(out), p(cnt), p(st), None, *extra)

    for case in common + host_only:
        a = {**base, **case}
        assert call(L.astroz_cuda_propagate_maneuvers, a, False) == -20, case
        if case in common:
            assert call(L.astroz_cuda_propagate_maneuvers_device, a, True) == -20, case
    assert (times == 7.0).all() and (out == 7.0).all() and (cnt == 3).all() and (st == 9).all()
