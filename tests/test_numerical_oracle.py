"""The scalar restatement of the reference's numerical propagation (tests/numerical_oracle) against independent truth:
the Prince-Dormand order conditions, the reference's own tests, analytic Kepler orbits, RK4's convergence order, scipy's
DOP853 with an acceleration written here in numpy, and the J2 energy / angular-momentum integrals.  K7 is checked
against this restatement in tests/test_numerical_host_emulation.py (CPU) and tests/test_gpu_numerical.py (device)."""
import math

import numpy as np
import pytest

from tests import numerical_oracle as N

MU_REF_TESTS = 398600.4418   # the reference's unit tests (Propagator.zig:80, Integrator.zig:302-377)
MU, R_EQ, J2 = 398600.5, 6378.137, 0.00108262998905   # WGS-84 (src/constants.zig:55-58)

# The published rationals, independent of both the oracle's and the product's double tables
A_ROWS = {
    1: {0: (1, 18)}, 2: {0: (1, 48), 1: (1, 16)}, 3: {0: (1, 32), 2: (3, 32)}, 4: {0: (5, 16), 2: (-75, 64), 3: (75, 64)},
    5: {0: (3, 80), 3: (3, 16), 4: (3, 20)},
}
C_Q = [(0, 1), (1, 18), (1, 12), (1, 8), (5, 16), (3, 8), (59, 400), (93, 200), (5490023248, 9719169821), (13, 20),
       (1201146811, 1299019798), (1, 1), (1, 1)]


def test_tableau_row_sums_and_quadrature_order():
    c, a, b8, b7 = N.tableau()
    for i in range(13):
        # c_i = sum_j a_ij; the published rationals are rounded to ~10 digits, so the sums agree to that, not to 1 ulp
        assert abs(a[i].sum() - c[i]) < 1e-12, i
        assert c[i] == C_Q[i][0] / C_Q[i][1]
    for i, row in A_ROWS.items():
        for j, (p, q) in row.items():
            assert a[i, j] == p / q
    # quadrature conditions sum b_i c_i^(k-1) = 1/k: order 8 for b8, order 7 for b7.  The rationals are approximations
    # of the exact (irrational) coefficients to about 1e-17 relative; the bound 1e-13 leaves room for the products.
    for k in range(1, 9):
        assert abs(float(np.sum(b8 * c ** (k - 1))) - 1.0 / k) < 1e-13, k
    for k in range(1, 8):
        assert abs(float(np.sum(b7 * c ** (k - 1))) - 1.0 / k) < 1e-13, k
    # the 7th-order weights fail the 8th condition: that gap is the error estimate
    assert abs(float(np.sum(b7 * c ** 7)) - 1.0 / 8) > 1e-6
    # a few order conditions beyond quadrature: sum_i b_i sum_j a_ij c_j = 1/6 (third order), exact for b8 and b7
    for b in (b8, b7):
        assert abs(float(b @ (a @ c[:12])) - 1.0 / 6) < 1e-13
        assert abs(float(b @ (c * (a @ c[:12]))) - 1.0 / 8) < 1e-13
        assert abs(float(b @ (a @ (c[:12] ** 2))) - 1.0 / 12) < 1e-13


def test_reference_unit_tests_restated():
    """Propagator.zig:76-112 and Integrator.zig:300-385, same inputs and the same assertions."""
    r0 = 7000.0
    v0 = math.sqrt(MU_REF_TESTS / r0)
    period = 2.0 * math.pi * math.sqrt(r0 ** 3 / MU_REF_TESTS)
    # rk4 twobody orbit: radius conserved to 1e-4, back within 50 km after one period at dt 10 s
    _, tr, st, _ = N.propagate([r0, 0, 0, 0, v0, 0], 0, period, 10.0, MU_REF_TESTS, integrator="rk4")
    f = tr[0, -1]
    assert st[0] == 0
    assert abs(np.linalg.norm(f[:3]) - r0) / r0 < 1e-4 and abs(f[0] - r0) < 50 and abs(f[1]) < 50
    # rk4 / dp87 basic: one 60 s step moves the state, DP87 towards smaller x
    s = [7000, 0, 0, 0, 7.5, 0]
    _, tr, _, _ = N.propagate(s, 0, 60, 60, MU_REF_TESTS, integrator="rk4")
    assert tr[0, 1, 0] != 7000
    _, tr, _, _ = N.propagate(s, 0, 60, 60, MU_REF_TESTS)
    assert tr[0, 1, 0] < 7000
    # dp87 vs rk4 accuracy over one period (one DP87 interval of a whole period, rtol 1e-12, atol 1e-14)
    _, rk, _, _ = N.propagate([r0, 0, 0, 0, v0, 0], 0, period, 10.0, MU_REF_TESTS, integrator="rk4")
    _, dp, _, _ = N.propagate([r0, 0, 0, 0, v0, 0], 0, period, period, MU_REF_TESTS, rtol=1e-12, atol=1e-14)
    assert abs(np.linalg.norm(dp[0, -1, :3]) - r0) < abs(np.linalg.norm(rk[0, -1, :3]) - r0)
    # dp87 energy conservation over 3600 s at rtol 1e-10: relative energy error < 1e-8
    _, tr, _, _ = N.propagate(s, 0, 3600, 3600, MU_REF_TESTS, rtol=1e-10, atol=1e-12)
    e = lambda y: 0.5 * np.dot(y[3:], y[3:]) - MU_REF_TESTS / np.linalg.norm(y[:3])  # noqa: E731
    assert abs(e(tr[0, -1]) - e(tr[0, 0])) / abs(e(tr[0, 0])) < 1e-8


def _kepler_state(a, e, M, mu=MU):
    """Perifocal state of an ellipse at mean anomaly M (Newton on Kepler's equation to machine precision)."""
    E = M if e < 0.8 else math.pi
    for _ in range(50):
        E -= (E - e * math.sin(E) - M) / (1 - e * math.cos(E))
    nu_c, nu_s = (math.cos(E) - e) / (1 - e * math.cos(E)), math.sqrt(1 - e * e) * math.sin(E) / (1 - e * math.cos(E))
    p = a * (1 - e * e)
    r = p / (1 + e * nu_c)
    h = math.sqrt(mu * p)
    return np.array([r * nu_c, r * nu_s, 0.0, -mu / h * nu_s, mu / h * (e + nu_c), 0.0])


@pytest.mark.parametrize("e", [0.0, 0.1, 0.7])
def test_two_body_against_kepler(e):
    """Ten periods at DP87 rtol 1e-12 / atol 1e-12 against the analytic ellipse.  Local errors are held near 1e-12
    relative per step and accumulate mostly along-track over ~10^3-10^4 steps, so the bound is 1e-6 relative to a for
    the position (1e-7 was observed for e = 0.7), and the radius-independent 1e-9 relative on the energy."""
    a = 8000.0 if e < 0.5 else 26600.0
    n = math.sqrt(MU / a ** 3)
    period = 2 * math.pi / n
    y0 = _kepler_state(a, e, 0.3)
    t, tr, st, steps = N.propagate(y0, 0.0, 10 * period, period / 8, MU, rtol=1e-12, atol=1e-12)
    assert st[0] == 0 and steps[0, 0] > 0
    err = max(np.linalg.norm(tr[0, k, :3] - _kepler_state(a, e, 0.3 + n * t[k])[:3]) for k in range(len(t)))
    assert err < 1e-6 * a, err
    energy = 0.5 * np.sum(tr[0, :, 3:] ** 2, axis=1) - MU / np.linalg.norm(tr[0, :, :3], axis=1)
    assert np.max(np.abs(energy / (-MU / (2 * a)) - 1)) < 1e-9


def test_rk4_converges_at_fourth_order():
    """Halving dt cuts the global error by 2^4 = 16 (e = 0.1, one period in 128, 256, 512 equal steps, so no short last
    step blurs the ratio).  The h^5 term still adds about 10% at these step sizes (measured 18.7, then 17.4), so the
    ratios must lie in 15-19.5 and fall towards 16."""
    a, e = 7500.0, 0.1
    n = math.sqrt(MU / a ** 3)
    period = 2 * math.pi / n
    y0 = _kepler_state(a, e, 0.0)
    exact = _kepler_state(a, e, n * period)
    errs = []
    for dt in (period / 128, period / 256, period / 512):
        _, tr, _, _ = N.propagate(y0, 0, period, dt, MU, integrator="rk4")
        errs.append(np.linalg.norm(tr[0, -1, :3] - exact[:3]))
    ratios = [errs[k] / errs[k + 1] for k in range(2)]
    assert all(15.0 < q < 19.5 for q in ratios) and ratios[1] < ratios[0], errs


def _accel_np(y, j2=True, drag=None):
    """J2 and drag written from their closed forms, not in the reference's operation order.  The reference's J2 term
    (ForceModel.zig:67-79) is the negative of the textbook oblate-earth acceleration -grad(mu J2 R^2 (3 sin^2 lat - 1)
    / (2 r^3)); K7 reproduces the reference, so this model takes the same sign: +grad of that potential."""
    r = y[:3]
    rn = np.linalg.norm(r)
    acc = -MU * r / rn ** 3
    if j2:
        k = 1.5 * J2 * MU * R_EQ ** 2 / rn ** 5
        zz = 5 * r[2] ** 2 / rn ** 2
        acc = acc - k * np.array([r[0] * (zz - 1), r[1] * (zz - 1), r[2] * (zz - 3)])
    if drag:
        cd, area, mass = drag
        alt = rn - R_EQ
        if alt <= 1500:
            v = y[3:]
            # the reference's magnitude is 0.5 cd A rho |v| 1e3 / m (ForceModel.zig:107-109): linear in the speed
            acc = acc - 0.5 * cd * area / mass * 1.225 * np.exp(-alt / 7.249) * 1e3 * v
    return acc


@pytest.mark.parametrize("drag", [None, (2.2, 10.0, 500.0)])
def test_j2_and_drag_against_scipy_dop853(drag):
    """A LEO state with a 150 km perigee (where drag matters) over 6 hours, DP87 at rtol 1e-12 / atol 1e-12 vs scipy's
    DOP853 at rtol 1e-13 / atol 1e-12 on the numpy acceleration.  Both integrators hold local errors near 1e-12; over
    ~2,000 steps they drift apart along-track by about 1e-7 of the 7,000 km radius, so the bound is 1e-3 km / 1e-6
    km/s.  Drag moves this orbit by tens of km, far outside the bound, so the bound tests the drag model too."""
    from scipy.integrate import solve_ivp

    a = R_EQ + 1000.0
    rp = R_EQ + 150.0
    e = 1 - rp / a
    y0 = _kepler_state(a, e, -0.5)
    y0 = np.array([y0[0], y0[1] * 0.8, y0[1] * 0.6, y0[3], y0[4] * 0.8, y0[4] * 0.6])  # 36.9 deg inclination
    T = 6 * 3600.0
    kw = dict(drag_cd=drag[0], drag_area=drag[1], drag_mass=drag[2]) if drag else {}
    t, tr, st, _ = N.propagate(y0, 0, T, 600.0, MU, j2=J2, r_eq=R_EQ, rtol=1e-12, atol=1e-12, **kw)
    assert st[0] == 0
    sol = solve_ivp(lambda _, y: np.concatenate([y[3:], _accel_np(y, True, drag)]), (0, T), y0, method="DOP853",
                    t_eval=t, rtol=1e-13, atol=1e-12)
    ref = sol.y.T
    assert np.max(np.abs(tr[0, :, :3] - ref[:, :3])) < 1e-3
    assert np.max(np.abs(tr[0, :, 3:] - ref[:, 3:])) < 1e-6
    if drag:
        _, nodrag, _, _ = N.propagate(y0, 0, T, 600.0, MU, j2=J2, r_eq=R_EQ, rtol=1e-12, atol=1e-12)
        assert np.max(np.abs(nodrag[0, -1, :3] - tr[0, -1, :3])) > 1.0


def test_j2_conserves_energy_and_polar_angular_momentum():
    """The reference's J2 (see _accel_np for its sign) is conservative and axisymmetric:
    E = v^2/2 - mu/r - mu J2 R^2 / (2 r^3) (3 sin^2(lat) - 1) and h_z are
    integrals.  One day of a 51.6 deg LEO at the default tolerances (rtol 1e-9): each accepted step adds a relative error
    near 1e-10 of the state, ~2,000 steps -> bound 1e-8 relative on both."""
    y0 = np.array([6778.0, 0.0, 0.0, 0.0, 7.6686 * math.cos(0.9006), 7.6686 * math.sin(0.9006)])
    _, tr, st, _ = N.propagate(y0, 0, 86400.0, 60.0, MU, j2=J2, r_eq=R_EQ)
    assert st[0] == 0
    r = np.linalg.norm(tr[0, :, :3], axis=1)
    sl2 = (tr[0, :, 2] / r) ** 2
    E = 0.5 * np.sum(tr[0, :, 3:] ** 2, axis=1) - MU / r - MU * J2 * R_EQ ** 2 / (2 * r ** 3) * (3 * sl2 - 1)
    hz = tr[0, :, 0] * tr[0, :, 4] - tr[0, :, 1] * tr[0, :, 3]
    assert np.max(np.abs(E / E[0] - 1)) < 1e-8
    assert np.max(np.abs(hz / hz[0] - 1)) < 1e-8


def _loop_times(t0, duration, dt):
    t, out = t0, [t0]
    while t < t0 + duration:
        t += min(dt, t0 + duration - t)
        out.append(t)
    return np.array(out)


@pytest.mark.parametrize("t0,duration,dt", [(0.0, 0.0, 10.0), (5.0, 3.0, 10.0), (0.0, 25.0, 10.0), (0.0, 1.0, 0.1),
                                            (1e5, 86400.0, 7.0), (-30.0, -5.0, 1.0)])
def test_sampling_edges(t0, duration, dt):
    """duration 0, dt > duration, a remainder, the float sums of 0.1 s steps (the last of which is 1e-16 s), a negative
    duration: the oracle's and the library's times are the loop's own float sums, bit for bit."""
    from astroz_b200.numerical import numerical_times

    ref = _loop_times(t0, duration, dt)
    assert np.array_equal(N.times(t0, duration, dt), ref)
    assert np.array_equal(numerical_times(t0, duration, dt), ref)
    if duration == 1.0:
        assert len(ref) == 12 and ref[-1] == 1.0 and ref[-2] < 1.0


def test_status_cases():
    # stopped: a state at the centre has a NaN error norm at every step size, so DP87 shrinks h to hMin and the
    # reference would retry that attempt forever; the first sample is kept, the rest zero-filled
    t, tr, st, steps = N.propagate([0.0, 0, 0, 0, 0, 0], 0, 300.0, 60.0, MU)
    assert st[0] == 1 and steps[0, 0] == 0 and steps[0, 1] > 0
    assert not tr[0].any() and len(t) == 6
    t, tr, st, steps = N.propagate([1e-3, 0, 0, 0, 0, 0], 0, 300.0, 60.0, MU)
    assert st[0] == 1 and tr[0, 0, 0] == 1e-3 and not tr[0, 1:].any()
    # substep limit: one interval of 1e6 s at rtol 1e-14 needs more than 10,000 accepted steps
    _, tr, st, steps = N.propagate([7000, 0, 0, 0, 7.5, 0], 0, 1e6, 1e6, MU, rtol=1e-14, atol=1e-14)
    assert st[0] == 2 and steps[0, 0] == 10000 and np.all(np.isfinite(tr))
    # RK4 non-finite: a state starting at the origin divides by zero
    _, tr, st, _ = N.propagate([0, 0, 0, 0, 0, 0], 0, 100.0, 10.0, MU, integrator="rk4")
    assert st[0] == 3 and not np.all(np.isfinite(tr[0, -1]))


def test_threaded_restatement_equals_single_thread():
    rng = np.random.default_rng(5)
    y = np.array([_kepler_state(7000 + 500 * rng.random(), 0.01 * rng.random(), rng.random() * 6) for _ in range(40)])
    area = 1.0 + rng.random(40)
    many = N.propagate(y, 0, 3000, 60, MU, j2=J2, r_eq=R_EQ, drag_cd=2.2, drag_area=area, drag_mass=100, threads=7)
    single = N.propagate(y, 0, 3000, 60, MU, j2=J2, r_eq=R_EQ, drag_cd=2.2, drag_area=area, drag_mass=100)
    for a, b in zip(many[1:], single[1:]):
        assert np.array_equal(a, b)
