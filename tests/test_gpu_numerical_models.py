"""K7 with model lists on the device (numerical_models_kernel, astroz_b200/csrc/az_numerical.cu): against the scalar
restatement for every model and mixed lists with both integrators, host vs device calls over pageable and pinned buffers
and several chunks, batch independence, the status cases, and the list path with K7's fixed force set."""
import numpy as np
import pytest

from astroz_b200 import numerical as P
from tests.numerical_oracle import models as M
from tests.test_numerical_models_cpu import (AU, J2, MOON_MU, MU, R_EQ, SUN_MU, _steps, fixtures, same, single_lists,
                                             spice_list, sun_moon_tables)

pytestmark = pytest.mark.gpu
EXP_FREE = {"two_body", "j2", "j3", "j4", "srp", "srp_table", "third_body", "third_body_table", "spice",
            "spice_reordered"}


@pytest.fixture(scope="module")
def dev():
    import astroz_b200

    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return 0


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_models_match_the_restatement(dev, integrator):
    """Without Drag or ImprovedDrag the device is bit-identical to the restatement with K7's step factor.  With them the
    device's exp differs from the C library's in the last place; those runs are held to K7's drag bound: 1e-6 km /
    1e-9 km/s relative to the orbit's scale, equal status."""
    y = fixtures()
    K = len(_steps(0.0, 10800.0, 60.0))
    for name, models in single_lists(len(y), K).items():
        _, tr, st, steps = P.propagate_models_batch(y, 0.0, 10800.0, 60.0, models, integrator=integrator)
        _, ref, rst, rsteps = M.propagate(y, 0.0, 10800.0, 60.0, models, integrator=integrator, k7_step_factor=True)
        assert np.array_equal(st, rst), name
        if name in EXP_FREE:
            assert same(tr, ref) and np.array_equal(steps, rsteps), name
            continue
        scale = np.maximum(1.0, np.abs(ref[..., :3]).max(axis=(1, 2)) / 7000.0)[:, None, None]
        assert np.max(np.abs(tr[..., :3] - ref[..., :3]) / scale) < 1e-6, name
        assert np.max(np.abs(tr[..., 3:] - ref[..., 3:]) / scale) < 1e-9, name


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_mixed_list_with_every_kind(dev, integrator):
    y = fixtures()
    K = len(_steps(0.0, 7200.0, 60.0))
    sun, moon = sun_moon_tables(K, 5)
    rng = np.random.default_rng(11)
    models = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.J3(MU, -2.53215306e-6, R_EQ), P.J4(MU, -1.61098761e-6, R_EQ),
              P.Drag(R_EQ, 1.225, 7.249, 2.2, rng.uniform(1, 10, len(y)), 400.0, 1500.0),
              P.ImprovedDrag(R_EQ, rng.uniform(2, 2.4, len(y)), 5.0, 300.0, 1500.0, 160.0),
              P.SolarRadiationPressure(1.4, rng.uniform(5, 25, len(y)), 800.0, R_EQ, sun), P.ThirdBody(SUN_MU, sun),
              P.ThirdBody(MOON_MU, moon)]
    _, tr, st, _ = P.propagate_models_batch(y, 0.0, 7200.0, 60.0, models, integrator=integrator)
    _, ref, rst, _ = M.propagate(y, 0.0, 7200.0, 60.0, models, integrator=integrator, k7_step_factor=True)
    assert np.array_equal(st, rst) and (st == 0).all()
    scale = np.maximum(1.0, np.abs(ref[..., :3]).max(axis=(1, 2)) / 7000.0)[:, None, None]
    assert np.max(np.abs(tr[..., :3] - ref[..., :3]) / scale) < 1e-6
    assert np.max(np.abs(tr[..., 3:] - ref[..., 3:]) / scale) < 1e-9


def test_list_with_k7_forces_equals_the_fixed_entry_point(dev):
    y = fixtures()
    area = np.linspace(1, 20, len(y))
    models = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.Drag(R_EQ, 1.225, 7.249, 2.2, area, 300.0, 1500.0)]
    for integ in ("rk4", "dp87"):
        a = P.propagate_models_batch(y, 0.0, 21600.0, 60.0, models, integrator=integ)
        b = P.propagate_numerical_batch(y, 0.0, 21600.0, 60.0, MU, j2=J2, r_eq=R_EQ, drag_cd=2.2, drag_area=area,
                                        drag_mass=300.0, integrator=integ)
        assert same(a[1], b[1]) and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
    for models, kw in (([P.TwoBody(MU)], {}), ([P.TwoBody(MU), P.J2(MU, J2, R_EQ)], dict(j2=J2, r_eq=R_EQ))):
        a = P.propagate_models_batch(y, 0.0, 21600.0, 60.0, models)
        b = P.propagate_numerical_batch(y, 0.0, 21600.0, 60.0, MU, **kw)
        assert same(a[1], b[1]) and np.array_equal(a[3], b[3])


def _dispersed(n, seed=1):
    rng = np.random.default_rng(seed)
    return np.array(fixtures()[:5])[rng.integers(0, 5, n)] * (1 + 1e-4 * rng.standard_normal((n, 6)))


def test_host_and_device_calls_give_the_same_bytes(dev):
    """2,000 states, RK4 over 4,000 samples: 384 MB of trajectories, two chunks of the host call; per-state SRP and drag
    coefficients and Sun / Moon tables.  Pageable and pinned destinations and inputs, and the device call, agree."""
    import torch

    import astroz_b200

    rng = np.random.default_rng(2)
    n = 2000
    y = _dispersed(n)
    args = (0.0, 39990.0, 10.0)
    K = len(_steps(*args))
    sun, moon = sun_moon_tables(K, 60, dt=10.0)
    cr, area, mass = rng.uniform(1, 2, n), rng.uniform(1, 20, n), rng.uniform(100, 900, n)
    models = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.SolarRadiationPressure(cr, area, mass, R_EQ, sun),
              P.ThirdBody(SUN_MU, sun), P.ThirdBody(MOON_MU, moon),
              P.ImprovedDrag(R_EQ, 2.2, area, mass, 1500.0, 150.0)]
    _, ref, st, steps = P.propagate_models_batch(y, *args, models, integrator="rk4")
    assert ref.nbytes > 256 << 20
    pinned = astroz_b200.pinned_empty(ref.shape)
    _, out, s2, c2 = P.propagate_models_batch(y, *args, models, integrator="rk4", out=pinned)
    assert same(out, ref) and np.array_equal(s2, st) and np.array_equal(c2, steps)
    # pinned inputs too
    py = astroz_b200.pinned_empty(y.shape)
    py[:] = y
    pcols = []
    for a in (cr, area, mass):
        b = astroz_b200.pinned_empty(a.shape)
        b[:] = a
        pcols.append(b)
    pmodels = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.SolarRadiationPressure(*pcols, R_EQ, sun),
               P.ThirdBody(SUN_MU, sun), P.ThirdBody(MOON_MU, moon),
               P.ImprovedDrag(R_EQ, 2.2, pcols[1], pcols[2], 1500.0, 150.0)]
    _, out2, _, _ = P.propagate_models_batch(py, *args, pmodels, integrator="rk4", out=pinned)
    assert same(out2, ref)
    d = torch.device("cuda", 0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(d)  # noqa: E731
    dmodels = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.SolarRadiationPressure(T(cr), T(area), T(mass), R_EQ, T(sun)),
               P.ThirdBody(SUN_MU, T(sun)), P.ThirdBody(MOON_MU, T(moon)),
               P.ImprovedDrag(R_EQ, 2.2, T(area), T(mass), 1500.0, 150.0)]
    dout = torch.empty(ref.shape, dtype=torch.float64, device=d)
    dst = torch.empty(n, dtype=torch.uint8, device=d)
    dsteps = torch.empty((n, 2), dtype=torch.int64, device=d)
    P.propagate_models_batch_device(T(y), *args, dmodels, dout, dst, dsteps, integrator="rk4")
    torch.cuda.synchronize()
    assert same(dout.cpu().numpy(), ref) and np.array_equal(dst.cpu().numpy(), st)
    assert np.array_equal(dsteps.cpu().numpy().astype(np.uint64), steps)
    with pytest.raises(ValueError, match="CUDA tensors"):
        P.propagate_models_batch_device(T(y), *args, models, dout, dst, integrator="rk4")


def test_dp87_several_chunks_and_device_call(dev):
    """DP87 with the SPICE list and tables over two chunks of the host call: equal to the device call and to the
    restatement (no exp in the list: bit for bit)."""
    import torch

    n = 3000
    y = _dispersed(n, 5)
    args = (0.0, 86400.0, 30.0)    # 2,881 samples: 138 kB per state, 1,941 states per 256 MB chunk
    K = len(_steps(*args))
    sun, moon = sun_moon_tables(K, 20, dt=30.0)
    models = spice_list(sun, moon)
    _, ref, st, steps = P.propagate_models_batch(y, *args, models)
    assert ref.nbytes > 256 << 20
    d = torch.device("cuda", 0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(d)  # noqa: E731
    dout = torch.empty(ref.shape, dtype=torch.float64, device=d)
    dst = torch.empty(n, dtype=torch.uint8, device=d)
    P.propagate_models_batch_device(T(y), *args, spice_list(T(sun), T(moon)), dout, dst)
    torch.cuda.synchronize()
    assert same(dout.cpu().numpy(), ref) and np.array_equal(dst.cpu().numpy(), st)
    pick = np.array([0, 1, 1940, 1941, 1942, 2999])
    _, o, s, c = M.propagate(y[pick], *args, models, k7_step_factor=True, threads=6)
    assert same(ref[pick], o) and np.array_equal(st[pick], s) and np.array_equal(steps[pick], c)


def test_batch_independence(dev):
    y = fixtures()
    K = len(_steps(0.0, 7200.0, 60.0))
    sun, moon = sun_moon_tables(K, 9)
    area = np.linspace(1, 30, len(y))
    models = lambda a: [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.ImprovedDrag(R_EQ, 2.2, a, 300.0, 1500.0, 150.0),  # noqa
                        P.SolarRadiationPressure(1.5, a, 600.0, R_EQ, sun), P.ThirdBody(MOON_MU, moon)]
    _, tr, st, steps = P.propagate_models_batch(y, 0.0, 7200.0, 60.0, models(area))
    perm = np.array([3, 1, 1, 5, 0, 5, 2, 4, 3])
    _, t2, s2, c2 = P.propagate_models_batch(y[perm], 0.0, 7200.0, 60.0, models(area[perm]))
    assert same(t2, tr[perm]) and np.array_equal(s2, st[perm]) and np.array_equal(c2, steps[perm])
    for i in range(len(y)):
        _, t1, s1, c1 = P.propagate_models_batch(y[i:i + 1], 0.0, 7200.0, 60.0, models(area[i:i + 1]))
        assert same(t1[0], tr[i]) and s1[0] == st[i] and np.array_equal(c1[0], steps[i])


def test_status_cases(dev):
    """DP87 stopped (a state at the centre), RK4 non-finite (a per-state mass of 0), and the substep limit; each equal to
    the restatement."""
    y = np.array([[7000.0, 0, 0, 0, 7.5, 0], [0.0, 0, 0, 0, 0, 0]])
    tb = [P.TwoBody(MU), P.ThirdBody(MOON_MU, (384400.0, 0, 0))]
    _, tr, st, _ = P.propagate_models_batch(y, 0.0, 600.0, 60.0, tb)
    _, ref, rst, _ = M.propagate(y, 0.0, 600.0, 60.0, tb, k7_step_factor=True)
    assert st.tolist() == [P.OK, P.STOPPED] and np.array_equal(st, rst) and same(tr, ref)
    assert (tr[1, 1:] == 0).all()
    srp = [P.TwoBody(MU), P.SolarRadiationPressure(1.5, 20.0, np.array([1000.0, 0.0]), R_EQ)]
    y2 = np.array([[7000.0, 0, 0, 0, 7.5, 0], [7100.0, 0, 0, 0, 7.4, 0]])
    _, tr, st, _ = P.propagate_models_batch(y2, 0.0, 600.0, 60.0, srp, integrator="rk4")
    _, ref, rst, _ = M.propagate(y2, 0.0, 600.0, 60.0, srp, integrator="rk4", k7_step_factor=True)
    assert st.tolist() == [P.OK, P.NON_FINITE] and np.array_equal(st, rst)
    assert np.array_equal(tr, ref, equal_nan=True)
    y3 = np.array([[7000.0, 0, 0, 0, 7.5, 0]])
    lst = [P.TwoBody(MU), P.ThirdBody(SUN_MU, (AU, 0, 0))]
    _, tr, st, steps = P.propagate_models_batch(y3, 0.0, 1.2e6, 1e6, lst, rtol=1e-14, atol=1e-14)
    _, ref, rst, rsteps = M.propagate(y3, 0.0, 1.2e6, 1e6, lst, rtol=1e-14, atol=1e-14, k7_step_factor=True)
    assert st[0] == P.SUBSTEP_LIMIT and np.array_equal(st, rst)
    assert np.array_equal(steps, rsteps) and same(tr, ref)
