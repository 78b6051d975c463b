"""K7 on the device (astroz_b200/csrc/az_numerical.cu): against the scalar restatement on a mixed batch for both
integrators and all four force sets, under reordering and duplication, host vs device calls over every kind of
destination and several chunks, the reference-shaped frontend call, and argument errors."""
import numpy as np
import pytest

from tests import numerical_oracle as N
from tests.test_numerical_host_emulation import J2, MU, R_EQ, STIFF, fixtures

pytestmark = pytest.mark.gpu
FORCES = {"none": {}, "j2": {"j2": J2, "r_eq": R_EQ}, "drag": {"r_eq": R_EQ}, "j2drag": {"j2": J2, "r_eq": R_EQ}}


@pytest.fixture(scope="module")
def num():
    import astroz_b200
    from astroz_b200 import numerical

    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return numerical


def _batch():
    y = fixtures()   # the 150 km perigee state once more, with the largest area
    return np.concatenate([y, y[2:3]]), np.linspace(1.0, 30.0, len(y) + 1)


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
@pytest.mark.parametrize("forces", list(FORCES))
def test_k7_matches_the_restatement(num, integrator, forces):
    """Against the restatement with K7's step factor (three square roots instead of pow, the one operation K7 forms
    differently): without drag the device is bit-identical (no contraction, IEEE sqrt and division on both sides) in
    states, steps and status, including the stopped state at the centre and RK4's non-finite one.  With drag the device's
    exp differs from glibc's in the last place: 1e-6 km / 1e-9 km/s relative to the orbit's scale and equal counts,
    except the stiff crawl (row STIFF), whose error norm hovers around 1.0 so last-bit differences flip some decisions:
    equal status, counts within 1 %."""
    y, area = _batch()
    kw = dict(FORCES[forces])
    if "drag" in forces:
        kw.update(drag_cd=2.2, drag_area=area, drag_mass=300.0)
    t, tr, st, steps = num.propagate_numerical_batch(y, 0.0, 21600.0, 60.0, MU, integrator=integrator, **kw)
    rt, ref, rst, rsteps = N.propagate(y, 0.0, 21600.0, 60.0, MU, integrator=integrator, k7_step_factor=True, **kw)
    assert np.array_equal(t, rt) and np.array_equal(st, rst)
    assert st[6] == (num.STOPPED if integrator == "dp87" else num.NON_FINITE)
    if "drag" not in forces:
        assert np.array_equal(steps, rsteps) and np.array_equal(tr, ref, equal_nan=True)
        return
    calm = np.isfinite(ref).all(axis=(1, 2)) & (np.arange(len(y)) != STIFF)
    assert np.array_equal(steps[calm], rsteps[calm])
    assert np.all(np.abs(steps[STIFF].astype(float) - rsteps[STIFF]) <= 0.01 * rsteps[STIFF].sum())
    scale = np.maximum(1.0, np.abs(ref[calm][..., :3]).max(axis=(1, 2)) / 7000.0)[:, None, None]
    assert np.max(np.abs(tr[calm][..., :3] - ref[calm][..., :3]) / scale) < 1e-6
    assert np.max(np.abs(tr[calm][..., 3:] - ref[calm][..., 3:]) / scale) < 1e-9


def test_k7_substep_limit(num):
    """The 10,000-substep cap on the device: bit-identical to the restatement with K7's step factor (no drag, no exp)."""
    y = np.array([[7000.0, 0, 0, 0, 7.5, 0], [6778.0, 0, 0, 0, 7.67, 0.1]])
    _, tr, st, steps = num.propagate_numerical_batch(y, 0.0, 1.2e6, 1e6, MU, rtol=1e-14, atol=1e-14)
    _, ref, rst, rsteps = N.propagate(y, 0.0, 1.2e6, 1e6, MU, rtol=1e-14, atol=1e-14, k7_step_factor=True)
    assert (st == num.SUBSTEP_LIMIT).all() and np.array_equal(st, rst)
    assert np.array_equal(steps, rsteps) and np.array_equal(tr, ref)


def test_batch_independence(num):
    y, area = _batch()
    kw = dict(j2=J2, r_eq=R_EQ, drag_cd=2.2, drag_mass=300.0)
    _, tr, st, steps = num.propagate_numerical_batch(y, 0.0, 7200.0, 60.0, MU, drag_area=area, **kw)
    perm = np.array([3, 1, 1, 7, 0, 5, 2, 4, 3, 6, 6, 8])
    _, t2, s2, c2 = num.propagate_numerical_batch(y[perm], 0.0, 7200.0, 60.0, MU, drag_area=area[perm], **kw)
    assert np.array_equal(t2, tr[perm]) and np.array_equal(s2, st[perm]) and np.array_equal(c2, steps[perm])
    for i in range(len(y)):
        _, t1, s1, c1 = num.propagate_numerical_batch(y[i:i + 1], 0.0, 7200.0, 60.0, MU, drag_area=area[i], **kw)
        assert np.array_equal(t1[0], tr[i]) and s1[0] == st[i] and np.array_equal(c1[0], steps[i])


def test_host_and_device_calls_give_the_same_bytes(num):
    """2,000 two-body + J2 RK4 states over 4,000 samples: 384 MB of trajectories, two chunks of the host call and twelve
    ring pieces for a pageable destination; pinned, registered and pageable destinations and the device call agree."""
    import torch

    import astroz_b200

    rng = np.random.default_rng(1)
    n = 2000
    y = np.array(fixtures()[:5])[rng.integers(0, 5, n)] * (1 + 1e-4 * rng.standard_normal((n, 6)))
    args = (0.0, 39990.0, 10.0, MU)
    _, ref, st, steps = num.propagate_numerical_batch(y, *args, j2=J2, r_eq=R_EQ, integrator="rk4")
    assert ref.nbytes > 256 << 20
    pinned = astroz_b200.pinned_empty(ref.shape)
    _, out, _, _ = num.propagate_numerical_batch(y, *args, j2=J2, r_eq=R_EQ, integrator="rk4", out=pinned)
    assert np.array_equal(out, ref)
    reg = np.empty(ref.shape)
    astroz_b200.host_register(reg)
    try:
        num.propagate_numerical_batch(y, *args, j2=J2, r_eq=R_EQ, integrator="rk4", out=reg)
        assert np.array_equal(reg, ref)
    finally:
        astroz_b200.host_unregister(reg)
    dev = torch.device("cuda", 0)
    ds = torch.from_numpy(y).to(dev)
    dout = torch.empty(ref.shape, dtype=torch.float64, device=dev)
    dst = torch.empty(n, dtype=torch.uint8, device=dev)
    dsteps = torch.empty((n, 2), dtype=torch.int64, device=dev)
    num.propagate_numerical_batch_device(ds, *args, dout, dst, dsteps, j2=J2, r_eq=R_EQ, integrator="rk4")
    torch.cuda.synchronize()
    assert np.array_equal(dout.cpu().numpy(), ref) and np.array_equal(dst.cpu().numpy(), st)
    assert np.array_equal(dsteps.cpu().numpy().astype(np.uint64), steps)
    # drag arrays as device tensors, DP87
    yd, area = _batch()
    kw = dict(j2=J2, r_eq=R_EQ, drag_cd=2.2, drag_mass=300.0)
    _, h, hs, hc = num.propagate_numerical_batch(yd, 0.0, 3600.0, 60.0, MU, drag_area=area, **kw)
    m = len(yd)
    dd = [torch.full((m,), 2.2, dtype=torch.float64, device=dev), torch.from_numpy(area).to(dev),
          torch.full((m,), 300.0, dtype=torch.float64, device=dev)]
    o = torch.empty(h.shape, dtype=torch.float64, device=dev)
    s = torch.empty(m, dtype=torch.uint8, device=dev)
    num.propagate_numerical_batch_device(torch.from_numpy(yd).to(dev), 0.0, 3600.0, 60.0, MU, o, s, j2=J2, r_eq=R_EQ,
                                         drag_cd=dd[0], drag_area=dd[1], drag_mass=dd[2])
    torch.cuda.synchronize()
    assert np.array_equal(o.cpu().numpy(), h) and np.array_equal(s.cpu().numpy(), hs)


def test_frontend_is_row_zero_of_the_batch(num):
    from astroz_b200 import frontend

    y = fixtures()[2]
    times, states = frontend.propagate_numerical(tuple(y), 0.0, 5400.0, 60.0, frontend.EARTH_MU, j2=frontend.EARTH_J2,
                                                 r_eq=frontend.EARTH_R_EQ, drag_cd=2.2, drag_area=4.0, drag_mass=300.0)
    t, tr, _, _ = num.propagate_numerical_batch([y], 0.0, 5400.0, 60.0, MU, j2=J2, r_eq=R_EQ, drag_cd=2.2,
                                                drag_area=4.0, drag_mass=300.0)
    assert type(times) is list and type(states) is list and type(states[0]) is tuple and type(states[0][0]) is float
    assert times == t.tolist() and np.array_equal(np.array(states), tr[0])
    with pytest.raises(ValueError, match="exactly 6"):
        frontend.propagate_numerical([1, 2, 3], 0.0, 10.0, 1.0, MU)
    with pytest.raises(ValueError, match="r_eq is required"):
        frontend.propagate_numerical(tuple(y), 0.0, 10.0, 1.0, MU, j2=J2)
    with pytest.raises(ValueError, match="drag_area and drag_mass"):
        frontend.propagate_numerical(tuple(y), 0.0, 10.0, 1.0, MU, r_eq=R_EQ, drag_cd=2.2)
    with pytest.raises(ValueError, match="integrator"):
        frontend.propagate_numerical(tuple(y), 0.0, 10.0, 1.0, MU, integrator="rk45")
    with pytest.raises(RuntimeError, match="stopped"):
        frontend.propagate_numerical((0.0,) * 6, 0.0, 120.0, 60.0, MU)
    # positional, as a migrated astroz call passes them; None selects the default tolerances
    pos = frontend.propagate_numerical(tuple(y), 0.0, 5400.0, 60.0, frontend.EARTH_MU, frontend.EARTH_J2,
                                       frontend.EARTH_R_EQ, 2.2, 4.0, 300.0, "dp87", None, None)
    assert pos == (times, states)


def test_empty_batch_and_errors(num):
    t, tr, st, steps = num.propagate_numerical_batch(np.zeros((0, 6)), 0.0, 100.0, 10.0, MU)
    assert tr.shape == (0, 11, 6) and st.shape == (0,) and len(t) == 11
    with pytest.raises(num.AstrozCudaError):
        num.propagate_numerical_batch(np.zeros((1, 6)), 0.0, 100.0, 0.0, MU)
    with pytest.raises(num.AstrozCudaError):
        num.propagate_numerical_batch(np.zeros((1, 6)), 0.0, 100.0, 10.0, MU, r_eq=R_EQ, drag_cd=1.0, drag_area=1.0,
                                      drag_mass=1.0, device=-1)
