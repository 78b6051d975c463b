"""K7 maneuvers on the device (maneuvers_kernel, astroz_b200/csrc/az_numerical.cu): against the scalar restatement
(tests/numerical_oracle/maneuvers.c) with both integrators, empty schedules against the model-list kernel, host vs device
calls over pageable and pinned buffers and several chunks, batch independence, the TRUNCATED rerun, and a catalogue's
states from propagate_pairs at each epoch with per-state burn sweeps."""
import math

import numpy as np
import pytest

from astroz_b200 import numerical as P
from tests.numerical_oracle import maneuvers as R
from tests.test_maneuvers_cpu import MU, SPACECRAFT, SPACECRAFT_SCHEDULES, T0_55909, TWO_BODY, Y55909, random_orbits, \
    same
from tests.test_numerical_models_cpu import J2, R_EQ

pytestmark = pytest.mark.gpu
EXP_FREE = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.ThirdBody(4902.8, (300000.0, 200000.0, 10000.0))]


@pytest.fixture(scope="module")
def dev():
    import astroz_b200

    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return 0


def sweeps(rng, n, kinds=("absolute", "prograde"), span=9000.0):
    out = []
    for i in range(n):
        s = []
        if "absolute" in kinds:
            s.append(P.Absolute(rng.uniform(-50, span), rng.uniform(-0.02, 0.02, 3)))
        if "prograde" in kinds:
            s += [P.Prograde(rng.uniform(0, span), rng.uniform(-0.05, 0.05)) for _ in range(2)]
        if "phase" in kinds and i % 2 == 0:   # phasing orbits whose perigee stays above the atmosphere's dense part
            s.append(P.Phase(rng.uniform(0, span), rng.uniform(-0.1, 0.1), rng.uniform(0.5, 1.5)))
        if "plane" in kinds:
            s.append(P.PlaneChange(rng.uniform(0, span), rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2)))
        out.append(s[::-1] if i % 3 == 0 else s)   # some lists unsorted
    return out


def within_drag_bound(a, b):
    """K7's drag bound: 1e-6 km / 1e-9 km/s relative to the orbit's scale"""
    assert np.isfinite(a).all() and np.isfinite(b).all()
    scale = np.maximum(1.0, np.abs(b[..., :3]).max(axis=(1, 2)) / 7000.0)[:, None, None]
    return np.max(np.abs(a[..., :3] - b[..., :3]) / scale) < 1e-6 and \
        np.max(np.abs(a[..., 3:] - b[..., 3:]) / scale) < 1e-9


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_exp_free_lists_with_absolute_and_prograde_burns_are_bit_identical(dev, integrator):
    rng = np.random.default_rng(4)
    y = random_orbits(rng, 64)
    sched = sweeps(rng, 64)
    ref = R.propagate(y, 50.0, 10800.0, 30.0, EXP_FREE, sched, integrator=integrator, k7_forms=True, threads=8)
    got = P.propagate_maneuvers_batch(y, 50.0, 10800.0, 30.0, EXP_FREE, sched, integrator=integrator,
                                      max_samples=ref[0].shape[1])
    for a, b in zip(got, ref):
        assert same(a, b)


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_drag_phasing_and_plane_changes_within_the_drag_bound(dev, integrator):
    rng = np.random.default_rng(9)
    y = random_orbits(rng, 48)
    y[:16] = [[(R_EQ + 450.0) * math.cos(a), (R_EQ + 450.0) * math.sin(a), 0.0, 0.0, 0.0,
               math.sqrt(MU / (R_EQ + 450.0))] for a in np.linspace(0, 6, 16)]   # circular, inside the drag cut-off
    sched = sweeps(rng, 48, kinds=("absolute", "prograde", "phase", "plane"))
    ref = R.propagate(y, 0.0, 21600.0, 20.0, SPACECRAFT, sched, integrator=integrator, k7_forms=True, threads=8)
    got = P.propagate_maneuvers_batch(y, 0.0, 21600.0, 20.0, SPACECRAFT, sched, integrator=integrator,
                                      max_samples=ref[0].shape[1])
    assert np.array_equal(got[2], ref[2]) and np.array_equal(got[3], ref[3]) and (ref[3][:16] == 0).all()
    assert np.array_equal(got[0], ref[0]) or np.max(np.abs(got[0] - ref[0])) < 1e-6
    assert within_drag_bound(got[1], ref[1])


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_spacecraft_schedules_match_the_restatement(dev, integrator):
    y = np.stack([Y55909] * 3)
    ref = R.propagate(y, T0_55909, 86400.0, 1.0, SPACECRAFT, SPACECRAFT_SCHEDULES, integrator=integrator,
                      k7_forms=True, threads=3)
    got = P.propagate_maneuvers_batch(y, T0_55909, 86400.0, 1.0, SPACECRAFT, SPACECRAFT_SCHEDULES,
                                      integrator=integrator)
    assert np.array_equal(got[2], ref[2]) and np.array_equal(got[3], ref[3])
    w = ref[0].shape[1]
    assert (got[0][:, w:] == 0).all() and np.max(np.abs(got[0][:, :w] - ref[0])) < 1e-6
    assert within_drag_bound(got[1][:, :w], ref[1])


@pytest.mark.parametrize("integrator", ["rk4", "dp87"])
def test_empty_schedules_give_the_model_list_bytes(dev, integrator):
    """Bit for bit up to the abnormal-orbit stop: a state whose perigee lies inside the atmosphere blows up under RK4's
    60 s steps, and the maneuver loop ends it at the first sample with positive energy, where K7 keeps integrating."""
    rng = np.random.default_rng(6)
    y = random_orbits(rng, 300)
    t, traj, st, steps = P.propagate_models_batch(y, 0.0, 14400.0, 60.0, SPACECRAFT, integrator=integrator)
    times, got, cnt, gst, gsteps = P.propagate_maneuvers_batch(y, 0.0, 14400.0, 60.0, SPACECRAFT, [],
                                                               integrator=integrator)
    full = gst != P.ABNORMAL
    assert full.sum() > 280 and same(got[full], traj[full]) and np.array_equal(gst[full], st[full])
    assert np.array_equal(gsteps[full], steps[full]) and (cnt[full] == len(t)).all()
    assert same(times[full], np.broadcast_to(t, times[full].shape))
    for i in np.flatnonzero(~full):
        c = int(cnt[i])
        last = traj[i, c - 1]
        r, v = np.linalg.norm(last[:3]), np.linalg.norm(last[3:])
        assert same(got[i, :c], traj[i, :c]) and (got[i, c:] == 0).all() and (0.5 * v * v - MU / r > 0 or r > 1e5)
        assert integrator == "dp87" or gsteps[i, 0] == c - 1   # one RK4 step per sample after the first


def test_host_and_device_calls_give_the_same_bytes(dev):
    """3,000 states over 2,900 samples of 56 bytes: two chunks of the host call.  Pageable and pinned destinations, and
    the device call on its own stream, agree."""
    import torch

    import astroz_b200

    rng = np.random.default_rng(2)
    n = 3000
    y = random_orbits(rng, n)
    area = rng.uniform(0.01, 5.0, n)
    models = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.Drag(R_EQ, 1.225, 7.249, 2.2, area, 300.0, 1000.0)]
    sched = sweeps(rng, n, kinds=("absolute", "prograde", "plane"), span=20000.0)
    args = (0.0, 28000.0, 10.0)
    ref = P.propagate_maneuvers_batch(y, *args, models, sched, max_samples=2900)
    assert ref[1].nbytes + ref[0].nbytes > 256 << 20
    pinned_y = astroz_b200.pinned_empty(y.shape)
    pinned_y[:] = y
    got = P.propagate_maneuvers_batch(pinned_y, *args, models, sched, max_samples=2900)
    for a, b in zip(got, ref):
        assert same(a, b)
    d = torch.device("cuda", 0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(d)  # noqa: E731
    dmodels = [P.TwoBody(MU), P.J2(MU, J2, R_EQ), P.Drag(R_EQ, 1.225, 7.249, 2.2, T(area), 300.0, 1000.0)]
    times = torch.empty((n, 2900), dtype=torch.float64, device=d)
    out = torch.empty((n, 2900, 6), dtype=torch.float64, device=d)
    cnt = torch.empty(n, dtype=torch.int64, device=d)
    st = torch.empty(n, dtype=torch.uint8, device=d)
    steps = torch.empty((n, 2), dtype=torch.int64, device=d)
    s = torch.cuda.Stream(device=d)
    torch.cuda.synchronize()
    P.propagate_maneuvers_batch_device(T(y), *args, dmodels, sched, times, out, cnt, st, steps,
                                       stream=s.cuda_stream)
    s.synchronize()
    assert same(times.cpu().numpy(), ref[0]) and same(out.cpu().numpy(), ref[1])
    assert np.array_equal(cnt.cpu().numpy().astype(np.uint64), ref[2]) and np.array_equal(st.cpu().numpy(), ref[3])
    assert np.array_equal(steps.cpu().numpy().astype(np.uint64), ref[4])
    with pytest.raises(ValueError, match="CUDA tensors"):
        P.propagate_maneuvers_batch_device(T(y), *args, models, sched, times, out, cnt, st)


def test_batch_independence(dev):
    rng = np.random.default_rng(8)
    y = random_orbits(rng, 200)
    sched = sweeps(rng, 200, kinds=("prograde", "phase", "plane"))
    full = P.propagate_maneuvers_batch(y, 0.0, 10800.0, 30.0, SPACECRAFT, sched, integrator="dp87", max_samples=900)
    idx = np.array([199, 3, 77, 150, 0])
    part = P.propagate_maneuvers_batch(y[idx], 0.0, 10800.0, 30.0, SPACECRAFT, [sched[i] for i in idx],
                                       integrator="dp87", max_samples=900)
    for a, b in zip(part, full):
        assert same(a, b[idx])


def test_truncated_states_rerun_to_the_ample_bytes(dev):
    rng = np.random.default_rng(12)
    y = random_orbits(rng, 40)
    sched = sweeps(rng, 40, kinds=("prograde",))
    # a phasing coast of three periods at the apogee of a raised orbit: longer than the estimate, which takes the
    # coast at the initial radius
    y[5] = [7000.0, 0.0, 0.0, 0.0, math.sqrt(MU / 7000.0), 0.0]
    sched[5] = [P.Prograde(0.0, 1.0), P.Phase(2000.0, 0.4, 3.0)]
    off, imp = P.pack_schedules(sched, len(y))
    ample = P.propagate_maneuvers_batch(y, 0.0, 7200.0, 30.0, TWO_BODY, sched, max_samples=200000)
    short = P.propagate_maneuvers_batch(y, 0.0, 7200.0, 30.0, TWO_BODY, sched, max_samples=100)
    assert (short[3] == P.TRUNCATED).any() and np.array_equal(short[2], ample[2])
    auto = P.propagate_maneuvers_batch(y, 0.0, 7200.0, 30.0, TWO_BODY, sched)
    w = int(ample[2].max())
    assert P._estimate_samples(y, 0.0, 7200.0, 30.0, off, imp, MU) < ample[2][5] == w
    assert auto[0].shape[1] >= w and np.array_equal(auto[3], ample[3]) and not (auto[3] == P.TRUNCATED).any()
    assert same(auto[0][:, :w], ample[0][:, :w]) and same(auto[1][:, :w], ample[1][:, :w])
    assert same(auto[4], ample[4])


def test_catalogue_states_from_propagate_pairs_with_burn_sweeps(dev):
    """Near-earth members of the mixed catalogue, each at its own epoch (TEME, propagate_pairs), each with its own sweep
    of prograde burn times and magnitudes, against the restatement."""
    from astroz_b200 import Constellation, synth

    tles = synth.mixed_catalog(512, n_geo=24, n_molniya=16, n_gps=8)
    c = Constellation(tles, device=0)
    near = np.flatnonzero(np.asarray(c.classes) == 0)[:96]
    ep = c.epochs[near]
    p, v, _ = c.propagate_pairs(near, np.floor(ep), ep - np.floor(ep))
    y = np.concatenate([p, v], axis=1)
    sched = [[P.Prograde(60.0 * (1 + k % 50), 0.001 * (1 + k % 7))] + ([P.PlaneChange(3000.0, 0.01, 0.0)]
                                                                        if k % 4 == 0 else []) for k in range(len(y))]
    for integ in ("rk4", "dp87"):
        ref = R.propagate(y, 0.0, 7200.0, 60.0, SPACECRAFT, sched, integrator=integ, k7_forms=True, threads=8)
        got = P.propagate_maneuvers_batch(y, 0.0, 7200.0, 60.0, SPACECRAFT, sched, integrator=integ,
                                          max_samples=ref[0].shape[1])
        assert np.array_equal(got[2], ref[2]) and np.array_equal(got[3], ref[3]) and (got[3] == 0).all()
        assert within_drag_bound(got[1], ref[1])
