"""Deep-space element fits on the device (fit_deep_kernel through the _mixed exports): near-earth rows byte-identical to
the near-earth call, the 1,536 config-3 deep-space sets fitted from their own K2 grid, the residual invariant through
create_from_elements + propagate_pairs, batch invariance and host vs device bytes, and GPS-like K7 trajectories
against the CPU restatement."""
import numpy as np
import pytest

from tests import fit_oracle as R
from tests.fit_oracle import deep as D

pytestmark = pytest.mark.gpu

N_OBS = 1440
MU, J2, REQ = 398600.8, 0.001082616, 6378.135   # WGS72


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def config3():
    """BASELINE config 3 (13,478 sets, 1,536 deep space), 1,440 observations each from the K1 / K2 grid."""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.constellation import Constellation, Layout

    el = synth.elements_from_tles(synth.mixed_catalog(13478))
    c = Constellation.from_elements(*el)
    jd, fr = synth.time_grid(N_OBS)
    pos, vel = c.propagate(jd, fr, layout=Layout.satelliteMajor)
    c.deinit()
    n = el.shape[1]
    deep = 1440.0 / el[1] > 225.0
    return el, deep, np.repeat(np.arange(n), N_OBS), np.tile(jd, n), np.tile(fr, n), \
        np.array(pos).reshape(-1, 3), np.array(vel).reshape(-1, 3)


@pytest.fixture(scope="module")
def deep_case(config3):
    """The deep-space sets alone: (elements, guess, sat, jd, fr, pos, vel), B* held at its generating value (one day of
    GEO or GPS observations does not constrain drag: with B* free, a quarter of them stop at the step limit)."""
    el, deep, sat, jd, fr, pos, vel = config3
    idx = np.flatnonzero(deep)
    rows = deep[sat]
    remap = np.full(el.shape[1], -1)
    remap[idx] = np.arange(len(idx))
    guess = R.perturbed(el, seed=3)[:, idx]
    guess[7] = el[7, idx]
    return el[:, idx], guess, remap[sat[rows]], jd[rows], fr[rows], pos[rows], vel[rows]


@pytest.fixture(scope="module")
def deep_fit(deep_case):
    from astroz_b200.fit import fit_elements

    el, guess, sat, jd, fr, pos, vel = deep_case
    return fit_elements(guess, sat, jd, fr, pos, vel, fit_bstar=False, deep_space=True)


def test_near_earth_rows_are_the_near_earth_call_bytes(config3):
    from astroz_b200.fit import fit_elements

    el, deep, sat, jd, fr, pos, vel = config3
    guess = R.perturbed(el, seed=3)
    near = fit_elements(guess, sat, jd, fr, pos, vel)
    mixed = fit_elements(guess, sat, jd, fr, pos, vel, deep_space=True)
    assert (near.status[deep] == R.DEEP_SPACE).all() and not (mixed.status == R.DEEP_SPACE).any()
    ne = ~deep
    assert mixed.elements[:, ne].tobytes() == near.elements[:, ne].tobytes()
    assert mixed.rms_pos[ne].tobytes() == near.rms_pos[ne].tobytes()
    assert mixed.rms_vel[ne].tobytes() == near.rms_vel[ne].tobytes()
    assert mixed.iterations[ne].tobytes() == near.iterations[ne].tobytes()
    assert mixed.status[ne].tobytes() == near.status[ne].tobytes()


def test_round_trip_of_config3_deep_space_sets(deep_case, deep_fit):
    el, guess, *_ = deep_case
    res = deep_fit
    assert len(res.status) == 1536
    print(f"deep-space round trip: status {np.bincount(res.status, minlength=5).tolist()}, iterations "
          f"{np.bincount(res.iterations).tolist()}, RMS max {res.rms_pos.max():.2e} km")
    # SDP4 raises a mean eccentricity below 1e-6 to 1e-6, so the model is flat in (e cos, e sin) there: 3 GEO sets of
    # config 3 have e < 1e-6, and 2 of them stop at the step limit (RMS 1e-4 and 0.1 km on the CPU restatement as
    # well).  Every set with e >= 1e-6 converges.
    tiny = el[2] < 1e-6
    assert tiny.sum() == 3
    assert (res.status[~tiny] == R.CONVERGED).all(), np.bincount(res.status, minlength=5)
    assert (res.status[tiny] <= R.ITERATION_LIMIT).all() and (res.status[tiny] == R.CONVERGED).sum() >= 1
    assert (res.rms_pos[~tiny] < 1e-6).all(), res.rms_pos[~tiny].max()
    assert np.isfinite(res.elements).all() and (res.elements[0] == el[0]).all()
    assert np.abs(res.elements[1] - el[1]).max() < 1e-8


def _rms(c, sat, jd, fr, pos, vel, n):
    p, v, st = c.propagate_pairs(sat, jd, fr)
    assert (np.asarray(st) == 0).all()
    dp = np.bincount(sat, ((np.asarray(p) - pos) ** 2).sum(1), minlength=n)
    dv = np.bincount(sat, ((np.asarray(v) - vel) ** 2).sum(1), minlength=n)
    cnt = np.bincount(sat, minlength=n)
    return np.sqrt(dp / cnt), np.sqrt(dv / cnt)


def test_residual_invariant(deep_case, deep_fit):
    """The fitted columns through create_from_elements + propagate_pairs give back the reported RMS.  The handle
    initialises its deep-space records with the host's libm, the fit with the device's; on this exact problem the RMS
    is rounding (~1e-8 km), so the agreement is absolute.  Measured on an H100: see the printed line."""
    from astroz_b200.constellation import Constellation

    el, guess, sat, jd, fr, pos, vel = deep_case
    res = deep_fit
    c = Constellation.from_elements(*res.elements)
    rp, rv = _rms(c, sat, jd, fr, pos, vel, el.shape[1])
    c.deinit()
    print(f"residual invariant: max |RMS difference| {np.abs(rp - res.rms_pos).max():.2e} km, "
          f"{np.abs(rv - res.rms_vel).max():.2e} km/s")
    assert np.abs(rp - res.rms_pos).max() < 1e-7
    assert np.abs(rv - res.rms_vel).max() < 1e-10


def test_batch_invariance_and_host_vs_device(deep_case, deep_fit):
    import torch

    from astroz_b200.fit import fit_elements, fit_elements_device

    el, guess, sat, jd, fr, pos, vel = deep_case
    res = deep_fit
    n = el.shape[1]
    for j in (0, 1100, 1535):
        m = sat == j
        one = fit_elements(guess[:, [j]], np.zeros(m.sum(), dtype=np.int64), jd[m], fr[m], pos[m], vel[m],
                           fit_bstar=False, deep_space=True)
        assert one.elements[:, 0].tobytes() == res.elements[:, j].tobytes()
        assert one.rms_pos[0] == res.rms_pos[j] and one.iterations[0] == res.iterations[j]
    pick = np.random.default_rng(7).permutation(n)[:48]
    rows = (sat[:, None] == pick[None, :]).any(1)
    remap = np.full(n, -1)
    remap[pick] = np.arange(len(pick))
    sub = fit_elements(guess[:, pick], remap[sat[rows]], jd[rows], fr[rows], pos[rows], vel[rows], fit_bstar=False,
                       deep_space=True)
    assert sub.elements.tobytes() == res.elements[:, pick].tobytes()
    assert sub.rms_pos.tobytes() == res.rms_pos[pick].tobytes()
    assert sub.iterations.tobytes() == res.iterations[pick].tobytes()
    dev = torch.device("cuda", 0)
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a)).to(dev, dt)  # noqa: E731
    offsets = np.searchsorted(sat, np.arange(n + 1)).astype(np.int32)
    fitted = torch.empty((8, n), dtype=torch.float64, device=dev)
    rms = torch.empty((n, 2), dtype=torch.float64, device=dev)
    iters = torch.empty(n, dtype=torch.int32, device=dev)
    status = torch.empty(n, dtype=torch.uint8, device=dev)
    fit_elements_device(t(guess), t(offsets, torch.int32), t(jd), t(fr), t(pos), t(vel), fitted, rms, iters, status,
                        fit_bstar=False, deep_space=True)
    torch.cuda.synchronize()
    assert fitted.cpu().numpy().tobytes() == res.elements.tobytes()
    assert rms[:, 0].cpu().numpy().tobytes() == res.rms_pos.tobytes()
    assert iters.cpu().numpy().astype(np.uint32).tobytes() == res.iterations.tobytes()
    assert status.cpu().numpy().tobytes() == res.status.tobytes()


def test_gps_like_k7_trajectories_against_restatement():
    """200 GPS-like states from K6, propagated one day at 1 min by K7 (TwoBody + J2), fitted with B* held, against the
    restatement on 20 of them."""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.constellation import Constellation
    from astroz_b200.fit import fit_elements
    from astroz_b200.numerical import propagate_numerical_batch

    el = synth.elements_from_tles(synth.mixed_catalog(13478))
    el = el[:, (np.abs(el[1] - 2.0056) < 0.001) & (el[2] < 0.05)][:, :200]
    n = el.shape[1]
    assert n == 200
    c = Constellation.from_elements(*el)
    ep = el[0]
    p0, v0, _ = c.propagate_pairs(np.arange(n), ep, np.zeros(n))
    c.deinit()
    states = np.concatenate([np.asarray(p0), np.asarray(v0)], axis=1)
    times, traj, st, _ = propagate_numerical_batch(states, 0.0, 86400.0, 60.0, MU, j2=J2, r_eq=REQ)
    assert (st == 0).all()
    m = len(times)
    sat = np.repeat(np.arange(n), m)
    jd, fr = np.repeat(ep, m), np.tile(times / 86400.0, n)
    pos, vel = traj[:, :, :3].reshape(-1, 3), traj[:, :, 3:].reshape(-1, 3)
    res = fit_elements(el, sat, jd, fr, pos, vel, fit_bstar=False, deep_space=True)
    print(f"GPS-like K7 J2 trajectories: status {np.bincount(res.status, minlength=5).tolist()}, SDP4 fit RMS median "
          f"{np.median(res.rms_pos):.4f} km, max {res.rms_pos.max():.4f} km")
    assert np.isfinite(res.elements).all() and (res.status <= R.ITERATION_LIMIT).all()
    pick = np.arange(0, n, n // 20)[:20]
    rows = (sat[:, None] == pick[None, :]).any(1)
    remap = np.full(n, -1)
    remap[pick] = np.arange(20)
    off = R.csr(20, remap[sat[rows]])
    rf, rrms, riters, rst = D.fit_mixed(el[:, pick], off, jd[rows], fr[rows], pos[rows], vel[rows], fit_bstar=False,
                                        threads=8)
    f = res.elements[:, pick]
    dn = np.abs(f[1] - rf[1]).max() / np.abs(rf[1]).max()
    de = np.abs(f[2] - rf[2]).max() / max(np.abs(rf[2]).max(), 1e-6)
    drms = np.abs(res.rms_pos[pick] / rrms[:, 0] - 1.0).max()
    print(f"against the restatement: status {res.status[pick].tolist()} vs {rst.tolist()}; n {dn:.1e}, "
          f"e {de:.1e} relative, RMS {drms:.1e} relative")
    assert res.status[pick].tolist() == rst.tolist()
    # The cost minimum is flat at SDP4's model error against a J2 trajectory (km), as for the near-earth fit of K7
    # trajectories: both fits stop where a step changes the cost by 1e-10 of it.  Bounds as the near-earth test's.
    assert dn <= 1e-6 and de <= 1e-5 and drms <= 1e-6
