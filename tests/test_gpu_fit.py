"""K8 on the device: element fits at catalogue scale, the residual invariant against create_from_elements +
propagate_pairs, batch invariance, host vs device bytes, a non-exact problem (J2 trajectories) against the CPU
restatement, and the statuses."""
import numpy as np
import pytest

from tests import fit_oracle as R

pytestmark = pytest.mark.gpu

N_SATS = 2000
N_OBS = 1440
MU, J2, REQ = 398600.8, 0.001082616, 6378.135   # WGS72 (src/constants.zig:41-50)


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def grid_case():
    """2,000 config-2 satellites, 1,440 observations each from the K1 grid (positions and velocities)."""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.constellation import Constellation, Layout

    tles = synth.near_earth_catalog(N_SATS)
    el = synth.elements_from_tles(tles)
    c = Constellation.from_elements(*el)
    jd, fr = synth.time_grid(N_OBS)
    pos, vel = c.propagate(jd, fr, layout=Layout.satelliteMajor)
    pos, vel = np.array(pos).reshape(-1, 3), np.array(vel).reshape(-1, 3)
    c.deinit()
    sat = np.repeat(np.arange(N_SATS), N_OBS)
    return el, sat, np.tile(jd, N_SATS), np.tile(fr, N_SATS), pos, vel


@pytest.fixture(scope="module")
def grid_fit(grid_case):
    from astroz_b200.fit import fit_elements

    el, sat, jd, fr, pos, vel = grid_case
    guess = R.perturbed(el, seed=3)
    return guess, fit_elements(guess, sat, jd, fr, pos, vel)


def _rms(c, sat, jd, fr, pos, vel, n):
    p, v, st = c.propagate_pairs(sat, jd, fr)
    dp = np.bincount(sat, ((np.asarray(p) - pos) ** 2).sum(1), minlength=n)
    dv = np.bincount(sat, ((np.asarray(v) - vel) ** 2).sum(1), minlength=n)
    cnt = np.bincount(sat, minlength=n)
    return np.sqrt(dp / cnt), np.sqrt(dv / cnt)


def test_round_trip_at_catalogue_scale(grid_case, grid_fit):
    el, *_ = grid_case
    guess, res = grid_fit
    ok = res.status == 0
    # A few low-perigee, high-drag sets (perigee < 220 km, B* > 5e-5) start so far off with B* doubled that 25 steps do
    # not bring them back (5 of these 2,000); they return their best iterate.  Every other set converges.
    assert ok.mean() >= 0.995, np.bincount(res.status)
    assert (res.status[~ok] == 1).all() and (res.iterations[~ok] == 25).all()
    assert (res.rms_pos[ok] < 1e-6).all(), res.rms_pos[ok].max()
    assert np.isfinite(res.elements).all() and np.isfinite(res.rms_pos).all() and (res.elements[0] == el[0]).all()
    assert np.abs(res.elements[1, ok] - el[1, ok]).max() < 1e-8


def test_residual_invariant_round_trip(grid_case, grid_fit):
    """The fitted columns through create_from_elements and propagate_pairs give back the reported RMS.  On this exact
    problem the RMS is rounding (1e-10 .. 1e-8 km), and the handle's own element init (host libm) and time model
    (reference epoch + offset) move it by rounding too: agreement to 1e-8 km absolute."""
    from astroz_b200.constellation import Constellation

    el, sat, jd, fr, pos, vel = grid_case
    _, res = grid_fit
    c = Constellation.from_elements(*res.elements)
    rp, rv = _rms(c, sat, jd, fr, pos, vel, N_SATS)
    c.deinit()
    assert np.abs(rp - res.rms_pos).max() < 1e-8
    assert np.abs(rv - res.rms_vel).max() < 1e-11


def test_batch_invariance_and_host_vs_device(grid_case, grid_fit):
    import torch

    from astroz_b200.fit import fit_elements, fit_elements_device

    el, sat, jd, fr, pos, vel = grid_case
    guess, res = grid_fit
    k = 64
    pick = np.array([0, 7, 1999, 1000] + list(range(100, 100 + k - 4)))
    rows = (sat[:, None] == pick[None, :]).any(1)
    # alone, one at a time
    for j in pick[:4]:
        m = sat == j
        one = fit_elements(guess[:, [j]], np.zeros(m.sum(), dtype=np.int64), jd[m], fr[m], pos[m], vel[m])
        assert one.elements[:, 0].tobytes() == res.elements[:, j].tobytes()
        assert one.rms_pos[0] == res.rms_pos[j] and one.rms_vel[0] == res.rms_vel[j]
        assert one.iterations[0] == res.iterations[j] and one.status[0] == res.status[j]
    # a permuted sub-batch, its observations interleaved across satellites (each satellite's own order kept: the
    # order of a satellite's observations is part of its input)
    perm = np.random.default_rng(5).permutation(k)
    remap = np.full(N_SATS, -1)
    remap[pick[perm]] = np.arange(k)
    shuffle = np.lexsort((remap[sat[rows]], np.tile(np.arange(N_OBS), k)))
    sub = fit_elements(guess[:, pick[perm]], remap[sat[rows]][shuffle], jd[rows][shuffle], fr[rows][shuffle],
                       pos[rows][shuffle], vel[rows][shuffle])
    assert sub.elements.tobytes() == res.elements[:, pick[perm]].tobytes()
    assert sub.rms_pos.tobytes() == res.rms_pos[pick[perm]].tobytes()
    assert sub.iterations.tobytes() == res.iterations[pick[perm]].tobytes()
    # the device call gives the host call's bytes
    dev = torch.device("cuda", 0)
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a)).to(dev, dt)  # noqa: E731
    offsets = np.searchsorted(sat, np.arange(N_SATS + 1)).astype(np.int32)
    fitted = torch.empty((8, N_SATS), dtype=torch.float64, device=dev)
    rms = torch.empty((N_SATS, 2), dtype=torch.float64, device=dev)
    iters = torch.empty(N_SATS, dtype=torch.int32, device=dev)
    status = torch.empty(N_SATS, dtype=torch.uint8, device=dev)
    fit_elements_device(t(guess), t(offsets, torch.int32), t(jd), t(fr), t(pos), t(vel), fitted, rms, iters, status)
    torch.cuda.synchronize()
    assert fitted.cpu().numpy().tobytes() == res.elements.tobytes()
    assert rms[:, 0].cpu().numpy().tobytes() == res.rms_pos.tobytes()
    assert iters.cpu().numpy().astype(np.uint32).tobytes() == res.iterations.tobytes()
    assert status.cpu().numpy().tobytes() == res.status.tobytes()


def k7_case(n, seed=0):
    """TEME states at epoch from K6, propagated one day at 1 min by K7 (TwoBody + J2, DP87): (elements, sat, jd, fr,
    pos, vel), the elements being the config-2 sets the states came from."""
    from astroz_b200 import synth
    from astroz_b200.constellation import Constellation
    from astroz_b200.numerical import propagate_numerical_batch

    el = synth.elements_from_tles(synth.near_earth_catalog(n, seed=13478 + seed))
    c = Constellation.from_elements(*el)
    ep = el[0]
    p0, v0, _ = c.propagate_pairs(np.arange(n), ep, np.zeros(n))
    c.deinit()
    states = np.concatenate([np.asarray(p0), np.asarray(v0)], axis=1)
    times, traj, st, _ = propagate_numerical_batch(states, 0.0, 86400.0, 60.0, MU, j2=J2, r_eq=REQ)
    assert (st == 0).all()
    m = len(times)
    sat = np.repeat(np.arange(n), m)
    return el, sat, np.repeat(ep, m), np.tile(times / 86400.0, n), traj[:, :, :3].reshape(-1, 3), \
        traj[:, :, 3:].reshape(-1, 3)


def test_non_exact_problem_against_restatement(record_property):
    _lib()
    from astroz_b200.fit import fit_elements

    n = 500
    el, sat, jd, fr, pos, vel = k7_case(n)
    res = fit_elements(el, sat, jd, fr, pos, vel)
    assert (res.status == 0).all(), np.bincount(res.status)
    assert np.isfinite(res.elements).all()
    # the RMS measures SGP4's model error against a J2 trajectory over one day
    record_property("k7_rms_pos_km_median_max", (float(np.median(res.rms_pos)), float(res.rms_pos.max())))
    print(f"K7 J2 trajectories: SGP4 fit RMS median {np.median(res.rms_pos):.4f} km, max {res.rms_pos.max():.4f} km")
    pick = np.arange(0, n, n // 20)[:20]
    rows = (sat[:, None] == pick[None, :]).any(1)
    remap = np.full(n, -1)
    remap[pick] = np.arange(20)
    off = R.csr(20, remap[sat[rows]])
    rf, rrms, riters, rst = R.fit(el[:, pick], off, jd[rows], fr[rows], pos[rows], vel[rows], threads=8)
    assert (rst == 0).all()
    f = res.elements[:, pick]
    dn = np.abs(f[1] - rf[1]).max() / np.abs(rf[1]).max()
    de = np.abs(f[2] - rf[2]).max() / np.abs(rf[2]).max()
    drms = np.abs(res.rms_pos[pick] / rrms[:, 0] - 1.0).max()
    print(f"against the restatement: n {dn:.1e}, e {de:.1e} relative, RMS {drms:.1e} relative")
    # The minimum is flat at this RMS: both fits stop once a step changes the cost by 1e-10 of it, at points that
    # differ by ~1e-7 in e.  Converged elements within 1e-6 relative (angles: of a turn), RMS within 1e-6 relative.
    assert dn <= 1e-6 and de <= 1e-6
    for c in (3, 4):
        assert np.abs((f[c] - rf[c] + 180.0) % 360.0 - 180.0).max() <= 360.0 * 1e-6
    assert np.abs((f[5] + f[6] - rf[5] - rf[6] + 180.0) % 360.0 - 180.0).max() <= 360.0 * 1e-6
    assert drms <= 1e-6


def test_residual_invariant_non_exact():
    """On the J2 trajectories the RMS is SGP4's model error (km): create_from_elements + propagate_pairs give it back
    to 1e-9 relative.  (Not to the bit: the handle initialises its elements with the host's libm and forms tsince from
    its reference epoch plus a per-satellite offset, which moves each state by ~1e-11 km.)"""
    _lib()
    from astroz_b200.constellation import Constellation
    from astroz_b200.fit import fit_elements

    n = 100
    el, sat, jd, fr, pos, vel = k7_case(n, seed=1)
    res = fit_elements(el, sat, jd, fr, pos, vel)
    c = Constellation.from_elements(*res.elements)
    rp, rv = _rms(c, sat, jd, fr, pos, vel, n)
    c.deinit()
    print(f"residual invariant: max relative RMS difference {np.abs(rp / res.rms_pos - 1.0).max():.2e}")
    assert np.abs(rp / res.rms_pos - 1.0).max() < 1e-9
    assert np.abs(rv / res.rms_vel - 1.0).max() < 1e-9


def test_statuses(grid_case, grid_fit):
    from astroz_b200.fit import fit_elements

    el, sat, jd, fr, pos, vel = grid_case
    guess, res = grid_fit
    a, b = 10, 11
    geo = guess[:, [a]].copy()
    geo[1] = 1.0027   # geostationary mean motion: deep space
    cols = np.concatenate([guess[:, [a]], geo, guess[:, [b]]], axis=1)
    ma, mb = sat == a, sat == b
    s3 = np.concatenate([np.zeros(ma.sum()), np.ones(ma.sum()), np.full(mb.sum(), 2)]).astype(np.int64)
    cat = lambda x: np.concatenate([x[ma], x[ma], x[mb]])  # noqa: E731
    out = fit_elements(cols, s3, cat(jd), cat(fr), cat(pos), cat(vel))
    assert out.status.tolist() == [0, 3, 0]
    assert out.elements[:, 0].tobytes() == res.elements[:, a].tobytes()
    assert out.elements[:, 2].tobytes() == res.elements[:, b].tobytes()
    assert out.rms_pos[[0, 2]].tobytes() == res.rms_pos[[a, b]].tobytes()
    assert (out.elements[:, 1] == geo[:, 0]).all() and out.rms_pos[1] == 0 and out.iterations[1] == 0
    # two positions: 6 scalar residuals < 7 variables
    few = fit_elements(guess[:, [a]], np.zeros(2, dtype=np.int64), jd[ma][:2], fr[ma][:2], pos[ma][:2])
    assert few.status.tolist() == [4]
    # observations of another satellite (another orbital plane): the step budget runs out, outputs stay finite
    inc = el[3]
    other = int(np.argmax(np.abs(inc - inc[a])))
    mo = sat == other
    wrong = fit_elements(guess[:, [a]], np.zeros(mo.sum(), dtype=np.int64), jd[mo], fr[mo], pos[mo], vel[mo],
                         max_iter=8)
    assert wrong.status.tolist() == [1] and wrong.iterations[0] == 8
    assert np.isfinite(wrong.elements).all() and np.isfinite(wrong.rms_pos).all() and wrong.rms_pos[0] > 1.0
