"""K18 sensor tasking on the device (task_score_kernel, task_score_deep_kernel, task_select_kernel): the device against
the host build of the same source on a mixed scene of radar and optical sensors over a day; pageable / pinned /
device-call and row-permutation byte identity; a closed loop that observes the planned tasks from a truth drawn from
each row's covariance and checks the pointing, the search window and K12's gate."""
import numpy as np
import pytest
from scipy import stats

from tests.fit_oracle import conjunction_mc as mc
from tests.fit_oracle import covariance as K
from tests.fit_oracle import obs as O
from tests.fit_oracle import tasking as TK

pytestmark = pytest.mark.gpu
# The Jacobians are forward differences over 1e-8-scale steps, and the device contracts their arithmetic into FMAs
# where the host build does not: gains agree to about 1e-6 relative, so ties are judged at 1e-5.
REL = 1e-5


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def emul():
    _lib()
    L = TK.emul_library()
    if L is None:
        pytest.skip("nvcc unavailable")
    return L


@pytest.fixture(scope="module")
def scene():
    """about 1,000 mixed rows x 6 radars + 3 optical sites x 1 day at 2 minutes"""
    return TK.scene(n_per=250, T=720, step_min=2.0, radar=O.RADAR_SITES, optical=TK.OPTICAL_SITES, seed=5)


def _plan(sc, **kw):
    from astroz_b200.tasking import plan

    sens = [_sensor(sc, k) for k in range(sc.S)]
    return plan(sc.el, sens, sc.jd, sc.fr, sun=sc.sun, covariance=sc.P, model=sc.model, **kw)


def _sensor(sc, k):
    from astroz_b200.tasking import Sensor

    lim = sc.limits[k]
    return Sensor(int(sc.kind[k]), *sc.stations[sc.station[k]], sigma=tuple(sc.sigma[k]), el_min=np.rad2deg(lim[0]),
                  range_max=lim[1], sun_el_max=np.rad2deg(lim[2]), exclusion=np.rad2deg(lim[3]))


def test_device_against_the_host_build(emul, scene):
    """visibility counts, failures and statuses equal; task gains and posteriors within 1e-5 relative; the schedules equal up to the
    first slot where two candidates' gains lie within that tolerance (reported and asserted to be such a tie)"""
    dev = _plan(scene)
    host = TK.emul(emul, scene)
    assert np.array_equal(dev.row_status, host["row_status"])
    assert np.array_equal(dev.n_visible, host["n_visible"])
    assert np.array_equal(dev.n_failed, host["n_failed"])
    hrow = np.where(host["task_row"] == TK.IDLE, -1, host["task_row"].astype(np.int64))
    diff = np.nonzero(np.any(dev.task_row != hrow, axis=0))[0]
    first = int(diff[0]) if len(diff) else scene.T
    print(f"schedules equal over slots [0, {first}) of {scene.T}; tasks {np.sum(hrow >= 0)}")
    same = slice(0, first)
    assert np.array_equal(dev.n_candidates[:, same], host["n_candidates"][:, same])
    g1, g2 = dev.task_gain[:, same], host["task_gain"][:, same]
    rel = np.abs(g1 - g2) / np.maximum(np.abs(g2), 1e-300)
    print(f"task gains: largest relative difference {rel.max():.2e}")
    assert np.all(rel <= REL)
    if first < scene.T:   # the first difference must be a tie within the tolerance
        k = int(np.nonzero(dev.task_row[:, first] != hrow[:, first])[0][0])
        a, b = dev.task_gain[k, first], host["task_gain"][k, first]
        assert abs(a - b) <= REL * abs(b), (first, k, a, b)
    if first == scene.T:
        scale = np.abs(host["posterior"]).max(axis=1, keepdims=True)
        dp = np.abs(dev.posterior - host["posterior"]) / np.maximum(scale, 1e-300)
        print(f"posteriors: largest difference {dp.max():.2e} of the row's largest word")
        assert np.all(dp <= REL)


def test_call_forms_and_row_permutation_are_byte_identical(scene):
    """pageable, pinned and the device call give identical bytes; permuted rows give the same schedule relabelled"""
    import torch

    from astroz_b200.tasking import plan, plan_device, plan_scratch_bytes

    sc = TK.scene(n_per=60, T=180, step_min=4.0, radar=O.RADAR_SITES[:3], optical=TK.OPTICAL_SITES[:2], seed=9)
    a = _plan(sc)
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory().numpy()  # noqa: E731
    sens = [_sensor(sc, k) for k in range(sc.S)]
    b = plan(pin(sc.el), sens, pin(sc.jd), pin(sc.fr), sun=pin(sc.sun), covariance=pin(sc.P), model=pin(sc.model))
    for f in ("task_row", "task_gain", "task_value", "task_spread", "n_candidates", "posterior", "n_tasks",
              "n_visible", "n_failed", "row_status"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    d = torch.device("cuda", 0)
    tt = lambda x, dt=torch.float64: torch.from_numpy(np.ascontiguousarray(x)).to(dt).to(d)  # noqa: E731
    n, S, T = sc.n, sc.S, sc.T
    out = dict(task_row=torch.zeros((S, T), dtype=torch.int32, device=d),
               task_gain=torch.zeros((S, T), dtype=torch.float64, device=d),
               task_value=torch.zeros((S, T, 4), dtype=torch.float64, device=d),
               task_spread=torch.zeros((S, T, 4), dtype=torch.float64, device=d),
               n_candidates=torch.zeros((S, T), dtype=torch.int32, device=d),
               posterior=torch.zeros((n, 28), dtype=torch.float64, device=d),
               n_tasks=torch.zeros(n, dtype=torch.int32, device=d), n_visible=torch.zeros(n, dtype=torch.int32, device=d),
               n_failed=torch.zeros(n, dtype=torch.int32, device=d), row_status=torch.zeros(n, dtype=torch.uint8, device=d))
    scratch = torch.zeros(plan_scratch_bytes(n, S), dtype=torch.uint8, device=d)
    plan_device(tt(sc.el), tt(sc.P), tt(sc.model, torch.uint8), tt(sc.kind, torch.uint8),
                tt(sc.station.astype(np.int32), torch.int32), tt(sc.sigma), tt(sc.limits), tt(sc.stations),
                tt(sc.jd), tt(sc.fr), tt(sc.sun), scratch, *out.values())
    torch.cuda.synchronize()
    assert np.array_equal(out["task_row"].cpu().numpy().astype(np.int64), a.task_row)
    for f in ("task_gain", "task_value", "task_spread", "posterior"):
        assert np.array_equal(out[f].cpu().numpy(), getattr(a, f)), f
    for f in ("n_candidates", "n_tasks", "n_visible", "n_failed", "row_status"):
        assert np.array_equal(out[f].cpu().numpy().astype(np.int64), getattr(a, f).astype(np.int64)), f
    perm = np.random.default_rng(2).permutation(n)
    c = plan(sc.el[:, perm], sens, sc.jd, sc.fr, sun=sc.sun, covariance=sc.P[perm], model=sc.model[perm])
    relabel = np.where(c.task_row >= 0, perm[np.maximum(c.task_row, 0)], -1)
    assert np.array_equal(relabel, a.task_row)
    assert np.array_equal(c.task_gain, a.task_gain)
    assert np.array_equal(c.posterior, a.posterior[perm])


def test_closed_loop_pointing_window_and_gate():
    """truth = each row plus a draw from its P; the planned tasks observed from the truth with noise at the sensors'
    sigmas: every innovation lies within 4 x sqrt(spread^2 + sigma^2) per component, and as a one-observation track
    the tasked row is inside K12's 0.99 gate for a fraction consistent with 0.99"""
    from astroz_b200.constellation import Constellation
    from astroz_b200.correlate import correlate
    from astroz_b200.fit import observe

    sc = TK.scene(n_per=100, T=240, step_min=3.0, radar=O.RADAR_SITES[:4], optical=TK.OPTICAL_SITES, seed=21)
    p = _plan(sc)
    rng = np.random.default_rng(4)
    truth = sc.el.copy()
    for s in range(sc.n):
        deep = bool(sc.model[s])
        Pm = K.unpack7(sc.P[s])
        w, V = np.linalg.eigh(Pm)
        x = mc.vars_of(sc.el[:, s], deep) + V @ (np.sqrt(np.maximum(w, 0)) * rng.standard_normal(7))
        truth[:, s] = K.elements_of(x, sc.el[0, s], deep)
    sat, jd, fr, kind, station, value, sigma = p.tasks()
    m = len(sat)
    assert m > 200
    c = Constellation.from_elements(*truth)
    pos, vel, st = c.propagate_pairs(sat, jd, fr)
    c.deinit()
    states = np.concatenate([np.asarray(pos), np.asarray(vel)], axis=1)
    meas = observe(states, jd, fr, kind, station, p.stations)
    used = np.isfinite(sigma)
    meas[used] += rng.standard_normal(used.sum()) * sigma[used]
    inn = meas - value
    wrap = np.where(kind == O.RADAR, 1, 0)
    inn[np.arange(m), wrap] = (inn[np.arange(m), wrap] + np.pi) % (2 * np.pi) - np.pi
    partner = np.where(kind == O.RADAR, 2, 1)
    inn[np.arange(m), wrap] *= np.cos(value[np.arange(m), partner])
    tt, kk = np.nonzero(p.task_row.T >= 0)   # the order of tasks()
    spread = p.task_spread[kk, tt]
    sig = np.where(used[:, :4], sigma[:, :4], 0.0)
    sig[np.arange(m), wrap] *= np.cos(value[np.arange(m), partner])
    bound = 4 * np.sqrt(spread ** 2 + sig ** 2)
    # a row's first task is predicted under the covariance the truth was drawn from; later ones under its posterior
    first = np.unique(sat, return_index=True)[1]
    u4 = used[first, :4]
    ratio = np.abs(inn[first, :4])[u4] / bound[first][u4]
    print(f"tasks {m}, first tasks {len(first)}, largest innovation / 4-sigma window {ratio.max():.3f}")
    assert np.all(ratio <= 1.0)
    res = correlate(sc.el, np.arange(m), jd, fr, kind, meas, sigma, station, p.stations, covariance=sc.P,
                    model=sc.model, gate_probability=0.99, best=8)
    d2_own = np.array([res.d2[j][list(res.rows[j]).index(sat[j])] if sat[j] in res.rows[j] else np.inf
                       for j in range(m)])
    inside = np.mean(d2_own <= res.gate_d2)
    lo = stats.binom.ppf(1e-4, m, 0.99) / m
    print(f"inside the 0.99 gate {inside:.4f} of {m}, binomial 1e-4 lower bound {lo:.4f}")
    assert inside >= lo
