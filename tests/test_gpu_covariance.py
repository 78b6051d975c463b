"""K10 state covariance on the device (covariance_kernel, covariance_deep_kernel): the device against the host build of
the same source on ~2,000 mixed rows fitted by the device, the nominal state against from_elements + propagate_pairs,
the hat-matrix invariant of a device fit, a Monte Carlo through propagate_pairs, and batch / order / chunk and host /
device-call independence."""
import numpy as np
import pytest

from tests import fit_oracle as R
from tests.fit_oracle import covariance as K

pytestmark = pytest.mark.gpu
SIG = np.array([1e-3] * 3 + [1e-6] * 3)


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def emul():
    _lib()
    L = K.emul_library()
    if L is None:
        pytest.skip("nvcc unavailable")
    return L


def _pairs_states(el, sat, jd, fr):
    from astroz_b200.constellation import Constellation

    c = Constellation.from_elements(*el)
    p, v, st = c.propagate_pairs(sat, jd, fr)
    c.deinit()
    return np.concatenate([np.asarray(p), np.asarray(v)], axis=1), np.asarray(st)


@pytest.fixture(scope="module")
def fitted():
    """~2,000 mixed rows (config-3 style: GEO, Molniya, GPS among LEO) fitted on the device to library-made TEME states
    with noise, one day at 30 min, deep_space=True"""
    _lib()
    from astroz_b200 import synth
    from astroz_b200.fit import OBS_TEME_STATE, fit_observations

    el = synth.elements_from_tles(synth.mixed_catalog(2048, n_geo=128, n_molniya=32, n_gps=32))
    n, t = el.shape[1], 49
    jd0 = np.floor(el[0] - 0.5) + 0.5
    sat = np.repeat(np.arange(n), t)
    jd = jd0[sat]
    fr = (el[0] - jd0)[sat] + np.tile(np.arange(t) / 48.0, n)
    st, status = _pairs_states(el, sat, jd, fr)
    rng = np.random.default_rng(3)
    val = st + rng.standard_normal(st.shape) * SIG
    keep = status == 0
    res = fit_observations(R.perturbed(el, seed=4), sat[keep], jd[keep], fr[keep],
                           np.full(keep.sum(), OBS_TEME_STATE), val[keep], np.tile(SIG, (keep.sum(), 1)),
                           deep_space=True)
    return res, (sat[keep], jd[keep], fr[keep])


def _queries(el, count, days, seed):
    rng = np.random.default_rng(seed)
    n = el.shape[1]
    sat = np.repeat(np.arange(n), count)
    t = rng.uniform(-days, days, len(sat))
    jd = np.floor(el[0][sat] + t - 0.5) + 0.5
    return sat, jd, (el[0][sat] + t) - jd


def _bstar_held_for_deep_rows(res):
    """res.covariance with the B* row and column zeroed on its deep-space rows: a deep-space fit with B* free has a B*
    column of rounding noise (SDP4's drag barely moves those orbits over a 1e-8 step) under a huge B* variance, so its
    Sigma would be that noise, differently rounded in each build"""
    P = res.covariance.copy()
    bstar = np.array([q for q, (j, k) in enumerate(zip(*np.triu_indices(7))) if j == 6 or k == 6])
    P[np.ix_(np.flatnonzero(res.deep_space), bstar)] = 0.0
    return P


@pytest.mark.parametrize("frame", [0, 1])
def test_device_matches_the_host_build(emul, fitted, frame):
    """Equal status bytes; states within 1e-8 km and 1e-11 km/s (measured 3.4e-9 km, 3.0e-12 km/s: the device build
    contracts into FMAs where the host build does not); Sigma within 1e-3 of its scale on near-earth rows (measured
    3.2e-4 against J's 7.2e-7: a fitted P is strongly correlated, so J P J^T cancels) and 2e-6 on deep-space rows
    (measured 4.6e-7); J within 3e-6 (measured 7.2e-7).  The deep-space rows go in with their B* row
    held (_bstar_held_for_deep_rows), so covariance_deep_kernel's P load, nvar choice and J P J^T are all compared."""
    from astroz_b200.covariance import propagate_covariance

    res, _ = fitted
    el = res.elements
    P = _bstar_held_for_deep_rows(res)
    model = res.deep_space.astype(np.uint8)
    sat, jd, fr = _queries(el, 8, 3.0, seed=1)
    got = propagate_covariance(el, sat, jd, fr, covariance=P, model=model, frame=frame, jacobian=True)
    off = np.arange(el.shape[1] + 1, dtype=np.uint32) * 8
    st, sig, jac, status = K.emul(emul, el, P, model, off, jd, fr, frame)
    assert (got.status == status).all()
    ok = (status == 0) & (np.abs(sig).max(axis=1) > 0)
    deep = res.deep_space[sat]
    assert ok.sum() > 0.9 * len(sat) and (ok & deep).sum() >= 400
    assert (got.jacobian[deep & ok][:, :, 6] == 0).all()
    dpos = np.abs(got.state[:, :3] - st[:, :3]).max()
    dvel = np.abs(got.state[:, 3:] - st[:, 3:]).max()
    S, RS = K.unpack6(got.covariance), K.unpack6(sig)
    es = np.abs(S - RS).max(axis=(1, 2)) / np.where(ok, np.abs(RS).max(axis=(1, 2)), 1.0)
    ej = np.abs(got.jacobian - jac).max(axis=(1, 2)) / np.where(ok, np.abs(jac).max(axis=(1, 2)), 1.0)
    print(f"frame {frame}: {(ok & ~deep).sum()} near-earth and {(ok & deep).sum()} deep-space queries, state "
          f"{dpos:.2e} km {dvel:.2e} km/s; Sigma near-earth {es[ok & ~deep].max():.2e} deep {es[ok & deep].max():.2e}, "
          f"J near-earth {ej[ok & ~deep].max():.2e} deep {ej[ok & deep].max():.2e} of scale")
    assert dpos < 1e-8 and dvel < 1e-11
    assert es[ok & ~deep].max() < 1e-3 and es[ok & deep].max() < 2e-6 and ej[ok].max() < 3e-6


def test_nominal_state_matches_propagate_pairs(fitted):
    """The nominal TEME state against from_elements + propagate_pairs, within K8's residual invariant of 2.4e-9 km and
    9.4e-13 km/s (measured 3.8e-10 km, 3.9e-13 km/s: propagate_pairs forms the near-earth tsince from the handle's
    reference epoch, so the two differ by rounding)"""
    from astroz_b200.covariance import propagate_covariance

    res, _ = fitted
    el = res.elements
    sat, jd, fr = _queries(el, 4, 3.0, seed=2)
    got = propagate_covariance(res, sat, jd, fr)
    ref, st = _pairs_states(el, sat, jd, fr)
    ok = (got.status == 0) & (st == 0)
    dp = np.abs(got.state[ok, :3] - ref[ok, :3]).max()
    dv = np.abs(got.state[ok, 3:] - ref[ok, 3:]).max()
    print(f"nominal vs propagate_pairs: {dp:.2e} km, {dv:.2e} km/s over {ok.sum()} queries")
    assert dp < 2.4e-9 and dv < 9.4e-13


def test_hat_matrix_invariant_of_a_device_fit(fitted):
    """sum over a row's observations of tr(W Sigma) = its number of fitted variables (7), for every converged
    near-earth row (deep-space rows fitted with B* free have a nearly singular normal matrix: SDP4's drag barely moves
    them, and the sum loses its digits to the huge B* variance; their figure is printed)"""
    from astroz_b200.covariance import propagate_covariance

    res, (sat, jd, fr) = fitted
    got = propagate_covariance(res, sat, jd, fr)
    good = (res.status == 0) & (np.abs(res.covariance).max(axis=1) > 0)
    diag = K.unpack6(got.covariance)[:, range(6), range(6)] / SIG ** 2
    total = np.bincount(sat, weights=diag.sum(axis=1), minlength=res.elements.shape[1])
    deep = np.abs(total[good & res.deep_space] - 7.0)
    print(f"deep-space rows: median |sum - 7| = {np.median(deep) if len(deep) else 0:.2e}, max {deep.max() if len(deep) else 0:.2e}")
    rows = np.flatnonzero(good & ~res.deep_space)
    worst = np.abs(total[rows] - 7.0).max()
    print(f"hat-matrix invariant over {len(rows)} near-earth rows: max |sum - 7| = {worst:.2e}")
    assert len(rows) > 1500 and worst < 1e-3


def test_monte_carlo_through_propagate_pairs(fitted):
    """100,000 draws of a LEO row's variables from N(x, P) through from_elements + propagate_pairs at +1 day: the RTN
    variances within 5 sigma of their sampling spread"""
    from astroz_b200.covariance import RTN, propagate_covariance

    res, _ = fitted
    s = int(np.flatnonzero((res.status == 0) & ~res.deep_space & (np.abs(res.covariance).max(axis=1) > 0))[0])
    el = res.elements[:, s]
    jd = np.array([np.floor(el[0] + 1.0 - 0.5) + 0.5])
    fr = (el[0] + 1.0) - jd
    one = propagate_covariance(res, [s], jd, fr, frame=RTN)
    P = K.unpack7(res.covariance[s])
    w, V = np.linalg.eigh(P)
    draws = 100000
    xs = R_vars(el) + (np.random.default_rng(9).standard_normal((draws, 7)) * np.sqrt(np.clip(w, 0, None))) @ V.T
    els = K.elements_of(xs, el[0], False)
    st, status = _pairs_states(els, np.arange(draws), np.full(draws, jd[0]), np.full(draws, fr[0]))
    assert (status == 0).all()
    Rm = K.rtn(one.state)[0]
    d = st - st.mean(axis=0)
    d = np.concatenate([d[:, :3] @ Rm.T, d[:, 3:] @ Rm.T], axis=1)
    ratio = np.diag(d.T @ d / (draws - 1)) / np.diag(one.matrix(0))
    print(f"+1 day sample / linear RTN variances {np.array2string(ratio, precision=4)}")
    assert np.abs(ratio - 1.0).max() < 5.0 * np.sqrt(2.0 / (draws - 1))


def R_vars(el):
    from tests.fit_oracle import obs as O

    return O.fit_vars(el, False)


def test_batch_order_chunk_and_call_independence(fitted):
    """A query's bytes do not depend on its batch, the order of the batch or where the chunk boundaries fall; the
    host call with pageable and pinned buffers and the _device call give the same bytes"""
    import torch

    from astroz_b200.covariance import RTN, propagate_covariance, propagate_covariance_device

    res, _ = fitted
    el = res.elements
    n = el.shape[1]
    rng = np.random.default_rng(5)
    counts = rng.integers(0, 600, n)
    counts[:3] = (5000, 1, 300)
    sat = np.repeat(np.arange(n), counts)
    t = rng.uniform(-3.0, 3.0, len(sat))
    jd = np.floor(el[0][sat] + t - 0.5) + 0.5
    fr = (el[0][sat] + t) - jd
    full = propagate_covariance(res, sat, jd, fr, frame=RTN, jacobian=True)
    perm = rng.permutation(len(sat))
    shuf = propagate_covariance(res, sat[perm], jd[perm], fr[perm], frame=RTN, jacobian=True)
    for a, b in ((full.state, shuf.state), (full.covariance, shuf.covariance), (full.jacobian, shuf.jacobian),
                 (full.status, shuf.status)):
        assert a[perm].tobytes() == b.tobytes()
    for lo, hi in ((0, 1), (3, 200), (0, 100000)):   # sub-batches shift every chunk boundary
        q = (sat >= lo) & (sat < hi) & (rng.random(len(sat)) < 0.7)
        part = propagate_covariance(res, sat[q], jd[q], fr[q], frame=RTN, jacobian=True)
        assert part.covariance.tobytes() == full.covariance[q].tobytes()
        assert part.jacobian.tobytes() == full.jacobian[q].tobytes() and part.state.tobytes() == full.state[q].tobytes()
    # the calls: grouped queries, pageable, pinned and device buffers
    cov = np.ascontiguousarray(res.covariance)
    model = res.deep_space.astype(np.uint8)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    from astroz_b200 import _lib as L
    import ctypes as C

    m = len(sat)
    outs = []
    for pinned in (False, True):
        mk = (lambda *s, dtype=torch.float64: torch.zeros(*s, dtype=dtype).pin_memory()) if pinned else \
            (lambda *s, dtype=torch.float64: torch.zeros(*s, dtype=dtype))
        ins = [torch.from_numpy(np.ascontiguousarray(a)) for a in (el, cov, model, off, jd, fr)]
        if pinned:
            ins = [x.pin_memory() for x in ins]
        st, sg, jc, stt = mk(m, 6), mk(m, 21), mk(m, 42), mk(m, dtype=torch.uint8)
        p = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731
        rc = L.lib().astroz_cuda_propagate_covariance(p(ins[0]), n, 1, p(ins[1]), p(ins[2]), p(ins[3]), p(ins[4]),
                                                       p(ins[5]), m, RTN, 0, p(st), p(sg), p(jc), p(stt))
        assert rc == 0
        outs.append([x.numpy().copy() for x in (st, sg, jc, stt)])
    dev = torch.device("cuda:0")
    d_in = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (el, cov, model)]
    d_off = torch.from_numpy(off.astype(np.int32)).to(dev)
    d_jd, d_fr = torch.from_numpy(jd).to(dev), torch.from_numpy(fr).to(dev)
    d_st, d_sg = torch.zeros(m, 6, dtype=torch.float64, device=dev), torch.zeros(m, 21, dtype=torch.float64, device=dev)
    d_jc, d_stt = torch.zeros(m, 6, 7, dtype=torch.float64, device=dev), torch.zeros(m, dtype=torch.uint8, device=dev)
    propagate_covariance_device(d_in[0], d_in[1], d_in[2], d_off, d_jd, d_fr, d_st, d_sg, d_jc, d_stt, frame=RTN)
    torch.cuda.synchronize()
    outs.append([x.cpu().numpy().reshape(y.shape) for x, y in zip((d_st, d_sg, d_jc, d_stt), outs[0])])
    ref = [full.state, full.covariance, full.jacobian.reshape(m, 42), full.status]
    for o in outs:
        for a, b in zip(o, ref):
            assert a.tobytes() == b.tobytes()
