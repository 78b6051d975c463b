"""K19 reentry prediction on the device (reentry_kernel, reentry_deep_kernel): the device against the host build of the
same source on a mixed scene of low-perigee rows with covariance and a few transfer orbits, and host / pinned /
device-call byte identity with a row permutation relabelling the result."""
import numpy as np
import pytest

from tests.fit_oracle import reentry as ro
from tests.test_reentry_cpu import leo

pytestmark = pytest.mark.gpu


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def emul():
    _lib()
    L = ro.emul_library()
    if L is None:
        pytest.skip("nvcc unavailable")
    return L


def scene(n_leo=256, n_gto=4, seed=4):
    """low-perigee rows (perigee 120-220 km, apogee up to 600 km) with a diagonal covariance of fitted-row size, and
    transfer orbits (deep-space model) with perigees near 150 km"""
    rng = np.random.default_rng(seed)
    cols, model = [], []
    for _ in range(n_leo):
        hp = rng.uniform(120, 220)
        cols.append(leo(hp, hp + rng.uniform(5, 380), incl=rng.uniform(0, 100), node=rng.uniform(0, 360),
                        argp=rng.uniform(0, 360), ma=rng.uniform(0, 360), bstar=rng.uniform(5e-5, 5e-4)))
        model.append(0)
    for _ in range(n_gto):
        cols.append(leo(rng.uniform(140, 160), 35786.0, incl=rng.uniform(5, 28), node=rng.uniform(0, 360),
                        argp=rng.uniform(0, 360), ma=rng.uniform(0, 360), bstar=1e-4))
        model.append(1)
    el = np.ascontiguousarray(np.stack(cols, 1))
    n = el.shape[1]
    P = np.zeros((n, 28))
    diag = [0, 7, 13, 18, 22, 25, 27]
    sd = np.array([1e-7, 1e-6, 1e-6, 1e-5, 1e-5, 1e-5, 3e-5])
    P[:, diag] = (sd * rng.uniform(0.5, 2.0, (n, 7))) ** 2
    P[:, 27] *= el[7, :] ** 2 / 1e-4 ** 2 * 1e-2   # B* spread of ~10 %
    return el, P, np.array(model, np.uint8)


KW = dict(interface_km=80.0, horizon_days=30.0, density_sigma=0.2, samples=64, seed=11, record=64, states=True)


def test_device_matches_the_host_build(emul):
    from astroz_b200 import reentry

    el, P, md = scene()
    n = el.shape[1]
    rows = np.arange(n)
    r = reentry.predict(el, rows, covariance=P, model=md, **KW)
    assert (r.status == 0).all()
    sub = np.r_[np.arange(0, 256, 4), np.arange(256, n)]   # every fourth LEO row and every transfer orbit
    rec, states, nst, counts, out, st = ro.emul(emul, el, P, md, sub, samples=64, seed=11, sigma=0.2, record=64,
                                                horizon_days=30.0, threads=16)
    assert np.array_equal(st, r.status[sub]) and np.array_equal(nst, r.nominal_status[sub])
    assert np.array_equal(counts, r.counts[sub])
    # attempts: the host build's libm and the device's round exp, sin and cos differently in the last place, and over
    # thousands of adaptive steps the step sequences part: on H100 48 % of the counts are equal and the worst differs by
    # 6.0 %, so the bound is 10 %
    att_dev = np.r_[r.record[sub, 6:8].sum(1), r.sample_words[sub, :, 3].reshape(-1)]
    att_host = np.r_[rec[:, 6:8].sum(1), out[:, :, 3].reshape(-1)]
    same = att_dev == att_host
    rel_att = np.abs(att_dev - att_host) / np.maximum(att_host, 1.0)
    dt_d = np.r_[r.record[sub, 0], r.sample_words[sub, :, 0].reshape(-1)]
    dt_h = np.r_[rec[:, 0], out[:, :, 0].reshape(-1)]
    fin = np.isfinite(dt_h)
    assert np.array_equal(np.isfinite(dt_d), fin)
    lat_d = np.r_[r.record[sub, 1], r.sample_words[sub, :, 1].reshape(-1)][fin]
    lat_h = np.r_[rec[:, 1], out[:, :, 1].reshape(-1)][fin]
    lon_d = np.r_[r.record[sub, 2], r.sample_words[sub, :, 2].reshape(-1)][fin]
    lon_h = np.r_[rec[:, 2], out[:, :, 2].reshape(-1)][fin]
    ddt = np.abs(dt_d[fin] - dt_h[fin]) * 60.0
    dlat = np.abs(lat_d - lat_h)
    dlon = np.abs((lon_d - lon_h + 180.0) % 360.0 - 180.0)
    print(f"{fin.sum()} crossings of {len(dt_h)}: attempts equal on {same.mean():.4%}, worst relative difference "
          f"{rel_att.max():.3e}; worst |dt| {ddt.max():.3e} s (99th percentile {np.percentile(ddt, 99):.3e}), "
          f"|lat| {dlat.max():.3e} deg, |lon| {dlon.max():.3e} deg")
    assert rel_att.max() < 0.1
    assert ddt.max() < 1.0 and dlat.max() < 0.01 and dlon.max() < 0.01


def test_call_forms_and_permutation():
    import torch

    from astroz_b200 import reentry

    el, P, md = scene(n_leo=40, n_gto=2, seed=9)
    n = el.shape[1]
    rows = np.arange(n)
    kw = dict(KW, samples=40, record=40)
    a = reentry.predict(el, rows, covariance=P, model=md, **kw)
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory().numpy()  # noqa: E731
    b = reentry.predict(pin(el), rows, covariance=pin(P), model=md, **kw)
    for f in ("record", "states", "nominal_status", "counts", "sample_words", "status"):
        assert np.array_equal(getattr(a, f).view(np.uint8), getattr(b, f).view(np.uint8)), f
    dev = torch.device("cuda", 0)
    m = n
    T = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x), dtype=dt, device=dev)  # noqa: E731
    rec, st = torch.zeros((m, 8), dtype=torch.float64, device=dev), torch.zeros((m, 6), dtype=torch.float64, device=dev)
    nst, stat = torch.zeros(m, dtype=torch.uint8, device=dev), torch.zeros(m, dtype=torch.uint8, device=dev)
    counts = torch.zeros((m, 3), dtype=torch.int64, device=dev)
    so = torch.zeros((m, 40, 4), dtype=torch.float64, device=dev)
    scratch = torch.zeros(reentry.predict_scratch_bytes(m), dtype=torch.uint8, device=dev)
    reentry.predict_device(T(el, torch.float64), T(P, torch.float64), T(md, torch.uint8), T(rows, torch.int32), None,
                           T(np.full(m, 40), torch.int64), None, T(np.full(m, 11), torch.int64), rec, st, nst, counts,
                           so, stat, scratch, interface_km=80.0, horizon_days=30.0, density_sigma=0.2)
    torch.cuda.synchronize()
    assert np.array_equal(rec.cpu().numpy().view(np.uint8), a.record.view(np.uint8))
    assert np.array_equal(so.cpu().numpy().view(np.uint8), a.sample_words.view(np.uint8))
    assert np.array_equal(counts.cpu().numpy().astype(np.uint64), a.counts)
    perm = np.random.default_rng(1).permutation(n)
    c = reentry.predict(el, perm, covariance=P, model=md, **kw)
    assert np.array_equal(c.record.view(np.uint8), a.record[perm].view(np.uint8))
    assert np.array_equal(c.counts, a.counts[perm])
