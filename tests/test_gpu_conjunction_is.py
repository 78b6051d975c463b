"""K15 importance-sampled collision probability on the device (is_proposal_kernel, conjunction_is_kernel,
conjunction_is_deep_kernel): the device against the host build on ~1,000 candidates among device-fitted mixed rows, a
zero shift against K14's device call, unbiasedness against K14's plain draws, the relative error down the Pc ladder, and
split ranges and host / pinned / device-call byte identity."""
import numpy as np
import pytest

from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import conjunction_is as ci
from tests.test_gpu_conjunction import _candidates, fitted  # noqa: F401  (module fixture: the fitted catalogue)

pytestmark = pytest.mark.gpu


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def emul():
    _lib()
    L = ci.emul_library()
    if L is None:
        pytest.skip("nvcc unavailable")
    return L


def _is(cat, cand, samples, record=0, first=0, seed=None, shift=None, **kw):
    from astroz_b200.collision import importance_sampling

    el, P, model = cat
    pr, se, jd, fr, w, r = cand
    seed = np.arange(len(pr)) * 3 + 1 if seed is None else seed
    return importance_sampling(el, pr, se, jd, fr, window_min=w, hbr_km=r, samples=samples, first=first, seed=seed,
                               record=record, shift=shift, covariance=P, model=model, **kw)


HOST = 32


def test_device_matches_the_host_build(emul, fitted):  # noqa: F811
    """~1,000 candidates: statuses and kinds equal the host build's and the linear shifts agree within a measured
    tolerance; with the host's shift passed as GIVEN, dt |dv| and the miss within K14's device allowance of 1e-6 km on
    the engineered crossings, log w within 1e-9 (1 + |log w|), and the counts equal wherever no miss lies within
    1e-6 km of the radius"""
    res, P = fitted
    cat, cand, engineered = _candidates(res, P, 1000, seed=2)
    cand = cand[:5] + (np.full(len(cand[0]), 0.5),)
    seed = np.arange(len(cand[0])) * 3 + 1
    lin = _is(cat, cand, HOST)
    h = ci.emul(emul, *cat, *cand, HOST, 0, seed, record=HOST)
    assert np.array_equal(lin.status, h["status"])
    ok = h["status"] == 0
    assert ok.sum() > 0.9 * len(ok)
    assert np.array_equal(lin.kind[ok], h["kind"][ok])
    linear = ok & (h["kind"] == ci.LINEAR)
    c_h = h["proposal"][:, :14]
    scale = np.abs(c_h).max(axis=1) + 1.0
    err = (np.abs(lin.shift - c_h).max(axis=1) / scale)[linear]
    print(f"linear proposals: {linear.sum()} of {ok.sum()}, kinds {np.bincount(lin.kind[ok], minlength=3)}; "
          f"|dc| / (1 + |c|) worst {err.max():.2e}, median {np.median(err):.2e}")
    assert err.max() <= 1e-3   # measured 2.2e-4 (forward-difference J of device vs host cells)
    given = _is(cat, cand, HOST, record=HOST, shift=c_h)
    assert np.array_equal(given.status, h["status"]) and (given.kind[ok] == ci.GIVEN).all()
    out = h["out"]
    nan_d, nan_h = np.isnan(given.sample_dt), np.isnan(out[:, :, 0])
    assert np.array_equal(nan_d, nan_h)
    rec = h["record"]
    both = engineered[:, None] & ~nan_h
    dt = np.abs(given.sample_dt - out[:, :, 0]) * 60.0 * rec[:, 2:3]
    dmiss = np.abs(given.sample_miss - out[:, :, 1])
    dlw = np.abs(given.sample_log_weight - out[:, :, 2]) / (1.0 + np.abs(out[:, :, 2]))
    print(f"GIVEN vs host build: dt |dv| {dt[both].max():.2e} km, miss {dmiss[both].max():.2e} km (engineered); "
          f"log w {np.nanmax(dlw):.2e}")
    assert dt[both].max() <= 1e-6 and dmiss[both].max() <= 1e-6 and np.nanmax(dlw) <= 1e-9
    clear = ok & (np.nanmin(np.abs(out[:, :, 1] - cand[5][:, None]), axis=1, initial=1.0) > 1e-6)
    diff = np.flatnonzero((given.counts[clear, :4] != h["counts"][clear, :4]).any(axis=1))
    print(f"counts: {clear.sum()} candidates clear of the radius, {len(diff)} differ")
    assert len(diff) == 0


def test_zero_shift_equals_k14(fitted):  # noqa: F811
    """A given shift of 0 draws K14's samples: hits, edge, failed and the (dt, miss) words bit for bit, V_hit = hits
    2^128, V2_hit the same, log w = 0"""
    from astroz_b200.collision import monte_carlo

    res, P = fitted
    cat, cand, _ = _candidates(res, P, 400, seed=3)
    seed = np.arange(400) * 3 + 1
    k14 = monte_carlo(cat[0], *cand[:4], window_min=cand[4], hbr_km=cand[5], samples=2000, seed=seed, record=40,
                      covariance=cat[1], model=cat[2])
    got = _is(cat, cand, 2000, record=40, shift=np.zeros(14))
    for f in ("hits", "edge", "failed", "status"):
        assert np.array_equal(getattr(got, f), getattr(k14, f)), f
    assert got.sample_dt.tobytes() == k14.sample_dt.tobytes() and got.sample_miss.tobytes() == k14.sample_miss.tobytes()
    ok = got.status == 0
    hits = got.hits.astype(object)
    for lo in (4, 8):
        v = [sum(int(x) << (64 * q) for q, x in enumerate(row)) for row in got.counts[:, lo:lo + 4]]
        assert all(a == int(b) << 128 for a, b in zip(v, hits))
    assert (got.sample_log_weight[ok][~np.isnan(got.sample_dt[ok])] == 0.0).all()
    assert (got.overflow == 0).all()


def _assess(el, P, hbr, model=None, w=1.0):
    from astroz_b200.collision import conjunctions

    jd = np.floor(el[0, 0] - 0.5) + 0.5
    md = np.zeros(2, np.uint8) if model is None else model
    return conjunctions(el, [0], [1], jd, el[0, 0] - jd, window_min=w, hbr_km=hbr, covariance=P, model=md).record[0]


def _one(el, P, hbr, model, w, samples, seed, first=0, shift=None):
    from astroz_b200.collision import importance_sampling

    jd = np.floor(el[0, 0] - 0.5) + 0.5
    return importance_sampling(el, [0], [1], jd, el[0, 0] - jd, window_min=w, hbr_km=hbr, samples=samples, seed=seed,
                               first=first, shift=shift, covariance=P, model=model)


def _k14(el, P, hbr, model, w, samples, seed):
    from astroz_b200.collision import monte_carlo

    jd = np.floor(el[0, 0] - 0.5) + 0.5
    return monte_carlo(el, [0], [1], jd, el[0, 0] - jd, window_min=w, hbr_km=hbr, samples=samples, seed=seed,
                       covariance=P, model=model)


def test_unbiased_against_plain_draws():
    """IS at 10^6 samples against K14's plain draws: the high-Pc LEO crossing and the slow GEO pair against 10^7, a LEO
    crossing at Pc ~ 1e-5 against 10^9, each within 4 combined standard errors (K14's failed draws: none here)"""
    _lib()
    el, P, hbr = cc.high_pc_leo(lambda el, P, hbr: _assess(el, P, hbr))
    geo = (cc.pair(cc.geo(), 0.05), cc.P_words(2, scale=0.2, bstar=False, deep=np.ones(2, bool)), 0.05)
    tail = ci.leo_at_pc(lambda el, P, hbr: _assess(el, P, hbr), 1e-5)
    for label, (e, p, r), model, w, plain in [("high-Pc LEO", (el, P, hbr), np.zeros(2, np.uint8), 1.0, 10 ** 7),
                                              ("GEO slow pair", geo, np.ones(2, np.uint8), 30.0, 10 ** 7),
                                              ("LEO Pc 1e-5", tail, np.zeros(2, np.uint8), 1.0, 10 ** 9)]:
        s = _one(e, p, r, model, w, 10 ** 6, 23)
        k = _k14(e, p, r, model, w, plain, 29)
        f, n = float(k.hits[0]) / plain, plain
        se_k = np.sqrt(max(f * (1 - f), 1.0 / n) / n)
        z = (s.pc[0] - f) / np.hypot(s.std_error[0], se_k)
        k11 = _assess(e, p, r, model, w)[12]
        print(f"{label}: IS {s.pc[0]:.5e} +- {s.std_error[0]:.2e} (kind {s.kind[0]}, hit fraction "
              f"{s.proposal_hit_fraction[0]:.3f}), K14 {f:.5e} +- {se_k:.2e} over {n:.0e}, K11 {k11:.5e}; z {z:+.2f}")
        assert s.status[0] == 0 and k.status[0] == 0 and k.failed[0] == 0 and s.failed[0] == 0
        assert abs(z) <= 4.0


def test_tail_ladder():
    """LEO crossings at K11 Pc 1e-6 .. 1e-10 (sigma 200 m, R 20 m): 10^6 IS samples give a relative standard error
    <= 10 % (the linear-model expectation is ~1.5 %); the ratio to K11's Pc is printed"""
    _lib()
    for target in (1e-6, 1e-7, 1e-8, 1e-9, 1e-10):
        el, P, hbr = ci.leo_at_pc(lambda el, P, hbr: _assess(el, P, hbr), target)
        k11 = _assess(el, P, hbr)[12]
        s = _one(el, P, hbr, np.zeros(2, np.uint8), 1.0, 10 ** 6, 31)
        rel = s.std_error[0] / s.pc[0]
        print(f"K11 Pc {k11:.3e}: IS {s.pc[0]:.4e}, relative error {rel:.4f}, ratio to K11 {s.pc[0] / k11:.4f}, "
              f"|c|^2 {-2 * s.log_scale[0]:.2f}, hit fraction {s.proposal_hit_fraction[0]:.4f}, kind {s.kind[0]}")
        assert s.kind[0] == ci.LINEAR and rel <= 0.10


def test_split_ranges_and_call_forms(fitted):  # noqa: F811
    """10^8 samples equal ten 10^7 ranges combined; pageable, pinned and _device calls give identical bytes"""
    import torch

    from astroz_b200.collision import importance_sampling_device, importance_sampling_scratch_bytes

    el, P, hbr = ci.leo_at_pc(lambda el, P, hbr: _assess(el, P, hbr), 1e-7)
    model = np.zeros(2, np.uint8)
    whole = _one(el, P, hbr, model, 1.0, 10 ** 8, 5)
    acc = None
    for k in range(10):
        part = _one(el, P, hbr, model, 1.0, 10 ** 7, 5, first=k * 10 ** 7)
        acc = part if acc is None else acc.combine(part)
    assert np.array_equal(whole.counts, acc.counts) and whole.pc[0] == acc.pc[0]
    print(f"10^8 samples: Pc {whole.pc[0]:.6e} +- {whole.std_error[0]:.2e}, hits {whole.hits[0]}")

    res, Pf = fitted
    cat, cand, _ = _candidates(res, Pf, 400, seed=4)
    base = _is(cat, cand, 3000, record=40)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()  # noqa: E731
    pinned = _is((pin(cat[0]), pin(cat[1]), cat[2]), (cand[0], cand[1], pin(cand[2]), pin(cand[3]), pin(cand[4]),
                                                      pin(cand[5])), 3000, record=40)
    assert np.array_equal(pinned.counts, base.counts) and pinned.sample_dt.tobytes() == base.sample_dt.tobytes()
    perm = np.random.default_rng(5).permutation(np.concatenate([np.arange(400), [7, 7, 300]]))
    shuf = _is(cat, tuple(c[perm] for c in cand), 3000, record=40, seed=(np.arange(400) * 3 + 1)[perm])
    assert np.array_equal(shuf.counts, base.counts[perm]) and np.array_equal(shuf.shift, base.shift[perm])
    assert shuf.sample_log_weight.tobytes() == base.sample_log_weight[perm].tobytes()
    dev = torch.device("cuda:0")
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
    m = len(cand[0])
    counts = torch.zeros((m, 12), dtype=torch.int64, device=dev)
    prop = torch.zeros((m, 15), dtype=torch.float64, device=dev)
    kind = torch.zeros(m, dtype=torch.uint8, device=dev)
    out = torch.zeros((m, 40, 3), dtype=torch.float64, device=dev)
    stat = torch.zeros(m, dtype=torch.uint8, device=dev)
    scratch = torch.empty(importance_sampling_scratch_bytes(m), dtype=torch.uint8, device=dev)
    importance_sampling_device(t(cat[0]), t(cat[1]), t(cat[2], torch.uint8), t(cand[0], torch.int32),
                               t(cand[1], torch.int32), t(cand[2]), t(cand[3]), t(cand[4]), t(cand[5]),
                               t(np.full(m, 3000), torch.int64), None, t(np.arange(m) * 3 + 1, torch.int64), None,
                               counts, prop, kind, out, stat, scratch)
    torch.cuda.synchronize()
    assert np.array_equal(counts.cpu().numpy().astype(np.uint64), base.counts)
    assert prop.cpu().numpy()[:, :14].tobytes() == base.shift.tobytes()
    assert np.array_equal(kind.cpu().numpy(), base.kind) and np.array_equal(stat.cpu().numpy(), base.status)
    assert out.cpu().numpy()[:, :, 2].tobytes() == base.sample_log_weight.tobytes()
