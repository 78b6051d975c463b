"""K14 Monte Carlo collision probability on the device (conjunction_mc_kernel, conjunction_mc_deep_kernel): the
in-repo Philox against curand's, the device against the host build of the same source on ~1,000 candidates among
device-fitted mixed rows, zero P against K11's device call, the hit fraction of 10^7 draws against K11's Pc, and split
ranges, batch / order / duplicates and host / pinned / device-call byte identity."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests.fit_oracle import conjunction as cj
from tests.fit_oracle import conjunction_cases as cc
from tests.fit_oracle import conjunction_mc as mc
from tests.test_gpu_conjunction import _candidates, fitted  # noqa: F401  (module fixture: the fitted catalogue)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "astroz_b200", "csrc")


def _lib():
    from astroz_b200 import _lib as L

    if L.device_count() <= 0:
        pytest.skip("no CUDA device")
    return L


@pytest.fixture(scope="module")
def emul():
    _lib()
    L = mc.emul_library()
    if L is None:
        pytest.skip("nvcc unavailable")
    return L


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    _lib()
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc unavailable")
    so = str(tmp_path_factory.mktemp("probe") / "libprobe_philox.so")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                    "-Xcompiler", "-fPIC", "-shared", "-I" + CSRC, "-o", so,
                    os.path.join(ROOT, "tests", "device_probe", "probe_philox.cu")], check=True, capture_output=True)
    return C.CDLL(so)


def test_philox_matches_curand(probe):
    """2^20 counters x 3 keys: the in-repo Philox4x32-10 equals curand_Philox4x32_10 bit for bit on the device, and
    the numpy statement's words on a subset"""
    rng = np.random.default_rng(2)
    n = 2 ** 20
    ctr = rng.integers(0, 2 ** 32, (n, 4), dtype=np.uint64).astype(np.uint32)
    ctr[:1000] = np.stack([np.arange(1000) % 7, np.arange(1000), np.zeros(1000), np.zeros(1000)], axis=1)
    for key in ([0, 0], [0xFFFFFFFF, 0xFFFFFFFF], [0xA4093822, 0x299F31D0]):
        keys = np.tile(np.array(key, np.uint32), (n, 1))
        ours, theirs = np.zeros_like(ctr), np.zeros_like(ctr)
        p = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
        assert probe.probe_philox(p(ctr), p(keys), n, p(ours), p(theirs)) == 0
        assert np.array_equal(ours, theirs)
        assert np.array_equal(ours[:4096], mc.philox(ctr[:4096], keys[:4096]))


def _mc(cat, cand, samples, record=0, first=0, seed=None, **kw):
    from astroz_b200.collision import monte_carlo

    el, P, model = cat
    pr, se, jd, fr, w, r = cand
    seed = np.arange(len(pr)) * 3 + 1 if seed is None else seed
    return monte_carlo(el, pr, se, jd, fr, window_min=w, hbr_km=r, samples=samples, first=first, seed=seed,
                       record=record, covariance=P, model=model, **kw)


HOST = 32


def test_device_matches_the_host_build(emul, fitted):  # noqa: F811
    """~1,000 candidates (engineered crossings, LEO-deep partners, random pairs): the device's first 32 of 20,000
    samples against the host build.  Statuses and failed samples equal; dt |dv| and the miss within 1e-6 km on the
    engineered crossings (K11's device allowance); counts of a 32-sample run equal wherever no miss lies within 1e-6 km
    of the radius"""
    res, P = fitted
    cat, cand, engineered = _candidates(res, P, 1000, seed=2)
    cand = cand[:5] + (np.full(len(cand[0]), 0.5),)
    seed = np.arange(len(cand[0])) * 3 + 1
    got = _mc(cat, cand, 20000, record=HOST)
    small = _mc(cat, cand, HOST)
    counts, out, status = mc.emul(emul, *cat, *cand, HOST, 0, seed, record=HOST)
    assert np.array_equal(got.status, status) and np.array_equal(small.status, status)
    ok = status == 0
    assert ok.sum() > 0.9 * len(status)
    nan_d, nan_h = np.isnan(got.sample_dt), np.isnan(out[:, :, 0])
    assert np.array_equal(nan_d, nan_h)
    rec = cj.emul(cj.emul_library(), *cat, *cand)[0]     # the nominal relative speed
    both = engineered[:, None] & ~nan_h
    dt = np.abs(got.sample_dt - out[:, :, 0]) * 60.0 * rec[:, 2:3]
    dmiss = np.abs(got.sample_miss - out[:, :, 1])
    print(f"device vs host build: {(~nan_h[ok]).sum()} samples, dt |dv| {dt[both].max():.2e} km, miss "
          f"{dmiss[both].max():.2e} km (engineered); all samples miss {np.nanmax(dmiss):.2e} km")
    assert dt[both].max() <= 1e-6 and dmiss[both].max() <= 1e-6
    clear = ok & (np.nanmin(np.abs(out[:, :, 1] - cand[5][:, None]), axis=1, initial=1.0) > 1e-6)
    hd = np.stack([small.hits, small.edge, small.failed], axis=1)
    diff = np.flatnonzero((hd[clear] != counts[clear]).any(axis=1))
    print(f"counts: {clear.sum()} candidates clear of the radius, {len(diff)} differ")
    assert len(diff) == 0


def test_zero_P_against_k11(fitted):  # noqa: F811
    """P = 0: every sample is the nominal pair; its dt and miss against K11's device record words 0 and 1.  The two
    kernels contract their search and miss arithmetic differently (K14's sampler reads the sample's set from a runtime
    slot index), so the words are not all bit-equal: a secant end can move within the 1e-9 min bracket, |d dt| |dv|
    within K11's device allowance of 1e-6 km, and the miss, stationary at the TCA, within 1e-10 km"""
    from astroz_b200.collision import conjunctions

    res, P = fitted
    cat, cand, _ = _candidates(res, P, 600, seed=3)
    cat = (cat[0], np.zeros_like(cat[1]), cat[2])
    k11 = conjunctions(cat[0], *cand[:4], window_min=cand[4], hbr_km=cand[5], covariance=cat[1], model=cat[2])
    got = _mc(cat, cand, 4, record=4)
    ok = np.isin(k11.status, (0, 3))
    assert np.array_equal(got.status[ok], np.zeros(ok.sum(), np.uint8))
    assert (got.sample_dt[ok] == got.sample_dt[ok, :1]).all()     # every sample is the nominal pair
    dt = np.abs(got.sample_dt[ok, 0] - k11.record[ok, 0]) * 60.0 * k11.record[ok, 2]
    dmiss = np.abs(got.sample_miss[ok, 0] - k11.record[ok, 1])
    print(f"zero P vs K11 on {ok.sum()} candidates: dt bit-equal on {(dt == 0).mean():.4f}, miss on "
          f"{(dmiss == 0).mean():.4f}; worst |d dt| |dv| {dt.max():.2e} km, miss {dmiss.max():.2e} km")
    assert dt.max() <= 1e-6 and dmiss.max() <= 1e-10
    assert (got.edge[ok] == 4 * (k11.status[ok] == 3)).all()


def test_statistics_against_k11():
    """10^7 draws: the high-Pc LEO crossing's hit fraction within 4 binomial sigma + 0.01 of K11's Pc (the allowance
    tests/test_conjunction_cpu.py measures); the slow GEO pair's hit fraction / Pc ratio printed"""
    from astroz_b200.collision import conjunctions, monte_carlo

    _lib()

    def k11(el, P, hbr, model, w):
        jd = np.floor(el[0, 0] - 0.5) + 0.5
        return conjunctions(el, [0], [1], jd, el[0, 0] - jd, window_min=w, hbr_km=hbr, covariance=P, model=model)

    el, P, hbr = cc.high_pc_leo(lambda el, P, hbr: k11(el, P, hbr, np.zeros(2, np.uint8), 1.0).record[0])
    for label, el, P, hbr, model, w in [
            ("high-Pc LEO", el, P, hbr, np.zeros(2, np.uint8), 1.0),
            ("GEO slow pair", cc.pair(cc.geo(), 0.05), cc.P_words(2, scale=0.2, bstar=False, deep=np.ones(2, bool)),
             0.05, np.ones(2, np.uint8), 30.0)]:
        pc = k11(el, P, hbr, model, w).pc[0]
        jd = np.floor(el[0, 0] - 0.5) + 0.5
        r = monte_carlo(el, [0], [1], jd, el[0, 0] - jd, window_min=w, hbr_km=hbr, samples=10 ** 7, seed=17,
                        covariance=P, model=model)
        f, n = r.pc[0], r.valid[0]
        lo, hi = r.interval()
        print(f"{label}: K11 Pc {pc:.5e}, hit fraction {f:.5e} over {int(n)} samples (Wilson 95% [{lo[0]:.5e}, "
              f"{hi[0]:.5e}]), edge {int(r.edge[0])}, failed {int(r.failed[0])}, ratio {f / pc:.4f}")
        assert r.status[0] == 0 and n > 0.99e7
        if label == "high-Pc LEO":
            assert abs(f - pc) <= 4 * np.sqrt(pc * (1 - pc) / n) + 0.01


def test_split_ranges_batch_and_call_forms(fitted):  # noqa: F811
    """One candidate at 10^8 samples equals the sum of ten 10^7 ranges; a candidate's bytes do not depend on the batch,
    its position or duplicates; pageable, pinned and _device calls give identical bytes"""
    import torch

    from astroz_b200.collision import monte_carlo, monte_carlo_device, monte_carlo_scratch_bytes

    el, P, hbr = cc.high_pc_leo(lambda el, P, hbr: cj.emul(cj.emul_library(), el, P, np.zeros(2, np.uint8), [0], [1],
                                                           np.floor(el[0, 0] - 0.5) + 0.5,
                                                           el[0, 0] - (np.floor(el[0, 0] - 0.5) + 0.5), 1.0,
                                                           hbr)[0][0])
    jd = np.floor(el[0, 0] - 0.5) + 0.5
    one = lambda n, first: monte_carlo(el, [0], [1], jd, el[0, 0] - jd, window_min=1.0, hbr_km=hbr,  # noqa: E731
                                       samples=n, first=first, seed=5, covariance=P, model=np.zeros(2, np.uint8))
    whole = one(10 ** 8, 0)
    parts = [one(10 ** 7, k * 10 ** 7) for k in range(10)]
    for f in ("hits", "edge", "failed"):
        assert getattr(whole, f)[0] == sum(getattr(p, f)[0] for p in parts)
    print(f"10^8 samples: hits {whole.hits[0]}, Pc {whole.pc[0]:.6f}")

    res, Pf = fitted
    cat, cand, _ = _candidates(res, Pf, 400, seed=4)
    base = _mc(cat, cand, 3000, record=40)
    perm = np.random.default_rng(5).permutation(np.concatenate([np.arange(400), [7, 7, 300]]))
    seed = (np.arange(400) * 3 + 1)[perm]
    shuf = _mc(cat, tuple(c[perm] for c in cand), 3000, record=40, seed=seed)
    for f in ("hits", "edge", "failed", "status"):
        assert np.array_equal(getattr(shuf, f), getattr(base, f)[perm])
    assert shuf.sample_dt.tobytes() == base.sample_dt[perm].tobytes()
    assert shuf.sample_miss.tobytes() == base.sample_miss[perm].tobytes()
    for i in (0, 123, 399):
        single = _mc(cat, tuple(c[i:i + 1] for c in cand), 3000, record=40, seed=[i * 3 + 1])
        assert single.hits[0] == base.hits[i] and single.sample_dt.tobytes() == base.sample_dt[i:i + 1].tobytes()
    # pinned host buffers
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()  # noqa: E731
    pinned = _mc((pin(cat[0]), pin(cat[1]), cat[2]), (cand[0], cand[1], pin(cand[2]), pin(cand[3]), pin(cand[4]),
                                                      pin(cand[5])), 3000, record=40)
    assert pinned.sample_dt.tobytes() == base.sample_dt.tobytes() and np.array_equal(pinned.hits, base.hits)
    # the device call
    dev = torch.device("cuda:0")
    t = lambda a, dt=torch.float64: torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device=dev)  # noqa: E731
    m = len(cand[0])
    counts = torch.zeros((m, 3), dtype=torch.int64, device=dev)
    out = torch.zeros((m, 40, 2), dtype=torch.float64, device=dev)
    stat = torch.zeros(m, dtype=torch.uint8, device=dev)
    scratch = torch.empty(monte_carlo_scratch_bytes(m), dtype=torch.uint8, device=dev)
    monte_carlo_device(t(cat[0]), t(cat[1]), t(cat[2], torch.uint8), t(cand[0], torch.int32), t(cand[1], torch.int32),
                       t(cand[2]), t(cand[3]), t(cand[4]), t(cand[5]), t(np.full(m, 3000), torch.int64), None,
                       t(np.arange(m) * 3 + 1, torch.int64), counts, out, stat, scratch)
    torch.cuda.synchronize()
    c = counts.cpu().numpy().astype(np.uint64)
    assert np.array_equal(c[:, 0], base.hits) and np.array_equal(c[:, 2], base.failed)
    assert out.cpu().numpy()[:, :, 0].tobytes() == base.sample_dt.tobytes()
    assert np.array_equal(stat.cpu().numpy(), base.status)
    # a bad pair on the device call
    monte_carlo_device(t(cat[0]), t(cat[1]), t(cat[2], torch.uint8), t([0, 5], torch.int32), t([1, 5], torch.int32),
                       t(cand[2][:2]), t(cand[3][:2]), t(cand[4][:2]), t(cand[5][:2]), t([100, 100], torch.int64),
                       None, None, counts[:2], out[:2], stat[:2], scratch)
    torch.cuda.synchronize()
    assert stat[:2].cpu().numpy()[1] == 5 and (counts[1].cpu().numpy() == 0).all()
    assert np.isnan(out[1].cpu().numpy()).all()
