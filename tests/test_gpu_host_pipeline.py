"""The two-slot chunk pipeline of the host-buffer calls (astroz_b200/csrc/az_hostcopy.cu, ChunkPipeline) over three or
more chunks, so that each device slot is reused: the numerical host call and astroz_cuda_sgp4_array into pageable,
registered and pinned result blocks."""
import numpy as np
import pytest

from tests.golden import tles as G
from tests.test_numerical_host_emulation import J2, MU, R_EQ, fixtures

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def az():
    import astroz_b200

    astroz_b200.lib()
    assert astroz_b200.device_count() >= 1, "GPU tests need a CUDA device"
    return astroz_b200


def test_numerical_host_call_reuses_its_slots(az):
    """4,000 two-body + J2 RK4 states over 4,000 samples: 768 MB of trajectories, three chunks of at most 256 MB, so the
    third chunk reuses the first one's slot.  Pageable and pinned destinations give the device call's bytes."""
    import torch

    from astroz_b200 import numerical as num

    rng = np.random.default_rng(7)
    n = 4000
    y = np.array(fixtures()[:5])[rng.integers(0, 5, n)] * (1 + 1e-4 * rng.standard_normal((n, 6)))
    args = (0.0, 39990.0, 10.0, MU)
    kw = dict(j2=J2, r_eq=R_EQ, integrator="rk4")
    _, ref, st, steps = num.propagate_numerical_batch(y, *args, **kw)   # pageable destination
    assert ref.shape == (n, 4000, 6) and ref.nbytes > 2 * (256 << 20)
    dev = torch.device("cuda", 0)
    dout = torch.empty(ref.shape, dtype=torch.float64, device=dev)
    dst = torch.empty(n, dtype=torch.uint8, device=dev)
    dsteps = torch.empty((n, 2), dtype=torch.int64, device=dev)
    num.propagate_numerical_batch_device(torch.from_numpy(y).to(dev), *args, dout, dst, dsteps, **kw)
    torch.cuda.synchronize()
    assert np.array_equal(dout.cpu().numpy(), ref) and np.array_equal(dst.cpu().numpy(), st)
    assert np.array_equal(dsteps.cpu().numpy().astype(np.uint64), steps)
    del dout
    pinned = az.pinned_empty(ref.shape)
    pinned.fill(-1.0)
    _, out, st2, steps2 = num.propagate_numerical_batch(y, *args, out=pinned, **kw)
    assert out is pinned and np.array_equal(out, ref)
    assert np.array_equal(st2, st) and np.array_equal(steps2, steps)


def test_sgp4_array_into_every_kind_of_result_block(az):
    """astroz_cuda_sgp4_array over three chunks of 1.5 M epochs from pageable epoch arrays, into a pageable, a registered
    and a pinned result block: the same bytes in all three."""
    from astroz_b200._lib import check, dptr, lib
    from astroz_b200.api import Satrec, WGS72

    sat = Satrec.twoline2rv(*G.ISS, WGS72)
    n = 4_500_007
    jd = np.full(n, sat.jdsatepoch)
    fr = sat.jdsatepochF + np.arange(n) * (1.0 / 86400.0)
    epoch = sat.jdsatepoch + sat.jdsatepochF

    def run(out):
        out.fill(-1.0)
        check(lib().astroz_cuda_sgp4_array(sat._h, dptr(jd), dptr(fr), epoch, dptr(out), n))
        return out

    pageable = run(np.empty((n, 6)))
    assert np.isfinite(pageable).all()
    reg = np.empty((n, 6))
    az.host_register(reg)
    try:
        assert np.array_equal(run(reg), pageable)
    finally:
        az.host_unregister(reg)
    assert np.array_equal(run(az.pinned_empty((n, 6))), pageable)
    # the Python call fills a pinned block of its own
    _, r, v = sat.sgp4_array(jd, fr)
    assert np.array_equal(r, pageable[:, :3]) and np.array_equal(v, pageable[:, 3:])
