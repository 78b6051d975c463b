"""Reentry prediction on the device: carry each catalogue row and its covariance draws down through the atmosphere to
the interface height (K19, astroz_b200/csrc/az_reentry.cu).

    from astroz_b200.reentry import predict
    fit = fit_observations(...)                                  # FitResult with covariance and deep_space
    r = predict(fit, rows, interface_km=80.0, horizon_days=30.0, samples=1000, density_sigma=0.3, seed=1)
    r.jd, r.fr, r.lat_deg, r.lon_deg, r.window(), r.fraction_reentered()

Each trajectory starts at its row's epoch from the TEME state of a set (the row's own for the nominal, a draw from the
row's covariance for a sample) and is integrated by the numerical propagator's Dormand-Prince 8(7) under two-body, J2
and drag quadratic in the speed relative to a co-rotating atmosphere, with Vallado's piecewise-exponential density at
the WGS-84 geodetic height.  The first crossing of the interface height gives the epoch, the footprint (geodetic
latitude and east longitude), the speed and the flight-path angle.  density_scale is the one solar-activity input;
density_sigma spreads each sample's density by a log-normal factor.  Lunisolar and higher zonal terms are not modelled,
so transfer-orbit predictions are indicative only.  Everything below the interface (lift, breakup, ablation, impact
footprints) is out of scope.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._abi import DEFINES as D
from ._lib import WGS72, check, lib
from .collision import _catalogue

OK, INIT_FAILED, NOT_PSD, BAD_ROW = (D["ASTROZ_REENTRY_OK"], D["ASTROZ_REENTRY_INIT_FAILED"],
                                     D["ASTROZ_REENTRY_NOT_PSD"], D["ASTROZ_REENTRY_BAD_ROW"])
REENTERED, ABOVE, TRAJ_INIT_FAILED, NONPHYSICAL, STOPPED = (
    D["ASTROZ_REENTRY_TRAJ_REENTERED"], D["ASTROZ_REENTRY_TRAJ_ABOVE"], D["ASTROZ_REENTRY_TRAJ_INIT_FAILED"],
    D["ASTROZ_REENTRY_TRAJ_NONPHYSICAL"], D["ASTROZ_REENTRY_TRAJ_STOPPED"])
_RECORD = D["ASTROZ_REENTRY_RECORD_WORDS"]
_SAMPLE = D["ASTROZ_REENTRY_SAMPLE_WORDS"]
_COUNT = D["ASTROZ_REENTRY_COUNT_WORDS"]
_STATE = D["ASTROZ_REENTRY_STATE_WORDS"]


@dataclass
class ReentryResult:
    record: np.ndarray               # (m, 8) the nominal's words (astroz_b200.h, K19)
    jd: np.ndarray                   # (m,) the nominal's crossing epoch as jd + fr: the row's epoch ...
    fr: np.ndarray                   # (m,) ... and dt / 1440 (inf while above at the horizon, NaN when failed)
    states: np.ndarray | None        # (m, 6) TEME state at the nominal crossing, or None
    nominal_status: np.ndarray       # (m,) uint8 REENTERED, ABOVE, TRAJ_INIT_FAILED, NONPHYSICAL, STOPPED
    counts: np.ndarray               # (m, 3) uint64: samples reentered, above, failed
    samples: np.ndarray              # (m,) uint64: samples drawn
    sample_words: np.ndarray | None  # (m, record, 4) dt [min], latitude, longitude [deg], attempts (NaN: none)
    status: np.ndarray               # (m,) uint8 OK, INIT_FAILED, NOT_PSD, BAD_ROW

    dt_min = property(lambda self: self.record[:, 0])
    lat_deg = property(lambda self: self.record[:, 1])
    lon_deg = property(lambda self: self.record[:, 2])
    speed_km_s = property(lambda self: self.record[:, 3])
    flight_path_deg = property(lambda self: self.record[:, 4])
    ballistic = property(lambda self: self.record[:, 5])
    reentered = property(lambda self: self.counts[:, 0])
    above = property(lambda self: self.counts[:, 1])
    failed = property(lambda self: self.counts[:, 2])

    def fraction_reentered(self) -> np.ndarray:
        """reentered / (samples - failed): the share of scored samples that cross before the horizon; NaN with none"""
        v = self.samples.astype(np.float64) - self.failed.astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where((v > 0) & (self.status == OK), self.reentered.astype(np.float64) / v, np.nan)

    def window(self, lo: float = 0.05, hi: float = 0.95) -> tuple[np.ndarray, np.ndarray]:
        """The (lo, hi) sample quantiles of the reentry epoch [JD] over the recorded samples that did not fail: the
        row's epoch (jd) plus each sample's dt.  ABOVE samples count as +inf, so a quantile past the horizon is inf
        rather than dropped; NaN where no recorded sample was scored."""
        if self.sample_words is None:
            raise ValueError("window() needs the samples' words: call predict with record > 0")
        dt = self.sample_words[:, :, 0]
        qlo, qhi = np.full(len(dt), np.nan), np.full(len(dt), np.nan)
        for i, row in enumerate(dt):
            v = np.sort(row[~np.isnan(row)])   # inf (ABOVE) sorts last
            if len(v):
                qlo[i], qhi[i] = (v[min(int(np.floor(q * len(v))), len(v) - 1)] for q in (lo, hi))
        return self.jd + qlo / 1440.0, self.jd + qhi / 1440.0


def _u64(a, m, name):
    a = np.asarray(a)
    if a.size and (not np.issubdtype(a.dtype, np.integer) or a.min() < 0):
        raise ValueError(f"{name} must hold integers >= 0")
    return np.ascontiguousarray(np.broadcast_to(a.astype(np.uint64), (m,)))


def predict(source, rows, *, interface_km=80.0, horizon_days=30.0, step_s=60.0, ballistic=None, density_scale=1.0,
            density_sigma=0.0, samples=0, seed=0, first=0, record: int = 0, states: bool = False, covariance=None,
            model=None, grav: int = WGS72, device: int = 0) -> ReentryResult:
    """Reentry prediction of m requests (astroz_cuda_reentry).

    source: a FitResult or an (8, n) array of element columns with covariance= (n, 28) words or (n, 7, 7) matrices and
    model= (n,) 0 / 1, as in astroz_b200.collision; a missing covariance means zero (the nominal plus density-only
    draws).  rows (m,): the catalogue rows.  ballistic: (m,) B [m^2/kg] or None (12.741621 B*).  samples, seed and
    first broadcast to rows; sample k of a row is K14's primary draw of k under its seed, with density factor
    exp(density_sigma z_7).  record > 0 returns the first `record` samples' words (needed by window()); states=True
    the nominal's TEME state at the crossing.  Counts over [0, 2N) are those over [0, N) plus those over [N, 2N)."""
    if covariance is None and not (hasattr(source, "covariance") and source.covariance is not None):
        n0 = source.elements.shape[1] if hasattr(source, "elements") else np.asarray(source).shape[-1]
        covariance = np.zeros((n0, 28))
    el, cov, md = _catalogue(source, covariance, model)
    n = el.shape[1]
    r = np.asarray(rows).reshape(-1)
    if r.size and (not np.issubdtype(r.dtype, np.integer) or r.min() < 0 or r.max() >= n):
        raise ValueError("rows must hold row indices in [0, n)")
    r = np.ascontiguousarray(r.astype(np.uint32))
    m = len(r)
    record = int(record)
    if record < 0:
        raise ValueError("record must be >= 0")
    bc = None if ballistic is None else np.ascontiguousarray(
        np.broadcast_to(np.asarray(ballistic, dtype=np.float64), (m,)))
    ns, fi, sd = _u64(samples, m, "samples"), _u64(first, m, "first"), _u64(seed, m, "seed")
    rec, nst, stat = np.zeros((m, _RECORD)), np.zeros(m, np.uint8), np.zeros(m, np.uint8)
    counts = np.zeros((m, _COUNT), np.uint64)
    st = np.zeros((m, _STATE)) if states else None
    out = np.zeros((m, record, _SAMPLE)) if record else None
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_reentry(vp(el), n, int(grav), vp(cov), vp(md), vp(r), vp(bc), vp(ns), vp(fi), vp(sd), m,
                                    float(interface_km), float(horizon_days), float(step_s), float(density_scale),
                                    float(density_sigma), record, int(device), vp(rec), vp(st), vp(nst), vp(counts),
                                    vp(out), vp(stat)))
    return ReentryResult(rec, el[0, r].copy(), rec[:, 0] / 1440.0, st, nst, counts, ns.copy(), out, stat)


def predict_scratch_bytes(m: int) -> int:
    """The scratch of predict_device for m requests"""
    b = C.c_uint64(0)
    check(lib().astroz_cuda_reentry_scratch_bytes(int(m), C.byref(b)))
    return int(b.value)


def predict_device(elements, covariance, model, rows, ballistic, samples, first, seed, record_out, states,
                   nominal_status, counts, sample_out, status, scratch, *, interface_km=80.0, horizon_days=30.0,
                   step_s=60.0, density_scale=1.0, density_sigma=0.0, grav: int = WGS72, stream: int = 0) -> None:
    """`predict` with torch CUDA tensors on one device: elements (8, n) float64, covariance (n, 28) float64, model (n,)
    uint8 or None, rows (m,) int32, ballistic (m,) float64 or None, samples (m,) int64, first / seed (m,) int64 or None
    (0); record_out (m, 8) float64, states (m, 6) float64 or None, nominal_status (m,) uint8, counts (m, 3) int64,
    sample_out (m, record, 4) float64 or None and status (m,) uint8 receive the results; scratch a uint8 tensor of at
    least predict_scratch_bytes(m) bytes.  The launches go on `stream` (a raw cudaStream_t value, 0 = the default
    stream).  Rows are not checked here: a row outside the catalogue gets BAD_ROW."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    m = int(rows.numel())
    record = int(sample_out.shape[1]) if sample_out is not None and sample_out.dim() == 3 else 0
    tensors = [("elements", elements, 8 * n, torch.float64), ("covariance", covariance, 28 * n, torch.float64),
               ("model", model, n, torch.uint8), ("rows", rows, m, torch.int32),
               ("ballistic", ballistic, m, torch.float64), ("samples", samples, m, torch.int64),
               ("first", first, m, torch.int64), ("seed", seed, m, torch.int64),
               ("record_out", record_out, _RECORD * m, torch.float64), ("states", states, _STATE * m, torch.float64),
               ("nominal_status", nominal_status, m, torch.uint8), ("counts", counts, _COUNT * m, torch.int64),
               ("sample_out", sample_out, _SAMPLE * record * m, torch.float64), ("status", status, m, torch.uint8)]
    for name, t, size, dtype in tensors:
        if t is None and name in ("model", "ballistic", "first", "seed", "states", "sample_out"):
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    if not isinstance(scratch, torch.Tensor) or not scratch.is_contiguous() or scratch.device != elements.device \
            or scratch.numel() * scratch.element_size() < predict_scratch_bytes(m):
        raise ValueError(f"scratch must be a contiguous tensor of predict_scratch_bytes({m}) bytes on {elements.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_reentry_device(
        ptr(elements), n, int(grav), ptr(covariance), ptr(model), ptr(rows), ptr(ballistic), ptr(samples), ptr(first),
        ptr(seed), m, float(interface_km), float(horizon_days), float(step_s), float(density_scale),
        float(density_sigma), record, int(elements.device.index), ptr(record_out), ptr(states), ptr(nominal_status),
        ptr(counts), ptr(sample_out), ptr(status), ptr(scratch), C.c_void_p(stream) if stream else None))
