"""Correlate sensor tracks with catalogue objects on the device: the Mahalanobis distance of every track to every
catalogue row under the row's covariance, and the best candidates per track (K12, astroz_b200/csrc/az_correlate.cu).

    from astroz_b200.correlate import correlate
    res = correlate(fit, track, jd, fr, kind, value, sigma, station, stations)   # fit: a FitResult with covariance
    res.rows, res.d2, res.n_gate, res.status
    sat = res.assigned()                 # the row of each track with exactly one row inside its gate, else -1
    keep = sat >= 0                      # ... ready for fit_observations(fit.elements, sat[track][keep], ...)

A track is a short run of observations of one unknown object (radar range / azimuth / elevation / range-rate, optical
angles, Earth-fixed or TEME states), in the observation layout of `fit_observations`.  For every (track, row) pair the
distance is d2 = z^T (I + G P G^T)^-1 z over the track's stacked weighted residuals z, with G the residuals' Jacobian in
the fit's variables and P the row's covariance: the shared element error of all the track's residuals is accounted
for.  The gate is the chi-square quantile of the track's used residual count at `gate_probability`.  Every pair is
scored; `assigned()` is the one assignment policy (exactly one row inside the gate).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._abi import DEFINES as D
from ._lib import WGS72, check, lib
from .covariance import _covariance_words
from .fit import _csr, _integers, _obs_columns, _stations

OK, UNCORRELATED, NO_ROW, BAD_TRACK = (D["ASTROZ_CORR_OK"], D["ASTROZ_CORR_UNCORRELATED"], D["ASTROZ_CORR_NO_ROW"],
                                       D["ASTROZ_CORR_BAD_TRACK"])
STATUS_NAMES = {OK: "at least one row inside the gate", UNCORRELATED: "no row inside the gate",
                NO_ROW: "no pair could be evaluated", BAD_TRACK: "empty, too long or no used residual"}
MAX_TRACK, MAX_BEST = D["ASTROZ_CORR_MAX_TRACK"], D["ASTROZ_CORR_MAX_BEST"]
_EMPTY = 0xFFFFFFFF


@dataclass
class CorrelationResult:
    rows: np.ndarray         # (t, best) int64: the nearest rows by d2 (then row index), -1 where a slot is empty
    d2: np.ndarray           # (t, best) their squared Mahalanobis distances, +inf where empty
    used: np.ndarray         # (t,) the track's used scalar residuals: the gate's degrees of freedom
    n_gate: np.ndarray       # (t,) rows with d2 <= gate_d2, over every row
    n_failed: np.ndarray     # (t,) pairs skipped because a cell failed or a sum was not finite
    status: np.ndarray       # (t,) uint8 ASTROZ_CORR_*
    row_status: np.ndarray   # (n,) uint8 ASTROZ_COV_OK / ASTROZ_COV_INIT_FAILED
    gate_d2: np.ndarray      # (t,) the chi-square gate of each track

    def assigned(self) -> np.ndarray:
        """(t,) the row of each track when exactly one row is inside its gate, -1 otherwise"""
        return np.where(self.n_gate == 1, self.rows[:, 0], -1)


def chi2_quantile(k: int, p: float) -> float:
    """The gate of k degrees of freedom at probability p, by the function the kernels evaluate"""
    x = C.c_double()
    check(lib().astroz_cuda_chi2_quantile(int(k), float(p), C.byref(x)))
    return x.value


def _catalogue(source, covariance, model):
    if hasattr(source, "elements") and hasattr(source, "deep_space"):
        el = np.ascontiguousarray(source.elements, dtype=np.float64)
        covariance = source.covariance if covariance is None else covariance
        model = source.deep_space if model is None else model
    else:
        el = np.ascontiguousarray(source, dtype=np.float64)
        if el.ndim != 2 or el.shape[0] != 8:
            raise ValueError("source must be a FitResult or an (8, n) array of element columns")
    n = el.shape[1]
    cov = None if covariance is None else _covariance_words(covariance, n)
    md = None
    if model is not None:
        mm = np.asarray(model).reshape(-1)
        if len(mm) != n or (mm.size and (mm.min() < 0 or mm.max() > 1)):
            raise ValueError("model must hold n values, 0 (near-earth) or 1 (deep space)")
        md = np.ascontiguousarray(mm.astype(np.uint8))
    return el, cov, md


def correlate(source, track, jd, fr, kind, value, sigma, station=None, stations=None, *,
              gate_probability: float = 0.999, best: int = 4, covariance=None, model=None, grav: int = WGS72,
              device: int = 0) -> CorrelationResult:
    """Correlate tracks with a catalogue (astroz_cuda_correlate).

    source: a FitResult (elements, covariance and deep_space are taken from it; covariance= or model= override them)
    or an (8, n) array of element columns with covariance= (n, 28) words or (n, 7, 7) matrices in the fit's variables
    (None: no covariance, every P zero) and model= (n,) 0 / 1 or bool.  Observation i (any order; grouped stably by
    track) belongs to track[i] in [0, t), t = max(track) + 1, and is described as in `fit_observations`.  Returns one
    result row per track id."""
    el, cov, md = _catalogue(source, covariance, model)
    n = el.shape[1]
    track = np.asarray(track).reshape(-1)
    t = int(track.max()) + 1 if track.size else 0
    order, offsets = _csr(t, track)
    m = len(order)
    kind_all = np.asarray(kind).reshape(-1)
    jd_s = np.ascontiguousarray(np.asarray(jd, dtype=np.float64).reshape(-1)[order])
    fr_s = np.ascontiguousarray(np.asarray(fr, dtype=np.float64).reshape(-1)[order])
    kind_s = np.ascontiguousarray(_integers(kind_all, "kind", 8)[order])
    val_s = np.ascontiguousarray(_obs_columns(value, len(kind_all), "value", 0.0)[order])
    sig_s = np.ascontiguousarray(_obs_columns(sigma, len(kind_all), "sigma", np.inf)[order])
    sta_s = None if station is None else np.ascontiguousarray(
        _integers(np.asarray(station).reshape(-1), "station", 32)[order])
    st = _stations(stations)
    if len(jd_s) != m or len(fr_s) != m or len(kind_s) != m or (sta_s is not None and len(sta_s) != m):
        raise ValueError("track, jd, fr, kind, value, sigma and station must describe the same observations")
    best = int(best)
    rows, d2 = np.zeros((t, best), dtype=np.uint32), np.zeros((t, best))
    used, n_gate, n_failed = (np.zeros(t, dtype=np.uint32) for _ in range(3))
    status, row_status = np.zeros(t, dtype=np.uint8), np.zeros(n, dtype=np.uint8)
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_correlate(vp(el), n, int(grav), vp(cov), vp(md), vp(offsets), t, vp(jd_s), vp(fr_s),
                                      vp(kind_s), vp(val_s), vp(sig_s), vp(sta_s), m, vp(st), len(st),
                                      float(gate_probability), best, int(device), vp(rows), vp(d2), vp(used),
                                      vp(n_gate), vp(n_failed), vp(status), vp(row_status)))
    gates = {k: chi2_quantile(k, gate_probability) for k in np.unique(used) if k > 0}
    gate_d2 = np.array([gates.get(k, np.nan) for k in used])
    return CorrelationResult(np.where(rows == _EMPTY, -1, rows.astype(np.int64)), d2, used, n_gate, n_failed, status,
                             row_status, gate_d2)


def correlate_scratch_bytes(n: int, t: int, best: int) -> int:
    """Bytes of the scratch `correlate_device` needs"""
    out = C.c_uint64()
    check(lib().astroz_cuda_correlate_scratch_bytes(int(n), int(t), int(best), C.byref(out)))
    return out.value


def correlate_device(elements, covariance, model, offsets, jd, fr, kind, value, sigma, station, stations, scratch,
                     rows, d2, used, n_gate, n_failed, status, row_status, *, gate_probability: float = 0.999,
                     grav: int = WGS72, stream: int = 0) -> None:
    """`correlate` with torch CUDA tensors on one device, observations already grouped by track: elements (8, n)
    float64, covariance (n, 28) float64 or None, model (n,) uint8 or None, offsets (t + 1,) int32, jd / fr (m,)
    float64, kind (m,) uint8, value / sigma (m, 6) float64, station (m,) int32 or None, stations (k, 3) float64 or None,
    scratch a uint8 tensor of at least correlate_scratch_bytes(n, t, best) bytes; rows (t, best) int32, d2 (t, best)
    float64, used / n_gate / n_failed (t,) int32, status (t,) uint8 and row_status (n,) uint8 receive the results
    (rows: 0xFFFFFFFF, read as -1 in int32, where a slot is empty).  best is rows.shape[1].  Launches on `stream` (a
    raw cudaStream_t value, 0 = the default stream); nothing is checked beyond shapes: a bad track gets BAD_TRACK."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    t = int(offsets.numel()) - 1
    m = int(jd.numel())
    best = int(rows.shape[1]) if rows.dim() == 2 else 0
    k = 0 if stations is None else int(stations.numel()) // 3
    tensors = [("elements", elements, 8 * n, torch.float64), ("covariance", covariance, 28 * n, torch.float64),
               ("model", model, n, torch.uint8), ("offsets", offsets, t + 1, torch.int32),
               ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64), ("kind", kind, m, torch.uint8),
               ("value", value, 6 * m, torch.float64), ("sigma", sigma, 6 * m, torch.float64),
               ("station", station, m, torch.int32), ("stations", stations, 3 * k, torch.float64),
               ("rows", rows, best * t, torch.int32), ("d2", d2, best * t, torch.float64),
               ("used", used, t, torch.int32), ("n_gate", n_gate, t, torch.int32),
               ("n_failed", n_failed, t, torch.int32), ("status", status, t, torch.uint8),
               ("row_status", row_status, n, torch.uint8)]
    for name, x, size, dtype in tensors:
        if x is None and name in ("covariance", "model", "station", "stations"):
            continue
        if not isinstance(x, torch.Tensor) or x.dtype != dtype or not x.is_contiguous() or int(x.numel()) != size \
                or x.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    need = correlate_scratch_bytes(n, t, max(best, 1))
    if not isinstance(scratch, torch.Tensor) or scratch.dtype != torch.uint8 or scratch.device != elements.device \
            or int(scratch.numel()) < need:
        raise ValueError(f"scratch must be a uint8 tensor of at least {need} bytes on {elements.device}")
    ptr = lambda x: None if x is None else C.c_void_p(x.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_correlate_device(
        ptr(elements), n, int(grav), ptr(covariance), ptr(model), ptr(offsets), t, ptr(jd), ptr(fr), ptr(kind),
        ptr(value), ptr(sigma), ptr(station), ptr(stations), float(gate_probability), best,
        int(elements.device.index), ptr(scratch), ptr(rows), ptr(d2), ptr(used), ptr(n_gate), ptr(n_failed),
        ptr(status), ptr(row_status), C.c_void_p(stream) if stream else None))
