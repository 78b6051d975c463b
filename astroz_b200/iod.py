"""Initial orbits for tracks no catalogue row predicts, on the device (K13, astroz_b200/csrc/az_iod.cu).

    from astroz_b200.iod import initial_orbits, fit_tracks
    res = initial_orbits(track, jd, fr, kind, value, sigma, station, stations)
    res.elements, res.state, res.method, res.status       # (8, t) SGP4 / SDP4 sets at each track's middle observation
    res, fit = fit_tracks(track, jd, fr, kind, value, sigma, station, stations)   # ... refined, with covariance

A track that `correlate` returns UNCORRELATED is a new or lost object.  For each track this builds candidate orbits
from every method its observations allow -- the state observations themselves, Gibbs and Herrick-Gibbs on radar
position triplets, Lambert between two radar positions, Gauss on optical triplets (every admissible root) -- scores
each two-body against every observation of the track, and converts the winner's state at the track's epoch (its
middle observation) to SGP4 / SDP4 mean elements with the element fit's own solver.  The sets go straight into
`fit_observations`; `fit_tracks` does both.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._abi import DEFINES as D
from ._lib import WGS72, check, lib
from .fit import _csr, _integers, _obs_columns, _stations

OK, TOO_FEW, NO_CANDIDATE, CONVERSION_FAILED, BAD_TRACK = (
    D["ASTROZ_IOD_OK"], D["ASTROZ_IOD_TOO_FEW"], D["ASTROZ_IOD_NO_CANDIDATE"], D["ASTROZ_IOD_CONVERSION_FAILED"],
    D["ASTROZ_IOD_BAD_TRACK"])
STATUS_NAMES = {OK: "converted", TOO_FEW: "fewer observations than any method needs",
                NO_CANDIDATE: "every candidate rejected", CONVERSION_FAILED: "the mean-element conversion failed",
                BAD_TRACK: "empty, too long, no used residual or out of time order"}
METHOD_STATE, METHOD_GIBBS, METHOD_HERRICK_GIBBS, METHOD_LAMBERT, METHOD_GAUSS, METHOD_NONE = (
    D["ASTROZ_IOD_METHOD_STATE"], D["ASTROZ_IOD_METHOD_GIBBS"], D["ASTROZ_IOD_METHOD_HERRICK_GIBBS"],
    D["ASTROZ_IOD_METHOD_LAMBERT"], D["ASTROZ_IOD_METHOD_GAUSS"], D["ASTROZ_IOD_METHOD_NONE"])
METHOD_NAMES = {METHOD_STATE: "state", METHOD_GIBBS: "Gibbs", METHOD_HERRICK_GIBBS: "Herrick-Gibbs",
                METHOD_LAMBERT: "Lambert", METHOD_GAUSS: "Gauss", METHOD_NONE: "none"}
MAX_TRACK = D["ASTROZ_IOD_MAX_TRACK"]


@dataclass
class IodResult:
    elements: np.ndarray     # (8, t) converted sets: epoch JD (the track's epoch), n rev/day, e, i, RAAN, w, M deg, B*
    state: np.ndarray        # (t, 6) TEME state at the epoch [km, km/s]
    wrms: np.ndarray         # (t,) two-body score of the winner, sqrt(F / used residuals)
    method: np.ndarray       # (t,) uint8 METHOD_*
    candidates: np.ndarray   # (t,) candidates scored
    conv_dr: np.ndarray      # (t,) km: the converted set's position residual at the epoch
    conv_dv: np.ndarray      # (t,) km/s
    deep_space: np.ndarray   # (t,) bool: an SDP4 (period > 225 min) set
    status: np.ndarray       # (t,) uint8 ASTROZ_IOD_*


def initial_orbits(track, jd, fr, kind, value, sigma, station=None, stations=None, *, bstar=None, grav: int = WGS72,
                   device: int = 0) -> IodResult:
    """Initial orbits of tracks (astroz_cuda_initial_orbits).

    Observation i (any order; grouped stably by track, then sorted stably by time) belongs to track[i] in [0, t),
    t = max(track) + 1, and is described as in `fit_observations`.  bstar: (t,) B* of each converted set (default 0).
    Returns one result row per track id."""
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
    bs = None
    if bstar is not None:
        bs = np.ascontiguousarray(np.broadcast_to(np.asarray(bstar, dtype=np.float64), (t,)))
    el, state, wrms = np.zeros((8, t)), np.zeros((t, 6)), np.zeros(t)
    method, cand = np.zeros(t, dtype=np.uint8), np.zeros(t, dtype=np.uint32)
    conv, deep, status = np.zeros((t, 2)), np.zeros(t, dtype=np.uint8), np.zeros(t, dtype=np.uint8)
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_initial_orbits(vp(offsets), t, vp(jd_s), vp(fr_s), vp(kind_s), vp(val_s), vp(sig_s),
                                           vp(sta_s), m, vp(st), len(st), vp(bs), int(grav), int(device), vp(el),
                                           vp(state), vp(wrms), vp(method), vp(cand), vp(conv), vp(deep), vp(status)))
    return IodResult(el, state, wrms, method, cand, conv[:, 0].copy(), conv[:, 1].copy(), deep == 1, status)


def initial_orbits_scratch_bytes(t: int) -> int:
    """Bytes of the scratch `initial_orbits_device` needs"""
    out = C.c_uint64()
    check(lib().astroz_cuda_initial_orbits_scratch_bytes(int(t), C.byref(out)))
    return out.value


def initial_orbits_device(offsets, jd, fr, kind, value, sigma, station, stations, bstar, scratch, elements, state,
                          wrms, method, candidates, conv, deep_space, status, *, grav: int = WGS72,
                          stream: int = 0) -> None:
    """`initial_orbits` with torch CUDA tensors on one device, observations grouped by track and in time order within
    each: offsets (t + 1,) int32, jd / fr (m,) float64, kind (m,) uint8, value / sigma (m, 6) float64, station (m,)
    int32 or None, stations (k, 3) float64 or None, bstar (t,) float64 or None, scratch a uint8 tensor of at least
    initial_orbits_scratch_bytes(t) bytes; elements (8, t), state (t, 6), wrms (t,), conv (t, 2) float64, method (t,)
    uint8, candidates (t,) int32, deep_space and status (t,) uint8 receive the results.  Launches on `stream` (a raw
    cudaStream_t value, 0 = the default stream); nothing is checked beyond shapes: a bad track gets BAD_TRACK."""
    import torch

    if not isinstance(offsets, torch.Tensor) or not offsets.is_cuda:
        raise ValueError("offsets must be a CUDA int32 tensor of shape (t + 1,)")
    dev = offsets.device
    t = int(offsets.numel()) - 1
    m = int(jd.numel())
    k = 0 if stations is None else int(stations.numel()) // 3
    tensors = [("offsets", offsets, t + 1, torch.int32), ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64),
               ("kind", kind, m, torch.uint8), ("value", value, 6 * m, torch.float64),
               ("sigma", sigma, 6 * m, torch.float64), ("station", station, m, torch.int32),
               ("stations", stations, 3 * k, torch.float64), ("bstar", bstar, t, torch.float64),
               ("elements", elements, 8 * t, torch.float64), ("state", state, 6 * t, torch.float64),
               ("wrms", wrms, t, torch.float64), ("method", method, t, torch.uint8),
               ("candidates", candidates, t, torch.int32), ("conv", conv, 2 * t, torch.float64),
               ("deep_space", deep_space, t, torch.uint8), ("status", status, t, torch.uint8)]
    for name, x, size, dtype in tensors:
        if x is None and name in ("station", "stations", "bstar"):
            continue
        if not isinstance(x, torch.Tensor) or x.dtype != dtype or not x.is_contiguous() or int(x.numel()) != size \
                or x.device != dev:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {dev}")
    need = initial_orbits_scratch_bytes(t)
    if not isinstance(scratch, torch.Tensor) or scratch.dtype != torch.uint8 or scratch.device != dev \
            or int(scratch.numel()) < need:
        raise ValueError(f"scratch must be a uint8 tensor of at least {need} bytes on {dev}")
    ptr = lambda x: None if x is None else C.c_void_p(x.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_initial_orbits_device(
        ptr(offsets), t, ptr(jd), ptr(fr), ptr(kind), ptr(value), ptr(sigma), ptr(station), ptr(stations), ptr(bstar),
        int(grav), int(dev.index), ptr(scratch), ptr(elements), ptr(state), ptr(wrms), ptr(method), ptr(candidates),
        ptr(conv), ptr(deep_space), ptr(status), C.c_void_p(stream) if stream else None))


def fit_tracks(track, jd, fr, kind, value, sigma, station=None, stations=None, *, bstar=None, max_iter: int = 25,
               grav: int = WGS72, device: int = 0):
    """`initial_orbits`, then `fit_observations` of every converted track to its own observations (deep-space sets
    under SDP4, B* held at the given value): the one call from a track to a catalogue row with covariance.  Returns
    (IodResult, FitResult); the FitResult has one row per track, and a track whose status is not OK keeps its (zero)
    row with status INIT_FAILED."""
    from .fit import INIT_FAILED, FitResult, fit_observations

    res = initial_orbits(track, jd, fr, kind, value, sigma, station, stations, bstar=bstar, grav=grav, device=device)
    t = res.status.shape[0]
    ok = np.flatnonzero(res.status == OK)
    track = np.asarray(track).reshape(-1)
    fit = FitResult(np.zeros((8, t)), np.zeros(t), np.zeros(t), np.zeros(t, np.uint32),
                    np.full(t, INIT_FAILED, np.uint8), np.zeros(t), np.zeros(t, np.uint32), np.zeros((t, 28)),
                    np.zeros(t, bool))
    if len(ok):
        row = np.full(t, -1)
        row[ok] = np.arange(len(ok))
        take = row[track] >= 0
        sub = fit_observations(res.elements[:, ok], row[track][take], np.asarray(jd).reshape(-1)[take],
                               np.asarray(fr).reshape(-1)[take], np.asarray(kind).reshape(-1)[take],
                               np.asarray(value)[take], np.asarray(sigma)[take],
                               None if station is None else np.asarray(station).reshape(-1)[take], stations,
                               fit_bstar=False, max_iter=max_iter, grav=grav, device=device, deep_space=True)
        fit.elements[:, ok] = sub.elements
        for name in ("rms_pos", "rms_vel", "iterations", "status", "wrms", "n_residuals", "covariance", "deep_space"):
            getattr(fit, name)[ok] = getattr(sub, name)
    return res, fit
