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

    from astroz_b200.iod import fit_links
    links = fit_links(track, jd, fr, kind, value, sigma, station, stations)   # every pair within 1.5 days
    pairs, elements, covariance, deep_space = links.linked()                 # new catalogue rows from two tracks each

Where one short track is not enough (the 55-minute optical arcs of deep-space objects), `link_tracks` determines an
orbit from two tracks together: Lambert transfers between the tracks' anchor observations over range hypotheses,
scored two-body against both tracks and refined on the ranges, converted like a single track's (K17, az_link.cu).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._abi import DEFINES as D
from ._lib import WGS72, check, lib
from .fit import OBS_OPTICAL, _csr, _integers, _obs_columns, _stations

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


def _sorted_obs(track, jd, fr, kind, value, sigma, station):
    """the observations grouped stably by track (offsets (t + 1,)), as the host calls take them"""
    track = np.asarray(track).reshape(-1)
    t = int(track.max()) + 1 if track.size else 0
    order, offsets = _csr(t, track)
    kind_all = np.asarray(kind).reshape(-1)
    out = dict(jd=np.ascontiguousarray(np.asarray(jd, dtype=np.float64).reshape(-1)[order]),
               fr=np.ascontiguousarray(np.asarray(fr, dtype=np.float64).reshape(-1)[order]),
               kind=np.ascontiguousarray(_integers(kind_all, "kind", 8)[order]),
               value=np.ascontiguousarray(_obs_columns(value, len(kind_all), "value", 0.0)[order]),
               sigma=np.ascontiguousarray(_obs_columns(sigma, len(kind_all), "sigma", np.inf)[order]),
               station=None if station is None else np.ascontiguousarray(
                   _integers(np.asarray(station).reshape(-1), "station", 32)[order]))
    m = len(order)
    if any(len(out[k]) != m for k in ("jd", "fr", "kind")) or (out["station"] is not None and len(out["station"]) != m):
        raise ValueError("track, jd, fr, kind, value, sigma and station must describe the same observations")
    return t, offsets, out


def initial_orbits(track, jd, fr, kind, value, sigma, station=None, stations=None, *, bstar=None, grav: int = WGS72,
                   device: int = 0) -> IodResult:
    """Initial orbits of tracks (astroz_cuda_initial_orbits).

    Observation i (any order; grouped stably by track, then sorted stably by time) belongs to track[i] in [0, t),
    t = max(track) + 1, and is described as in `fit_observations`.  bstar: (t,) B* of each converted set (default 0).
    Returns one result row per track id."""
    t, offsets, o = _sorted_obs(track, jd, fr, kind, value, sigma, station)
    jd_s, fr_s, kind_s, val_s, sig_s, sta_s = (o[k] for k in ("jd", "fr", "kind", "value", "sigma", "station"))
    m = len(jd_s)
    st = _stations(stations)
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


# ---- track linking (K17, astroz_b200/csrc/az_link.cu) ---------------------------------------------------------------
LINK_OK, LINK_TOO_FEW, LINK_NO_CANDIDATE, LINK_CONVERSION_FAILED, LINK_BAD_TRACK, LINK_BAD_PAIR = (
    D["ASTROZ_LINK_OK"], D["ASTROZ_LINK_TOO_FEW"], D["ASTROZ_LINK_NO_CANDIDATE"], D["ASTROZ_LINK_CONVERSION_FAILED"],
    D["ASTROZ_LINK_BAD_TRACK"], D["ASTROZ_LINK_BAD_PAIR"])
LINK_STATUS_NAMES = {LINK_OK: "converted", LINK_TOO_FEW: "a track without an anchor observation",
                     LINK_NO_CANDIDATE: "no admissible transfer",
                     LINK_CONVERSION_FAILED: "the mean-element conversion failed",
                     LINK_BAD_TRACK: "empty, too long, no used residual or out of time order",
                     LINK_BAD_PAIR: "a pair index out of range, one track twice, or anchors at the same time"}
LINK_RETROGRADE, LINK_RIGHT_BRANCH = D["ASTROZ_LINK_RETROGRADE"], D["ASTROZ_LINK_RIGHT_BRANCH"]
LINK_R_MIN, LINK_R_MAX = 6578.0, 50000.0   # km: 200 km above the equator to past the GEO belt


@dataclass
class LinkResult:
    pairs: np.ndarray        # (p, 2) the pairs as given
    elements: np.ndarray     # (8, p) converted sets: epoch JD (the later anchor), n rev/day, e, i, RAAN, w, M, B*
    state: np.ndarray        # (p, 6) TEME state at the epoch [km, km/s]
    rho: np.ndarray          # (p, 2) the winner's ranges [km], the track with the earlier anchor first
    revs: np.ndarray         # (p,) uint8 complete revolutions of the transfer
    flags: np.ndarray        # (p,) uint8 LINK_RETROGRADE (normal -z) | LINK_RIGHT_BRANCH
    wrms: np.ndarray         # (p,) two-body score over both tracks, sqrt(F / used)
    used: np.ndarray         # (p,) uint32 used residuals of both tracks
    hypotheses: np.ndarray   # (p,) uint32 admissible transfers scored
    conv_dr: np.ndarray      # (p,) km
    conv_dv: np.ndarray      # (p,) km/s
    deep_space: np.ndarray   # (p,) bool
    status: np.ndarray       # (p,) uint8 ASTROZ_LINK_*


def link_tracks(track, jd, fr, kind, value, sigma, station=None, stations=None, pairs=None, *,
                r_min: float = LINK_R_MIN, r_max: float = LINK_R_MAX, max_revs: int = 1, bstar=None,
                grav: int = WGS72, device: int = 0) -> LinkResult:
    """Orbits from pairs of tracks (astroz_cuda_link_tracks).

    Observations as in `initial_orbits`; pairs (p, 2) track ids.  For each pair: Lambert transfers between the tracks'
    anchor observations over a grid of range hypotheses in [r_min, r_max] km (geocentric) and 0 .. max_revs
    revolutions, the best scored two-body against both tracks and refined on its ranges, then converted to an SGP4 /
    SDP4 set at the later anchor's time with B* = bstar (p,) (default 0).  One result row per pair."""
    t, offsets, o = _sorted_obs(track, jd, fr, kind, value, sigma, station)
    m = len(o["jd"])
    st = _stations(stations)
    pr = np.asarray(pairs if pairs is not None else np.zeros((0, 2)), dtype=np.int64).reshape(-1, 2)
    if pr.size and (pr.min() < 0 or pr.max() > 0xFFFFFFFF):
        raise ValueError("pairs must be track ids in [0, t)")
    pr32 = np.ascontiguousarray(pr, dtype=np.uint32)
    p = len(pr32)
    bs = None
    if bstar is not None:
        bs = np.ascontiguousarray(np.broadcast_to(np.asarray(bstar, dtype=np.float64), (p,)))
    el, state, rho, wrms = np.zeros((8, p)), np.zeros((p, 6)), np.zeros((p, 2)), np.zeros(p)
    revs, flags, deep, status = (np.zeros(p, dtype=np.uint8) for _ in range(4))
    used, hyp, conv = np.zeros(p, dtype=np.uint32), np.zeros(p, dtype=np.uint32), np.zeros((p, 2))
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_link_tracks(vp(offsets), t, vp(o["jd"]), vp(o["fr"]), vp(o["kind"]), vp(o["value"]),
                                        vp(o["sigma"]), vp(o["station"]), m, vp(st), len(st), vp(pr32), p, vp(bs),
                                        float(r_min), float(r_max), int(max_revs), int(grav), int(device), vp(el),
                                        vp(state), vp(rho), vp(revs), vp(flags), vp(wrms), vp(used), vp(hyp),
                                        vp(conv), vp(deep), vp(status)))
    return LinkResult(pr, el, state, rho, revs, flags, wrms, used, hyp, conv[:, 0].copy(), conv[:, 1].copy(),
                      deep == 1, status)


def link_tracks_scratch_bytes(p: int) -> int:
    """Bytes of the scratch `link_tracks_device` needs"""
    out = C.c_uint64()
    check(lib().astroz_cuda_link_tracks_scratch_bytes(int(p), C.byref(out)))
    return out.value


def link_tracks_device(offsets, jd, fr, kind, value, sigma, station, stations, pairs, bstar, scratch, elements, state,
                       rho, revs, flags, wrms, used, hypotheses, conv, deep_space, status, *, r_min: float = LINK_R_MIN,
                       r_max: float = LINK_R_MAX, max_revs: int = 1, grav: int = WGS72, stream: int = 0) -> None:
    """`link_tracks` with torch CUDA tensors on one device, observations grouped by track and in time order within
    each: as `initial_orbits_device`, plus pairs (p, 2) int32 and bstar (p,) float64 or None; scratch a uint8 tensor of
    at least link_tracks_scratch_bytes(p) bytes; elements (8, p), state (p, 6), rho (p, 2), wrms (p,), conv (p, 2)
    float64, revs, flags, deep_space, status (p,) uint8, used and hypotheses (p,) int32 receive the results.  Nothing
    is checked beyond shapes and scalars: a bad track gets BAD_TRACK, a bad pair BAD_PAIR."""
    import torch

    if not isinstance(offsets, torch.Tensor) or not offsets.is_cuda:
        raise ValueError("offsets must be a CUDA int32 tensor of shape (t + 1,)")
    dev = offsets.device
    t = int(offsets.numel()) - 1
    m = int(jd.numel())
    p = int(pairs.numel()) // 2 if isinstance(pairs, torch.Tensor) else -1
    k = 0 if stations is None else int(stations.numel()) // 3
    tensors = [("offsets", offsets, t + 1, torch.int32), ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64),
               ("kind", kind, m, torch.uint8), ("value", value, 6 * m, torch.float64),
               ("sigma", sigma, 6 * m, torch.float64), ("station", station, m, torch.int32),
               ("stations", stations, 3 * k, torch.float64), ("pairs", pairs, 2 * p, torch.int32),
               ("bstar", bstar, p, torch.float64), ("elements", elements, 8 * p, torch.float64),
               ("state", state, 6 * p, torch.float64), ("rho", rho, 2 * p, torch.float64),
               ("revs", revs, p, torch.uint8), ("flags", flags, p, torch.uint8), ("wrms", wrms, p, torch.float64),
               ("used", used, p, torch.int32), ("hypotheses", hypotheses, p, torch.int32),
               ("conv", conv, 2 * p, torch.float64), ("deep_space", deep_space, p, torch.uint8),
               ("status", status, p, torch.uint8)]
    for name, x, size, dtype in tensors:
        if x is None and name in ("station", "stations", "bstar"):
            continue
        if not isinstance(x, torch.Tensor) or x.dtype != dtype or not x.is_contiguous() or int(x.numel()) != size \
                or x.device != dev:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {dev}")
    need = link_tracks_scratch_bytes(p)
    if not isinstance(scratch, torch.Tensor) or scratch.dtype != torch.uint8 or scratch.device != dev \
            or int(scratch.numel()) < need:
        raise ValueError(f"scratch must be a uint8 tensor of at least {need} bytes on {dev}")
    ptr = lambda x: None if x is None else C.c_void_p(x.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_link_tracks_device(
        ptr(offsets), t, ptr(jd), ptr(fr), ptr(kind), ptr(value), ptr(sigma), ptr(station), ptr(stations), ptr(pairs),
        p, ptr(bstar), float(r_min), float(r_max), int(max_revs), int(grav), int(dev.index), ptr(scratch),
        ptr(elements), ptr(state), ptr(rho), ptr(revs), ptr(flags), ptr(wrms), ptr(used), ptr(hypotheses), ptr(conv),
        ptr(deep_space), ptr(status), C.c_void_p(stream) if stream else None))


def anchor_times(track, jd, fr, kind, sigma):
    """(t,) jd + fr of each track's anchor observation (NaN without one): its middle observation, in time order, among
    those whose line of sight is used in full (both optical angles; radar range, azimuth and elevation; a state's
    position)"""
    track = np.asarray(track).reshape(-1)
    t = int(track.max()) + 1 if track.size else 0
    jdf = np.asarray(jd, dtype=np.float64).reshape(-1) + np.asarray(fr, dtype=np.float64).reshape(-1)
    kind = np.asarray(kind).reshape(-1)
    sig = _obs_columns(sigma, len(kind), "sigma", np.inf)
    need = np.where(kind == OBS_OPTICAL, 2, 3)
    ok = np.all(np.isfinite(sig[:, :3]) | (np.arange(3)[None, :] >= need[:, None]), axis=1)
    order = np.lexsort((jdf, track))
    tr_s, ok_s, t_s = track[order], ok[order], jdf[order]
    sel = np.flatnonzero(ok_s)
    out = np.full(t, np.nan)
    if len(sel):
        ids = tr_s[sel]
        first = np.searchsorted(ids, np.arange(t))
        count = np.searchsorted(ids, np.arange(t), side="right") - first
        has = count > 0
        out[has] = t_s[sel[first[has] + count[has] // 2]]
    return out


def candidate_pairs(anchor_t, max_gap_days: float) -> np.ndarray:
    """(p, 2) every pair of tracks (lower id first) whose anchors are at most max_gap_days apart and not equal"""
    ids = np.flatnonzero(np.isfinite(anchor_t))
    order = ids[np.argsort(anchor_t[ids], kind="stable")]
    ts = anchor_t[order]
    n = np.searchsorted(ts, ts + max_gap_days, side="right") - np.arange(len(ts)) - 1   # later partners of each
    a = np.repeat(np.arange(len(ts)), n)
    b = a + 1 + np.arange(len(a)) - np.repeat(np.cumsum(n) - n, n)
    a, b = order[a], order[b]
    keep = anchor_t[a] != anchor_t[b]
    pr = np.stack([np.minimum(a, b), np.maximum(a, b)], axis=1)[keep]
    return pr[np.lexsort((pr[:, 1], pr[:, 0]))] if len(pr) else pr.reshape(0, 2)


def best_links(pairs, wrms, status, best: int) -> np.ndarray:
    """Ascending indices of the OK links (status LINK_OK) that are among the `best` links of least wrms of either of
    their tracks: every OK link is ranked once within each of its two tracks over all of that track's OK links (ties
    by link index)."""
    pairs = np.asarray(pairs).reshape(-1, 2)
    ok = np.flatnonzero(np.asarray(status) == LINK_OK)
    link = np.concatenate([ok, ok])
    tid = np.concatenate([pairs[ok, 0], pairs[ok, 1]])
    order = np.lexsort((link, np.asarray(wrms)[link], tid))
    tid_s = tid[order]
    rank = np.arange(len(order)) - np.searchsorted(tid_s, tid_s)
    return np.unique(link[order][rank < best])


@dataclass
class LinkFit:
    links: LinkResult        # link_tracks on every candidate pair
    fitted: np.ndarray       # (q,) indices into links of the pairs that were fitted
    fit: object              # FitResult of those pairs, one row each (both tracks' observations, B* held)
    gate: np.ndarray         # (q,) chi-square gate of each fitted pair
    consistent: np.ndarray   # (q,) bool: converged and wrms^2 n_residuals <= gate

    def linked(self):
        """The mutually-best consistent pairs: (pairs (k, 2), elements (8, k), covariance (k, 28), deep_space (k,)),
        each pair being the consistent link of least fitted wrms of both its tracks; rows ready to append to a
        catalogue (elements and covariance as fit_observations gives them)."""
        idx = np.flatnonzero(self.consistent)
        pr = self.links.pairs[self.fitted[idx]]
        w = self.fit.wrms[idx]
        best = {}
        for q in np.lexsort((np.arange(len(idx)), w)):
            for tid in pr[q]:
                best.setdefault(int(tid), q)
        keep = np.array([q for q in range(len(idx)) if best[int(pr[q, 0])] == q and best[int(pr[q, 1])] == q], int)
        sel = idx[keep] if len(keep) else np.zeros(0, int)
        return (pr[keep].reshape(-1, 2), self.fit.elements[:, sel], self.fit.covariance[sel],
                self.fit.deep_space[sel])


def fit_links(track, jd, fr, kind, value, sigma, station=None, stations=None, *, pairs=None, max_gap_days: float = 1.5,
              best: int = 4, gate_probability: float = 0.99, r_min: float = LINK_R_MIN, r_max: float = LINK_R_MAX,
              max_revs: int = 1, max_iter: int = 25, grav: int = WGS72, device: int = 0) -> LinkFit:
    """Link uncorrelated tracks into orbits: `link_tracks` on `pairs` (default: every pair whose anchors are within
    max_gap_days), then `fit_observations` (mixed, B* held at 0) over both tracks' observations for each OK link that
    is among the `best` links of least two-body wrms of either of its tracks (`best_links`).  A fitted link is
    consistent when the fit converged and wrms^2 n_residuals <= the chi-square quantile of n_residuals - 6 degrees of
    freedom at gate_probability.  `LinkFit.linked()` gives the mutually-best ones."""
    from .correlate import chi2_quantile
    from .fit import CONVERGED, fit_observations

    track = np.asarray(track).reshape(-1)
    t = int(track.max()) + 1 if track.size else 0
    if pairs is None:
        pairs = candidate_pairs(anchor_times(track, jd, fr, kind, sigma), max_gap_days)
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    res = link_tracks(track, jd, fr, kind, value, sigma, station, stations, pairs, r_min=r_min, r_max=r_max,
                      max_revs=max_revs, grav=grav, device=device)
    fitted = best_links(res.pairs, res.wrms, res.status, best)
    from .fit import FitResult

    if not len(fitted):
        empty = FitResult(np.zeros((8, 0)), np.zeros(0), np.zeros(0), np.zeros(0, np.uint32), np.zeros(0, np.uint8),
                          np.zeros(0), np.zeros(0, np.uint32), np.zeros((0, 28)), np.zeros(0, bool))
        return LinkFit(res, fitted, empty, np.zeros(0), np.zeros(0, bool))
    # both tracks' observations, repeated once per fitted pair that uses them
    order, offsets = _csr(t, track)
    obs_of = lambda j: order[offsets[j]:offsets[j + 1]]  # noqa: E731
    take = [np.concatenate([obs_of(a), obs_of(b)]) for a, b in pairs[fitted]]
    rows = np.repeat(np.arange(len(fitted)), [len(x) for x in take])
    take = np.concatenate(take)
    val, sig = np.asarray(value).reshape(len(track), -1), np.asarray(sigma).reshape(len(track), -1)
    fit = fit_observations(res.elements[:, fitted], rows, np.asarray(jd).reshape(-1)[take],
                           np.asarray(fr).reshape(-1)[take], np.asarray(kind).reshape(-1)[take], val[take], sig[take],
                           None if station is None else np.asarray(station).reshape(-1)[take], stations,
                           fit_bstar=False, max_iter=max_iter, grav=grav, device=device, deep_space=True)
    n_res = fit.n_residuals.astype(np.int64)
    gate = np.array([chi2_quantile(int(k) - 6, gate_probability) if k > 6 else 0.0 for k in n_res])
    consistent = (fit.status == CONVERGED) & (n_res > 6) & (fit.wrms ** 2 * n_res <= gate)
    return LinkFit(res, fitted, fit, gate, consistent)
