"""Fit SGP4 mean elements to TEME ephemerides on the device (K8, astroz_b200/csrc/az_fit.cu).

    from astroz_b200.fit import fit_elements
    res = fit_elements(tle_pairs, sat, jd, fr, pos, vel)          # or an (8, n) array of element columns
    res.elements, res.rms_pos, res.status; res.to_tle_pairs()

The reverse of propagation: for each satellite, the near-earth mean elements at its epoch whose SGP4 states best match
its observations (GPS or precise-ephemeris states, a numerical trajectory, a Monte-Carlo member) in the weighted least-
squares sense.  Levenberg-Marquardt over n, e cos w, e sin w, i, RAAN, M + w and B* (optional), every trial element set
propagated by the library's own near-earth path, one GPU warp per satellite.  The fitted columns, passed to
`Constellation.from_elements` and propagated at the observation times, give back the reported RMS.

Deep-space sets (period > 225 min: GEO, GPS, Molniya) are fitted with `deep_space=True`, under SDP4 with equinoctial
variables (n, e cos(w + RAAN), e sin(w + RAAN), tan(i/2) cos RAAN, tan(i/2) sin RAAN, M + w + RAAN, B*), which stay well
conditioned at i = 0 and e = 0.  Near-earth rows of such a batch are fitted exactly as without it.  By default deep-space
sets are returned unfitted with status DEEP_SPACE.

`fit_observations` fits the same way to what sensors report -- TEME or Earth-fixed states (GPS), radar range / azimuth /
elevation / range-rate, optical right ascension / declination -- each observation with its own kind, station and
sigmas, and returns the formal covariance of the fitted variables.  `observe` evaluates the measurement model alone.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._abi import DEFINES as D
from ._lib import WGS72, check, lib

# per-satellite status bytes
CONVERGED, ITERATION_LIMIT, INIT_FAILED, DEEP_SPACE, TOO_FEW_OBSERVATIONS = (
    D["ASTROZ_FIT_CONVERGED"], D["ASTROZ_FIT_ITERATION_LIMIT"], D["ASTROZ_FIT_INIT_FAILED"], D["ASTROZ_FIT_DEEP_SPACE"],
    D["ASTROZ_FIT_TOO_FEW_OBSERVATIONS"])
STATUS_NAMES = {CONVERGED: "converged", ITERATION_LIMIT: "iteration limit", INIT_FAILED: "initial set fails init",
                DEEP_SPACE: "deep space, not fitted (deep_space=False)", TOO_FEW_OBSERVATIONS: "too few observations"}


def parse_tle(line1: str, line2: str) -> np.ndarray:
    """The eight element columns of one TLE line pair, read by the library's parser (the numbers `create` uses)."""
    out = np.zeros(8)
    check(lib().astroz_cuda_parse_tle(line1.encode(), line2.encode(), out.ctypes.data_as(C.POINTER(C.c_double))))
    return out


def _initial_columns(initial) -> np.ndarray:
    if isinstance(initial, (list, tuple)) and initial and isinstance(initial[0], (list, tuple)) \
            and isinstance(initial[0][0], str):
        return np.ascontiguousarray(np.stack([parse_tle(l1, l2) for l1, l2 in initial], axis=1))
    el = np.ascontiguousarray(initial, dtype=np.float64)
    if el.ndim != 2 or el.shape[0] != 8:
        raise ValueError("initial must be TLE line pairs or an (8, n) array: epoch JD, n rev/day, e, i, RAAN, w, M "
                         "deg, B*")
    return el


def _jd_to_year_doy(jd: float) -> tuple[int, float]:
    """Inverse of the TLE epoch rule (src/Datetime.zig:222-231): doy 1.0 = Jan 1 00:00 of the year."""
    year = int(np.floor((jd - 1721058.5) / 365.25)) + 1
    for y in (year + 1, year, year - 1):
        jan0 = 367.0 * y - np.floor(7 * y / 4) + 30 + 1721013.5   # JD of Jan 0.0 (1901..2099)
        if jd >= jan0 + 1.0:
            return y, jd - jan0
    raise ValueError("epoch outside 1901..2099")


# observation kinds (ASTROZ_OBS_*) and their value counts
OBS_TEME_STATE, OBS_ECEF_STATE, OBS_RADAR, OBS_OPTICAL = (
    D["ASTROZ_OBS_TEME_STATE"], D["ASTROZ_OBS_ECEF_STATE"], D["ASTROZ_OBS_RADAR"], D["ASTROZ_OBS_OPTICAL"])
OBS_COUNTS = {OBS_TEME_STATE: 6, OBS_ECEF_STATE: 6, OBS_RADAR: 4, OBS_OPTICAL: 2}
_OBS_VALUES = D["ASTROZ_OBS_VALUES"]
_COV_WORDS = D["ASTROZ_FIT_COVARIANCE_WORDS"]
_TRIU = np.triu_indices(7)   # the covariance words, row by row over the upper triangle


@dataclass
class FitResult:
    elements: np.ndarray     # (8, n) fitted columns, epoch unchanged
    rms_pos: np.ndarray      # (n,) km: sqrt(mean |r_obs - r_fit|^2) (fit_elements; zero from fit_observations)
    rms_vel: np.ndarray      # (n,) km/s (0 without velocities)
    iterations: np.ndarray   # (n,) uint32 LM steps tried
    status: np.ndarray       # (n,) uint8 ASTROZ_FIT_*
    wrms: np.ndarray | None = None          # (n,) sqrt(cost / used residuals), fit_observations only
    n_residuals: np.ndarray | None = None   # (n,) uint32 used scalar residuals, fit_observations only
    covariance: np.ndarray | None = None    # (n, 28) upper triangle of the fitted variables' covariance
    deep_space: np.ndarray | None = None    # (n,) bool: the library fitted the row in the deep-space (equinoctial)
    #                                         variables (its deep-space pass ran on it), fit_observations only

    def covariance_matrix(self, s: int) -> np.ndarray:
        """The 7 x 7 covariance of satellite s in the fit's own variables and order -- near-earth: n [rev/day], e cos w,
        e sin w, i, RAAN, M + w [rad], B* [1/ER]; deep space: n, e cos(w + RAAN), e sin(w + RAAN), tan(i/2) cos RAAN,
        tan(i/2) sin RAAN, M + w + RAAN, B*.  All zeros: the normal matrix was not positive definite or s was not
        fitted; the B* row and column are zero when B* was held."""
        if self.covariance is None:
            raise ValueError("no covariance: the result of fit_elements (fit_observations returns one)")
        P = np.zeros((7, 7))
        P[_TRIU] = self.covariance[s]
        return P + np.triu(P, 1).T

    def element_covariance(self, s: int) -> np.ndarray:
        """Satellite s's covariance mapped to (n rev/day, e, i, RAAN, w, M [rad], B*) by the analytic Jacobian of the
        variables -> elements map, near-earth or equinoctial as the row was fitted.  It is singular at e = 0 (w and M
        are not defined there) and, for a deep-space row, at i = 0 (neither is RAAN)."""
        P = self.covariance_matrix(s)
        J = element_jacobian(self.elements[:, s], bool(self.deep_space[s]))
        return J @ P @ J.T

    def to_tle_pairs(self, satnums=None) -> list[tuple[str, str]]:
        """The fitted sets as checksummed TLE line pairs (satellite numbers 0, 1, ... unless given), rendered by the
        formatting `frontend.omm_to_tle_pairs` uses."""
        from .frontend import tle_line_pair

        n = self.elements.shape[1]
        nums = range(n) if satnums is None else satnums
        out = []
        for s, num in zip(range(n), nums):
            e = self.elements[:, s]
            year, doy = _jd_to_year_doy(float(e[0]))
            out.append(tle_line_pair(int(num), year, doy, e[3], e[4], e[2], e[5], e[6], e[1], e[7]))
        return out


def element_jacobian(el, deep: bool) -> np.ndarray:
    """d(n, e, i, RAAN, w, M, B*) / d(fit variables) at the element columns el (8,): the fit's variables -> elements
    map (near-earth, or equinoctial for deep), differentiated analytically.  Angles in rad."""
    d2r = np.pi / 180.0
    e, inc, node, argp = el[2], el[3] * d2r, el[4] * d2r, el[5] * d2r
    J = np.zeros((7, 7))
    J[0, 0] = J[6, 6] = 1.0
    peri = argp + node if deep else argp          # the angle of (e cos, e sin)
    k, h = e * np.cos(peri), e * np.sin(peri)
    J[1, 1], J[1, 2] = k / e, h / e               # e = |(k, h)|
    dpk, dph = -h / e ** 2, k / e ** 2            # d(peri) / d(k, h)
    if not deep:
        J[2, 3] = J[3, 4] = 1.0                   # i, RAAN
        J[4, 1], J[4, 2] = dpk, dph               # w = peri
        J[5, 1], J[5, 2], J[5, 5] = -dpk, -dph, 1.0   # M = lambda - w
        return J
    t = np.tan(0.5 * inc)
    q, p = t * np.cos(node), t * np.sin(node)
    J[2, 3], J[2, 4] = 2.0 / (1.0 + t * t) * q / t, 2.0 / (1.0 + t * t) * p / t   # i = 2 atan |(q, p)|
    J[3, 3], J[3, 4] = -p / t ** 2, q / t ** 2                                    # RAAN = atan2(p, q)
    J[4, 1], J[4, 2], J[4, 3], J[4, 4] = dpk, dph, -J[3, 3], -J[3, 4]             # w = peri - RAAN
    J[5, 1], J[5, 2], J[5, 5] = -dpk, -dph, 1.0                                   # M = lambda - peri
    return J


def _csr(n: int, sat):
    sat = np.asarray(sat)
    if sat.ndim != 1 or (len(sat) and (sat.min() < 0 or sat.max() >= n)):
        raise ValueError("sat must be a 1-D array of satellite indices in [0, n)")
    order = np.argsort(sat, kind="stable")
    offsets = np.searchsorted(sat[order], np.arange(n + 1)).astype(np.uint32)
    return order, offsets


def fit_elements(initial, sat, jd, fr, pos, vel=None, *, pos_sigma: float = 1.0, vel_sigma: float = 1e-3,
                 fit_bstar: bool = True, max_iter: int = 25, grav: int = WGS72, device: int = 0,
                 deep_space: bool = False) -> FitResult:
    """Fit n satellites at once.

    initial: TLE line pairs or an (8, n) array of element columns (epoch JD, n rev/day, e, i, RAAN, w, M deg, B*).
    sat[m], jd[m], fr[m], pos[m, 3] (TEME km), vel[m, 3] (TEME km/s, optional): the observations, in any order; they
    are sorted stably by satellite.  pos_sigma [km] and vel_sigma [km/s] weight the residuals.  deep_space: fit the
    deep-space sets too (astroz_cuda_fit_elements_mixed) instead of returning them with status DEEP_SPACE."""
    el = _initial_columns(initial)
    n = el.shape[1]
    order, offsets = _csr(n, sat)
    take = lambda a, w: np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, w)[order])  # noqa: E731
    jd_s, fr_s = take(jd, 1).ravel(), take(fr, 1).ravel()
    pos_s = take(pos, 3)
    vel_s = None if vel is None else take(vel, 3)
    m = len(order)
    if len(jd_s) != m or len(fr_s) != m or len(pos_s) != m or (vel_s is not None and len(vel_s) != m):
        raise ValueError("sat, jd, fr, pos and vel must describe the same observations")
    fitted, rms = np.zeros((8, n)), np.zeros((n, 2))
    iters, status = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
    vp = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    call = lib().astroz_cuda_fit_elements_mixed if deep_space else lib().astroz_cuda_fit_elements
    check(call(vp(el), n, int(grav), vp(offsets), vp(jd_s), vp(fr_s), vp(pos_s), vp(vel_s), m, float(pos_sigma),
               float(vel_sigma), int(bool(fit_bstar)), int(max_iter), int(device), vp(fitted), vp(rms), vp(iters),
               vp(status)))
    return FitResult(fitted, rms[:, 0].copy(), rms[:, 1].copy(), iters, status)


def fit_elements_device(elements, offsets, jd, fr, pos, vel, fitted, rms, iterations, status, *,
                        pos_sigma: float = 1.0, vel_sigma: float = 1e-3, fit_bstar: bool = True, max_iter: int = 25,
                        grav: int = WGS72, stream: int = 0, deep_space: bool = False) -> None:
    """`fit_elements` with torch CUDA tensors on one device, observations already grouped by satellite: elements (8, n)
    float64, offsets (n + 1,) int32 (non-decreasing, offsets[n] = m), jd / fr (m,) float64, pos / vel (m, 3) float64
    (vel may be None); fitted (8, n) float64, rms (n, 2) float64, iterations (n,) int32 and status (n,) uint8 receive
    the results.  One launch on `stream` (a raw cudaStream_t value, 0 = the default stream); two with deep_space, the
    deep-space fit after the near-earth one."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    m = int(jd.numel())
    tensors = [("elements", elements, 8 * n, torch.float64), ("offsets", offsets, n + 1, torch.int32),
               ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64), ("pos", pos, 3 * m, torch.float64),
               ("vel", vel, 3 * m, torch.float64), ("fitted", fitted, 8 * n, torch.float64),
               ("rms", rms, 2 * n, torch.float64), ("iterations", iterations, n, torch.int32),
               ("status", status, n, torch.uint8)]
    for name, t, size, dtype in tensors:
        if t is None and name == "vel":
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    call = lib().astroz_cuda_fit_elements_mixed_device if deep_space else lib().astroz_cuda_fit_elements_device
    check(call(
        ptr(elements), n, int(grav), ptr(offsets), ptr(jd), ptr(fr), ptr(pos), ptr(vel), float(pos_sigma),
        float(vel_sigma), int(bool(fit_bstar)), int(max_iter), int(elements.device.index), ptr(fitted), ptr(rms),
        ptr(iterations), ptr(status), C.c_void_p(stream) if stream else None))


def _integers(a, name: str, bits: int) -> np.ndarray:
    """a as unsigned integers of `bits` bits, refusing what does not fit (a cast would wrap 256 to 0)"""
    a = np.asarray(a)
    if a.size and (not np.issubdtype(a.dtype, np.integer) or a.min() < 0 or int(a.max()) >= 1 << bits):
        raise ValueError(f"{name} must hold integers in [0, 2**{bits})")
    return a.astype(np.uint8 if bits == 8 else np.uint32)


def _obs_columns(a, m: int, name: str, fill: float) -> np.ndarray:
    a = np.asarray(a, dtype=np.float64)
    a = a.reshape(m, -1) if a.ndim != 2 else a
    if a.shape[0] != m or a.shape[1] > _OBS_VALUES:
        raise ValueError(f"{name} must be (m, c) with c <= {_OBS_VALUES}")
    out = np.full((m, _OBS_VALUES), fill)
    out[:, :a.shape[1]] = a
    return out


def _stations(stations) -> np.ndarray:
    st = np.zeros((0, 3)) if stations is None else np.ascontiguousarray(stations, dtype=np.float64).reshape(-1, 3)
    return np.ascontiguousarray(st)


def fit_observations(initial, sat, jd, fr, kind, value, sigma, station=None, stations=None, *, fit_bstar: bool = True,
                     max_iter: int = 25, grav: int = WGS72, device: int = 0, deep_space: bool = False) -> FitResult:
    """Fit n satellites to sensor observations (astroz_cuda_fit_observations[_mixed]).

    initial: as fit_elements.  Observation i (any order; sorted stably by satellite): sat[i], jd[i] + fr[i], kind[i]
    (OBS_TEME_STATE, OBS_ECEF_STATE, OBS_RADAR, OBS_OPTICAL), value[i] and sigma[i] ((m, c), c <= 6: missing columns
    and sigma = inf mean "not used"), station[i] (radar and optical: a row of stations (k, 3) = geodetic lat deg, lon
    deg, height km on WGS84).  Units: km, km/s, rad.  Returns a FitResult with wrms, n_residuals and covariance."""
    el = _initial_columns(initial)
    n = el.shape[1]
    order, offsets = _csr(n, sat)
    m = len(order)
    jd_s = np.ascontiguousarray(np.asarray(jd, dtype=np.float64).reshape(-1)[order])
    fr_s = np.ascontiguousarray(np.asarray(fr, dtype=np.float64).reshape(-1)[order])
    kind_s = np.ascontiguousarray(_integers(np.asarray(kind).reshape(-1), "kind", 8)[order])
    val_s = np.ascontiguousarray(_obs_columns(value, len(np.asarray(kind).reshape(-1)), "value", 0.0)[order])
    sig_s = np.ascontiguousarray(_obs_columns(sigma, len(np.asarray(kind).reshape(-1)), "sigma", np.inf)[order])
    sta_s = None if station is None else np.ascontiguousarray(
        _integers(np.asarray(station).reshape(-1), "station", 32)[order])
    st = _stations(stations)
    if len(jd_s) != m or len(fr_s) != m or len(kind_s) != m or (sta_s is not None and len(sta_s) != m):
        raise ValueError("sat, jd, fr, kind, value, sigma and station must describe the same observations")
    fitted, wrms, nres = np.zeros((8, n)), np.zeros(n), np.zeros(n, dtype=np.uint32)
    cov = np.zeros((n, _COV_WORDS))
    iters, status, model = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.uint8)
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    call = lib().astroz_cuda_fit_observations_mixed if deep_space else lib().astroz_cuda_fit_observations
    check(call(vp(el), n, int(grav), vp(offsets), vp(jd_s), vp(fr_s), vp(val_s), vp(sig_s), vp(sta_s), vp(kind_s), m,
               vp(st), len(st), int(bool(fit_bstar)), int(max_iter), int(device), vp(fitted), vp(wrms), vp(nres),
               vp(cov), vp(iters), vp(status), vp(model)))
    return FitResult(fitted, np.zeros(n), np.zeros(n), iters, status, wrms, nres, cov, model == 1)


def fit_observations_device(elements, offsets, jd, fr, kind, value, sigma, station, stations, fitted, wrms,
                            n_residuals, covariance, iterations, status, model, *, fit_bstar: bool = True,
                            max_iter: int = 25, grav: int = WGS72, stream: int = 0,
                            deep_space: bool = False) -> None:
    """`fit_observations` with torch CUDA tensors on one device, observations grouped by satellite: elements (8, n)
    float64, offsets (n + 1,) int32, jd / fr (m,) float64, kind (m,) uint8, value / sigma (m, 6) float64, station (m,)
    int32 or None, stations (k, 3) float64 or None; fitted (8, n), wrms (n,), covariance (n, 28) float64, n_residuals and
    iterations (n,) int32, status and model (n,) uint8 receive the results (model: 1 where the row was fitted in the
    deep-space variables).  One launch on `stream` (two with deep_space)."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    m = int(jd.numel())
    k = 0 if stations is None else int(stations.numel()) // 3
    tensors = [("elements", elements, 8 * n, torch.float64), ("offsets", offsets, n + 1, torch.int32),
               ("jd", jd, m, torch.float64), ("fr", fr, m, torch.float64), ("kind", kind, m, torch.uint8),
               ("value", value, 6 * m, torch.float64), ("sigma", sigma, 6 * m, torch.float64),
               ("station", station, m, torch.int32), ("stations", stations, 3 * k, torch.float64),
               ("fitted", fitted, 8 * n, torch.float64), ("wrms", wrms, n, torch.float64),
               ("n_residuals", n_residuals, n, torch.int32), ("covariance", covariance, _COV_WORDS * n, torch.float64),
               ("iterations", iterations, n, torch.int32), ("status", status, n, torch.uint8),
               ("model", model, n, torch.uint8)]
    for name, t, size, dtype in tensors:
        if t is None and name in ("station", "stations"):
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    call = lib().astroz_cuda_fit_observations_mixed_device if deep_space else lib().astroz_cuda_fit_observations_device
    check(call(ptr(elements), n, int(grav), ptr(offsets), ptr(jd), ptr(fr), ptr(value), ptr(sigma), ptr(station),
               ptr(kind), ptr(stations), int(bool(fit_bstar)), int(max_iter), int(elements.device.index),
               ptr(fitted), ptr(wrms), ptr(n_residuals), ptr(covariance), ptr(iterations), ptr(status), ptr(model),
               C.c_void_p(stream) if stream else None))


def observe(states, jd, fr, kinds, station_idx=None, stations=None, *, device: int = 0) -> np.ndarray:
    """The measurement model alone (astroz_cuda_observe): TEME states (m, 6) [km, km/s] at jd + fr -> (m, 6) values of
    each observation's kind (radar: range, azimuth, elevation, range-rate; optical: right ascension, declination;
    angles in rad, azimuth and right ascension in [0, 2 pi)), zero past the kind's count.  Residuals for outlier
    editing are value - observe(...) row by row."""
    s = np.ascontiguousarray(states, dtype=np.float64).reshape(-1, 6)
    m = len(s)
    jd_ = np.ascontiguousarray(np.broadcast_to(np.asarray(jd, dtype=np.float64), (m,)))
    fr_ = np.ascontiguousarray(np.broadcast_to(np.asarray(fr, dtype=np.float64), (m,)))
    k_ = np.ascontiguousarray(_integers(np.broadcast_to(np.asarray(kinds), (m,)), "kinds", 8))
    sta = None if station_idx is None else np.ascontiguousarray(
        _integers(np.broadcast_to(np.asarray(station_idx), (m,)), "station_idx", 32))
    st = _stations(stations)
    out = np.zeros((m, _OBS_VALUES))
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_observe(vp(s), vp(jd_), vp(fr_), vp(k_), vp(sta), m, vp(st), len(st), int(device),
                                    vp(out)))
    return out
