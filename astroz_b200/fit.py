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


@dataclass
class FitResult:
    elements: np.ndarray     # (8, n) fitted columns, epoch unchanged
    rms_pos: np.ndarray      # (n,) km: sqrt(mean |r_obs - r_fit|^2)
    rms_vel: np.ndarray      # (n,) km/s (0 without velocities)
    iterations: np.ndarray   # (n,) uint32 LM steps tried
    status: np.ndarray       # (n,) uint8 ASTROZ_FIT_*

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
