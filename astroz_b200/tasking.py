"""Sensor tasking on the device: which catalogue row each sensor should observe at each slot, chosen greedily by the
information one observation gives about the row's elements, with each tasked row's covariance carried forward
(K18, astroz_b200/csrc/az_tasking.cu).

    from astroz_b200.tasking import Sensor, plan
    sensors = [Sensor("radar", 42.6, -71.5, 0.12, sigma=(0.01, 1.7e-4, 1.7e-4, 1e-5), el_min=10.0),
               Sensor("optical", 32.4, -110.7, 2.5, sigma=(4.8e-6, 4.8e-6), el_min=20.0, sun_el_max=-12.0)]
    p = plan(fit, sensors, jd, fr)        # fit: a FitResult with covariance; jd + fr the slot times
    p.task_row, p.task_gain, p.posterior
    sat, jd, fr, kind, station, value, sigma = p.tasks()   # K8's observation layout, stations = p.stations

At every slot each sensor takes the row of largest gain g = 1/2 log det(I + G P G^T) (nats) among the rows it can see,
g > gain_min, not taken by a lower-numbered sensor in the slot; the taken row's covariance becomes the Kalman posterior
of that one observation before the next slot.  The plan is greedy per slot: there is no look-ahead.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._abi import DEFINES as D
from ._lib import WGS72, check, lib
from .correlate import _catalogue

RADAR, OPTICAL = D["ASTROZ_OBS_RADAR"], D["ASTROZ_OBS_OPTICAL"]
MAX_SENSORS = D["ASTROZ_TASK_MAX_SENSORS"]
IDLE = 0xFFFFFFFF
_KINDS = {"radar": RADAR, "optical": OPTICAL, RADAR: RADAR, OPTICAL: OPTICAL}


@dataclass
class Sensor:
    """One sensor: kind "radar" or "optical", its station (geodetic latitude and longitude in degrees, height in km
    on WGS84), sigma in the observation layout's units (radar range km, azimuth rad, elevation rad, range-rate km/s;
    optical RA rad, Dec rad; inf: not measured), and its limits in degrees: the minimum elevation, the maximum Sun
    elevation at the station and the minimum angle between the line of sight and the Sun (the last two read for
    optical sensors only), with the maximum range in km."""
    kind: str | int
    lat: float
    lon: float
    h: float
    sigma: tuple = (0.01, 1.7e-4, 1.7e-4, 1e-5)
    el_min: float = 10.0
    range_max: float = float("inf")
    sun_el_max: float = -12.0
    exclusion: float = 40.0


@dataclass
class TaskingPlan:
    task_row: np.ndarray      # (S, T) int64 row observed by sensor k at slot t, -1 when the sensor idles
    task_gain: np.ndarray     # (S, T) the gain in nats (0 idle)
    task_value: np.ndarray    # (S, T, 4) the predicted measurement: the pointing
    task_spread: np.ndarray   # (S, T, 4) its predicted 1-sigma per component: the search window
    n_candidates: np.ndarray  # (S, T) rows that qualified when the sensor chose
    posterior: np.ndarray     # (n, 28) each row's covariance after its planned observations
    n_tasks: np.ndarray       # (n,) planned observations per row
    n_visible: np.ndarray     # (n,) visible (sensor, slot) cells
    n_failed: np.ndarray      # (n,) failed cells
    row_status: np.ndarray    # (n,) uint8 ASTROZ_COV_OK / ASTROZ_COV_INIT_FAILED
    kind: np.ndarray          # (S,) uint8 ASTROZ_OBS_RADAR / ASTROZ_OBS_OPTICAL
    sigma: np.ndarray         # (S, 4)
    stations: np.ndarray      # (S, 3) sensor k's station is row k
    jd: np.ndarray            # (T,)
    fr: np.ndarray            # (T,)

    def tasks(self):
        """The schedule as observations in K8's layout, slot-major: (sat, jd, fr, kind, station, value (m, 6),
        sigma (m, 6)), the predicted value in place of a measurement; `stations` of the plan are their stations."""
        t, k = np.nonzero(self.task_row.T >= 0)
        value, sigma = np.zeros((len(k), 6)), np.full((len(k), 6), np.inf)
        value[:, :4] = self.task_value[k, t]
        sigma[:, :4] = self.sigma[k]
        optical = self.kind[k] == OPTICAL
        value[optical, 2:4] = 0.0
        sigma[optical, 2:4] = np.inf
        return (self.task_row[k, t], self.jd[t], self.fr[t], self.kind[k].copy(), k.astype(np.uint32), value, sigma)


def sun_direction(jd, fr=0.0) -> np.ndarray:
    """(T, 3) the geocentric Sun in AU, mean equator and equinox of date (used as TEME), by the Astronomical Almanac's
    low-precision formulae (about 0.01 deg from 1950 to 2050)"""
    n = (np.asarray(jd, dtype=np.float64) - 2451545.0) + np.asarray(fr, dtype=np.float64)
    n = np.atleast_1d(n)
    L = np.deg2rad(280.460 + 0.9856474 * n)
    g = np.deg2rad(357.528 + 0.9856003 * n)
    lam = L + np.deg2rad(1.915) * np.sin(g) + np.deg2rad(0.020) * np.sin(2 * g)
    eps = np.deg2rad(23.439 - 4e-7 * n)
    R = 1.00014 - 0.01671 * np.cos(g) - 0.00014 * np.cos(2 * g)
    return np.stack([R * np.cos(lam), R * np.cos(eps) * np.sin(lam), R * np.sin(eps) * np.sin(lam)], axis=1)


def _sensors(sensors):
    S = len(sensors)
    kind = np.zeros(S, np.uint8)
    sigma, limits, stations = np.full((S, 4), np.inf), np.zeros((S, 4)), np.zeros((S, 3))
    for k, s in enumerate(sensors):
        if s.kind not in _KINDS:
            raise ValueError("a sensor kind must be 'radar' or 'optical'")
        kind[k] = _KINDS[s.kind]
        sg = np.asarray(s.sigma, dtype=np.float64).reshape(-1)
        if len(sg) > 4:
            raise ValueError("a sensor has at most 4 sigmas")
        sigma[k, :len(sg)] = sg
        limits[k] = (np.deg2rad(s.el_min), s.range_max, np.deg2rad(s.sun_el_max), np.deg2rad(s.exclusion))
        stations[k] = (s.lat, s.lon, s.h)
    return kind, np.arange(S, dtype=np.uint32), sigma, limits, stations


def plan(source, sensors, jd, fr, *, sun=None, gain_min: float = 0.0, covariance=None, model=None,
         grav: int = WGS72, device: int = 0) -> TaskingPlan:
    """Plan sensor tasks over the slots jd + fr (astroz_cuda_tasking).

    source: a FitResult (elements, covariance and deep_space taken from it; covariance= or model= override them) or
    an (8, n) array of element columns with covariance= (n, 28) words or (n, 7, 7) matrices and model= (n,) 0 / 1.
    sensors: a list of Sensor.  sun: (T, 3) the Sun's direction in TEME per slot, any length; None: sun_direction."""
    el, cov, md = _catalogue(source, covariance, model)
    n = el.shape[1]
    kind, station, sigma, limits, stations = _sensors(sensors)
    S = len(kind)
    jd = np.ascontiguousarray(np.atleast_1d(np.asarray(jd, dtype=np.float64)).reshape(-1))
    fr = np.ascontiguousarray(np.broadcast_to(np.asarray(fr, dtype=np.float64), jd.shape))
    T = len(jd)
    sun = sun_direction(jd, fr) if sun is None else np.asarray(sun, dtype=np.float64)
    sun = np.ascontiguousarray(sun.reshape(-1, 3))
    if len(sun) != T:
        raise ValueError("sun must hold one row per slot")
    task_row, n_cand = np.zeros((S, T), np.uint32), np.zeros((S, T), np.uint32)
    task_gain, task_value, task_spread = np.zeros((S, T)), np.zeros((S, T, 4)), np.zeros((S, T, 4))
    post = np.zeros((n, 28))
    n_tasks, n_vis, n_fail = (np.zeros(n, np.uint32) for _ in range(3))
    row_status = np.zeros(n, np.uint8)
    vp = lambda a: None if a is None or a.size == 0 else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_tasking(vp(el), n, int(grav), vp(cov), vp(md), vp(kind), vp(station), vp(sigma),
                                    vp(limits), S, vp(stations), len(stations), vp(jd), vp(fr), T, vp(sun),
                                    float(gain_min), int(device), vp(task_row), vp(task_gain), vp(task_value),
                                    vp(task_spread), vp(n_cand), vp(post), vp(n_tasks), vp(n_vis), vp(n_fail),
                                    vp(row_status)))
    return TaskingPlan(np.where(task_row == IDLE, -1, task_row.astype(np.int64)), task_gain, task_value, task_spread,
                       n_cand, post, n_tasks, n_vis, n_fail, row_status, kind, sigma, stations, jd, fr)


def plan_scratch_bytes(n: int, s: int) -> int:
    """Bytes of the scratch `plan_device` needs for n rows and s sensors"""
    out = C.c_uint64()
    check(lib().astroz_cuda_tasking_scratch_bytes(int(n), int(s), C.byref(out)))
    return out.value


def plan_device(elements, covariance, model, kind, station, sigma, limits, stations, jd, fr, sun, scratch, task_row,
                task_gain, task_value, task_spread, n_candidates, posterior, n_tasks, n_visible, n_failed,
                row_status, *, gain_min: float = 0.0, grav: int = WGS72, stream: int = 0) -> None:
    """`plan` with torch CUDA tensors on one device: elements (8, n) float64, covariance (n, 28) float64 or None,
    model (n,) uint8 or None, kind (S,) uint8, station (S,) int32, sigma / limits (S, 4) float64 (limits in rad and
    km, ASTROZ_TASK_LIMIT_* order), stations (k, 3) float64, jd / fr (T,) float64, sun (T, 3) float64 or None (no
    optical sensor), scratch a uint8 tensor of at least plan_scratch_bytes(n, S) bytes; task_row / n_candidates
    (S, T) int32 (task_row -1 idle), task_gain (S, T), task_value / task_spread (S, T, 4), posterior (n, 28) float64,
    n_tasks / n_visible / n_failed (n,) int32 and row_status (n,) uint8 receive the results.  Launches on `stream` (a
    raw cudaStream_t value, 0 = the default stream); nothing is checked beyond shapes."""
    import torch

    n = int(elements.shape[1]) if elements.dim() == 2 and elements.shape[0] == 8 else -1
    if n < 0 or elements.dtype != torch.float64 or not elements.is_cuda:
        raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
    S, T = int(kind.numel()), int(jd.numel())
    k = int(stations.numel()) // 3
    tensors = [("elements", elements, 8 * n, torch.float64), ("covariance", covariance, 28 * n, torch.float64),
               ("model", model, n, torch.uint8), ("kind", kind, S, torch.uint8), ("station", station, S, torch.int32),
               ("sigma", sigma, 4 * S, torch.float64), ("limits", limits, 4 * S, torch.float64),
               ("stations", stations, 3 * k, torch.float64), ("jd", jd, T, torch.float64),
               ("fr", fr, T, torch.float64), ("sun", sun, 3 * T, torch.float64),
               ("task_row", task_row, S * T, torch.int32), ("task_gain", task_gain, S * T, torch.float64),
               ("task_value", task_value, 4 * S * T, torch.float64),
               ("task_spread", task_spread, 4 * S * T, torch.float64),
               ("n_candidates", n_candidates, S * T, torch.int32), ("posterior", posterior, 28 * n, torch.float64),
               ("n_tasks", n_tasks, n, torch.int32), ("n_visible", n_visible, n, torch.int32),
               ("n_failed", n_failed, n, torch.int32), ("row_status", row_status, n, torch.uint8)]
    for name, x, size, dtype in tensors:
        if x is None and name in ("covariance", "model", "sun"):
            continue
        if not isinstance(x, torch.Tensor) or x.dtype != dtype or not x.is_contiguous() or int(x.numel()) != size \
                or x.device != elements.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {elements.device}")
    need = plan_scratch_bytes(n, max(S, 1))
    if not isinstance(scratch, torch.Tensor) or scratch.dtype != torch.uint8 or scratch.device != elements.device \
            or int(scratch.numel()) < need:
        raise ValueError(f"scratch must be a uint8 tensor of at least {need} bytes on {elements.device}")
    ptr = lambda x: None if x is None else C.c_void_p(x.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_tasking_device(
        ptr(elements), n, int(grav), ptr(covariance), ptr(model), ptr(kind), ptr(station), ptr(sigma), ptr(limits), S,
        ptr(stations), ptr(jd), ptr(fr), T, ptr(sun), float(gain_min), int(elements.device.index), ptr(scratch),
        ptr(task_row), ptr(task_gain), ptr(task_value), ptr(task_spread), ptr(n_candidates), ptr(posterior),
        ptr(n_tasks), ptr(n_visible), ptr(n_failed), ptr(row_status), C.c_void_p(stream) if stream else None))
