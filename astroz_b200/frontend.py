"""High-level entry points of the reference's Python package over the CUDA path:

    from astroz_b200.frontend import Constellation, propagate, screen     # was: from astroz import ...

Mirrors `astroz.Constellation`, `astroz.propagate` and `astroz.screen`
(bindings/python/astroz/__init__.py:305-660): same arguments, same output shapes (time-major
`(n_times, n_satellites, 3)`), same row order (near-earth satellites first, deep-space after, :373-375), the
same time convention (`times` in minutes from `start_time`, near-earth tsince = times[t] + (start - epoch) * 1440,
:513-526) and the same loaders for TLE text and OMM JSON.  Differences, all deliberate:

* sources that need the network (CelesTrak group names, URLs, `norad_id=`) raise: this build has no egress and the
  catalogue download is outside the propagation path;
* the deep-space rows of `propagate()` are filled (the reference leaves them uninitialised, SURVEY.md appendix C);
* `lambert()` returns the true solution of Lambert's problem; the reference's velocities miss r2 (SURVEY.md appendix C);
* geodetic output is what the core produces -- latitude / longitude in radians, altitude in km
  (src/Constellation.zig:497) -- like the reference's actual return value, not its docstring.
"""
from __future__ import annotations

import json
import math
from datetime import datetime, timezone
from pathlib import Path

import numpy as np

from ._lib import WGS72
from .constellation import Constellation as DeviceConstellation
from .constellation import OutputMode

_OUTPUT = {"teme": OutputMode.teme, "ecef": OutputMode.ecef, "geodetic": OutputMode.geodetic}


def _start_jd(start_time) -> float:
    """`start_time` (datetime, default: now, UTC) as a Julian date (__init__.py:282-286)."""
    if start_time is None:
        start_time = datetime.now(timezone.utc)
    return 2440587.5 + start_time.timestamp() / 86400.0


def parse_tle_pairs(text: str) -> list[tuple[str, str]]:
    """(line1, line2) pairs of a 2- or 3-line element-set listing; name lines and orphans are skipped
    (__init__.py:184-200)."""
    rows = [ln.strip() for ln in text.strip().splitlines() if ln.strip()]
    pairs, i = [], 0
    while i < len(rows):
        if rows[i].startswith("1 ") and i + 1 < len(rows) and rows[i + 1].startswith("2 "):
            pairs.append((rows[i], rows[i + 1]))
            i += 2
        else:
            i += 1
    return pairs


def _checksum(body: str) -> str:
    return str(sum(int(ch) if ch.isdigit() else (1 if ch == "-" else 0) for ch in body) % 10)


def _implied_decimal(x: float) -> str:
    """8-column TLE field with an implied leading decimal point and a signed power-of-ten digit."""
    if x == 0:
        return " 00000+0"
    mag = abs(x)
    exp = math.floor(math.log10(mag)) + 1
    digits = int(round(mag * 10.0 ** (5 - exp)))
    if digits == 100000:   # 0.999995.. rounds up to the next power of ten
        digits, exp = 10000, exp + 1
    return f"{'-' if x < 0 else ' '}{digits:05d}{exp:+d}"


def tle_line_pair(norad: int, year: int, doy: float, incl: float, raan: float, ecc: float, argp: float, ma: float,
                  mean_motion: float, bstar: float, *, classification: str = "U", designator: str = "00000A  ",
                  ndot: float = 0.0, nddot: float = 0.0, ephemeris_type: int = 0, element_set_no: int = 0,
                  rev_at_epoch: int = 0) -> tuple[str, str]:
    """One element set as a checksummed TLE line pair, with TLE column precision (angles in degrees, day of year from
    1.0 at Jan 1 00:00, B* in 1 / earth radii)."""
    ndot_txt = ("-" if ndot < 0 else " ") + f"{abs(ndot):.8f}"[1:]
    head = (f"1 {norad:05d}{classification} {designator} {year % 100:02d}{doy:012.8f} {ndot_txt} "
            f"{_implied_decimal(nddot)} {_implied_decimal(bstar)} {ephemeris_type} {element_set_no:4d}")
    head = head[:68].ljust(68)
    ecc_txt = f"{ecc:.7f}"[2:]
    tail = (f"2 {norad:05d} {incl:8.4f} {raan:8.4f} {ecc_txt} {argp:8.4f} {ma:8.4f} {mean_motion:11.8f}"
            f"{rev_at_epoch:5d}")
    tail = tail[:68].ljust(68)
    return head + _checksum(head), tail + _checksum(tail)


def omm_to_tle_pairs(json_text: str) -> list[tuple[str, str]]:
    """OMM JSON (one record or an array) rendered as TLE line pairs, with TLE column precision -- the reference
    converts OMM input the same way before initialising (__init__.py:203-279), so an OMM catalogue propagates to
    the same values here as there."""
    data = json.loads(json_text)
    records = [data] if isinstance(data, dict) else data
    pairs = []
    for rec in records:
        norad = int(rec["NORAD_CAT_ID"])
        cls = (rec.get("CLASSIFICATION_TYPE") or "U")[0]
        obj = rec.get("OBJECT_ID") or "00000A"
        if "-" in obj:  # "1998-067A" -> "98067A"
            launch_year, piece = obj.split("-", 1)
            designator = f"{launch_year[-2:]}{piece:<6s}"
        else:
            designator = f"{obj:<8s}"
        when = datetime.fromisoformat(rec["EPOCH"]).replace(tzinfo=None)
        doy = (when - datetime(when.year, 1, 1)).total_seconds() / 86400.0 + 1.0
        pairs.append(tle_line_pair(
            norad, when.year, doy, rec["INCLINATION"], rec["RA_OF_ASC_NODE"], rec["ECCENTRICITY"],
            rec["ARG_OF_PERICENTER"], rec["MEAN_ANOMALY"], rec["MEAN_MOTION"], rec["BSTAR"], classification=cls,
            designator=designator, ndot=rec.get("MEAN_MOTION_DOT") or 0, nddot=rec.get("MEAN_MOTION_DDOT") or 0,
            ephemeris_type=rec.get("EPHEMERIS_TYPE") or 0, element_set_no=rec.get("ELEMENT_SET_NO") or 0,
            rev_at_epoch=rec.get("REV_AT_EPOCH") or 0))
    return pairs


def _load(source, norad_id):
    """(text, "tle" | "json") for the offline sources of __init__.py:163-181."""
    if norad_id is not None:
        raise RuntimeError("norad_id= needs a CelesTrak download; this build has no network access")
    if source is None:
        raise ValueError("Must specify 'source' or 'norad_id'")
    if source.startswith(("http://", "https://")):
        raise RuntimeError("URL sources need network access, which this build does not have")
    if "1 " in source and "2 " in source:
        return source, "tle"
    if source.lstrip().startswith(("[", "{")):
        return source, "json"
    if Path(source).exists():
        text = Path(source).read_text()
        return text, ("json" if text.lstrip().startswith(("[", "{")) else "tle")
    raise RuntimeError(f"'{source}' is not TLE text, OMM JSON or a file; CelesTrak group names need network access")


class Constellation:
    """Pre-parsed element sets for repeated propagation / screening (`astroz.Constellation`, __init__.py:305-408).
    Near-earth members occupy rows [0, n_sgp4), deep-space members the rows after them."""

    def __init__(self, source=None, *, norad_id=None, device: int = 0):
        text, fmt = _load(source, norad_id)
        pairs = omm_to_tle_pairs(text) if fmt == "json" else parse_tle_pairs(text)
        self._total_sats = len(pairs)
        if not pairs:
            raise ValueError("no element sets found in source")
        probe = DeviceConstellation(pairs, WGS72, device)
        deep = probe.classes != 0
        probe.deinit()
        ordered = [p for p, d in zip(pairs, deep) if not d] + [p for p, d in zip(pairs, deep) if d]
        self._dev = DeviceConstellation(ordered, WGS72, device)
        self._n_sgp4 = self._dev.numSgp4
        self._n_sdp4 = self._dev.numSdp4

    @property
    def num_satellites(self) -> int:
        return self._total_sats

    @property
    def epochs(self) -> list:
        return self._dev.epochs.tolist()


def _as_constellation(source, norad_id) -> Constellation:
    return source if isinstance(source, Constellation) else Constellation(source, norad_id=norad_id)


def propagate(source, times, *, start_time=None, output="ecef", velocities=False, norad_id=None):
    """`astroz.propagate(source, times, start_time=None, output="ecef", velocities=False)` (__init__.py:411-532):
    positions `(n_times, n_satellites, 3)` (and velocities, km/s) at `times` minutes from `start_time`."""
    const = _as_constellation(source, norad_id)
    times = np.ascontiguousarray(times, dtype=np.float64)
    if output not in _OUTPUT:
        raise ValueError("output must be 'ecef', 'teme' or 'geodetic'")  # sgp4.zig:198-206
    mode = _OUTPUT[output]
    n_sats, nt = const.num_satellites, len(times)
    start = _start_jd(start_time)
    pos = np.empty((nt, n_sats, 3))
    vel = np.empty((nt, n_sats, 3)) if velocities else None
    dev = const._dev
    if const._n_sgp4 and nt:
        offsets = (start - dev.epochs[:const._n_sgp4]) * 1440.0  # __init__.py:513-514
        dev.propagate_into(times, pos, vel, epoch_offsets=offsets, outputMode=mode, reference_jd=start,
                           time_major=True, output_stride=n_sats, want_velocities=velocities)
    if const._n_sdp4 and nt:
        jd = np.full(nt, start)
        dev.propagate_sdp4_into(jd, times / 1440.0, pos, vel, outputMode=mode, time_major=True, output_stride=n_sats,
                                sat_offset=const._n_sgp4)
    return (pos, vel) if velocities else pos


def screen(source, times, threshold=10.0, *, target=None, start_time=None, norad_id=None):
    """`astroz.screen(source, times, threshold=10.0, target=None, start_time=None)` (__init__.py:535-660).
    With `target`: (min_distances[n], min_t_indices[n]) from the fused propagate + screen kernel.  Without: all-vs-all
    (pairs[n, 2], t_indices[n]) from the cell-list kernel; the position block never leaves the GPU."""
    const = _as_constellation(source, norad_id)
    times = np.ascontiguousarray(times, dtype=np.float64)
    dev = const._dev
    start = _start_jd(start_time)
    if const._n_sdp4 == 0:
        offsets = (start - dev.epochs) * 1440.0
        if target is not None:
            dist, tidx = dev.screen_conjunction(times, int(target), float(threshold), epoch_offsets=offsets,
                                                reference_jd=start)
            return np.asarray(dist), np.asarray(tidx, dtype=np.uint32)
        return dev.screen_all(times, float(threshold), epoch_offsets=offsets)
    # mixed catalogue: propagate everything (TEME), then the cell-list screen on the device copy of the block
    import torch
    pos = propagate(const, times, start_time=start_time, output="teme")
    block = torch.from_numpy(pos).cuda(dev.device)
    return dev.coarse_screen_device(block, float(threshold))


# WGS-84 (src/constants.zig:55-58), the values the reference exports as EARTH_MU / EARTH_R_EQ / EARTH_J2
EARTH_MU = 398600.5
EARTH_R_EQ = 6378.137
EARTH_J2 = 0.00108262998905
# gravitational parameters of the Sun and the Moon [km^3/s^2] (src/constants.zig:97, :170), the values the reference
# exports as SUN_MU / MOON_MU (bindings/python/src/main.zig:73-74): the mu of a ThirdBody model (astroz_b200.numerical)
SUN_MU = 1.32712e11
MOON_MU = 4902.80


def propagate_numerical(state, t0, duration, dt, mu, j2=None, r_eq=None, drag_cd=None, drag_area=None, drag_mass=None,
                        integrator=None, rtol=None, atol=None):
    """`astroz.propagate_numerical(state, t0, duration, dt, mu, ...)` (bindings/python/src/propagator.zig:13-193): the
    trajectory of one state as (list of times, list of (x, y, z, vx, vy, vz) tuples), integrated on the device as a batch
    of one.  Every argument after mu is positional-or-keyword and None selects its default, as the reference's parser
    does (:28-52, :76-79).  Raises the reference's ValueErrors; where the reference would never return it raises instead:
    ValueError for dt <= 0 with a loop to run, RuntimeError when a Dormand-Prince step is rejected at its minimum size
    (the reference retries that step forever)."""
    from . import numerical

    if len(state) != 6:
        raise ValueError("state must have exactly 6 elements [x, y, z, vx, vy, vz]")
    initial = [float(x) for x in state]
    t0, duration, dt, mu = float(t0), float(duration), float(dt), float(mu)
    if (j2 is not None or drag_cd is not None) and r_eq is None:
        raise ValueError("r_eq is required when j2 or drag_cd is specified")
    if drag_cd is not None and (drag_area is None or drag_mass is None):
        raise ValueError("drag_area and drag_mass are required when drag_cd is specified")
    if integrator is None:
        integrator = "dp87"
    if integrator not in ("rk4", "dp87"):
        raise ValueError("integrator must be 'rk4' or 'dp87'")
    if not t0 < t0 + duration:
        return [t0], [tuple(initial)]   # the loop does not run, whatever dt is (Propagator.zig:36-40)
    if not dt > 0.0:
        raise ValueError("dt must be positive (the reference's sampling loop would not end)")
    times, traj, status, _ = numerical.propagate_numerical_batch(
        np.array([initial]), t0, duration, dt, mu, j2=j2, r_eq=r_eq, drag_cd=drag_cd, drag_area=drag_area,
        drag_mass=drag_mass, integrator=integrator, rtol=1e-9 if rtol is None else float(rtol),
        atol=1e-12 if atol is None else float(atol))
    if status[0] == numerical.STOPPED:
        raise RuntimeError("propagation stopped: a Dormand-Prince step was rejected at the minimum step size "
                           "(the reference retries it forever)")
    return [float(t) for t in times], [tuple(float(x) for x in row) for row in traj[0]]


_LAMBERT_ERROR = "Lambert solver failed (check inputs: tof>0, non-zero position vectors)"


def lambert(mu, r1, r2, tof):
    """`astroz.lambert(mu, r1, r2, tof)` (bindings/python/src/orbital_mechanics.zig:37-97): a dict with
    `departure_velocity` and `arrival_velocity` (3-tuples, km/s), `transfer_angle` (rad), `sma` (km) and `tof` (s).
    The reference's geometry: the short way, transfer angle acos(r1 . r2 / |r1| |r2|) in (0, pi), no revolutions, solved
    on the device with the normal r1 x r2.  The velocities are the true solution of Lambert's problem, not the
    reference's (whose departure velocity misses r2, SURVEY.md appendix C); `sma` is that transfer conic's semi-major
    axis, negative for a hyperbola.  ValueError with the reference's message for tof <= 0, a zero vector or
    |sin(transfer angle)| < 1e-12 (src/OrbitalMechanics.zig:122-158)."""
    from . import lambert as K9

    mu, tof = float(mu), float(tof)
    r1, r2 = [float(x) for x in r1], [float(x) for x in r2]
    if len(r1) != 3 or len(r2) != 3:
        raise ValueError("position vectors must have exactly 3 elements")
    n1, n2 = math.sqrt(sum(x * x for x in r1)), math.sqrt(sum(x * x for x in r2))
    if tof <= 0 or n1 <= 0 or n2 <= 0:
        raise ValueError(_LAMBERT_ERROR)
    cos_angle = max(-1.0, min(1.0, sum(a * b for a, b in zip(r1, r2)) / (n1 * n2)))
    angle = math.acos(cos_angle)
    if abs(math.sin(angle)) < 1e-12:
        raise ValueError(_LAMBERT_ERROR)
    normal = np.cross(r1, r2)
    v1, v2, status, _ = K9.lambert_batch([r1], [r2], [tof], mu, normal=normal)
    if status[0, 0] != K9.OK:
        raise ValueError(_LAMBERT_ERROR)
    dep = v1[0, 0]
    sma = 1.0 / (2.0 / n1 - float(dep @ dep) / mu)   # vis-viva
    return {"departure_velocity": tuple(float(x) for x in dep), "arrival_velocity": tuple(float(x) for x in v2[0, 0]),
            "transfer_angle": angle, "sma": sma, "tof": tof}


__all__ = ["Constellation", "propagate", "screen", "parse_tle_pairs", "omm_to_tle_pairs", "propagate_numerical", "lambert",
           "EARTH_MU", "EARTH_R_EQ", "EARTH_J2", "SUN_MU", "MOON_MU"]
