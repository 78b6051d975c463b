"""python-sgp4 compatible API -- mirror of bindings/python/astroz/api.py over the CUDA C-ABI.

    from astroz_b200.api import Satrec, SatrecArray, jday, WGS72

Same call shapes and return conventions as the reference (and python-sgp4):
  Satrec.twoline2rv(l1, l2, whichconst=WGS72) ; sat.sgp4(jd, fr) -> (e, r, v) ;
  sat.sgp4_array(jd, fr) -> (e[n], r[n,3], v[n,3]) ;
  SatrecArray(sats).sgp4(jd, fr, velocities=True) -> (e[ns,nt] uint8, r[ns,nt,3], v[ns,nt,3]).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import as_f64, check, dptr, lib
from .constellation import Constellation, Layout, OutputMode

WGS72OLD = 0  # python-sgp4 numbering (sgp4.api.WGS72OLD / WGS72 / WGS84), not the header's: _grav maps it
WGS72 = 1
WGS84 = 2
accelerated = True


def _grav(whichconst: int) -> int:
    """python-sgp4 gravity ids -> library ids (bindings/python/src/shared.zig getGravity)."""
    return _lib.WGS84 if whichconst == WGS84 else _lib.WGS72


def jday(year, mon, day, hr, minute, sec):
    """python-sgp4 compatible calendar -> (jd, fr) (src/Datetime.zig:235-240; Vallado jday)."""
    jd = (367.0 * year - math.floor(7 * (year + math.floor((mon + 9) / 12.0)) * 0.25)
          + math.floor(275 * mon / 9.0) + day + 1721013.5)
    fr = (sec + minute * 60.0 + hr * 3600.0) / 86400.0
    return jd, fr


def days2mdhms(year, days):
    """python-sgp4 compatible day-of-year -> (mon, day, hr, minute, sec) (src/Datetime.zig:244-253)."""
    lmonth = [31, 29 if year % 4 == 0 and (year % 100 != 0 or year % 400 == 0) else 28,
              31, 30, 31, 30, 31, 31, 30, 31, 30, 31]
    dayofyr = int(days // 1.0)
    i, inttemp = 1, 0
    while dayofyr > inttemp + lmonth[i - 1] and i < 12:
        inttemp += lmonth[i - 1]
        i += 1
    mon, day = i, dayofyr - inttemp
    temp = (days - dayofyr) * 24.0
    hr = int(temp // 1.0)
    temp = (temp - hr) * 60.0
    minute = int(temp // 1.0)
    sec = (temp - minute) * 60.0
    return mon, day, hr, minute, sec


class Satrec:
    """One satellite (near-earth or deep-space), python-sgp4 `Satrec` look-alike
    (bindings/python/src/satrec.zig:83-343)."""

    def __init__(self):
        self._h = C.c_void_p()
        self._free = None
        self.error = 0
        self.line1 = self.line2 = ""
        self.whichconst = WGS72
        self.jdsatepoch = self.jdsatepochF = 0.0
        self.is_deep_space = False
        self.t = 0.0

    @classmethod
    def twoline2rv(cls, line1: str, line2: str, whichconst: int = WGS72, device: int = 0) -> "Satrec":
        self = cls()
        self.line1, self.line2, self.whichconst = line1, line2, whichconst
        self._free = lib().astroz_cuda_sgp4_free
        rc = lib().astroz_cuda_sgp4_init(line1.encode(), line2.encode(), _grav(whichconst), int(device),
                                         C.byref(self._h))
        if rc == -1:
            raise ValueError("Failed to parse TLE lines")  # satrec.zig:111-115
        if rc in _lib.SGP4_ERROR:  # init failure is recorded, not raised (satrec.zig:128-147)
            self.error = _lib.SGP4_ERROR[rc]
            return self
        check(rc)
        ep = C.c_double()
        check(lib().astroz_cuda_sgp4_epoch(self._h, C.byref(ep)))
        self.jdsatepoch = math.floor(ep.value - 0.5) + 0.5   # satrec.zig:124-126
        self.jdsatepochF = ep.value - self.jdsatepoch
        self.is_deep_space = bool(lib().astroz_cuda_sgp4_is_deep_space(self._h))
        self._read_elements()
        return self

    def _read_elements(self) -> None:
        """python-sgp4 attribute set of the native Satrec (bindings/python/src/satrec.zig:385-494): TLE fields in
        python-sgp4 units (radians, rad/min) and the un-Kozai'd semi-major axis with its apsis altitudes (earth radii)."""
        l1 = self.line1
        sn = l1[2:7].strip()
        if sn[:1].isalpha():  # Alpha-5 catalog numbers, src/Tle.zig:281-290
            self.satnum = (ord(sn[0].upper()) - ord("A") + 10) * 10000 + int(sn[1:] or 0)
        else:
            self.satnum = int(sn) if sn.isdigit() else 0
        self.epochyr = int(l1[18:20])
        self.epochdays = float(l1[20:32])
        self.ndot = float(l1[33:43]) * (2.0 * math.pi) / (1440.0 * 1440.0)  # satrec.zig:420-424
        el = np.zeros(10)
        check(lib().astroz_cuda_sgp4_elements(self._h, dptr(el)))
        (self.ecco, self.inclo, self.nodeo, self.argpo, self.mo, self.no_kozai, self.bstar, self.a, self.no_unkozai,
         _) = el.tolist()
        self.alta = self.a * (1.0 + self.ecco) - 1.0
        self.altp = self.a * (1.0 - self.ecco) - 1.0

    def __del__(self):
        if self._free is not None and self._h:
            self._free(self._h)
            self._h = C.c_void_p()

    def _tsince(self, jd, fr):
        return ((jd + fr) - (self.jdsatepoch + self.jdsatepochF)) * 1440.0  # satrec.zig:176-179

    def sgp4(self, jd: float, fr: float):
        """(error, (x, y, z) km, (vx, vy, vz) km/s) in TEME."""
        if not self._h:
            return (self.error or 6), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0)
        self.t = self._tsince(float(jd), float(fr))
        r = np.zeros(3)
        v = np.zeros(3)
        rc = lib().astroz_cuda_sgp4_propagate(self._h, self.t, dptr(r), dptr(v))
        if rc in _lib.SGP4_ERROR:
            self.error = _lib.SGP4_ERROR[rc]
            return self.error, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0)
        check(rc)
        self.error = 0
        return 0, tuple(r.tolist()), tuple(v.tolist())

    def sgp4_array(self, jd, fr):
        """(e[n], r[n,3], v[n,3]); e is all zeros like the reference (api.py:171-180)."""
        jd, fr = as_f64(jd), as_f64(fr)
        n = jd.shape[0]
        if not (self._h and n):
            return np.zeros(n, dtype=np.uint8), np.zeros((n, 3)), np.zeros((n, 3))
        out = _lib.pinned_empty((n, 6))  # x y z vx vy vz records, filled by one device->host copy
        rc = lib().astroz_cuda_sgp4_array(self._h, dptr(jd), dptr(fr), self.jdsatepoch + self.jdsatepochF, dptr(out), n)
        if rc not in _lib.SGP4_ERROR:
            check(rc)
        return np.zeros(n, dtype=np.uint8), out[:, :3], out[:, 3:]

    def sgp4_array_into(self, jd, fr, positions, velocities) -> None:
        """Native `Satrec.sgp4_array_into(jd, fr, r, v)` (bindings/python/src/satrec.zig:256-343): fills caller-owned
        (n, 3) float64 arrays."""
        _, r, v = self.sgp4_array(jd, fr)
        n = r.shape[0]
        if positions.shape[0] < n or velocities.shape[0] < n:
            raise ValueError("output arrays too small")  # satrec.zig:290-297
        positions[:n] = r
        velocities[:n] = v


class SatrecArray:
    """Batch propagator, python-sgp4 `SatrecArray` look-alike (bindings/python/astroz/api.py:183-359).
    Near-earth and deep-space members are propagated in one device pass."""

    def __init__(self, satrecs, device: int = 0):
        self._sats = list(satrecs)
        if not self._sats:
            raise ValueError("SatrecArray needs at least one Satrec")
        wc = self._sats[0].whichconst
        self._c = Constellation([(s.line1, s.line2) for s in self._sats], _grav(wc), device)
        self._num_sats = len(self._sats)
        self._ref = None

    @property
    def num_satellites(self) -> int:
        return self._num_sats

    @property
    def epochs(self) -> list:
        """Epoch Julian date of each satellite (bindings/python/src/satrec.zig:807)."""
        return self._c.epochs.tolist()

    def propagate_into(self, times, positions, velocities=None, epoch_offsets=None) -> None:
        """Native `SatrecArray.propagate_into(times, positions, velocities=None, epoch_offsets=None)`
        (bindings/python/src/satrec.zig:896-988): near-earth members only, tsince = times[t] + epoch_offsets[sat]
        (zero offsets = minutes since each satellite's own epoch), TEME, written TIME-MAJOR (n_times, n_sats, 3)
        into caller-owned float64 arrays."""
        times = as_f64(times)
        ns, nt = self._c.numSgp4, times.shape[0]
        need = ns * nt * 3
        if positions.size < need:
            raise ValueError("positions array too small")   # satrec.zig:927-930
        if velocities is not None and velocities.size < need:
            raise ValueError("velocities array too small")  # satrec.zig:937-941
        if ns == 0 or nt == 0:
            return
        r, v = self._c.propagate_into(times, None, None, epoch_offsets=epoch_offsets, time_major=True,
                                      want_velocities=velocities is not None)
        positions.reshape(-1)[:need] = r.reshape(-1)
        if velocities is not None:
            velocities.reshape(-1)[:need] = v.reshape(-1)

    def sgp4(self, jd, fr, *, velocities: bool = True):
        jd, fr = as_f64(jd), as_f64(fr)
        nt = jd.shape[0]
        e = np.zeros((self._num_sats, nt), dtype=np.uint8)  # always zeros, api.py:294
        ref = float(jd[0] + fr[0])  # api.py:300: reference_jd = jd[0] + fr[0]
        if ref != self._ref:
            self._c.referenceEpochJd = ref
            self._ref = ref
        r, v = self._c.propagate(jd, fr, outputMode=OutputMode.teme, layout=Layout.satelliteMajor,
                                 velocities=velocities)
        if v is None:
            v = np.zeros((self._num_sats, nt, 3))
        return e, r, v


def sdp4_batch_propagate_into(satrecs, jd, fr, positions, velocities, output_stride: int = -1, sat_offset: int = 0):
    """Native `sdp4_batch_propagate_into(satrecs, jd, fr, positions, velocities, output_stride=-1, sat_offset=0)`
    (bindings/python/src/satrec.zig:505-644): deep-space Satrecs only, TEME, TIME-MAJOR, satellite s written at
    pos[t, sat_offset + s] of a block with `output_stride` satellites per epoch."""
    sats = list(satrecs)
    if not sats:
        return None
    for s in sats:
        if not isinstance(s, Satrec):
            raise TypeError("All items must be Satrec objects")
        if not s.is_deep_space:
            raise ValueError("Satrec at index is not a deep-space (SDP4) object")
    c = Constellation([(s.line1, s.line2) for s in sats], _grav(sats[0].whichconst))
    c.propagate_sdp4_into(jd, fr, positions, velocities, outputMode=OutputMode.teme, time_major=True,
                          output_stride=output_stride, sat_offset=sat_offset)
    return None


__all__ = ["sdp4_batch_propagate_into", "Satrec", "SatrecArray", "jday", "days2mdhms", "WGS72", "WGS84", "WGS72OLD", "accelerated"]
