"""Constellation -- host-side mirror of `astroz.Constellation` (src/Constellation.zig:76-308) over the
CUDA C-ABI.  Same names, argument meaning and error behaviour as the reference: `init` classifies each
TLE as SGP4 or SDP4, `propagate(jd, fr, ...)` fills (n_sats, n_times, 3) or (n_times, n_sats, 3) blocks
in TEME / ECEF / geodetic, failed cells are zero-filled, `reset_carry` exists for drop-in use.
"""
from __future__ import annotations

import ctypes as C
from enum import IntEnum

import numpy as np

from . import _lib
from ._abi import DEFINES as D
from ._lib import AstrozCudaError, as_f64, check, dptr, lib


class OutputMode(IntEnum):  # src/Constellation.zig:30-34
    teme = D["ASTROZ_MODE_TEME"]
    ecef = D["ASTROZ_MODE_ECEF"]
    geodetic = D["ASTROZ_MODE_GEODETIC"]


class Layout(IntEnum):  # src/Constellation.zig:37-42
    satelliteMajor = D["ASTROZ_LAYOUT_SATELLITE_MAJOR"]
    timeMajor = D["ASTROZ_LAYOUT_TIME_MAJOR"]


def _c_lines(tles):
    n = len(tles)
    a1 = (C.c_char_p * n)(*[(t[0] if isinstance(t[0], bytes) else t[0].encode()) for t in tles])
    a2 = (C.c_char_p * n)(*[(t[1] if isinstance(t[1], bytes) else t[1].encode()) for t in tles])
    return a1, a2


class Constellation:
    """Mixed SGP4/SDP4 constellation resident on one GPU.

    Parameters
    ----------
    tles : sequence of (line1, line2)
    grav : WGS72 (1, python default of the reference) or WGS84 (0)
    device : CUDA device index, or -1 for a multi-device handle over every visible GPU (ASTROZ_DEVICES caps the
             count, like the reference's ASTROZ_THREADS, src/Constellation.zig:61-74): one `propagate` call then
             runs all GPUs, each copying its satellite range over its own PCIe link into the caller's block.
    """

    def __init__(self, tles, grav: int = _lib.WGS72, device: int = 0):
        self._h = C.c_void_p()
        self._free = lib().astroz_cuda_constellation_free
        a1, a2 = _c_lines(tles)
        check(lib().astroz_cuda_constellation_create(a1, a2, len(tles), int(grav), int(device), C.byref(self._h)))
        n, ns, nd = C.c_uint32(), C.c_uint32(), C.c_uint32()
        check(lib().astroz_cuda_constellation_counts(self._h, C.byref(n), C.byref(ns), C.byref(nd)))
        self.numSatellites, self.numSgp4, self.numSdp4 = n.value, ns.value, nd.value
        self.device = int(device)
        self.grav = int(grav)

    @classmethod
    def init(cls, tles, grav: int = _lib.WGS72, device: int = 0) -> "Constellation":
        """Constellation.init(allocator, tles, grav)  (src/Constellation.zig:101)."""
        return cls(tles, grav, device)

    @classmethod
    def from_text(cls, text: str, grav: int = _lib.WGS72, device: int = 0) -> "Constellation":
        """Build from a 2/3-line element-set blob (src/Tle.zig:103-132)."""
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self._free = lib().astroz_cuda_constellation_free
        raw = text.encode()
        check(lib().astroz_cuda_constellation_create_from_text(raw, len(raw), int(grav), int(device), C.byref(self._h)))
        n, ns, nd = C.c_uint32(), C.c_uint32(), C.c_uint32()
        check(lib().astroz_cuda_constellation_counts(self._h, C.byref(n), C.byref(ns), C.byref(nd)))
        self.numSatellites, self.numSgp4, self.numSdp4 = n.value, ns.value, nd.value
        self.device, self.grav = int(device), int(grav)
        return self

    @classmethod
    def from_elements(cls, epoch_jd, mean_motion_rev_day, ecc, incl_deg, raan_deg, argp_deg, ma_deg, bstar,
                      grav: int = _lib.WGS72, device: int = 0) -> "Constellation":
        """Build from numeric mean elements (what Tle.parseOmm extracts from an OMM record, src/Tle.zig:134-215):
        no TLE text round trip, so e.g. Monte-Carlo draws keep their full fp64 values."""
        cols = [as_f64(a) for a in (epoch_jd, mean_motion_rev_day, ecc, incl_deg, raan_deg, argp_deg, ma_deg, bstar)]
        n = cols[0].shape[0]
        if any(c.shape[0] != n for c in cols):
            raise ValueError("element arrays must have the same length")
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self._free = lib().astroz_cuda_constellation_free
        check(lib().astroz_cuda_constellation_create_from_elements(*[dptr(c) for c in cols], n, int(grav), int(device),
                                                                    C.byref(self._h)))
        cn, ns, nd = C.c_uint32(), C.c_uint32(), C.c_uint32()
        check(lib().astroz_cuda_constellation_counts(self._h, C.byref(cn), C.byref(ns), C.byref(nd)))
        self.numSatellites, self.numSgp4, self.numSdp4 = cn.value, ns.value, nd.value
        self.device, self.grav = int(device), int(grav)
        return self

    @classmethod
    def from_device_elements(cls, elements, grav: int = _lib.WGS72) -> "Constellation":
        """Build from element columns that already live in HBM: `elements` is a CUDA float64 tensor of shape (8, n)
        whose rows are epoch_jd, mean_motion_rev_day, ecc, incl_deg, raan_deg, argp_deg, ma_deg, bstar (the order of
        `from_elements`).  Classification, Sgp4/Sdp4.initElements (src/Sgp4.zig:108-417, src/Sdp4.zig:174-657) and
        the table build (src/Constellation.zig:101-200) run on the device (K5); the element values never visit the
        host.  Results match `from_elements` to the last few ulps of the device's libm."""
        import torch
        if not (isinstance(elements, torch.Tensor) and elements.is_cuda and elements.dtype == torch.float64 and
                elements.dim() == 2 and elements.shape[0] == 8):
            raise ValueError("elements must be a CUDA float64 tensor of shape (8, n)")
        elements = elements.contiguous()
        n = int(elements.shape[1])
        device = elements.device.index or 0
        torch.cuda.current_stream(device).synchronize()  # the library reads the columns on its own stream
        self = cls.__new__(cls)
        self._h = C.c_void_p()
        self._free = lib().astroz_cuda_constellation_free
        ptrs = [C.c_void_p(elements[k].data_ptr()) for k in range(8)]
        check(lib().astroz_cuda_constellation_create_from_elements_device(*ptrs, n, int(grav), int(device),
                                                                           C.byref(self._h)))
        cn, ns, nd = C.c_uint32(), C.c_uint32(), C.c_uint32()
        check(lib().astroz_cuda_constellation_counts(self._h, C.byref(cn), C.byref(ns), C.byref(nd)))
        self.numSatellites, self.numSgp4, self.numSdp4 = cn.value, ns.value, nd.value
        self.device, self.grav = int(device), int(grav)
        return self

    @property
    def devices(self):
        """(device ordinals, first catalog row of each device's satellite range + [n]) behind this handle."""
        n = C.c_int32()
        check(lib().astroz_cuda_constellation_devices(self._h, C.byref(n), None, None))
        ids = (C.c_int32 * n.value)()
        rows = (C.c_uint32 * (n.value + 1))()
        check(lib().astroz_cuda_constellation_devices(self._h, C.byref(n), ids, rows))
        return list(ids), list(rows)

    def host_block(self, n_times: int, layout: int = Layout.satelliteMajor) -> np.ndarray:
        """A page-locked (n, n_times, 3) / (n_times, n, 3) result block placed for this handle: on a multi-device handle
        each GPU's satellite range sits on that GPU's NUMA node.  Released when the array is collected."""
        p = C.c_void_p()
        check(lib().astroz_cuda_constellation_host_block(self._h, int(n_times), int(layout), C.byref(p)))
        shape = self._shape(int(n_times), layout)
        nbytes = int(np.prod(shape)) * 8
        owner = _HostBlock(p.value, nbytes)
        return np.asarray(owner).view(np.float64).reshape(shape)

    def propagate_replicated(self, jd, fr, velocities: bool = True):
        """The north star's all-gather behind one (multi-device) handle: TEME, satellite-major; the whole
        (n, n_times, 3) block(s) end up in the HBM of every device of the handle, stored there from inside the
        propagation kernels over NVLink peer mappings.  Returns (devices, pos_ptrs, vel_ptrs): raw device pointers
        per device, owned by the handle."""
        jd, fr = as_f64(jd), as_f64(fr)
        ids, _ = self.devices
        pp = (C.c_void_p * len(ids))()
        pv = (C.c_void_p * len(ids))()
        check(lib().astroz_cuda_constellation_propagate_replicated(self._h, dptr(jd), dptr(fr), jd.shape[0],
                                                                    1 if velocities else 0, pp, pv))
        return ids, [int(p or 0) for p in pp], [int(p or 0) for p in pv]

    def deinit(self) -> None:
        """Constellation.deinit (src/Constellation.zig:202-210)."""
        if getattr(self, "_h", None) is not None and self._h:
            self._free(self._h)
            self._h = C.c_void_p()

    __del__ = deinit

    # ---- introspection ------------------------------------------------------------------------
    @classmethod
    def from_tle_text(cls, text: str, grav: int = _lib.WGS72, device: int = 0) -> "Constellation":
        """Name of the native `Sgp4Constellation.from_tle_text` (bindings/python/src/sgp4.zig:287-390)."""
        return cls.from_text(text, grav, device)

    @property
    def num_satellites(self) -> int:
        """`Sgp4Constellation.num_satellites` (bindings/python/src/sgp4.zig:413-420)."""
        return self.numSatellites

    @property
    def epochs(self) -> np.ndarray:
        out = np.empty(self.numSatellites)
        check(lib().astroz_cuda_constellation_epochs(self._h, dptr(out)))
        return out

    @property
    def classes(self) -> np.ndarray:
        """0 = SGP4, 1 = SDP4 non-resonant, 2 = SDP4 synchronous, 3 = SDP4 half-day."""
        out = np.empty(self.numSatellites, dtype=np.int32)
        check(lib().astroz_cuda_constellation_classes(self._h, out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    @property
    def referenceEpochJd(self) -> float:
        v = C.c_double()
        check(lib().astroz_cuda_constellation_get_reference_epoch(self._h, C.byref(v)))
        return v.value

    @referenceEpochJd.setter
    def referenceEpochJd(self, jd: float) -> None:
        check(lib().astroz_cuda_constellation_set_reference_epoch(self._h, float(jd)))

    def resetCarry(self) -> None:
        """Constellation.resetCarry (src/Constellation.zig:214-218); a no-op on the device path."""
        check(lib().astroz_cuda_constellation_reset_carry(self._h))

    reset_carry = resetCarry

    # ---- propagation --------------------------------------------------------------------------
    def _shape(self, n_times: int, layout: int, rows=None):
        rows = self.numSatellites if rows is None else rows
        return (rows, n_times, 3) if layout == Layout.satelliteMajor else (n_times, rows, 3)

    def propagate(self, jd, fr, resultsPos=None, resultsVel=None, outputMode: int = OutputMode.teme,
                  layout: int = Layout.timeMajor, velocities: bool = True):
        """Constellation.propagate(jd, fr, resultsPos, resultsVel, outputMode, layout)
        (src/Constellation.zig:245-308) with host buffers.  Buffers are allocated in pinned memory when
        not supplied.  Returns (pos, vel) shaped by `layout`; vel is None when velocities=False."""
        jd, fr = as_f64(jd), as_f64(fr)
        if jd.shape != fr.shape:
            raise ValueError("jd and fr must have the same length")
        nt = jd.shape[0]
        shape = self._shape(nt, layout)
        if resultsPos is None:
            resultsPos = _lib.pinned_empty(shape)
        if resultsVel is None and velocities:
            resultsVel = _lib.pinned_empty(shape)
        for buf in (resultsPos, resultsVel):
            if buf is not None and (buf.dtype != np.float64 or not buf.flags.c_contiguous or buf.size < nt * self.numSatellites * 3):
                # the reference reports a short buffer as SatelliteDecayed (src/Constellation.zig:255-257)
                raise AstrozCudaError(-12, "result buffer too small or not contiguous float64")
        check(lib().astroz_cuda_constellation_propagate(
            self._h, dptr(jd), dptr(fr), nt, dptr(resultsPos), dptr(resultsVel) if resultsVel is not None else None,
            int(outputMode), int(layout)))
        return resultsPos, resultsVel

    def propagate_device(self, jd, fr, pos, vel=None, status=None, outputMode: int = OutputMode.teme,
                         layout: int = Layout.satelliteMajor, out_num_sats: int | None = None,
                         out_sat_offset: int = 0, stream: int = 0) -> None:
        """Same computation, results left in HBM.  pos / vel / status are torch CUDA tensors (or anything
        with .data_ptr()) on this constellation's device; asynchronous on `stream` (a raw cudaStream_t
        value, 0 = the handle's own stream).  out_num_sats / out_sat_offset place this handle's rows inside a larger
        pos / vel block; status is this handle's own (numSatellites, n_times) uint8 block, satellite-major, satellite
        i at row i whatever the offset."""
        jd, fr = as_f64(jd), as_f64(fr)
        nt = jd.shape[0]
        rows = self.numSatellites if out_num_sats is None else int(out_num_sats)
        check(lib().astroz_cuda_constellation_propagate_device(
            self._h, dptr(jd), dptr(fr), nt, C.c_void_p(pos.data_ptr()),
            C.c_void_p(vel.data_ptr()) if vel is not None else None,
            C.c_void_p(status.data_ptr()) if status is not None else None,
            int(outputMode), int(layout), rows, int(out_sat_offset), C.c_void_p(stream) if stream else None))

    # ---- arbitrary (satellite, time) pairs -----------------------------------------------------------
    def propagate_pairs(self, sat, jd, fr, outputMode: int = OutputMode.teme, velocities: bool = True):
        """Propagate n queries (sat[i], jd[i] + fr[i]) in one call -- the batched form of
        `for s, jd, fr in obs: sats[s].sgp4(jd, fr)`.  sat[i] is a catalog row (the row numbering of `propagate`).
        Returns (pos[n, 3], vel[n, 3] or None, status[n] uint8) in the frame of `outputMode`, with the grid's time
        model, epilogues and failed-cell rules; a row outside the catalog raises (valueError), nothing is computed.
        Single-device handles only."""
        sat = np.ascontiguousarray(np.atleast_1d(np.asarray(sat)))
        jd, fr = as_f64(jd), as_f64(fr)
        if not (sat.ndim == jd.ndim == fr.ndim == 1) or not (sat.shape[0] == jd.shape[0] == fr.shape[0]):
            raise ValueError("sat, jd and fr must be 1-D arrays of the same length")
        if sat.size and not np.issubdtype(sat.dtype, np.integer):
            raise ValueError("sat must hold integer catalog rows")
        if sat.size and (sat.min() < 0 or sat.max() > 0xFFFFFFFF):
            raise ValueError("sat holds a negative or too large row index")
        sat = sat.astype(np.uint32, copy=False)
        n = sat.shape[0]
        pos = _lib.pinned_empty((n, 3))
        vel = _lib.pinned_empty((n, 3)) if velocities else None
        status = _lib.pinned_empty((n,), np.uint8)
        check(lib().astroz_cuda_constellation_propagate_pairs(
            self._h, C.c_void_p(sat.ctypes.data), dptr(jd), dptr(fr), n, int(outputMode), dptr(pos),
            dptr(vel) if vel is not None else None, C.c_void_p(status.ctypes.data)))
        return pos, vel, status

    def propagate_pairs_device(self, sat, jd, fr, pos, vel=None, status=None, outputMode: int = OutputMode.teme,
                               stream: int = 0) -> None:
        """`propagate_pairs` with torch CUDA tensors on this constellation's device: sat (int32 / uint32), jd, fr
        (float64) of n queries; pos / vel (n, 3) float64 and status (n,) uint8 receive the results (vel / status
        optional).  A row outside the catalog gets zeros and status 3 (ASTROZ_CELL_BAD_SATELLITE).  Asynchronous on
        `stream` (a raw cudaStream_t value, 0 = the handle's own stream), except that a catalog with deep-space members
        reads the queries' time range back first."""
        import torch

        n = int(sat.numel())
        if int(jd.numel()) != n or int(fr.numel()) != n:
            raise ValueError("sat, jd and fr must have the same length")
        if sat.dtype not in (torch.int32, getattr(torch, "uint32", torch.int32)) or jd.dtype != torch.float64 or \
                fr.dtype != torch.float64:
            raise ValueError("sat must be int32 / uint32, jd and fr float64")
        for name, t, per, dt in (("pos", pos, 3, torch.float64), ("vel", vel, 3, torch.float64),
                                 ("status", status, 1, torch.uint8)):
            if t is not None and (t.dtype != dt or not t.is_contiguous() or int(t.numel()) < n * per):
                raise ValueError(f"{name} must be a contiguous {dt} tensor with at least {n * per} elements")
        for t in (sat, jd, fr):
            if not t.is_contiguous():
                raise ValueError("sat, jd and fr must be contiguous")
        check(lib().astroz_cuda_constellation_propagate_pairs_device(
            self._h, C.c_void_p(sat.data_ptr()), C.c_void_p(jd.data_ptr()), C.c_void_p(fr.data_ptr()), n,
            int(outputMode), C.c_void_p(pos.data_ptr()), C.c_void_p(vel.data_ptr()) if vel is not None else None,
            C.c_void_p(status.data_ptr()) if status is not None else None, C.c_void_p(stream) if stream else None))

    def porkchop(self, chaser, target, dep_jd, dep_fr, arr_jd, arr_fr, *, mu: float | None = None, max_revs: int = 0):
        """Porkchop grids between catalog rows: pair p departs from row chaser[p] at each epoch dep_jd + dep_fr and
        arrives at row target[p] at each epoch arr_jd + arr_fr, both propagated by `propagate_pairs` (TEME).  Cell
        (p, d, a) is the transfer of least |dv1| + |dv2| over max_revs revolutions, prograde relative to the chaser
        (astroz_b200.lambert).  mu defaults to the handle's gravity model's.  Returns dv (P, D, A, 2) km/s, slot and
        status (P, D, A) uint8 (ASTROZ_LAMBERT_*; STATE_FAILED where an endpoint's propagation status is not 0).
        Single-device handles only."""
        rows = [np.ascontiguousarray(np.atleast_1d(np.asarray(x))) for x in (chaser, target)]
        for r in rows:
            if r.ndim != 1 or (r.size and (not np.issubdtype(r.dtype, np.integer) or r.min() < 0 or
                                           r.max() > 0xFFFFFFFF)):
                raise ValueError("chaser and target must be 1-D arrays of catalog rows")
        if rows[0].shape != rows[1].shape:
            raise ValueError("chaser and target must have the same length")
        chaser, target = (r.astype(np.uint32, copy=False) for r in rows)
        dep_jd, dep_fr, arr_jd, arr_fr = as_f64(dep_jd), as_f64(dep_fr), as_f64(arr_jd), as_f64(arr_fr)
        if dep_jd.shape != dep_fr.shape or arr_jd.shape != arr_fr.shape or dep_jd.ndim != 1 or arr_jd.ndim != 1:
            raise ValueError("dep_jd / dep_fr and arr_jd / arr_fr must be 1-D arrays of the same length")
        if max_revs < 0:
            raise ValueError("max_revs must be >= 0")
        if mu is None:
            mu = 398600.8 if self.grav == _lib.WGS72 else 398600.5   # src/constants.zig:41-58
        P, Dn, An = len(chaser), len(dep_jd), len(arr_jd)
        dv = np.zeros((P, Dn, An, 2))
        slot, status = np.zeros((P, Dn, An), dtype=np.uint8), np.zeros((P, Dn, An), dtype=np.uint8)
        check(lib().astroz_cuda_constellation_porkchop(
            self._h, C.c_void_p(chaser.ctypes.data), C.c_void_p(target.ctypes.data), P, dptr(dep_jd), dptr(dep_fr), Dn,
            dptr(arr_jd), dptr(arr_fr), An, float(mu), int(max_revs), dptr(dv), C.c_void_p(slot.ctypes.data),
            C.c_void_p(status.ctypes.data)))
        return dv, slot, status

    def propagate_gather(self, jd, fr, peer_pos=None, peer_vel=None, mc_pos: int = 0, mc_vel: int = 0,
                         out_num_sats: int | None = None, out_sat_offset: int = 0, stream: int = 0) -> None:
        """Fused propagate + all-gather (TEME, satellite-major): this constellation's rows are written into
        every GPU's copy of the block from inside the kernels.  peer_pos / peer_vel: lists of raw device
        pointers (ints) of the per-GPU mappings; mc_pos / mc_vel: NVLS multicast pointers (ints, 0 = use the
        peer lists)."""
        jd, fr = as_f64(jd), as_f64(fr)
        rows = self.numSatellites if out_num_sats is None else int(out_num_sats)
        n = len(peer_pos) if peer_pos else 0
        pp = (C.c_void_p * max(n, 1))(*[C.c_void_p(int(p)) for p in (peer_pos or [])])
        pv = (C.c_void_p * max(n, 1))(*[C.c_void_p(int(p)) for p in (peer_vel or [])]) if peer_vel else None
        check(lib().astroz_cuda_constellation_propagate_gather(
            self._h, dptr(jd), dptr(fr), jd.shape[0], pp if n else None, pv, n,
            C.c_void_p(mc_pos) if mc_pos else None, C.c_void_p(mc_vel) if mc_vel else None,
            rows, int(out_sat_offset), C.c_void_p(stream) if stream else None))

    def propagate_device_f32(self, jd, fr, pos, vel, phase64: bool = True, stream: int = 0) -> None:
        """BASELINE config 5 precision study: the near-earth satellites in fp32 arithmetic (phase64: secular
        angles in fp64 first).  pos / vel: (n_sats, n_times, 3) float64 CUDA tensors."""
        jd, fr = as_f64(jd), as_f64(fr)
        check(lib().astroz_cuda_constellation_propagate_device_f32(
            self._h, dptr(jd), dptr(fr), jd.shape[0], C.c_void_p(pos.data_ptr()), C.c_void_p(vel.data_ptr()),
            1 if phase64 else 0, C.c_void_p(stream) if stream else None))

    def synchronize(self) -> None:
        check(lib().astroz_cuda_constellation_synchronize(self._h))

    def set_timing(self, enabled: bool = True) -> None:
        """Record CUDA events around the kernels of every later call (off by default: the events cost stream time)."""
        check(lib().astroz_cuda_constellation_set_timing(self._h, 1 if enabled else 0))

    def last_kernel_ms(self):
        ms = (C.c_float * 3)()
        check(lib().astroz_cuda_constellation_last_kernel_ms(self._h, ms))
        return float(ms[0]), float(ms[1]), float(ms[2])

    # ---- stateless near-earth path (Constellation.propagateConstellation, :541-605) -----------------
    def propagate_into(self, times, positions=None, velocities=None, epoch_offsets=None, satellite_mask=None,
                       outputMode: int = OutputMode.teme, reference_jd: float = 0.0, time_major: bool = True,
                       output_stride: int = -1, want_velocities: bool = True):
        """Sgp4Constellation.propagate_into(times, positions, velocities, epoch_offsets=, satellite_mask=, output=,
        reference_jd=, time_major=, output_stride=) (bindings/python/src/sgp4.zig:171-268): tsince = times[t] +
        epoch_offsets[sat] for the near-earth satellites only, satellite i -> row i of a block with `output_stride`
        rows (default: the number of near-earth satellites); rows whose mask byte is 0 are left untouched."""
        times = as_f64(times)
        nt = times.shape[0]
        ns = self.numSgp4
        rows = ns if output_stride is None or output_stride <= 0 else int(output_stride)
        if rows < ns:
            raise ValueError("output_stride must be at least num_satellites")
        if epoch_offsets is None:
            off = np.zeros(ns)
        else:
            off = as_f64(epoch_offsets)
            if off.shape[0] < ns:
                raise ValueError("epoch_offsets must have at least num_satellites elements")  # sgp4.zig:144
            off = off[:ns].copy()
        layout = Layout.timeMajor if time_major else Layout.satelliteMajor
        shape = self._shape(nt, layout, rows=rows)
        mask = None
        if satellite_mask is not None:
            mask = np.ascontiguousarray(satellite_mask, dtype=np.uint8)
            if mask.shape[0] < ns:
                raise ValueError("satellite_mask must have at least num_satellites elements")  # sgp4.zig:167
        need = rows * nt * 3
        for name, arr in (("positions", positions), ("velocities", velocities)):
            # the C side writes rows*n_times*3 doubles through the raw pointer (satrec.zig:927-941 raises ValueError)
            if arr is not None and (not isinstance(arr, np.ndarray) or arr.dtype != np.float64 or
                                    not arr.flags.c_contiguous or not arr.flags.writeable or arr.size < need):
                raise ValueError(f"{name} must be a writable C-contiguous float64 array with at least "
                                 f"output_stride*n_times*3 = {need} elements")
        # rows the mask leaves out, or rows beyond the near-earth satellites, are never written: buffers this
        # wrapper allocates itself start at zero so the caller never sees uninitialised pinned memory
        partial = mask is not None or rows > ns
        if positions is None:
            positions = _lib.pinned_empty(shape)
            if partial:
                positions.fill(0.0)
        if velocities is None and want_velocities:
            velocities = _lib.pinned_empty(shape)
            if partial:
                velocities.fill(0.0)
        check(lib().astroz_cuda_sgp4_propagate_into(
            self._h, dptr(times), nt, dptr(off), dptr(positions),
            dptr(velocities) if velocities is not None else None, int(outputMode), float(reference_jd), int(layout),
            mask.ctypes.data_as(C.c_void_p) if mask is not None else None, rows))
        return positions, velocities

    def propagate_sdp4_into(self, jd, fr, positions, velocities=None, outputMode: int = OutputMode.teme,
                            time_major: bool = True, output_stride: int = -1, sat_offset: int = 0) -> None:
        """Constellation.propagateSdp4Constellation (src/Constellation.zig:611-674): the deep-space members only,
        member i -> row sat_offset + i of caller-owned float64 blocks with `output_stride` rows (default numSdp4),
        tsince = (jd + fr - epoch) * 1440."""
        jd, fr = as_f64(jd), as_f64(fr)
        nt = jd.shape[0]
        rows = self.numSdp4 if output_stride is None or output_stride <= 0 else int(output_stride)
        need = rows * nt * 3
        for arr in (positions, velocities):
            if arr is not None and (arr.dtype != np.float64 or not arr.flags.c_contiguous or arr.size < need):
                raise ValueError("output arrays must be C-contiguous float64 with output_stride*n_times*3 elements")
        check(lib().astroz_cuda_sdp4_propagate_into(
            self._h, dptr(jd), dptr(fr), nt, dptr(positions), dptr(velocities) if velocities is not None else None,
            int(outputMode), int(Layout.timeMajor if time_major else Layout.satelliteMajor), rows, int(sat_offset)))

    def screen_conjunction(self, times, target: int, threshold: float = 10.0, epoch_offsets=None,
                           reference_jd: float = 0.0):
        """Sgp4Constellation.screen_conjunction(times, target, threshold, epoch_offsets=, reference_jd=)
        -> (min_distances[n_sgp4] km, min_t_indices[n_sgp4] uint32): fused propagate + single-target screen
        (src/Constellation.zig:683-756).  Nothing but the 12 bytes per satellite leaves the GPU."""
        times = as_f64(times)
        ns = self.numSgp4
        off = np.zeros(ns) if epoch_offsets is None else as_f64(epoch_offsets)[:ns].copy()
        dist = np.empty(ns)
        tidx = np.empty(ns, dtype=np.uint32)
        check(lib().astroz_cuda_sgp4_screen(self._h, dptr(times), times.shape[0], dptr(off), int(target),
                                            float(threshold), float(reference_jd), dptr(dist),
                                            tidx.ctypes.data_as(C.POINTER(C.c_uint32))))
        return dist, tidx


    def coarse_screen_device(self, positions, threshold: float, layout: int = Layout.timeMajor, valid_mask=None,
                             max_results: int = 10_000_000):
        """coarse_screen(positions, num_sats, threshold, valid_mask) (bindings/python/src/conjunction.zig:11-149) on a
        DEVICE position block (torch CUDA tensor shaped by `layout`).  Returns (pairs[n, 2] uint32, t_indices[n]
        uint32) as numpy arrays, sorted by (t, s, other); raises if more than max_results hits were found."""
        import torch

        shape = tuple(positions.shape)
        ns, nt = (shape[0], shape[1]) if layout == Layout.satelliteMajor else (shape[1], shape[0])
        dev = positions.device
        pairs = torch.empty((max_results, 2), dtype=torch.int32, device=dev)
        tidx = torch.empty((max_results,), dtype=torch.int32, device=dev)
        cnt = C.c_uint64()
        torch.cuda.synchronize(dev)
        check(lib().astroz_cuda_constellation_coarse_screen_device(
            self._h, C.c_void_p(positions.data_ptr()), ns, nt, int(layout), float(threshold),
            C.c_void_p(valid_mask.data_ptr()) if valid_mask is not None else None,
            C.c_void_p(pairs.data_ptr()), C.c_void_p(tidx.data_ptr()), max_results, C.byref(cnt)))
        if cnt.value > max_results:
            raise AstrozCudaError(-20, f"{cnt.value} hits exceed max_results={max_results}")
        k = cnt.value
        return _sorted_hits(pairs[:k].cpu().numpy().view(np.uint32), tidx[:k].cpu().numpy().view(np.uint32))

    def screen_all(self, times, threshold: float = 10.0, epoch_offsets=None, max_results: int = 10_000_000):
        """The all-vs-all branch of astroz.screen(source, times, threshold)
        (bindings/python/astroz/__init__.py:535-650): propagate, keep the block in HBM, coarse-screen it there;
        only the hits come back.  Returns (pairs[n, 2], t_indices[n]) sorted by (t, s, other)."""
        times = as_f64(times)
        ns = self.numSgp4
        off = np.zeros(ns) if epoch_offsets is None else as_f64(epoch_offsets)[:ns].copy()
        pairs = np.empty((max_results, 2), dtype=np.uint32)
        tidx = np.empty(max_results, dtype=np.uint32)
        cnt = C.c_uint64()
        check(lib().astroz_cuda_sgp4_screen_all(
            self._h, dptr(times), times.shape[0], dptr(off), float(threshold),
            pairs.ctypes.data_as(C.POINTER(C.c_uint32)), tidx.ctypes.data_as(C.POINTER(C.c_uint32)), max_results,
            C.byref(cnt)))
        if cnt.value > max_results:
            raise AstrozCudaError(-20, f"{cnt.value} hits exceed max_results={max_results}")
        return _sorted_hits(pairs[:cnt.value], tidx[:cnt.value])


class _HostBlock:
    """Owner of a block from astroz_cuda_constellation_host_block (array interface; freed with the last view)."""

    def __init__(self, ptr: int, nbytes: int):
        self.ptr = ptr
        self.__array_interface__ = {"shape": (max(nbytes, 1),), "typestr": "|u1", "data": (ptr, False), "version": 3}

    def __del__(self):
        if getattr(self, "ptr", None):
            try:
                lib().astroz_cuda_host_free(C.c_void_p(self.ptr))
            except Exception:
                pass
            self.ptr = None


def _sorted_hits(pairs: np.ndarray, tidx: np.ndarray):
    """Deterministic order for the hit set: by epoch, then satellite, then partner (the reference's order up to
    ties inside one satellite's neighbourhood walk)."""
    if len(tidx) == 0:
        return pairs.reshape(0, 2).copy(), tidx.copy()
    order = np.lexsort((pairs[:, 1], pairs[:, 0], tidx))
    return np.ascontiguousarray(pairs[order]), np.ascontiguousarray(tidx[order])


def fp64_peak_tflops(device: int = 0) -> float:
    """Measured DFMA throughput of the device (the fp64 roofline denominator)."""
    v = C.c_double()
    check(lib().astroz_cuda_fp64_peak(int(device), C.byref(v)))
    return v.value


def fp64_pipe_peak_tflops(device: int = 0) -> float:
    """Arithmetic peak of the device's fp64 pipe: SMs x 64 lanes x 2 FLOP x max SM clock."""
    v = C.c_double()
    check(lib().astroz_cuda_fp64_pipe_peak(int(device), C.byref(v)))
    return v.value
