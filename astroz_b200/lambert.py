"""Lambert transfers on the device (K9, astroz_b200/csrc/az_lambert.cu).

    from astroz_b200.lambert import lambert_batch
    v1, v2, status, iterations = lambert_batch(r1, r2, tof, 398600.5, max_revs=3)   # (n, 7, 3), (n, 7, 3), (n, 7), (n, 7)

Batched multi-revolution solves of Lambert's problem by Izzo's algorithm, one problem per GPU thread: slot 0 is the
zero-revolution transfer, slot 2M - 1 the left and slot 2M the right branch of M revolutions.  A unit normal per problem
(default +z) sets the sense of motion: the short way when (r1 x r2) . n > 0, the long way when it is < 0.  Slots whose
status is not OK are zero-filled.  `porkchop_device` turns device-resident endpoint states into transfer-cost grids;
`Constellation.porkchop` runs the whole grid from a catalogue.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._abi import DEFINES as D
from ._lib import check, lib

# per-slot status bytes
OK, NO_SOLUTION, DEGENERATE, NOT_CONVERGED, STATE_FAILED = (
    D["ASTROZ_LAMBERT_OK"], D["ASTROZ_LAMBERT_NO_SOLUTION"], D["ASTROZ_LAMBERT_DEGENERATE"],
    D["ASTROZ_LAMBERT_NOT_CONVERGED"], D["ASTROZ_LAMBERT_STATE_FAILED"])
STATUS_NAMES = {OK: "ok", NO_SOLUTION: "no solution", DEGENERATE: "degenerate geometry",
                NOT_CONVERGED: "not converged", STATE_FAILED: "endpoint state failed"}
MAX_REVS = D["ASTROZ_LAMBERT_MAX_REVS"]


def _rows3(x, name, n=None) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1, 3))
    if n is not None and len(a) != n:
        raise ValueError(f"{name} must have shape (n, 3) or (3,)")
    return a


def lambert_batch(r1, r2, tof, mu: float, *, max_revs: int = 0, normal=None, device: int = 0):
    """Solve n problems at once.  r1, r2: (n, 3) km; tof: (n,) s; mu: km^3/s^2; normal: (n, 3) or (3,) (default +z).
    Returns v1, v2 (n, S, 3) km/s, status (n, S) uint8 and iterations (n, S) uint8, S = 2 max_revs + 1."""
    r1 = _rows3(r1, "r1")
    n = len(r1)
    r2 = _rows3(r2, "r2", n)
    tof = np.ascontiguousarray(np.broadcast_to(np.asarray(tof, dtype=np.float64), (n,)))
    nrm = None
    if normal is not None:
        nrm = np.ascontiguousarray(np.broadcast_to(np.asarray(normal, dtype=np.float64), (n, 3)))
    if not 0 <= int(max_revs) <= MAX_REVS:
        raise ValueError(f"max_revs must be in [0, {MAX_REVS}]")
    S = 2 * int(max_revs) + 1
    v1, v2 = np.zeros((n, S, 3)), np.zeros((n, S, 3))
    status, iters = np.zeros((n, S), dtype=np.uint8), np.zeros((n, S), dtype=np.uint8)
    vp = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_lambert(vp(r1), vp(r2), vp(tof), vp(nrm), n, float(mu), int(max_revs), int(device), vp(v1),
                                    vp(v2), vp(status), vp(iters)))
    return v1, v2, status, iters


def _check_tensors(specs, device):
    import torch

    for name, t, size, dtype in specs:
        if t is None:
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {device}")


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def lambert_batch_device(r1, r2, tof, v1, v2, status, mu: float, *, iterations=None, normal=None, max_revs: int = 0,
                         stream: int = 0) -> None:
    """`lambert_batch` with torch CUDA tensors on one device: r1 / r2 (n, 3), tof (n,), normal (n, 3) or None, float64;
    v1 / v2 (n, S, 3) float64, status and iterations (n, S) uint8 (iterations optional) receive the results.  One launch
    on `stream` (a raw cudaStream_t value, 0 = the default stream)."""
    import torch

    if int(max_revs) < 0:
        raise ValueError("max_revs must be >= 0")
    n = int(tof.numel())
    S = 2 * int(max_revs) + 1
    f64, u8 = torch.float64, torch.uint8
    _check_tensors([("r1", r1, 3 * n, f64), ("r2", r2, 3 * n, f64), ("tof", tof, n, f64), ("normal", normal, 3 * n, f64),
                    ("v1", v1, 3 * n * S, f64), ("v2", v2, 3 * n * S, f64), ("status", status, n * S, u8),
                    ("iterations", iterations, n * S, u8)], tof.device)
    check(lib().astroz_cuda_lambert_device(_ptr(r1), _ptr(r2), _ptr(tof), _ptr(normal), n, float(mu), int(max_revs),
                                           int(tof.device.index), _ptr(v1), _ptr(v2), _ptr(status), _ptr(iterations),
                                           C.c_void_p(stream) if stream else None))


def porkchop_device(dep_states, dep_status, arr_states, arr_status, dep_jd, dep_fr, arr_jd, arr_fr, mu: float, dv,
                    slot, status, *, max_revs: int = 0, stream: int = 0) -> None:
    """Porkchop grids from device-resident endpoint states (torch CUDA tensors on one device).  dep_states (P, D, 6) and
    arr_states (P, A, 6) float64: the chaser of pair p at each departure, the target at each arrival (km, km/s); their
    status bytes (P, D) / (P, A) uint8 (None: all valid; a nonzero byte gives the cell STATE_FAILED); dep_jd / dep_fr (D,)
    and arr_jd / arr_fr (A,) float64, shared by all pairs.  Cell (p, d, a): tof = ((arr_jd - dep_jd) + (arr_fr - dep_fr))
    * 86400 s, transfers prograde relative to the chaser, the slot of least |dv1| + |dv2| kept.  dv (P, D, A, 2) float64,
    slot and status (P, D, A) uint8 receive the results.  Asynchronous on `stream`."""
    import torch

    if int(max_revs) < 0:
        raise ValueError("max_revs must be >= 0")
    if dep_states.dim() != 3 or arr_states.dim() != 3 or dep_states.shape[0] != arr_states.shape[0]:
        raise ValueError("dep_states must be (P, D, 6) and arr_states (P, A, 6)")
    P, Dn, An = int(dep_states.shape[0]), int(dep_states.shape[1]), int(arr_states.shape[1])
    f64, u8 = torch.float64, torch.uint8
    _check_tensors([("dep_states", dep_states, P * Dn * 6, f64), ("dep_status", dep_status, P * Dn, u8),
                    ("arr_states", arr_states, P * An * 6, f64), ("arr_status", arr_status, P * An, u8),
                    ("dep_jd", dep_jd, Dn, f64), ("dep_fr", dep_fr, Dn, f64), ("arr_jd", arr_jd, An, f64),
                    ("arr_fr", arr_fr, An, f64), ("dv", dv, P * Dn * An * 2, f64), ("slot", slot, P * Dn * An, u8),
                    ("status", status, P * Dn * An, u8)], dep_states.device)
    check(lib().astroz_cuda_lambert_porkchop_device(
        _ptr(dep_states), _ptr(dep_status), _ptr(arr_states), _ptr(arr_status), P, _ptr(dep_jd), _ptr(dep_fr), Dn,
        _ptr(arr_jd), _ptr(arr_fr), An, float(mu), int(max_revs), int(dep_states.device.index), _ptr(dv), _ptr(slot),
        _ptr(status), C.c_void_p(stream) if stream else None))
