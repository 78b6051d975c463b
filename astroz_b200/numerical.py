"""Numerical propagation of batches of initial states on the device (K7, astroz_b200/csrc/az_numerical.cu).

    from astroz_b200.numerical import propagate_numerical_batch
    times, traj, status, steps = propagate_numerical_batch(states, 0.0, 86400.0, 60.0, 398600.5, j2=1.0826e-3,
                                                           r_eq=6378.137)

State i's trajectory is what the reference's `propagate_numerical(states[i], t0, duration, dt, mu, ...)`
(bindings/python/src/propagator.zig:13-193) returns for it alone: RK4 or Dormand-Prince 8(7), two-body plus optional J2
and exponential-atmosphere drag.  The states of a batch are independent (Monte-Carlo dispersions, debris clouds, a
catalogue's TEME states), so one call runs them all, one per GPU thread.  Units: km, km/s, s, km^3/s^2.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import AstrozCudaError, check, lib

FORCE_J2, FORCE_DRAG = 1, 2
INTEGRATORS = {"rk4": 0, "dp87": 1}
# per-state status bytes (ASTROZ_NUMERICAL_*)
OK, STOPPED, SUBSTEP_LIMIT, NON_FINITE = 0, 1, 2, 3


def numerical_times(t0: float, duration: float, dt: float) -> np.ndarray:
    """The sample times every state of a batch shares (the loop of src/propagators/Propagator.zig:32-45)."""
    count = C.c_uint64()
    check(lib().astroz_cuda_numerical_times(float(t0), float(duration), float(dt), None, C.byref(count)))
    times = np.empty(count.value)
    check(lib().astroz_cuda_numerical_times(float(t0), float(duration), float(dt), C.c_void_p(times.ctypes.data),
                                            C.byref(count)))
    return times


def _forces(j2, r_eq, drag_cd) -> int:
    return (FORCE_J2 if j2 is not None else 0) | (FORCE_DRAG if drag_cd is not None else 0)


def _scalar_ptr(x):
    return None if x is None else C.pointer(C.c_double(float(x)))


def _integrator(name: str) -> int:
    if name not in INTEGRATORS:
        raise ValueError("integrator must be 'rk4' or 'dp87'")
    return INTEGRATORS[name]


def propagate_numerical_batch(states, t0, duration, dt, mu, *, j2=None, r_eq=None, drag_cd=None, drag_area=None,
                              drag_mass=None, integrator="dp87", rtol=1e-9, atol=1e-12, device=0, out=None):
    """Integrate n initial states over the shared sample times.

    states: (n, 6) x y z vx vy vz.  j2 / r_eq: J2 is on when j2 is given; r_eq is needed for J2 and drag.  Drag is on when
    drag_cd is given; drag_cd / drag_area [m^2] / drag_mass [kg] are scalars or one value per state.
    out (optional): a caller-owned (n, samples, 6) float64 block (pinned or registered memory receives it by direct DMA).
    Returns (times[samples], traj[n, samples, 6], status[n] uint8, steps[n, 2] uint64 accepted / rejected)."""
    states = np.ascontiguousarray(states, dtype=np.float64)
    if states.ndim != 2 or states.shape[1] != 6:
        raise ValueError("states must have shape (n, 6)")
    n = states.shape[0]
    forces = _forces(j2, r_eq, drag_cd)
    drag = [None, None, None]
    if forces & FORCE_DRAG:
        if drag_area is None or drag_mass is None:
            raise ValueError("drag_area and drag_mass are required when drag_cd is specified")
        drag = [np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (n,))) for x in
                (drag_cd, drag_area, drag_mass)]
    times = numerical_times(t0, duration, dt)
    shape = (n, len(times), 6)
    if out is None:
        out = np.empty(shape)
    elif out.shape != shape or out.dtype != np.float64 or not out.flags.c_contiguous:
        raise ValueError(f"out must be a C-contiguous float64 array of shape {shape}")
    status = np.zeros(n, dtype=np.uint8)
    steps = np.zeros((n, 2), dtype=np.uint64)
    vp = lambda a: None if a is None else C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_propagate_numerical(
        vp(states), n, float(t0), float(duration), float(dt), float(mu), forces, _scalar_ptr(j2), _scalar_ptr(r_eq),
        *[vp(a) for a in drag], _integrator(integrator), float(rtol), float(atol), int(device), vp(out), vp(status),
        vp(steps)))
    return times, out, status, steps


def propagate_numerical_batch_device(states, t0, duration, dt, mu, out, status, steps=None, *, j2=None, r_eq=None,
                                     drag_cd=None, drag_area=None, drag_mass=None, integrator="dp87", rtol=1e-9,
                                     atol=1e-12, stream: int = 0) -> None:
    """`propagate_numerical_batch` with torch CUDA tensors on one device: states (n, 6) float64; drag_cd / drag_area /
    drag_mass (n,) float64 tensors when drag is on; out (n, samples, 6) float64, status (n,) uint8 and steps (n, 2)
    int64 (optional) receive the results.  Asynchronous on `stream` (a raw cudaStream_t value, 0 = the default
    stream)."""
    import torch

    n = int(states.shape[0]) if states.dim() == 2 else -1
    if n < 0 or states.shape[1] != 6 or states.dtype != torch.float64 or not states.is_cuda:
        raise ValueError("states must be a CUDA float64 tensor of shape (n, 6)")
    samples = len(numerical_times(t0, duration, dt))
    forces = _forces(j2, r_eq, drag_cd)
    tensors = [("states", states, n * 6, torch.float64), ("out", out, n * samples * 6, torch.float64),
               ("status", status, n, torch.uint8), ("steps", steps, n * 2, torch.int64)]
    if forces & FORCE_DRAG:
        if drag_area is None or drag_mass is None:
            raise ValueError("drag_area and drag_mass are required when drag_cd is specified")
        tensors += [("drag_cd", drag_cd, n, torch.float64), ("drag_area", drag_area, n, torch.float64),
                    ("drag_mass", drag_mass, n, torch.float64)]
    for name, t, size, dtype in tensors:
        if t is None and name == "steps":
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != states.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {states.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    drag = [drag_cd, drag_area, drag_mass] if forces & FORCE_DRAG else [None, None, None]
    check(lib().astroz_cuda_propagate_numerical_device(
        ptr(states), n, float(t0), float(duration), float(dt), float(mu), forces, _scalar_ptr(j2), _scalar_ptr(r_eq),
        *[ptr(t) for t in drag], _integrator(integrator), float(rtol), float(atol), int(states.device.index), ptr(out),
        ptr(status), ptr(steps), C.c_void_p(stream) if stream else None))


__all__ = ["propagate_numerical_batch", "propagate_numerical_batch_device", "numerical_times", "AstrozCudaError",
           "OK", "STOPPED", "SUBSTEP_LIMIT", "NON_FINITE"]
