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

from . import _abi
from ._abi import DEFINES as D
from ._lib import AstrozCudaError, check, lib

FORCE_J2, FORCE_DRAG = D["ASTROZ_FORCE_J2"], D["ASTROZ_FORCE_DRAG"]
INTEGRATORS = {"rk4": D["ASTROZ_INTEGRATOR_RK4"], "dp87": D["ASTROZ_INTEGRATOR_DP87"]}
# per-state status bytes
OK, STOPPED, SUBSTEP_LIMIT, NON_FINITE = (D["ASTROZ_NUMERICAL_OK"], D["ASTROZ_NUMERICAL_STOPPED"],
                                         D["ASTROZ_NUMERICAL_SUBSTEP_LIMIT"], D["ASTROZ_NUMERICAL_NON_FINITE"])


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


# ---- model lists: the force models of the reference's propagators module (src/propagators/ForceModel.zig) -------------
# flags of astroz_force_model_t
_PER_STATE = {"c": D["ASTROZ_MODEL_PER_STATE_C"], "area": D["ASTROZ_MODEL_PER_STATE_AREA"],
              "mass": D["ASTROZ_MODEL_PER_STATE_MASS"]}
_POS_TABLE = D["ASTROZ_MODEL_POS_TABLE"]
MAX_MODELS = D["ASTROZ_MAX_MODELS"]
AU_KM = 1.495978707e8   # src/constants.zig:28, SolarRadiationPressure's default Sun distance

_ForceModelC = _abi.structure("astroz_force_model_t")


class _Model:
    """A force model of a list: its scalar fields, its coefficients that may vary per state (c, area, mass: a scalar or
    one value per state) and its position (a fixed 3-vector or one row per output interval)."""
    kind = -1

    def __init__(self, scalars, coefs=None, pos=None):
        self._scalars, self._coefs, self._pos = scalars, coefs or {}, pos

    def __repr__(self):
        fields = {**self._scalars, **self._coefs, **({} if self._pos is None else {"pos": self._pos})}
        return f"{type(self).__name__}({', '.join(f'{k}={v!r}' for k, v in fields.items())})"


class TwoBody(_Model):
    """TwoBody(mu): ForceModel.zig:42-56"""
    kind = D["ASTROZ_MODEL_TWO_BODY"]

    def __init__(self, mu):
        super().__init__({"mu": float(mu)})


class _Zonal(_Model):
    def __init__(self, mu, coef, r_eq):
        super().__init__({"mu": float(mu), "coef": float(coef), "r_eq": float(r_eq)})


class J2(_Zonal):
    """J2(mu, j2, r_eq): ForceModel.zig:58-80"""
    kind = D["ASTROZ_MODEL_J2"]


class J3(_Zonal):
    """J3(mu, j3, r_eq): ForceModel.zig:113-143.  Its x / y terms carry an extra 1/r, as the reference's do."""
    kind = D["ASTROZ_MODEL_J3"]


class J4(_Zonal):
    """J4(mu, j4, r_eq): ForceModel.zig:145-176.  Divides by r^9, as the reference does."""
    kind = D["ASTROZ_MODEL_J4"]


class Drag(_Model):
    """Drag(r_eq, rho0, H, cd, area, mass, max_altitude): exponential atmosphere, ForceModel.zig:82-111.  cd, area [m^2]
    and mass [kg] are scalars or one value per state."""
    kind = D["ASTROZ_MODEL_DRAG"]

    def __init__(self, r_eq, rho0, H, cd, area, mass, max_altitude):
        super().__init__({"r_eq": float(r_eq), "rho0": float(rho0), "scale_height": float(H),
                          "max_altitude": float(max_altitude)}, {"c": cd, "area": area, "mass": mass})


class ImprovedDrag(_Model):
    """ImprovedDrag(r_eq, cd, area, mass, max_altitude, f107): five-layer atmosphere rotating with the Earth, scaled by
    F10.7, ForceModel.zig:268-349.  Zero below 100 km, as the reference.  cd, area [m^2] and mass [kg] are scalars or one
    value per state."""
    kind = D["ASTROZ_MODEL_IMPROVED_DRAG"]

    def __init__(self, r_eq, cd, area, mass, max_altitude, f107):
        super().__init__({"r_eq": float(r_eq), "max_altitude": float(max_altitude), "f107": float(f107)},
                         {"c": cd, "area": area, "mass": mass})


class SolarRadiationPressure(_Model):
    """SolarRadiationPressure(cr, area, mass, r_eq, sun_pos=None): ForceModel.zig:178-228, with a cylindrical shadow of
    radius r_eq.  cr, area [m^2] and mass [kg] are scalars or one value per state.  sun_pos [km] is a 3-vector (default
    (AU, 0, 0), as init sets it) or a (K, 3) table whose row k holds for output interval k (K = samples - 1)."""
    kind = D["ASTROZ_MODEL_SRP"]

    def __init__(self, cr, area, mass, r_eq, sun_pos=None):
        super().__init__({"r_eq": float(r_eq)}, {"c": cr, "area": area, "mass": mass},
                         (AU_KM, 0.0, 0.0) if sun_pos is None else sun_pos)


class ThirdBody(_Model):
    """ThirdBody(mu, pos): Battin's formula, ForceModel.zig:230-266.  pos [km] is a 3-vector or a (K, 3) table whose row
    k holds for output interval k (K = samples - 1)."""
    kind = D["ASTROZ_MODEL_THIRD_BODY"]

    def __init__(self, mu, pos):
        super().__init__({"mu": float(mu)}, pos=pos)


def _descriptors(models, n, K, array):
    """The astroz_force_model_t array of `models`.  array(x, shape, name) returns (pointer, keep-alive) for a per-state
    array or a position table, or None when x is a scalar / a fixed 3-vector."""
    models = list(models)
    if not models or not all(isinstance(m, _Model) for m in models):
        raise ValueError("models must be a non-empty list of TwoBody / J2 / J3 / J4 / Drag / ImprovedDrag / "
                         "SolarRadiationPressure / ThirdBody")
    if len(models) > MAX_MODELS:
        raise ValueError(f"at most {MAX_MODELS} models")
    descs = (_ForceModelC * len(models))()
    keep = []
    for d, m in zip(descs, models):
        d.kind = m.kind
        for k, v in m._scalars.items():
            setattr(d, k, v)
        for k, v in m._coefs.items():
            a = array(v, (n,), k)
            if a is None:
                setattr(d, k, float(v))
            else:
                d.flags |= _PER_STATE[k]
                setattr(d, k + "_per_state", a[0])
                keep.append(a[1])
        if m._pos is not None:
            a = array(m._pos, (K, 3), "pos")
            if a is None:
                d.pos[:] = [float(x) for x in m._pos]
            else:
                d.flags |= _POS_TABLE
                d.pos_table = a[0]
                keep.append(a[1])
    return descs, keep


def _host_array(x, shape, name):
    a = np.asarray(x, dtype=np.float64)
    if a.ndim == 0 or (name == "pos" and a.ndim == 1):
        if name == "pos" and a.shape != (3,):
            raise ValueError("a position is a 3-vector or a (K, 3) table")
        return None
    if a.shape != shape:
        raise ValueError(f"{name} must be a scalar{' or 3-vector' if name == 'pos' else ''} or have shape {shape}")
    a = np.ascontiguousarray(a)
    return C.c_void_p(a.ctypes.data), a


def propagate_models_batch(states, t0, duration, dt, models, *, integrator="dp87", rtol=1e-9, atol=1e-12, device=0,
                           out=None):
    """Integrate n initial states over the shared sample times under an ordered list of force models (at most 16):
    one model is used as it is, several are summed as the reference's Composite sums them, in list order.

    states: (n, 6).  models: TwoBody / J2 / J3 / J4 / Drag / ImprovedDrag / SolarRadiationPressure / ThirdBody, whose
    coefficients may be (n,) arrays and whose positions may be (K, 3) tables, K = samples - 1.
    Returns (times[samples], traj[n, samples, 6], status[n] uint8, steps[n, 2] uint64 accepted / rejected), as
    propagate_numerical_batch does."""
    states = np.ascontiguousarray(states, dtype=np.float64)
    if states.ndim != 2 or states.shape[1] != 6:
        raise ValueError("states must have shape (n, 6)")
    n = states.shape[0]
    times = numerical_times(t0, duration, dt)
    descs, keep = _descriptors(models, n, len(times) - 1, _host_array)
    shape = (n, len(times), 6)
    if out is None:
        out = np.empty(shape)
    elif out.shape != shape or out.dtype != np.float64 or not out.flags.c_contiguous:
        raise ValueError(f"out must be a C-contiguous float64 array of shape {shape}")
    status = np.zeros(n, dtype=np.uint8)
    steps = np.zeros((n, 2), dtype=np.uint64)
    vp = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_propagate_numerical_models(
        vp(states), n, float(t0), float(duration), float(dt), C.cast(descs, C.c_void_p), len(descs),
        _integrator(integrator), float(rtol), float(atol), int(device), vp(out), vp(status), vp(steps)))
    del keep
    return times, out, status, steps


def propagate_models_batch_device(states, t0, duration, dt, models, out, status, steps=None, *, integrator="dp87",
                                  rtol=1e-9, atol=1e-12, stream: int = 0) -> None:
    """`propagate_models_batch` with torch CUDA tensors on one device: states (n, 6) float64; per-state coefficients as
    (n,) float64 tensors and position tables as (K, 3) float64 tensors on the same device (scalars and fixed 3-vectors
    as Python numbers); out (n, samples, 6) float64, status (n,) uint8 and steps (n, 2) int64 (optional) receive the
    results.  Asynchronous on `stream` (a raw cudaStream_t value, 0 = the default stream)."""
    import torch

    n = int(states.shape[0]) if states.dim() == 2 else -1
    if n < 0 or states.shape[1] != 6 or states.dtype != torch.float64 or not states.is_cuda:
        raise ValueError("states must be a CUDA float64 tensor of shape (n, 6)")
    samples = len(numerical_times(t0, duration, dt))

    def tensor_or_none(x, shape, name):
        if not isinstance(x, torch.Tensor):
            return _host_array(x, shape, name)   # a scalar or a fixed 3-vector; a host array is refused below
        if x.dtype != torch.float64 or not x.is_contiguous() or tuple(x.shape) != shape or x.device != states.device:
            raise ValueError(f"{name} must be a contiguous float64 tensor of shape {shape} on {states.device}")
        return C.c_void_p(x.data_ptr()), x

    def array(x, shape, name):
        r = tensor_or_none(x, shape, name)
        if r is not None and not isinstance(r[1], torch.Tensor):
            raise ValueError(f"{name}: per-state arrays and position tables must be CUDA tensors here")
        return r

    descs, keep = _descriptors(models, n, samples - 1, array)
    for name, t, size, dtype in (("out", out, n * samples * 6, torch.float64), ("status", status, n, torch.uint8),
                                 ("steps", steps, n * 2, torch.int64)):
        if t is None and name == "steps":
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != states.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {states.device}")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_propagate_numerical_models_device(
        ptr(states), n, float(t0), float(duration), float(dt), C.cast(descs, C.c_void_p), len(descs),
        _integrator(integrator), float(rtol), float(atol), int(states.device.index), ptr(out), ptr(status), ptr(steps),
        C.c_void_p(stream) if stream else None))
    del keep


# ---- impulsive maneuvers: the loop of the reference's Spacecraft.propagate (src/Spacecraft.zig:172-323) -------------
# status bytes beyond the batch calls'
ABNORMAL, TRUNCATED = D["ASTROZ_MANEUVER_ABNORMAL"], D["ASTROZ_MANEUVER_TRUNCATED"]
EARTH_MU = 398600.5   # WGS-84 (src/constants.zig:55-58), the reference's default orbitingObject.mu
IMPULSE_DTYPE = np.dtype(_abi.structure("astroz_impulse_t"))


class _Impulse:
    """An impulse of a schedule: its time [s, the states' clock] and the kind's parameters."""
    kind = -1

    def __init__(self, t, *p):
        self.time, self.p = float(t), tuple(float(x) for x in p) + (0.0,) * (3 - len(p))

    def __repr__(self):
        return f"{type(self).__name__}({self.time!r}, {', '.join(repr(x) for x in self.p)})"


class Absolute(_Impulse):
    """Absolute(t, dv): velocity += dv (a 3-vector, km/s), calculations.impulse (calculations.zig:480-485)"""
    kind = D["ASTROZ_IMPULSE_ABSOLUTE"]

    def __init__(self, t, dv):
        dv = [float(x) for x in dv]
        if len(dv) != 3:
            raise ValueError("dv is a 3-vector")
        super().__init__(t, *dv)


class Prograde(_Impulse):
    """Prograde(t, dv): dv km/s along the velocity (Spacecraft.zig:260-263)"""
    kind = D["ASTROZ_IMPULSE_PROGRADE"]

    def __init__(self, t, dv):
        super().__init__(t, dv)


class Phase(_Impulse):
    """Phase(t, angle, orbits=1.0): the reference's phasing maneuver (Spacecraft.zig:237-252, :310-323): a prograde
    burn, a coast of `orbits` periods of the circular orbit at the burn's radius sampled every h, then the opposite
    burn.  angle in rad, orbits > 0."""
    kind = D["ASTROZ_IMPULSE_PHASE"]

    def __init__(self, t, angle, orbits=1.0):
        super().__init__(t, angle, orbits)


class PlaneChange(_Impulse):
    """PlaneChange(t, d_incl, d_raan): the reference's applyPlaneChange (Spacecraft.zig:272-307), nothing below 1e-10
    rad.  Its Δv points along (hx sin di, hy sin di, hz cos di) / |h|, the reference's "simplified" direction -- not
    the textbook plane change."""
    kind = D["ASTROZ_IMPULSE_PLANE_CHANGE"]

    def __init__(self, t, d_incl, d_raan):
        super().__init__(t, d_incl, d_raan)


def pack_schedules(schedules, n):
    """(offsets[n + 1] uint32, impulses[m] IMPULSE_DTYPE) of `schedules`: one list of impulses shared by every state,
    or n lists.  Impulse kinds and parameters are checked as the C ABI checks them."""
    schedules = list(schedules)
    if all(isinstance(b, _Impulse) for b in schedules):
        schedules = [schedules] * n
    elif len(schedules) != n:
        raise ValueError(f"schedules must be one list of impulses or {n} lists")
    lengths = [len(s) for s in schedules]
    offsets = np.zeros(n + 1, dtype=np.uint32)
    np.cumsum(lengths, out=offsets[1:])
    imp = np.zeros(int(offsets[-1]), dtype=IMPULSE_DTYPE)
    k = 0
    for s in schedules:
        for b in s:
            if not isinstance(b, _Impulse):
                raise ValueError("a schedule holds Absolute / Prograde / Phase / PlaneChange impulses")
            if not (np.isfinite(b.time) and all(np.isfinite(b.p))):
                raise ValueError(f"{b!r}: time and parameters must be finite")
            if b.kind == Phase.kind and not b.p[1] > 0:
                raise ValueError(f"{b!r}: orbits must be > 0")
            imp[k] = (b.time, b.kind, 0, b.p)
            k += 1
    return offsets, imp


def _estimate_samples(states, t0, duration, h, offsets, imp, mu):
    """Rows for a first call: the regular samples, 3 per burn (the partial step, the burn sample, one more regular step
    on the shifted grid) and every phasing coast at the state's initial radius with 10 % slack."""
    base = len(numerical_times(t0, duration, h)) + 3 * int(np.max(np.diff(offsets), initial=0))
    phase = np.flatnonzero(imp["kind"] == Phase.kind)
    if len(phase) == 0:
        return base
    owner = np.searchsorted(offsets, phase, side="right") - 1
    r = np.linalg.norm(states[owner, :3], axis=1)
    coast = np.ceil(1.1 * 2.0 * np.pi * np.sqrt(r ** 3 / mu) * imp["p"][phase, 1] / h) + 2
    extra = np.zeros(len(states))
    np.add.at(extra, owner, coast)
    return int(min(base + extra.max(), 0xfffffffe))


def _subset(models, idx):
    """The models with their per-state coefficients cut to the states idx"""
    import copy

    out = []
    for m in models:
        c = copy.copy(m)
        c._coefs = {k: (np.asarray(v)[idx] if np.ndim(v) == 1 else v) for k, v in m._coefs.items()}
        out.append(c)
    return out


def _maneuvers_call(states, t0, duration, h, models, offsets, imp, mu, integrator, rtol, atol, max_samples, device):
    n = states.shape[0]
    descs, keep = _descriptors(models, n, 0, _host_array)
    times = np.empty((n, max_samples))
    traj = np.empty((n, max_samples, 6))
    count = np.zeros(n, dtype=np.uint64)
    status = np.zeros(n, dtype=np.uint8)
    steps = np.zeros((n, 2), dtype=np.uint64)
    vp = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    check(lib().astroz_cuda_propagate_maneuvers(
        vp(states), n, float(t0), float(duration), float(h), float(mu), vp(offsets), vp(imp) if len(imp) else None,
        len(imp), C.cast(descs, C.c_void_p), len(descs), _integrator(integrator), float(rtol), float(atol),
        int(max_samples), int(device), vp(times), vp(traj), vp(count), vp(status), vp(steps)))
    del keep
    return times, traj, count, status, steps


def propagate_maneuvers_batch(states, t0, duration, h, models, schedules, *, mu=EARTH_MU, integrator="rk4", rtol=1e-9,
                              atol=1e-12, max_samples=None, device=0):
    """Propagate n states through impulse schedules, as the reference's Spacecraft.propagate does for one: step h
    from t0 to t0 + duration under the model list, the impulses of each schedule fired in list order when their time
    comes within the next step (an impulse before t0 fires at once), each burn sampled, stopping on an abnormal orbit.

    states: (n, 6) km, km/s.  models: as propagate_models_batch (fixed positions only).  schedules: one list of
    Absolute / Prograde / Phase / PlaneChange shared by every state, or n lists.  mu: the central body's parameter
    (phasing burns and the abnormal-orbit test).  integrator: "rk4" (the reference's) or "dp87".
    max_samples: the row length; None sizes the rows from an estimate and reruns the states that did not fit, once, at
    their own sample count (a state's result depends on its own inputs only, so the bytes are those of an ample call).
    Returns (times[n, S], traj[n, S, 6], n_samples[n] uint64, status[n] uint8, steps[n, 2] uint64).  Row i holds
    n_samples[i] samples and zeros after them (all S when the state was TRUNCATED); sample times repeat at burns and the
    last step can be negative after a phasing coast that passes t0 + duration."""
    states = np.ascontiguousarray(states, dtype=np.float64)
    if states.ndim != 2 or states.shape[1] != 6:
        raise ValueError("states must have shape (n, 6)")
    n = states.shape[0]
    offsets, imp = pack_schedules(schedules, n)
    models = list(models)
    if max_samples is not None:
        return _maneuvers_call(states, t0, duration, h, models, offsets, imp, mu, integrator, rtol, atol,
                               int(max_samples), device)
    first = _estimate_samples(states, t0, duration, h, offsets, imp, mu)
    times, traj, count, status, steps = _maneuvers_call(states, t0, duration, h, models, offsets, imp, mu, integrator,
                                                        rtol, atol, first, device)
    again = np.flatnonzero(status == TRUNCATED)
    if len(again) == 0:
        return times, traj, count, status, steps
    width = int(count[again].max())
    sub_off = np.zeros(len(again) + 1, dtype=np.uint32)
    np.cumsum(np.diff(offsets)[again], out=sub_off[1:])
    sub_imp = np.concatenate([imp[offsets[i]:offsets[i + 1]] for i in again]) if len(imp) else imp
    t2, y2, c2, s2, st2 = _maneuvers_call(np.ascontiguousarray(states[again]), t0, duration, h, _subset(models, again),
                                          sub_off, sub_imp, mu, integrator, rtol, atol, width, device)
    T = np.zeros((n, width))
    Y = np.zeros((n, width, 6))
    T[:, :first], Y[:, :first] = times, traj
    T[again], Y[again], count[again], status[again], steps[again] = t2, y2, c2, s2, st2
    return T, Y, count, status, steps


def propagate_maneuvers_batch_device(states, t0, duration, h, models, schedules, times, out, n_samples, status,
                                     steps=None, *, mu=EARTH_MU, integrator="rk4", rtol=1e-9, atol=1e-12,
                                     stream: int = 0) -> None:
    """`propagate_maneuvers_batch` with torch CUDA tensors on one device: states (n, 6) float64, per-state coefficients
    as (n,) float64 tensors; schedules as there (checked here, then uploaded); times (n, S) float64, out (n, S, 6)
    float64, n_samples (n,) int64, status (n,) uint8 and steps (n, 2) int64 (optional) receive the results, S being the
    row length.  One kernel, asynchronous on `stream` (a raw cudaStream_t value, 0 = the default stream)."""
    import torch

    n = int(states.shape[0]) if states.dim() == 2 else -1
    if n < 0 or states.shape[1] != 6 or states.dtype != torch.float64 or not states.is_cuda:
        raise ValueError("states must be a CUDA float64 tensor of shape (n, 6)")
    if not isinstance(times, torch.Tensor) or times.dim() != 2 or times.shape[0] != n:
        raise ValueError("times must be a tensor of shape (n, max_samples)")
    S = int(times.shape[1])
    for name, t, size, dtype in (("times", times, n * S, torch.float64), ("out", out, n * S * 6, torch.float64),
                                 ("n_samples", n_samples, n, torch.int64), ("status", status, n, torch.uint8),
                                 ("steps", steps, n * 2, torch.int64)):
        if t is None and name == "steps":
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or not t.is_contiguous() or int(t.numel()) != size \
                or t.device != states.device:
            raise ValueError(f"{name} must be a contiguous {dtype} tensor of {size} elements on {states.device}")

    def array(x, shape, name):
        if not isinstance(x, torch.Tensor):
            r = _host_array(x, shape, name)
            if r is not None:
                raise ValueError(f"{name}: per-state arrays must be CUDA tensors here")
            return None
        if x.dtype != torch.float64 or not x.is_contiguous() or tuple(x.shape) != shape or x.device != states.device:
            raise ValueError(f"{name} must be a contiguous float64 tensor of shape {shape} on {states.device}")
        return C.c_void_p(x.data_ptr()), x

    descs, keep = _descriptors(models, n, 0, array)
    offsets, imp = pack_schedules(schedules, n)
    d_off = torch.from_numpy(offsets.view(np.int32)).to(states.device)
    d_imp = torch.from_numpy(imp.view(np.uint8)).to(states.device)
    torch.cuda.current_stream(states.device).synchronize()   # the uploads have landed before `stream` reads them
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    check(lib().astroz_cuda_propagate_maneuvers_device(
        ptr(states), n, float(t0), float(duration), float(h), float(mu), ptr(d_off), ptr(d_imp) if len(imp) else None,
        len(imp), C.cast(descs, C.c_void_p), len(descs), _integrator(integrator), float(rtol), float(atol), S,
        int(states.device.index), ptr(times), ptr(out), ptr(n_samples), ptr(status), ptr(steps),
        C.c_void_p(stream) if stream else None))
    if stream:   # the schedules stay allocated until the kernel on `stream` has read them
        ext = torch.cuda.ExternalStream(stream, device=states.device)
        d_off.record_stream(ext)
        d_imp.record_stream(ext)
    del keep


__all__ = ["propagate_numerical_batch", "propagate_numerical_batch_device", "numerical_times", "AstrozCudaError",
           "OK", "STOPPED", "SUBSTEP_LIMIT", "NON_FINITE", "propagate_models_batch", "propagate_models_batch_device",
           "TwoBody", "J2", "J3", "J4", "Drag", "ImprovedDrag", "SolarRadiationPressure", "ThirdBody", "MAX_MODELS",
           "ABNORMAL", "TRUNCATED", "EARTH_MU", "Absolute", "Prograde", "Phase", "PlaneChange", "pack_schedules",
           "propagate_maneuvers_batch", "propagate_maneuvers_batch_device"]
